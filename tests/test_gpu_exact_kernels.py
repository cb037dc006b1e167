"""Kernel-level tests of the exact-fp32 CUDA-core kernels against fp64 references of the same operations, at every
dispatch variant and edge the kernels branch on:

* A. the exact-fp32 LSTM (lstm.cu on gemm_tall.cuh) through ``ops.SharedLSTM``;
* B. the exact-fp32 projection (proj.cu: tall GEMM, dz_kernel, small_wgrad_kernel, reduce GEMM, pool_kernel) through
  ``ops._proj_fwd`` / ``ops._proj_bwd`` without a weight image, and ``ops.TemporalPool``;
* C. small.cu: ``ops.ContextGate``, ``ops.FuseOut``, ``ops.obs_to_node_major``;
* D. CSR construction on the device and the SpMM step on graphs with empty rows, empty columns and no entries at all, and one
  model with an isolated region against the fp64 sparse oracle.

Bars: 2e-5 on forward values, 5e-5 on gradients (max-norm relative, ``O.max_rel_err``), the bars of the tensor-core
suites.  Every group has a negative control: a subtly wrong reference that must land outside its bar.
"""
import re

import numpy as np
import pytest
import scipy.sparse as sp
import torch
from torch import nn

import stmgcn_oracle as O
from helpers import DEV, FWD_TOL, GRAD_TOL, rel_err, sm_count
from kernel_cases import ACTS, fuse_rows, isolated_matrix, proj_inputs, proj_ref_out, proj_rows, round_tf32
from lstm_cases import LSTM_CASES, lstm_inputs, reference, step_local_error

pytestmark = pytest.mark.gpu
SPMM_TOL = 1e-5


def _report(what, errs, gerrs, control):
    worst_g = max(gerrs, key=gerrs.get) if gerrs else None
    print(f"{what}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items())
          + (f"; worst gradient {gerrs[worst_g]:.2e} ({worst_g})" if gerrs else "") + f"; control {control:.2e}")
    bad = {k: v for k, v in errs.items() if not v <= FWD_TOL}
    bad.update({k: v for k, v in gerrs.items() if not v <= GRAD_TOL})
    assert not bad, f"{what}: above the bar: {bad}"


# ======================================================================================================================
# A. exact-fp32 LSTM
# ======================================================================================================================
def _no_tensor_cores(monkeypatch, force_fma):
    """Route SharedLSTM as a user would (``tc`` unless forced) and record any call into the tensor-core forward."""
    from stmgcn_b200 import ops
    calls = []
    real = ops._lstm16_forward
    monkeypatch.setattr(ops, "_lstm16_forward", lambda *a: calls.append(1) or real(*a))
    monkeypatch.setattr(ops, "_LSTM_PATH", "fma" if force_fma else "tc")
    return calls


@pytest.mark.parametrize("case", LSTM_CASES, ids=[c[0] for c in LSTM_CASES])
def test_exact_lstm_matches_fp64(case, monkeypatch):
    """Forward step by step (every layer-step's c and h), h_top / h_n / c_n, then d_s and the four gradients of every
    layer of the loss (h_top . d_top).sum(), against the fp64 reference forced with the kernel's tape.  Negative
    control: the one-plane (bf16-rounded h and weights) reference lands outside the forward bar.

    Measured on an H100 80GB HBM3 (max over the nine cases): step-local forward 1.0e-6 (7.6e-6 in the saturated case),
    h_top / h_n / c_n 1.8e-6, gradients 1.1e-5 (weight_ih_l0 at T = 70, a sum over 294 000 row-steps), control
    2.4e-4 .. 2.7e-2.  Free-running instead of tape-forced, fp32 against fp64 differs by ~7e-5 in the saturated case
    (rounding amplified through 20 steps of a recurrence with weights in +-2; torch's own fp32 LSTM arithmetic is as far
    from fp64 on these inputs)."""
    from stmgcn_b200 import ops
    name, hid, lyr, t, c, n, b, state, force_fma = case
    if n is None:
        n = (2 * 32 * sm_count()) // b + 1
    rows = n * b
    calls = _no_tensor_cores(monkeypatch, force_fma)
    xo, s, h0, c0, ws, d_top = lstm_inputs(n, b, t, lyr, c, hid, state, seed=LSTM_CASES.index(case),
                                           saturate=name == "saturated")
    xo, s, d_top = xo.to(DEV), s.to(DEV), d_top.to(DEV)
    h0, c0 = (None, None) if h0 is None else (h0.to(DEV), c0.to(DEV))
    ws = [w.to(DEV) for w in ws]
    s_g = s.clone().requires_grad_(True)
    ws_g = [w.clone().requires_grad_(True) for w in ws]
    h_top, h_n, c_n = ops.SharedLSTM.apply(xo, s_g, h0, c0, lyr, hid, state, *ws_g)
    hs_k, cs_k = h_top.grad_fn.saved_tensors[4:6]                   # the exact path's own tape, (L, T, R, H)
    tape = dict(h=hs_k.detach().double(), c=cs_k.detach().double())
    if state:
        tape["h0"] = h0.double()
    h_top = h_top.reshape(rows, hid)
    (h_top * d_top).sum().backward()
    torch.cuda.synchronize()
    assert not calls, f"{name}: SharedLSTM took the tensor-core kernels"

    hs, cs, layers, s64 = reference(xo, s, h0, c0, ws, lyr, 2, tape)
    assert all(bool(torch.isfinite(v).all()) for v in (h_top, tape["c"], s_g.grad, *[w.grad for w in ws_g]))
    errs = {"step-local forward": step_local_error(tape, hs, cs), "h_top": rel_err(h_top, hs[-1][-1])}
    if state:
        errs["h_n"] = rel_err(h_n, torch.stack([h[-1] for h in hs]))
        errs["c_n"] = rel_err(c_n, torch.stack([v[-1] for v in cs]))
    flat = [w for layer in layers for w in layer]
    ref_grads = torch.autograd.grad((hs[-1][-1] * d_top.double()).sum(), [s64] + flat)
    gerrs = {"d_s": rel_err(s_g.grad, ref_grads[0])}
    for i, (g, r) in enumerate(zip(ws_g, ref_grads[1:])):
        l, j = divmod(i, 4)
        gerrs[f"{('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')[j]}_l{l}"] = rel_err(g.grad, r)
    if name == "saturated":
        assert float(tape["c"].abs().max()) > 15.0, "the saturated case does not drive c far enough"
    hs_o, cs_o, _, _ = reference(xo, s, h0, c0, ws, lyr, 1, tape, grad=False)
    control = step_local_error(tape, hs_o, cs_o)
    _report(f"exact LSTM {name} rows={rows}", errs, gerrs, control)
    assert control > FWD_TOL, f"{name}: the one-plane reference is within the bar ({control:.2e})"


@pytest.mark.parametrize("hid,lyr,c,limit", [(64, 2, 5, "input_dim=5 unsupported (max 4)"),
                                             (132, 2, 1, "lstm hidden=132 unsupported (need multiple of 4, <= 128)"),
                                             (6, 2, 1, "lstm hidden=6 unsupported (need multiple of 4, <= 128)"),
                                             (64, 9, 1, "layers=9 (max 8)")])
def test_exact_lstm_rejects_shapes_beyond_its_limits(hid, lyr, c, limit, monkeypatch):
    """C <= 4, H a multiple of 4 and <= 128, L <= 8 (lstm.cu check_dims): beyond them SharedLSTM raises, naming the
    limit, instead of running."""
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_LSTM_PATH", "fma")
    xo, s, _, _, ws, _ = lstm_inputs(2, 3, 4, lyr, c, hid, False, seed=0)
    with pytest.raises(RuntimeError, match=re.escape(limit)):
        ops.SharedLSTM.apply(xo.to(DEV), s.to(DEV), None, None, lyr, hid, False, *[w.to(DEV) for w in ws])


def test_exact_lstm_second_backward_raises(monkeypatch):
    """The exact path's backward overwrites its gate tape in place: a second backward over the same graph raises."""
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_LSTM_PATH", "fma")
    xo, s, _, _, ws, d_top = lstm_inputs(3, 4, 5, 2, 1, 64, False, seed=1)
    ws_g = [w.to(DEV).requires_grad_(True) for w in ws]
    h_top, _, _ = ops.SharedLSTM.apply(xo.to(DEV), s.to(DEV), None, None, 2, 64, False, *ws_g)
    loss = (h_top.reshape(12, 64) * d_top.to(DEV)).sum()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="second backward over the same graph is not supported"):
        loss.backward()


@pytest.mark.parametrize("lyr,t", [(3, 7), (1, 1)])
def test_exact_lstm_launch_sequence(lyr, t, monkeypatch):
    """The exact path's forward is one tall GEMM per (timestep, layer); its backward one pointwise kernel and one data
    GEMM per (timestep, layer), then one weight-gradient reduce GEMM per layer."""
    from stmgcn_b200 import _lib, ops
    monkeypatch.setattr(ops, "_LSTM_PATH", "fma")
    xo, s, _, _, ws, d_top = lstm_inputs(3, 4, t, lyr, 2, 36, False, seed=2)
    ws_g = [w.to(DEV).requires_grad_(True) for w in ws]
    n0 = _lib.launch_count()
    h_top, _, _ = ops.SharedLSTM.apply(xo.to(DEV), s.to(DEV), None, None, lyr, 36, False, *ws_g)
    n1 = _lib.launch_count()
    (h_top.reshape(12, 36) * d_top.to(DEV)).sum().backward()
    n2 = _lib.launch_count()
    assert (n1 - n0, n2 - n1) == (lyr * t, 2 * lyr * t + lyr)


# ======================================================================================================================
# B. exact-fp32 projection and temporal pooling
# ======================================================================================================================
PROJ_PAIRS = [(7, 7), (9, 9),          # p, q % 4 != 0: scalar tall GEMMs, small_wgrad
              (12, 12),                # cfg3 temporal GCN
              (32, 20), (128, 68),     # spatial projection with H / G != 64; (128, 68): TN = 128, reduce<256>
              (64, 300),               # q > 256: two tall-GEMM column panels, two reduce z-panels
              (100, 64)]               # U GEMM with ks * p > 256: several column panels
# the small_wgrad_kernel / reduce GEMM boundary: ks*p*q <= 2048 and 64 rows of (ks*p + q) floats <= 48 KB
BOUNDARY = [(3, 24, 24, True), (4, 24, 24, False),      # 1728 vs 2304 outputs
            (1, 180, 10, True), (1, 200, 10, False),    # 1800 / 2000 outputs; 47.5 KB vs 52.5 KB of shared memory
            (8, 25, 10, False)]                         # 2000 outputs, 52.5 KB: the scalar reduce<64> GEMM
PROJ_SHAPES = ([(ks, p, q) for p, q in PROJ_PAIRS for ks in range(1, 9)] + [(6, 24, 24)]   # cfg5 temporal: reduce
               + [(ks, p, q) for ks, p, q, _ in BOUNDARY])
PROJ_ROWS = [1, 33, 513, "waves"]


def small_wgrad_taken(ks, p, q):
    """The condition under which stmgcn_proj_bwd computes dW with small_wgrad_kernel (proj.cu)."""
    return ks * p * q <= 256 * 8 and 64 * (ks * p + q) * 4 <= 48 * 1024


@pytest.mark.parametrize("ks,p,q,small", BOUNDARY)
def test_small_wgrad_boundary_cases_sit_on_the_intended_side(ks, p, q, small):
    assert small_wgrad_taken(ks, p, q) == small


@pytest.mark.parametrize("rows_id", PROJ_ROWS)
@pytest.mark.parametrize("ks,p,q", PROJ_SHAPES)
def test_exact_projection_matches_fp64(ks, p, q, rows_id):
    """out = act(sum_k S_k W_k + b); dZ = d_out * [out > 0] (the kernel's own mask); db = sum dZ; dW_k = S_k^T dZ;
    U_k = dZ W_k^T, on the exact-fp32 kernels (no weight image).  ReLU and bias cycle through their four combinations
    with ks and the row count, so every shape and every row count meets each.  Negative control: the reference with the
    stack rounded to tf32 lands outside the forward bar.

    Measured on an H100 80GB HBM3 (max over all 248 cases): out 1.7e-6, gradients 2.0e-6, control 6.2e-5 .. 6.8e-4."""
    from stmgcn_b200 import ops
    rows = proj_rows(rows_id)
    relu, bias = ACTS[(ks + PROJ_ROWS.index(rows_id)) % 4]
    s, w, bv, d_out = proj_inputs(ks, p, q, rows, relu, bias, seed=1000 * ks + 10 * p + q + PROJ_ROWS.index(rows_id))
    s, w, d_out = s.to(DEV), w.to(DEV), d_out.to(DEV)
    bv = None if bv is None else bv.to(DEV)
    act = 1 if relu else 0
    s4 = s.reshape(ks, rows, 1, p)
    out = ops._proj_fwd(s4, w, bv, act, None, 1)
    dw, db, u = ops._proj_bwd(s4, w, act, out, d_out.reshape(rows, 1, q), None, 1.0, 1, bias, True)
    torch.cuda.synchronize()
    out = out.reshape(rows, q)

    s64, w64 = s.double(), w.double()
    b64 = None if bv is None else bv.double()
    ref_out = proj_ref_out(s64, w64, b64, relu)
    dz = d_out.double() * (out > 0) if relu else d_out.double()
    errs = {"out": rel_err(out, ref_out)}
    gerrs = {}
    if bias:
        gerrs["db"] = rel_err(db, dz.sum(0))
    dw_ref = torch.einsum("krp,rq->kpq", s64, dz)
    u_ref = torch.einsum("rq,kpq->krp", dz, w64.reshape(ks, p, q))
    for k in range(ks):
        gerrs[f"dW_{k}"] = rel_err(dw[k * p:(k + 1) * p], dw_ref[k])
        gerrs[f"U_{k}"] = rel_err(u[k].reshape(rows, p), u_ref[k])
    if relu and rows > 4:
        zero = out[4::5][:, ::3] if bias else out[4::5]
        assert bool((zero == 0).all()), "a zero pre-activation did not give a zero ReLU output"
    control = rel_err(out, proj_ref_out(round_tf32(s), w64, b64, relu))
    _report(f"proj ks={ks} p={p} q={q} rows={rows} relu={relu} bias={bias}", errs, gerrs, control)
    assert control > FWD_TOL, f"the tf32-rounded reference is within the bar ({control:.2e})"


def _cheb_stack64(lap64, x64, ks):
    n = x64.shape[0]
    flat = x64.reshape(n, -1)
    out = [flat]
    if ks > 1:
        out.append(lap64 @ flat)
    for _ in range(2, ks):
        out.append(2.0 * (lap64 @ out[-1]) - out[-2])
    return torch.stack(out).reshape((ks,) + tuple(x64.shape))


# (regions N, batch B, T, supports ks)
POOL_CASES = [(33, 5, 12, 4),       # cfg3-like temporal GCN: small_wgrad
              (50, 3, 7, 3),        # T = 7: scalar GEMMs
              (300, 2, 24, 6),      # cfg5-like: reduce<64>
              (20, 64, 9, 1),       # ks = 1 (no graph), scalar
              (2100, 1, 12, 4)]     # 2100 rows: grid-stride dz / small_wgrad, several pool region chunks


@pytest.mark.parametrize("relu,bias", ACTS)
@pytest.mark.parametrize("n,b,t,ks", POOL_CASES)
def test_temporal_pool_matches_fp64(n, b, t, ks, relu, bias):
    """ops.TemporalPool on Chebyshev supports (pool = sum_n (x + act(GCN_T x)), pool_kernel) and its backward
    (dz_kernel's broadcast gradient d_pool[b] * scale, bias and weight gradients) against fp64 autograd; then the same
    backward called with scale 0.37.  The graph has isolated regions and x is zero on one of them, so some ReLU
    pre-activations are exactly 0.  Negative control: the reference without the residual x of one region.

    Measured on an H100 80GB HBM3 (max over all 20 cases): pool 1.2e-6, gradients 2.0e-6, control 9.0e-4 .. 0.16."""
    from stmgcn_b200 import ops
    from stmgcn_b200.graph import GraphHandle, SupportSet
    a = isolated_matrix(n, seed=n + ks)
    a = a / max(1.0, float(np.abs(a).sum(1).max()), float(np.abs(a).sum(0).max()))     # spectral radius <= 1
    lap = torch.from_numpy(a)
    gen = torch.Generator().manual_seed(7 * n + t)
    x = torch.randn(n, b, t, generator=gen)
    iso = np.flatnonzero((a == 0).all(0) & (a == 0).all(1))
    if len(iso):
        x[int(iso[0])] = 0.0
    w = torch.randn(ks * t, t, generator=gen) / t ** 0.5
    bv = torch.randn(t, generator=gen) * 0.3
    bv[::3] = 0.0
    d_pool = torch.randn(b, t, generator=gen)
    graphs = [GraphHandle.from_dense(lap.to(DEV))] if ks > 1 else []
    sset = SupportSet("cheb", n, ks, graphs, torch.device(DEV))
    xd, d_pool = x.to(DEV), d_pool.to(DEV)
    w_g = w.to(DEV).requires_grad_(True)
    b_g = bv.to(DEV).requires_grad_(True) if bias else None
    act = 1 if relu else 0
    pool = ops.TemporalPool.apply(xd, w_g, b_g, sset, act)
    stack, _, out_k = pool.grad_fn.saved_tensors
    (pool * d_pool).sum().backward()
    dw2, db2, _ = ops._proj_bwd(stack, w_g.detach(), act, out_k, None, d_pool, 0.37, b, bias, False)
    torch.cuda.synchronize()

    w64 = w.double().to(DEV).requires_grad_(True)
    b64 = bv.double().to(DEV).requires_grad_(True) if bias else None
    s64 = _cheb_stack64(lap.double().to(DEV), xd.double(), ks)
    z = torch.einsum("knbp,kpq->nbq", s64, w64.reshape(ks, t, t))
    if bias:
        z = z + b64
    ref_pool = (xd.double() + (z.clamp_min(0) if relu else z)).sum(0)
    masked = z * (out_k > 0) if relu else z                        # the kernel's own ReLU mask for the backward
    grads = torch.autograd.grad(((xd.double() + masked).sum(0) * d_pool.double()).sum(), [w64] + ([b64] if bias else []))
    errs = {"pool": rel_err(pool, ref_pool)}
    gerrs = {"dW": rel_err(w_g.grad, grads[0]), "dW scale 0.37": rel_err(dw2, 0.37 * grads[0])}
    if bias:
        gerrs.update({"db": rel_err(b_g.grad, grads[1]), "db scale 0.37": rel_err(db2, 0.37 * grads[1])})
    if relu and len(iso):
        assert bool((out_k[int(iso[0])][:, ::3] == 0).all())
    control = rel_err(pool, ref_pool - xd.double()[n // 2])
    _report(f"TemporalPool N={n} B={b} T={t} ks={ks} relu={relu} bias={bias}", errs, gerrs, control)
    assert control > FWD_TOL, f"the reference without one region's residual is within the bar ({control:.2e})"


# ======================================================================================================================
# C. small.cu
# ======================================================================================================================
@pytest.mark.parametrize("b", [1, 64])
@pytest.mark.parametrize("t", [1, 12, 33, 129, 300])
def test_context_gate_matches_fp64(t, b):
    """ops.ContextGate: s = sigmoid(fc(relu(fc(pool / N)))) with the same fc twice, forward and backward (d_pool,
    d_fcw, d_fcb) against fp64 autograd.  T = 1, 12 | 33, 129 | 300 run 32 | 128 | 256 threads, and T = 300 makes every
    thread loop.  For T > 1 window 0's bias cancels a quarter of its first-layer pre-activations, so those a1 lie within
    rounding distance of 0; the reference takes the kernel's own ReLU mask.  Negative control: the reference with fcb applied in
    the first fc only lands outside the forward bar.

    Measured on an H100 80GB HBM3 (max over all ten cases): s 3.6e-7, a1 7.1e-7, gradients 5.7e-7, control 0.13 .. 0.70.
    (With T = 1 and B = 1 cancelled too, the only a1 was ~1e-8 and its max-norm error meaningless.)"""
    from stmgcn_b200 import ops
    n_regions = 50
    gen = torch.Generator().manual_seed(31 * t + b)
    pool = torch.randn(b, t, generator=gen) * n_regions
    fcw = torch.randn(t, t, generator=gen) / t ** 0.5
    fcb = (torch.rand(t, generator=gen) - 0.5)
    fcb[1::4] = -(fcw.double() @ (pool[0].double() / n_regions))[1::4].float()
    d_s = torch.randn(b, t, generator=gen)
    pool_g, fcw_g, fcb_g = (v.to(DEV).requires_grad_(True) for v in (pool, fcw, fcb))
    s = ops.ContextGate.apply(pool_g, fcw_g, fcb_g, n_regions)
    a1_k = s.grad_fn.saved_tensors[1]
    (s * d_s.to(DEV)).sum().backward()
    torch.cuda.synchronize()

    p64, w64, b64 = (v.double().to(DEV).requires_grad_(True) for v in (pool, fcw, fcb))
    a1 = (p64 / n_regions) @ w64.t() + b64
    ref_s = torch.sigmoid(a1.clamp_min(0) @ w64.t() + b64)
    s_masked = torch.sigmoid((a1 * (a1_k > 0)) @ w64.t() + b64)
    g = torch.autograd.grad((s_masked * d_s.double().to(DEV)).sum(), [p64, w64, b64])
    errs = {"s": rel_err(s, ref_s), "a1": rel_err(a1_k, a1)}
    gerrs = {"d_pool": rel_err(pool_g.grad, g[0]), "d_fcw": rel_err(fcw_g.grad, g[1]), "d_fcb": rel_err(fcb_g.grad, g[2])}
    control = rel_err(s, torch.sigmoid(a1.clamp_min(0) @ w64.t()))
    _report(f"gate T={t} B={b}", errs, gerrs, control)
    assert control > FWD_TOL, f"the reference with one fcb is within the bar ({control:.2e})"


@pytest.mark.parametrize("rows_id", ["small", "waves"])
@pytest.mark.parametrize("c_out", [1, 2, 33, 40])
@pytest.mark.parametrize("gdim", [1, 20, 64, 100])
@pytest.mark.parametrize("m", [1, 3, 8])
def test_fuse_out_matches_fp64(m, gdim, c_out, rows_id):
    """ops.FuseOut: y (B,N,C) = fc(sum_m g_m) and its backward (d_g_m, d_fcw, d_fcb) against fp64.  c_out > 32 runs the
    second bias-gradient lane loop; gdim 1 / 20 / 100 leave lanes idle.  g_m and d_y have nonzero means: with zero-mean
    inputs the single entry of d_fcw at M = G = C = 1 is a sum over 17 K rows that nearly cancels, and its max-norm error
    (3.2e-5, measured) reflects that sum's conditioning rather than the kernel.  Negative control: the reference without
    fcb.

    Measured on an H100 80GB HBM3 (max over all 96 cases): y 1.9e-7, gradients 1.5e-6, control 2.9e-3 .. 0.43."""
    from stmgcn_b200 import ops
    n, b = fuse_rows(rows_id)
    gen = torch.Generator().manual_seed(1000 * m + 10 * gdim + c_out)
    gs = [(0.3 + torch.randn(n, b, gdim, generator=gen)).to(DEV).requires_grad_(True) for _ in range(m)]
    fcw = (torch.randn(c_out, gdim, generator=gen) / gdim ** 0.5).to(DEV).requires_grad_(True)
    fcb = (torch.randn(c_out, generator=gen) * 0.3).to(DEV).requires_grad_(True)
    d_y = (0.5 + torch.randn(b, n, c_out, generator=gen)).to(DEV)
    y = ops.FuseOut.apply(fcw, fcb, *gs)
    (y * d_y).sum().backward()
    torch.cuda.synchronize()

    g64 = [g.detach().double().requires_grad_(True) for g in gs]
    w64, b64 = fcw.detach().double().requires_grad_(True), fcb.detach().double().requires_grad_(True)
    feat = sum(g64)
    ref_y = (feat @ w64.t() + b64).permute(1, 0, 2)
    grads = torch.autograd.grad((ref_y * d_y.double()).sum(), g64 + [w64, b64])
    errs = {"y": rel_err(y, ref_y)}
    gerrs = {f"d_g{k}": rel_err(gs[k].grad, grads[k]) for k in range(m)}
    gerrs.update({"d_fcw": rel_err(fcw.grad, grads[m]), "d_fcb": rel_err(fcb.grad, grads[m + 1])})
    control = rel_err(y, ref_y - b64)
    _report(f"fuse_out M={m} G={gdim} C={c_out} rows={n * b}", errs, gerrs, control)
    assert control > FWD_TOL, f"the reference without fcb is within the bar ({control:.2e})"


def test_fuse_out_beyond_shared_memory_raises_in_the_forward():
    """The backward accumulates C*G + C floats in 48 KB of shared memory, and the forward takes the same limit: C = 40,
    G = 400 (16 040 floats) raises in the forward, so no step runs a forward its backward would refuse."""
    from stmgcn_b200 import ops
    gs = [torch.randn(3, 2, 400, device=DEV, requires_grad=True)]
    fcw = torch.randn(40, 400, device=DEV, requires_grad=True)
    fcb = torch.randn(40, device=DEV, requires_grad=True)
    with pytest.raises(RuntimeError, match="fuse_out_fwd: C\\*G=16000 too large"):
        ops.FuseOut.apply(fcw, fcb, *gs)


@pytest.mark.parametrize("c", [1, 3])
def test_obs_to_node_major_is_exact(c):
    """xo (N,B,T,C) is the permuted observation tensor and xt (N,B,T) its sum over C in channel order, bit for bit."""
    from stmgcn_b200 import ops
    gen = torch.Generator().manual_seed(c)
    obs = torch.randn(5, 7, 33, c, generator=gen)
    xo, xt = ops.obs_to_node_major(obs.to(DEV))
    want_xo = obs.permute(2, 0, 1, 3)
    want_xt = want_xo[..., 0].clone()
    for k in range(1, c):
        want_xt = want_xt + want_xo[..., k]
    assert torch.equal(xo.cpu(), want_xo)
    assert torch.equal(xt.cpu(), want_xt)


# ======================================================================================================================
# D. graphs with empty rows and columns
# ======================================================================================================================
GRAPHS = [(n, kind) for n in (1, 33, 300) for kind in ("isolated", "zero")]


@pytest.mark.parametrize("n,kind", GRAPHS)
def test_graph_handles_with_empty_rows_and_columns_export_scipy_csr(n, kind):
    """GraphHandle.from_dense and from_csr on matrices with empty rows, empty columns, isolated indices, or no entries:
    export(False) / export(True) equal scipy's CSR and CSR^T exactly."""
    from stmgcn_b200.graph import GraphHandle
    a = isolated_matrix(n, seed=n, kind=kind)
    ref, ref_t = sp.csr_matrix(a), sp.csr_matrix(a.T)
    if kind == "isolated" and n > 1:
        assert (np.diff(ref.indptr) == 0).any() and (np.diff(ref_t.indptr) == 0).any()
    handles = {"dense": GraphHandle.from_dense(torch.from_numpy(a).to(DEV)),
               "csr": GraphHandle.from_csr(n, torch.from_numpy(ref.indptr).to(DEV), torch.from_numpy(ref.indices).to(DEV),
                                           torch.from_numpy(ref.data).to(DEV))}
    for src, g in handles.items():
        assert g.n == n and g.nnz == ref.nnz, src
        for transpose, want in ((False, ref), (True, ref_t)):
            rp, ci, va = (t.cpu().numpy() for t in g.export(transpose))
            assert np.array_equal(rp, want.indptr), (src, transpose)
            assert np.array_equal(ci, want.indices), (src, transpose)
            assert np.array_equal(va, want.data), (src, transpose)


@pytest.mark.parametrize("f", [7, 40])
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("n,kind", GRAPHS)
def test_spmm_step_on_empty_rows(n, kind, transpose, f):
    """Y = 2 op(A) X - Z + 0.5 U with ops.spmm_step (f = 7: scalar kernel; f = 40: float4 kernel) and, for f = 40,
    ops.spmm_step16 (X gathered from its bf16 copy), against fp64; on the rows of op(A) without entries Y must be
    exactly -Z + 0.5 U.  Negative control: each kernel's result against the other kernel's reference (X rounded to bf16
    or not) lands outside the bar.  Measured on an H100 80GB HBM3 (max over all cases): 1.7e-7, control 1.5e-3 .. 2.4e-3."""
    from stmgcn_b200 import ops
    from stmgcn_b200.graph import GraphHandle
    a = isolated_matrix(n, seed=3 * n + f, kind=kind)
    op = (a.T if transpose else a).astype(np.float64)
    empty = np.flatnonzero((op == 0).all(1))
    g = GraphHandle.from_dense(torch.from_numpy(a).to(DEV))
    gen = torch.Generator().manual_seed(n + f)
    x, z, u = (torch.randn(n, f, generator=gen).to(DEV) for _ in range(3))
    x16 = ops.to_bf16(x) if f % 8 == 0 else None
    ys = {"fp32": torch.empty_like(x)}
    ops.spmm_step(g, transpose, 2.0, x, -1.0, z, 0.5, u, ys["fp32"])
    if x16 is not None:
        ys["bf16"] = torch.empty_like(x)
        ops.spmm_step16(g, transpose, 2.0, x16, -1.0, z, 0.5, u, ys["bf16"], None)
    torch.cuda.synchronize()
    a64 = torch.from_numpy(op).to(DEV)
    refs = {"fp32": 2.0 * (a64 @ x.double()) - z.double() + 0.5 * u.double()}
    if x16 is not None:
        refs["bf16"] = 2.0 * (a64 @ x16.double()) - z.double() + 0.5 * u.double()
    rest = -z + 0.5 * u
    for mode, y in ys.items():
        err = rel_err(y, refs[mode])
        line = f"spmm {mode} n={n} {kind} transpose={transpose} f={f}: {err:.2e}, {len(empty)} empty rows"
        assert torch.equal(y[empty], rest[empty]), f"{mode}: an empty row is not beta Z + gamma U"
        if len(refs) == 2 and kind != "zero":
            control = rel_err(y, refs["bf16" if mode == "fp32" else "fp32"])
            line += f"; control {control:.2e}"
            assert control > SPMM_TOL, f"{mode}: the other kernel's reference is within the bar ({control:.2e})"
        print(line)
        assert err <= SPMM_TOL, line


@pytest.mark.parametrize("supports", ["sparse", "dense"])
def test_model_with_an_isolated_region_matches_sparse_oracle(supports):
    """ST_MGCN with one region of graph 0 that has no edge: its row and column of L~ are zero.  The supports come from
    Adj_Preprocessor("chebyshev").process_sparse, as CSR or as the dense Chebyshev stack of that L~ (dense() on the
    adjacency itself follows the reference's symmetric_normalize, whose D^-1/2 is infinite on such a region and makes
    the stack NaN).  H = 32 and G = 16: the exact-fp32 LSTM and projections.  Forward and every gradient against the
    fp64 sparse oracle at 1e-4, the bar of tests/test_gpu_parity.py.  Measured on an H100 80GB HBM3: forward 6.6e-7,
    gradients 1.4e-6."""
    import GCN
    from helpers import TOL, assert_close, build_model
    from stmgcn_b200 import synth
    shape = dict(n=60, m=2, k=2, t=6, b=3, c=1, hid=32, layers=2, gcn_hid=16)
    n = shape["n"]
    adjs = [synth.make_adjacency(n, g, 0.08) for g in range(shape["m"])]
    iso = 17
    adjs[0][iso, :] = 0.0
    adjs[0][:, iso] = 0.0
    adjs[0][iso - 1, iso + 1] = adjs[0][iso + 1, iso - 1] = 1.0                  # keep the ring's neighbours connected
    pre = GCN.Adj_Preprocessor("chebyshev", shape["k"])
    sparse = [pre.process_sparse(a) for a in adjs]
    laps = [s.laplacian_dense() for s in sparse]
    assert bool((laps[0][iso] == 0).all() and (laps[0][:, iso] == 0).all())
    if supports == "sparse":
        sups = [s.to(DEV) for s in sparse]
    else:
        sups = [torch.stack([torch.eye(n), lt, 2.0 * (lt @ lt) - torch.eye(n)]).to(DEV) for lt in laps]
    params = O.init_params(shape["m"], shape["t"], shape["c"], shape["hid"], shape["layers"], shape["gcn_hid"],
                           shape["k"] + 1, seed=5)
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(shape["b"], shape["t"], n, shape["c"], generator=gen)
    y = torch.randn(shape["b"], n, shape["c"], generator=gen)
    model = build_model(shape, DEV)
    model.load_state_dict(params)
    out = model(obs_seq=x.to(DEV), sta_adj_list=sups)
    loss = nn.MSELoss()(out, y.to(DEV))
    loss.backward()
    orc = O.SparseOracle({k_: v.numpy() for k_, v in params.items()}, [sp.csr_matrix(lt.numpy()) for lt in laps],
                         shape["k"] + 1, dtype=np.float64)
    o_ref, l_ref, g_ref = orc.loss_and_grads(x.numpy(), y.numpy())
    errs = [assert_close(out.detach().cpu().numpy(), o_ref, "forward")]
    for key, p in model.named_parameters():
        errs.append(assert_close(p.grad.cpu().numpy(), g_ref[key], f"grad {key}"))
    print(f"isolated region ({supports} supports): forward {errs[0]:.2e}, worst gradient {max(errs[1:]):.2e} "
          f"(bar {TOL:.0e})")
    assert abs(loss.item() - l_ref) <= 1e-5 * max(1.0, abs(l_ref))
