"""NaN and +-Inf through every kernel and the model, against torch's IEEE semantics (fp64 references: plain torch,
``O.lstm_planes_reference``, ``O.dense_st_mgcn``; their ReLU is torch.relu, whose backward passes the gradient at NaN).

Each kernel test compares a run with one poisoned value with a clean run on the same inputs and with the reference:
* no masking: every entry the reference computes as non-finite is non-finite in the kernel's result;
* no leaks: a poisoned value is a tracer (0 * NaN = NaN), so a stale shared-memory read, a padding row or a tile mix-up
  that pulls it into another row shows up as NaN there.  Entries that do not depend on it equal the clean run's bit for
  bit, or within LEAK_TOL (max-norm relative) where atomics sum them in an order that changes from run to run (the
  fused pooling, d_s, the parameter gradients).  Two clean runs differ by as much: measured on an H100 80GB HBM3,
  the other windows' d_s of the tensor-core LSTM moved by up to 1.5e-6 between runs, so the bar is 5e-6.

Named deviations from the dense reference, each asserted by a test whose name carries it (include/stmgcn_b200.h):
* spmm_stored_entries_only: the SpMM multiplies stored entries only, so a NaN in X reaches the rows with a stored entry
  in its column, not every row as in a dense product (0 * NaN).  The model's mean pool and gate spread a NaN to its
  whole window in both, so model-level results agree.
* inf_through_split_operands: the 3xTF32 / 3xBF16 splits form lo = x - hi = Inf - Inf = NaN, so an Inf operand gives
  NaN where torch gives +-Inf; relu(-Inf) = 0 in torch is NaN there.  Still non-finite wherever torch's is.
* products_skipped_with_a_zero_initial_state: without h0 the tensor-core LSTM skips W_hh . 0 at t = 0, so a NaN W_hh
  leaves step 0 finite where torch's matmul gives NaN (with T = 1, the whole result).  The exact-fp32 LSTM forms the
  product and matches torch.
"""
import math

import numpy as np
import pytest
import torch
from torch import nn

import stmgcn_oracle as O
from helpers import DEV, FWD_TOL, GRAD_TOL
from kernel_cases import fuse_rows, isolated_matrix, proj_rows, tc_shape
from lstm_cases import HID, lstm16_inputs, wave_regions

pytestmark = pytest.mark.gpu
LEAK_TOL = 5e-6
NAN = math.nan


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _assert_same(a, b, what, tol=0.0):
    """a == b bit for bit (tol = 0) or within tol max-norm relative; both must be finite."""
    assert bool(torch.isfinite(a).all()), f"{what}: non-finite entries {int((~torch.isfinite(a)).sum())}"
    if tol == 0.0:
        assert torch.equal(_bits(a), _bits(b)), f"{what}: {int((_bits(a) != _bits(b)).sum())} entries differ from the clean run"
        return 0.0
    err = O.max_rel_err(a.double().cpu().numpy(), b.double().cpu().numpy())
    assert err <= tol, f"{what}: {err:.2e} from the clean run (bar {tol:.0e})"
    return err


def _assert_mask(got, ref, what):
    """isfinite(got) == isfinite(ref), reported as masked (reference non-finite, kernel finite) and spurious entries."""
    g, r = torch.isfinite(got).cpu(), torch.isfinite(ref).cpu()
    masked, spurious = int((g & ~r).sum()), int((~g & r).sum())
    assert masked == 0 and spurious == 0, f"{what}: {masked} masked, {spurious} spurious non-finite entries"


def _finite_err(got, ref):
    """max-norm relative error over the entries where the reference is finite."""
    keep = torch.isfinite(ref)
    if not bool(keep.any()):
        return 0.0
    return O.max_rel_err(got[keep].double().cpu().numpy(), ref[keep].double().cpu().numpy())


def _others(t, rows, dim=0):
    """t without the given indices along ``dim``."""
    keep = torch.ones(t.shape[dim], dtype=torch.bool, device=t.device)
    keep[list(rows)] = False
    return t.index_select(dim, keep.nonzero().flatten())


# ======================================================================================================================
# A. kernels
# ======================================================================================================================
def _proj_run(s, w, bias, act, d_out, tc):
    """ops._proj_fwd / ops._proj_bwd, with the dZ workspace returned: (out, dz, dW, db, U)."""
    from stmgcn_b200 import _lib, ops
    ks, n, b, p = s.shape
    q = w.shape[1]
    img_f, img_b = ops._proj_images(w, ks, p, True) if tc else (None, None)
    assert (img_f is not None) == tc
    out = ops._proj_fwd(s, w, bias, act, None, b, img_f)
    dw = torch.zeros_like(w)
    db = torch.zeros(q, device=DEV)
    dz = torch.empty((n * b, q), device=DEV)
    u = torch.empty_like(s)
    wt = w.t().contiguous()
    _lib.check(ops.L.stmgcn_proj_bwd(s.data_ptr(), n * b * p, ks, n * b, p, wt.data_ptr(), q, act, out.data_ptr(),
                                     d_out.data_ptr(), None, 1.0, b, dz.data_ptr(), dw.data_ptr(), db.data_ptr(),
                                     u.data_ptr(), n * b * p, ops._p(img_b), ops._stream()), "proj_bwd")
    torch.cuda.synchronize()
    return out.reshape(n * b, q), dz, dw, db, u.reshape(ks, n * b, p)


def _proj_reference(s, w, bias, relu, d_out, out_k):
    """fp64 torch: out = act(sum_k S_k W_k + b); dZ = torch's ReLU backward at the kernel's own output (out <= 0 -> 0,
    NaN passes), so a rounding-distance sign flip is not charged to the kernel."""
    ks, rows, p = s.shape
    s64, w64 = s.double(), w.double().reshape(ks, p, -1)
    z = torch.einsum("krp,kpq->rq", s64, w64) + (bias.double() if bias is not None else 0.0)
    out = torch.relu(z) if relu else z
    dz = d_out.double().masked_fill(out_k <= 0, 0.0) if relu else d_out.double()
    return out, dz, torch.einsum("krp,rq->kpq", s64, dz).reshape(ks * p, -1), dz.sum(0), torch.einsum("rq,kpq->krp", dz, w64)


# (path, ks, p, q, rows id): tc at every support count on a multi-wave ragged size; FFMA over the scalar (p, q % 4 != 0)
# and the vector tall GEMM with small_wgrad_kernel on both sides of its boundary
PROJ_CASES = ([("tc", ks, 64, 64, "waves") for ks in range(1, 9)] + [("tc", 3, 64, 64, 129)]
              + [("fma", 3, 7, 7, "waves"), ("fma", 2, 32, 20, "waves"), ("fma", 3, 24, 24, 513), ("fma", 4, 24, 24, 513)])


def _proj_case(path, ks, p, q, rows_id, seed):
    if path == "tc":
        n, b = tc_shape(rows_id)
    else:
        n, b = proj_rows(rows_id), 1
    gen = torch.Generator().manual_seed(seed)
    s = torch.randn(ks, n, b, p, generator=gen)
    s[:, 1::5] = 0.0                                 # rows whose stack is exactly zero
    w = torch.randn(ks * p, q, generator=gen) / p ** 0.5
    bias = torch.randn(q, generator=gen) * 0.3
    d_out = torch.randn(n * b, q, generator=gen)
    return s.to(DEV), w.to(DEV), bias.to(DEV), d_out.to(DEV)


def _proj_check(path, relu, s, w, bias, d_out, poisoned, what):
    """Run clean and poisoned; masks of every result against the fp64 reference of the poisoned inputs; finite entries
    within the bars.  Returns (clean, poisoned) results."""
    act = 1 if relu else 0
    clean = _proj_run(s, w, bias, act, d_out, path == "tc")
    bad = _proj_run(*poisoned, bias, act, d_out, path == "tc")
    ks, _, _, p = s.shape
    ref = _proj_reference(poisoned[0].reshape(ks, -1, p), poisoned[1], bias, relu, d_out, bad[0])
    errs = {}
    for name, got, r in zip(("out", "dZ", "dW", "db", "U"), bad, ref):
        _assert_mask(got, r, f"{what} {name}")
        errs[name] = _finite_err(got, r)
    print(f"{what}: " + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert errs["out"] <= FWD_TOL and max(v for k, v in errs.items() if k != "out") <= GRAD_TOL, errs
    return clean, bad


@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("path,ks,p,q,rows_id", PROJ_CASES)
def test_projection_nan_in_the_stack_stays_in_its_row(path, ks, p, q, rows_id, relu):
    """NaN in S[k, r, i]: out row r is NaN and every other row is the clean run's bit for bit; dZ and U differ from the
    clean run only in row r, where torch's mask passes d_out (relu(NaN) = NaN); exactly row k*p + i of dW is NaN."""
    s, w, bias, d_out = _proj_case(path, ks, p, q, rows_id, seed=17 * ks + p + relu)
    rows = s.shape[1] * s.shape[2]
    k, r, i = ks - 1, rows - 2, p // 2
    s_bad = s.clone()
    s_bad.view(ks, rows, p)[k, r, i] = NAN
    (out_c, dz_c, _, _, u_c), (out, dz, dw, db, u) = _proj_check(path, relu, s, w, bias, d_out, (s_bad, w),
                                                                 f"proj {path} ks={ks} p={p} q={q} rows={rows} relu={relu}")
    assert bool(torch.isnan(out[r]).all())
    _assert_same(_others(out, [r]), _others(out_c, [r]), "out, other rows")
    _assert_same(_others(dz, [r]), _others(dz_c, [r]), "dZ, other rows")
    assert torch.equal(dz[r], d_out[r]), "dZ row r: the NaN output did not pass d_out"
    _assert_same(_others(u, [r], 1), _others(u_c, [r], 1), "U, other rows")
    assert bool(torch.isfinite(u[:, r]).all() and torch.isfinite(db).all())
    assert bool(torch.isnan(dw[k * p + i]).all()) and bool(torch.isfinite(_others(dw, [k * p + i])).all())


@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("path,ks,p,q,rows_id", PROJ_CASES)
def test_projection_nan_in_a_weight_reaches_its_column_in_every_row(path, ks, p, q, rows_id, relu):
    """NaN in W[k*p + i, j]: column j of out is NaN in every row, also where S is exactly zero; the other columns are
    the clean run's bit for bit."""
    s, w, bias, d_out = _proj_case(path, ks, p, q, rows_id, seed=19 * ks + q + relu)
    k, i, j = ks // 2, p - 1, q // 3
    w_bad = w.clone()
    w_bad[k * p + i, j] = NAN
    (out_c, _, _, _, _), (out, _, _, _, _) = _proj_check(path, relu, s, w, bias, d_out, (s, w_bad),
                                                         f"proj W {path} ks={ks} p={p} q={q} relu={relu}")
    assert bool(torch.isnan(out[:, j]).all())
    _assert_same(_others(out, [j], 1), _others(out_c, [j], 1), "out, other columns")


@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("sign", [1.0, -1.0])
@pytest.mark.parametrize("path,ks,p,q,rows_id", [c for c in PROJ_CASES if c[0] == "fma"])
def test_projection_inf_in_the_stack_on_the_exact_path(path, ks, p, q, rows_id, sign, relu):
    """+-Inf in S[k, r, i] on the FFMA kernels: out, dZ, dW, db and U non-finite exactly where torch's are (relu(-Inf)
    = 0 and masks its gradient); the other rows of out the clean run's bit for bit."""
    s, w, bias, d_out = _proj_case(path, ks, p, q, rows_id, seed=23 * ks + p + relu)
    rows = s.shape[1]
    r, i = rows // 2, 0
    s_bad = s.clone()
    s_bad[0, r, 0, i] = sign * math.inf
    (out_c, _, _, _, _), (out, _, _, _, _) = _proj_check(path, relu, s, w, bias, d_out, (s_bad, w),
                                                         f"proj {sign:+.0f}Inf ks={ks} p={p} q={q} relu={relu}")
    _assert_same(_others(out, [r]), _others(out_c, [r]), "out, other rows")


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_projection_inf_through_split_operands(sign):
    """Deviation inf_through_split_operands: the tensor-core projection splits S into tf32 hi + lo, lo = Inf - Inf =
    NaN, so row r of out is NaN in every column, where torch has +-Inf (and relu(-Inf) = 0).  One-sided contract: every
    entry torch makes non-finite is non-finite; the other rows are the clean run's bit for bit."""
    s, w, bias, d_out = _proj_case("tc", 2, 64, 64, 129, seed=29)
    r = 77
    s_bad = s.clone()
    s_bad.view(2, -1, 64)[1, r, 5] = sign * math.inf
    out_c = _proj_run(s, w, bias, 1, d_out, True)[0]
    out = _proj_run(s_bad, w, bias, 1, d_out, True)[0]
    ref = _proj_reference(s_bad.view(2, -1, 64), w, bias, True, d_out, out)[0]
    assert bool(torch.isnan(out[r]).all())
    assert not bool((~torch.isfinite(ref.cpu()) & torch.isfinite(out.cpu())).any())
    assert bool(torch.isfinite(ref[r]).any()), "torch's row has finite entries (relu(-Inf) = 0): nothing deviates"
    _assert_same(_others(out, [r]), _others(out_c, [r]), "out, other rows")


# ---- LSTM -------------------------------------------------------------------------------------------------------------
def _lstm_run(family, xo, s, h0, c0, ws, lyr, d_top):
    """Forward and backward of one family: 'tc1' / 'tc2' (lstm16.cu, one / two planes), 'fma' (lstm.cu).  Returns a
    dict of per-row results (rows along dim 0 after the leading dims named in ROW_DIM) and the weight gradients."""
    from stmgcn_b200 import ops
    n, b, t, c = xo.shape
    rows = n * b
    state = h0 is not None
    want = (True, state, state)
    if family == "fma":
        h_top, h_n, c_n, tape = ops._exact_forward(xo, s, h0, c0, lyr, HID, True, ws, True)
        res = dict(h=tape[2].clone(), c=tape[3].clone(), h_top=h_top.reshape(rows, HID).clone(), h_n=h_n.clone(),
                   c_n=c_n.clone())
        d_s, grads, (d_xo, dh0, dc0) = ops._exact_backward_ex(xo, s, tape, lyr, HID, d_top, want=want)
    else:
        planes = int(family[2])
        h_top, h_n, c_n, tape = ops._lstm16_forward(xo, s, h0, c0, lyr, True, ws, planes, True)
        res = dict(h=tape["hp"].transpose(2, 3).clone(), c=ops.from_blocked(tape["cs"], rows),
                   h_top=h_top.reshape(rows, HID).clone(), h_n=h_n.clone(), c_n=c_n.clone())
        d_s, grads, (d_xo, dh0, dc0) = ops._lstm16_backward_ex(xo, s, tape, lyr, planes, d_top, want=want)
    torch.cuda.synchronize()
    res["d_xo"] = d_xo.reshape(rows, t, c)
    if state:
        res["dh0"], res["dc0"] = dh0, dc0
    return res, d_s, grads


# the dimension of each result that indexes rows: h, c: (L, T, R, ...); h_n, c_n, dh0, dc0: (L, R, H)
ROW_DIM = dict(h=2, c=2, h_top=0, h_n=1, c_n=1, d_xo=0, dh0=1, dc0=1)


def _lstm_row_reference(family, xo, s, h0, c0, ws, lyr, d_top, r):
    """fp64 reference of row r alone (rows of the LSTM are independent): its tape, d_xo, dh0, dc0, its window's d_s
    and its contribution to the weight gradients.  The kernels sum finite contributions of the other rows to those,
    so the full results are non-finite exactly where these are."""
    b = s.shape[0]
    t, c = xo.shape[2], xo.shape[3]
    planes = 1 if family == "tc1" else 2
    x64 = xo.reshape(-1, t, c)[r:r + 1].double().requires_grad_(True)
    s64 = s.double().requires_grad_(True)
    layers = [tuple(w.double().requires_grad_(True) for w in ws[4 * l:4 * l + 4]) for l in range(lyr)]
    st = [None if v is None else v[:, r:r + 1].double().requires_grad_(True) for v in (h0, c0)]
    _, _, (hs, cs) = O.lstm_planes_reference(x64 * s64[r % b][None, :, None], layers, planes, st[0], st[1])
    leaves = [x64, s64] + [w for layer in layers for w in layer] + [v for v in st if v is not None]
    grads = torch.autograd.grad((hs[-1][-1] * d_top[r].double()).sum(), leaves, allow_unused=True)
    ref = dict(h=torch.stack([torch.stack(v) for v in hs])[:, :, 0], c=torch.stack([torch.stack(v) for v in cs])[:, :, 0],
               d_xo=grads[0][0], d_s=grads[1], w=grads[2:2 + 4 * lyr])
    if st[0] is not None:
        ref["dh0"], ref["dc0"] = grads[-2][:, 0], grads[-1][:, 0]
    return ref


def _lstm_poison_check(family, inputs, poisoned, lyr, r, what, row_local=True, tape_from=0):
    """Clean and poisoned runs, and the row-r reference of the poisoned inputs.  Row r's tape, d_xo, dh0, dc0, the
    window's d_s and the weight gradients: non-finite exactly where the reference's are.  ``row_local``: every other
    row's tape, h_top, h_n, c_n, d_xo, dh0 and dc0 are the clean run's bit for bit, the other windows' d_s within
    LEAK_TOL.  ``tape_from``: compare the tape masks from that step on.  Returns (clean results, poisoned results,
    reference)."""
    xo, s, h0, c0, ws, d_top = inputs
    b = s.shape[0]
    clean, d_s_c, _ = _lstm_run(family, xo, s, h0, c0, ws, lyr, d_top)
    bad, d_s, grads = _lstm_run(family, *poisoned, lyr, d_top)
    ref = _lstm_row_reference(family, *poisoned, lyr, d_top, r)
    h_r = bad["h"].select(2, r).float()
    if family != "fma":
        h_r = h_r.sum(2)                                             # planes summed: NaN if either plane is
    _assert_mask(h_r[:, tape_from:], ref["h"][:, tape_from:], f"{what}: h of row r")
    _assert_mask(bad["c"].select(2, r)[:, tape_from:], ref["c"][:, tape_from:], f"{what}: c of row r")
    _assert_mask(bad["d_xo"][r], ref["d_xo"], f"{what}: d_xo of row r")
    for key in ("dh0", "dc0"):
        if key in ref:
            _assert_mask(bad[key].select(1, r), ref[key], f"{what}: {key} of row r")
    _assert_mask(d_s[r % b], ref["d_s"][r % b], f"{what}: d_s of row r's window")
    for i, (g, rg) in enumerate(zip(grads, ref["w"])):
        _assert_mask(g, rg, f"{what}: weight gradient {i}")
    if row_local:
        for key, dim in ROW_DIM.items():
            if key in bad:
                _assert_same(_others(bad[key], [r], dim), _others(clean[key], [r], dim), f"{what}: {key}, other rows")
        err = _assert_same(_others(d_s, [r % b]), _others(d_s_c, [r % b]), f"{what}: d_s, other windows", LEAK_TOL)
        print(f"{what}: other windows' d_s {err:.1e} from the clean run")
    return clean, bad, ref


FAMILIES = ["tc1", "tc2", "fma"]


def _family_setup(monkeypatch, family):
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_LSTM_PATH", "fma" if family == "fma" else "tc")


def _position(rows, where):
    """'last_tile': a row of the last, partial 128-row tile; 'second_warpgroup': row 64 + 37 of a middle tile."""
    if where == "last_tile":
        return rows - 1 - (rows % 128) // 3
    return 128 * ((rows // 128) // 2) + 64 + 37


@pytest.mark.parametrize("where", ["last_tile", "second_warpgroup"])
@pytest.mark.parametrize("c,state", [(1, False), (3, True)])
@pytest.mark.parametrize("family", FAMILIES)
def test_lstm_nan_in_one_input_row_stays_in_that_row(family, c, state, where, monkeypatch):
    """NaN in xo[r, t = 5] (one channel): h and c of row r are NaN from step 5 on in every layer and finite before;
    every other row's tape, h_top, h_n, c_n, d_xo, dh0 and dc0 are the clean run's bit for bit; d_s is non-finite
    exactly in row r's window; the weight gradients are non-finite where the fp64 reference's are.  Multi-wave ragged
    size (several 128-row tiles per CTA), 3 layers, T = 12."""
    _family_setup(monkeypatch, family)
    b, t, lyr = 37, 12, 3
    n = wave_regions(b)
    inputs = lstm16_inputs(n, b, t, lyr, c, state, seed=7 * c + state)
    rows = n * b
    r = _position(rows, where)
    xo_bad = inputs[0].clone()
    xo_bad.view(rows, t, c)[r, 5, c - 1] = NAN
    what = f"lstm {family} C={c} state={state} r={r} of {rows}"
    _, bad, ref = _lstm_poison_check(family, inputs, (xo_bad,) + inputs[1:5], lyr, r, what)
    assert bool(torch.isfinite(ref["h"][:, :5]).all()) and bool(torch.isnan(ref["h"][:, 5:]).all())
    assert bool(torch.isnan(bad["c"][:, 5:, r]).all()) and bool(torch.isfinite(bad["c"][:, :5, r]).all())
    assert not bool(torch.isfinite(bad["h_top"][r]).any())


@pytest.mark.parametrize("which,layer", [("h0", 0), ("c0", 1)])
@pytest.mark.parametrize("family", FAMILIES)
def test_lstm_nan_in_one_initial_state_row_stays_in_that_row(family, which, layer, monkeypatch):
    """NaN in one entry of h0[layer, r] or c0[layer, r]: row r of that layer and the layers above is NaN from step 1 on;
    the layers below and every other row are the clean run's bit for bit."""
    _family_setup(monkeypatch, family)
    b, t, lyr = 64, 6, 3
    n = wave_regions(b)
    inputs = lstm16_inputs(n, b, t, lyr, 2, True, seed=11 + layer)
    r = _position(n * b, "second_warpgroup")
    h0, c0 = inputs[2].clone(), inputs[3].clone()
    (h0 if which == "h0" else c0)[layer, r, 9] = NAN
    _, bad, _ = _lstm_poison_check(family, inputs, inputs[:2] + (h0, c0, inputs[4]), lyr, r,
                                   f"lstm {family} NaN {which}[{layer}]")
    assert bool(torch.isnan(bad["c"][layer:, 1:, r]).all()) and bool(torch.isfinite(bad["c"][:layer, :, r]).all())


@pytest.mark.parametrize("state", [False, True])
@pytest.mark.parametrize("family", FAMILIES)
def test_lstm_nan_in_a_recurrent_weight_reaches_every_row(family, state, monkeypatch):
    """NaN in one W_hh entry of layer 1: every row of layers 1 and 2 is NaN from step 2 on (step 1 with an initial
    state); layer 0 is the clean run's bit for bit; every row's results are non-finite where the fp64 reference's are
    (checked on two rows).  The tensor-core tape without an initial state is compared from step 2: at step 0 those
    kernels skip W_hh . 0 (products_skipped_with_a_zero_initial_state), which delays the NaN by one step."""
    _family_setup(monkeypatch, family)
    b, t, lyr = 40, 7, 3
    n = 9
    inputs = lstm16_inputs(n, b, t, lyr, 1, state, seed=13 + state)
    ws = [w.clone() for w in inputs[4]]
    ws[5][2 * HID + 3, 17] = NAN                     # layer 1, W_hh: the g gate of unit 3, from h unit 17
    clean = None
    for r in (0, n * b - 1):
        clean, bad, ref = _lstm_poison_check(family, inputs, inputs[:4] + (ws,), lyr, r, f"lstm {family} W_hh",
                                             row_local=False, tape_from=2 if family != "fma" and not state else 0)
    assert bool(torch.isnan(bad["c"][1:, (1 if state else 2):]).all())
    _assert_same(bad["h"][0], clean["h"][0], "layer 0 tape h")
    _assert_same(bad["c"][0], clean["c"][0], "layer 0 tape c")


@pytest.mark.parametrize("family", FAMILIES)
def test_lstm_products_skipped_with_a_zero_initial_state(family, monkeypatch):
    """Deviation products_skipped_with_a_zero_initial_state: with T = 1 and no h0 the tensor-core kernels never form
    W_hh . 0, so a NaN W_hh leaves h_top finite where torch's matmul (0 * NaN) makes it NaN; the exact-fp32 kernels
    form the product and give NaN as torch does.  With an h0 of zeros every family gives NaN."""
    _family_setup(monkeypatch, family)
    b, t, lyr = 40, 1, 2
    xo, s, _, _, ws, d_top = lstm16_inputs(3, b, t, lyr, 1, False, seed=3)
    ws = [w.clone() for w in ws]
    ws[1][7, 7] = NAN                                # layer 0 W_hh
    res, _, _ = _lstm_run(family, xo, s, None, None, ws, lyr, d_top)
    ref = _lstm_row_reference(family, xo, s, None, None, ws, lyr, d_top, 0)
    assert not bool(torch.isfinite(ref["h"][-1, -1]).any())
    if family == "fma":
        _assert_mask(res["h_top"][0], ref["h"][-1, -1], "exact h_top")
    else:
        assert bool(torch.isfinite(res["h_top"]).all())
    zeros = xo.new_zeros(lyr, 3 * b, HID)
    res0, _, _ = _lstm_run(family, xo, s, zeros, zeros.clone(), ws, lyr, d_top)
    assert not bool(torch.isfinite(res0["h_top"]).any())


@pytest.mark.parametrize("family", ["tc1", "tc2"])
def test_lstm16_saturated_gates_keep_their_cap_and_trace_nan(family, monkeypatch):
    """The saturated inputs of test_gpu_lstm16 (pre-activations to +-70, capped exponentials): the clean run is finite
    with c beyond 15 (the NaN-keeping cap saturates as before), and a NaN in xo[r, 3] stays in row r."""
    _family_setup(monkeypatch, family)
    n, b, t, lyr, c = 5, 40, 20, 3, 1
    inputs = lstm16_inputs(n, b, t, lyr, c, True, seed=70, saturate=True)
    r = 150
    xo_bad = inputs[0].clone()
    xo_bad.view(n * b, t, c)[r, 3, 0] = NAN
    clean, _, _ = _lstm_poison_check(family, inputs, (xo_bad,) + inputs[1:5], lyr, r, f"lstm {family} saturated")
    assert all(bool(torch.isfinite(v).all()) for v in clean.values())
    assert float(clean["c"].abs().max()) > 15.0


# ---- gate, FuseOut, SpMM ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t", [12, 300])
def test_context_gate_nan_in_one_window(t):
    """NaN in pool[b, j]: s[b, :] is all NaN, the other windows' s and d_pool are the clean run's bit for bit; d_pool,
    d_fcw and d_fcb are non-finite exactly where fp64 torch's are (relu(NaN) = NaN, its backward passes)."""
    from stmgcn_b200 import ops
    b, n_regions = 64, 50
    gen = torch.Generator().manual_seed(t)
    pool = torch.randn(b, t, generator=gen) * n_regions
    fcw = torch.randn(t, t, generator=gen) / t ** 0.5
    fcb = torch.rand(t, generator=gen) - 0.5
    d_s = torch.randn(b, t, generator=gen).to(DEV)
    bad = pool.clone()
    bad[17, t // 2] = NAN
    res = []
    for p in (pool, bad):
        leaves = [v.to(DEV).requires_grad_(True) for v in (p, fcw, fcb)]
        s = ops.ContextGate.apply(*leaves, n_regions)
        (s * d_s).sum().backward()
        res.append((s.detach(),) + tuple(v.grad for v in leaves))
    torch.cuda.synchronize()
    (s_c, dp_c, _, dfb_c), (s, dp, dfw, dfb) = res
    leaves = [v.double().to(DEV).requires_grad_(True) for v in (bad, fcw, fcb)]
    ref_s = torch.sigmoid(torch.relu((leaves[0] / n_regions) @ leaves[1].t() + leaves[2]) @ leaves[1].t() + leaves[2])
    ref_g = torch.autograd.grad((ref_s * d_s.double()).sum(), leaves)
    for name, got, ref in zip(("s", "d_pool", "d_fcw", "d_fcb"), (s, dp, dfw, dfb), (ref_s,) + ref_g):
        _assert_mask(got, ref, f"gate T={t} {name}")
    assert bool(torch.isnan(s[17]).all())
    _assert_same(_others(s, [17]), _others(s_c, [17]), "s, other windows")
    _assert_same(_others(dp, [17]), _others(dp_c, [17]), "d_pool, other windows")


def test_fuse_out_nan_in_one_feature():
    """NaN in g_1[r, g]: output row r is NaN in every channel, the other rows are the clean run's bit for bit; only
    column g of d_fcw is NaN; d_g (which does not read the features) is the clean run's bit for bit and d_fcb within
    LEAK_TOL (atomics)."""
    from stmgcn_b200 import ops
    n, b = fuse_rows("waves")
    m, gdim, c_out = 3, 64, 2
    gen = torch.Generator().manual_seed(5)
    gs = [torch.randn(n, b, gdim, generator=gen).to(DEV) for _ in range(m)]
    fcw = (torch.randn(c_out, gdim, generator=gen) / 8).to(DEV)
    fcb = torch.randn(c_out, generator=gen).to(DEV)
    d_y = torch.randn(b, n, c_out, generator=gen).to(DEV)
    rn, rb, g = n - 2, 1, 40
    res = []
    for poison in (False, True):
        leaves = [fcw.clone().requires_grad_(True), fcb.clone().requires_grad_(True)]
        feats = [v.clone() for v in gs]
        if poison:
            feats[1][rn, rb, g] = NAN
        feats = [v.requires_grad_(True) for v in feats]
        y = ops.FuseOut.apply(*leaves, *feats)
        (y * d_y).sum().backward()
        res.append((y.detach(), leaves[0].grad, leaves[1].grad, feats[1].grad))
    torch.cuda.synchronize()
    (y_c, dw_c, db_c, dg_c), (y, dw, db, dg) = res
    assert bool(torch.isnan(y[rb, rn]).all())
    y_rows, yc_rows = y.reshape(b * n, c_out), y_c.reshape(b * n, c_out)
    _assert_same(_others(y_rows, [rb * n + rn]), _others(yc_rows, [rb * n + rn]), "y, other rows")
    assert bool(torch.isnan(dw[:, g]).all())
    _assert_same(_others(dw, [g], 1), _others(dw_c, [g], 1), "d_fcw, other columns", LEAK_TOL)
    err = _assert_same(db, db_c, "d_fcb", LEAK_TOL)
    _assert_same(dg, dg_c, "d_g")
    print(f"fuse_out rows={n * b}: d_fcb {err:.1e} from the clean run")


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("kernel", ["fp32_f7", "fp32_f40", "bf16_f40"])
def test_spmm_stored_entries_only(kernel, transpose):
    """Y = 2 op(A) X - Z + 0.5 U on a 300-region graph with empty rows and columns.  NaN in X[j, f] reaches exactly
    Y[i, f] for the stored entries op(A)[i, j]; NaN in one stored value of op(A) reaches all of row i; everything else
    is the clean run's bit for bit.  Deviation spmm_stored_entries_only: the dense fp64 product makes the whole column
    f NaN (0 * NaN), the kernel only the rows with a stored entry in column j."""
    from stmgcn_b200 import ops
    from stmgcn_b200.graph import GraphHandle
    n, f = 300, (7 if kernel == "fp32_f7" else 40)
    a = isolated_matrix(n, seed=41)
    op = torch.from_numpy(a.T.copy() if transpose else a)
    gen = torch.Generator().manual_seed(42)
    x, z, u = (torch.randn(n, f, generator=gen).to(DEV) for _ in range(3))

    def run(mat, xv):
        g = GraphHandle.from_dense(mat.to(DEV))
        y = torch.empty_like(xv)
        if kernel == "bf16_f40":
            ops.spmm_step16(g, transpose, 2.0, ops.to_bf16(xv), -1.0, z, 0.5, u, y, None)
        else:
            ops.spmm_step(g, transpose, 2.0, xv, -1.0, z, 0.5, u, y)
        torch.cuda.synchronize()
        return y

    y_c = run(torch.from_numpy(a), x)
    j = int(np.argmax((op != 0).sum(0).numpy()))            # the column of op(A) with the most stored entries
    fi = f - 1
    x_bad = x.clone()
    x_bad[j, fi] = NAN
    y = run(torch.from_numpy(a), x_bad)
    hit = (op[:, j] != 0).to(DEV)
    want = torch.zeros_like(y, dtype=torch.bool)
    want[hit, fi] = True
    assert torch.equal(~torch.isfinite(y), want), "NaN in X: non-finite entries are not exactly the stored column"
    assert torch.equal(_bits(y[~want]), _bits(y_c[~want]))
    dense = 2.0 * (op.double().to(DEV) @ x_bad.double()) - z.double() + 0.5 * u.double()
    assert bool(torch.isnan(dense[:, fi]).all()) and int(hit.sum()) < n, "the dense product does not deviate here"
    # NaN in the stored value op(A)[i, j2]
    i = int(np.argmax((op != 0).sum(1).numpy()))
    j2 = int(np.flatnonzero(op[i].numpy())[0])
    a_bad = a.copy()
    a_bad[(j2, i) if transpose else (i, j2)] = NAN
    y = run(torch.from_numpy(a_bad), x)
    assert bool(torch.isnan(y[i]).all())
    _assert_same(_others(y, [i]), _others(y_c, [i]), "Y, other rows")


# ======================================================================================================================
# B. the model
# ======================================================================================================================
PATHS = [("tc", 2), ("tc", 1), ("fma", 2)]
PATH_IDS = ["tc2", "tc1", "fma"]


def _path(monkeypatch, path):
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_LSTM_PATH", path[0])
    monkeypatch.setattr(ops, "_PLANES", path[1])


def _model_setup(m=2, c=1, n=60, seed=5):
    from helpers import build_model
    from stmgcn_b200 import synth
    shape = dict(n=n, m=m, k=2, t=6, b=3, c=c, hid=64, layers=2, gcn_hid=64)
    adjs = [synth.make_adjacency(n, g, 0.08) for g in range(m)]
    params = O.init_params(m, shape["t"], c, 64, 2, 64, shape["k"] + 1, seed=seed)
    model = build_model(shape, DEV)
    model.load_state_dict(params)
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(shape["b"], shape["t"], n, c, generator=gen)
    y = torch.randn(shape["b"], n, c, generator=gen)
    return shape, adjs, params, model, x, y


def _model_run(model, x, y, sups, obs_grad=False):
    for p in model.parameters():
        p.grad = None
    xd = x.to(DEV).requires_grad_(obs_grad)
    out = model(obs_seq=xd, sta_adj_list=sups)
    loss = nn.MSELoss()(out, y.to(DEV))
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    return out.detach(), loss.detach(), grads, (xd.grad if obs_grad else None)


def _oracle(params, x, y, sups, obs_grad=False):
    """fp64 dense oracle: (out, loss, parameter gradients, d obs)."""
    leaves = {k: v.detach().double().cpu().clone().requires_grad_(True) for k, v in params.items()}
    xd = x.double().cpu().requires_grad_(obs_grad)
    out = O.dense_st_mgcn(leaves, xd, [s.double().cpu() for s in sups])
    loss = torch.mean((out - y.double().cpu()) ** 2)
    grads = torch.autograd.grad(loss, list(leaves.values()) + ([xd] if obs_grad else []))
    return out.detach(), loss.detach(), dict(zip(leaves.keys(), grads)), (grads[-1] if obs_grad else None)


@pytest.mark.parametrize("path", PATHS, ids=PATH_IDS)
def test_model_loss_is_nan_on_process_supports_with_an_isolated_region(path, monkeypatch):
    """test_model_with_an_isolated_region_matches_sparse_oracle's graph, with the supports of Adj_Preprocessor.process
    (NaN row and column on the isolated region, as the reference's symmetric_normalize makes them) at H = G = 64: the
    loss is NaN and the output non-finite where the dense oracle's is.  Before ReLU propagated NaN, the spatial and
    temporal GCNs turned the NaN into 0 and the loss was finite."""
    import GCN
    _path(monkeypatch, path)
    shape, adjs, params, model, x, y = _model_setup()
    iso = 17
    adjs[0][iso, :] = 0.0
    adjs[0][:, iso] = 0.0
    adjs[0][iso - 1, iso + 1] = adjs[0][iso + 1, iso - 1] = 1.0
    sups = [GCN.Adj_Preprocessor("chebyshev", shape["k"]).process(a) for a in adjs]
    assert bool(torch.isnan(sups[0]).any())
    out, loss, _, _ = _model_run(model, x, y, [s.to(DEV) for s in sups])
    o_ref, l_ref, _, _ = _oracle(params, x, y, sups)
    assert math.isnan(float(l_ref))
    assert math.isnan(float(loss)), f"loss {float(loss)} is finite where the reference's is NaN"
    _assert_mask(out, o_ref, "output")


@pytest.mark.parametrize("path", PATHS, ids=PATH_IDS)
def test_model_nan_in_one_window_stays_in_that_window(path, monkeypatch):
    """NaN in obs[1, 2, 5, 0] with obs.requires_grad: window 1's outputs and obs gradient are non-finite where the dense
    oracle's are; the other windows' outputs and obs gradient equal the clean run's within LEAK_TOL (the fused pooling
    and d_s are sums of atomics); every parameter gradient's isfinite mask equals the oracle's."""
    _path(monkeypatch, path)
    shape, adjs, params, model, x, y = _model_setup()
    sups = [O.chebyshev_supports_dense(a, shape["k"]) for a in adjs]
    sups_d = [s.to(DEV) for s in sups]
    out_c, _, _, dx_c = _model_run(model, x, y, sups_d, obs_grad=True)
    x_bad = x.clone()
    x_bad[1, 2, 5, 0] = NAN
    out, loss, grads, dx = _model_run(model, x_bad, y, sups_d, obs_grad=True)
    o_ref, _, g_ref, dx_ref = _oracle(params, x_bad, y, sups, obs_grad=True)
    assert math.isnan(float(loss))
    _assert_mask(out, o_ref, "output")
    _assert_mask(dx, dx_ref, "obs gradient")
    assert not bool(torch.isfinite(out[1]).any())
    e_out = _assert_same(out[[0, 2]], out_c[[0, 2]], "output, other windows", LEAK_TOL)
    e_dx = _assert_same(dx[[0, 2]], dx_c[[0, 2]], "obs gradient, other windows", LEAK_TOL)
    for key, g in grads.items():
        _assert_mask(g, g_ref[key], f"grad {key}")
    print(f"model {path}: other windows from the clean run: output {e_out:.1e}, obs gradient {e_dx:.1e}")


@pytest.mark.parametrize("name", list(O.init_params(1, 6, 2, 64, 2, 64, 3)))
@pytest.mark.parametrize("path", PATHS, ids=PATH_IDS)
def test_model_nan_in_each_parameter(path, name, monkeypatch):
    """NaN in the middle entry of one parameter tensor, C = 2: the isfinite masks of the output and of every parameter
    gradient equal the dense oracle's (fc gives a per-channel pattern: a NaN fc.bias[c] or fc.weight[c, g] leaves the
    other channel finite)."""
    _path(monkeypatch, path)
    shape, adjs, params, model, x, y = _model_setup(m=1, c=2, n=40)
    sups = [O.chebyshev_supports_dense(a, shape["k"]) for a in adjs]
    params = {k: v.clone() for k, v in params.items()}
    params[name].view(-1)[params[name].numel() // 2] = NAN
    model.load_state_dict(params)
    out, _, grads, _ = _model_run(model, x, y, [s.to(DEV) for s in sups])
    o_ref, _, g_ref, _ = _oracle(params, x, y, sups)
    assert not bool(torch.isfinite(o_ref).all())
    _assert_mask(out, o_ref, f"NaN {name}: output")
    for key, g in grads.items():
        _assert_mask(g, g_ref[key], f"NaN {name}: grad {key}")


def test_graphed_step_recovers_after_a_poisoned_batch():
    """A CUDA-graph replay on a batch with a NaN returns a NaN loss; a clean batch replayed afterwards gives the loss and
    output of the clean replay before it within LEAK_TOL and its gradients within 2e-5, the bar test_gpu_graphs.py holds
    replays to (weight_ih_l0's gradient, a sum with cancellation over every row and step, moved by 1.2e-6 and 2.2e-6
    between two clean replays on an H100): nothing of the NaN stays in the workspaces or the weight images."""
    from stmgcn_b200 import graphs
    shape, adjs, _, model, x, y = _model_setup(m=3)
    sups = [O.chebyshev_supports_dense(a, shape["k"]).to(DEV) for a in adjs]
    xd, yd = x.to(DEV), y.to(DEV)
    gstep = graphs.GraphedStep(model, nn.MSELoss(), xd, yd, sups)

    def replay(xv):
        loss = float(gstep(xv, yd).detach())
        return loss, gstep.out.clone(), {k: p.grad.detach().clone() for k, p in model.named_parameters()}

    l0, out0, g0 = replay(xd)
    x_bad = xd.clone()
    x_bad[2, 4, 11, 0] = NAN
    l_bad, out_bad, _ = replay(x_bad)
    assert math.isnan(l_bad) and not bool(torch.isfinite(out_bad[2]).any())
    l1, out1, g1 = replay(xd)
    assert abs(l1 - l0) <= LEAK_TOL * abs(l0), (l1, l0)
    errs = [_assert_same(out1, out0, "output after the poisoned replay", LEAK_TOL)]
    errs += [_assert_same(g1[k], g0[k], f"grad {k} after the poisoned replay", 2e-5) for k in g0]
    print(f"graphed step after a poisoned replay: worst {max(errs):.1e} from the clean replay")


# ======================================================================================================================
# C. large finite magnitudes
# ======================================================================================================================
@pytest.mark.parametrize("path", [("tc", 2), ("fma", 2)], ids=["tc2", "fma"])
def test_model_on_raw_counts_matches_the_sparse_oracle(path, monkeypatch):
    """Non-negative integer counts up to 3000 (the reference's Data_Container without norm_opt), forward and every
    gradient against the fp64 sparse oracle at 1e-4.  The two weights that read the counts directly, the gate's fc and
    layer 0's W_ih, are scaled by 1e-3, as training on counts would make them: at unit scale both saturate, and fp32
    sigmoid' = s (1 - s) has no digits left there (0 where fp64 has e^-20)."""
    from helpers import TOL, assert_close
    _path(monkeypatch, path)
    shape, adjs, params, model, _, _ = _model_setup(seed=8)
    for m in range(shape["m"]):
        params[f"rnn_list.{m}.fc.weight"] *= 1e-3
        params[f"rnn_list.{m}.lstm.weight_ih_l0"] *= 1e-3
    model.load_state_dict(params)
    gen = torch.Generator().manual_seed(8)
    x = torch.randint(0, 3001, (shape["b"], shape["t"], shape["n"], 1), generator=gen).float()
    y = torch.randint(0, 3001, (shape["b"], shape["n"], 1), generator=gen).float()
    sups = [O.chebyshev_supports_dense(a, shape["k"]) for a in adjs]
    out, loss, grads, _ = _model_run(model, x, y, [s.to(DEV) for s in sups])
    orc = O.SparseOracle({k: v.numpy() for k, v in params.items()}, [O.laplacian_csr_from_supports(s) for s in sups],
                         shape["k"] + 1, dtype=np.float64)
    o_ref, l_ref, g_ref = orc.loss_and_grads(x.numpy(), y.numpy())
    errs = {"out": assert_close(out.cpu().numpy(), o_ref, "forward")}
    for key, g in grads.items():
        errs[key] = assert_close(g.cpu().numpy(), g_ref[key], f"grad {key}")
    print(f"raw counts {path}: forward {errs['out']:.2e}, worst gradient "
          f"{max(v for k, v in errs.items() if k != 'out'):.2e} (bar {TOL:.0e}); loss {float(loss):.6e} vs {l_ref:.6e}")
    assert abs(float(loss) - l_ref) <= TOL * abs(l_ref)


@pytest.mark.parametrize("scale", [1e6, 1e30])
@pytest.mark.parametrize("path", PATHS, ids=PATH_IDS)
def test_model_at_huge_obs_scales_is_finite_where_fp32_torch_is(path, scale, monkeypatch):
    """obs = |N(0, 1)| * scale: the output and every parameter gradient are finite exactly where the fp32 dense oracle's
    are (no overflow the reference does not have, no NaN from Inf - Inf or 0 * Inf)."""
    _path(monkeypatch, path)
    shape, adjs, params, model, x, y = _model_setup(seed=9)
    x = x.abs() * scale
    sups = [O.chebyshev_supports_dense(a, shape["k"]) for a in adjs]
    out, _, grads, _ = _model_run(model, x, y, [s.to(DEV) for s in sups])
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    o_ref = O.dense_st_mgcn(leaves, x, [s.float() for s in sups])
    g_ref = dict(zip(leaves, torch.autograd.grad(torch.mean((o_ref - y) ** 2), list(leaves.values()))))
    _assert_mask(out, o_ref, f"scale {scale:.0e}: output")
    for key, g in grads.items():
        _assert_mask(g, g_ref[key], f"scale {scale:.0e}: grad {key}")
