"""Gradients at the model's inputs and recurrent state on the GPU: d obs_seq, d h0 / d c0 and the seeds d h_n / d c_n.

Kernel level: stmgcn_lstm16_bwd_ex (tensor cores) and stmgcn_lstm_bwd_ex (exact fp32) against the fp64 reference of
their arithmetic forced with the kernel's own tape, as in test_gpu_lstm16.py / test_gpu_exact_kernels.py, with the loss
<h_top, d_top> + <h_n, dh_n> + <c_n, dc_n>; the new entry points with every extra NULL against the old ones; the memory
contract of test_gpu_abi_contract.py for every new entry point.  Module level: the drop-in modules against the
reference's own gradients (tests/golden/inputgrad_ref.npz) and the dense fp64 oracle, and d obs at cfg3 size.
"""
import numpy as np
import pytest
import torch
from torch import nn

import stmgcn_oracle as O
from abi_harness import Buf, bits, drive, lstm16_ex_calls, lstm_ex_calls, obs_grad_calls, run_captured, run_contract
from helpers import DEV, GOLDEN, GRAD_TOL, TOL, lib, rel_err
from lstm_cases import (CASES, EXACT_CASES, HID, exact_run, grad_errors, lstm16_inputs, lstm16_run, lstm_inputs, seeds,
                        state_gradients, wave_regions)
from model_cases import CHUNK, cheb_workload, dense_grads, forced_errors, gpu_run, small_model

pytestmark = pytest.mark.gpu


# ======================================================================================================================
# tensor-core kernels
# ======================================================================================================================
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_tensor_core_input_and_state_gradients(case, planes):
    """d_xo, dh0, dc0 (also at a zero initial state: dh0 without h0), d_s and every weight gradient of the seeded loss
    against the tape-forced fp64 reference.  Negative control: the same backward without the seeds lands outside the
    bar.

    One exception to the 5e-5 bar: the weight gradients of the saturated case with two planes, held to 2e-4.  There the
    seeds reach every layer's saturated gates, and the layer-1 bias gradient, a sum of tiny cancelling terms, came out
    1.8e-4 off (measured on an H100); its d_xo / dh0 / dc0 / d_s were within 5e-6.  The two-plane reference multiplies
    exactly while the kernel's three bf16 passes keep ~16 bits of each product (see test_gpu_lstm16's saturated case);
    with one plane, whose reference rounds like the kernel, the same case holds 5e-5."""
    name, n, b, t, lyr, c, state = case
    if n is None:
        n = wave_regions(b)
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n, b, t, lyr, c, state, seed=10 * CASES.index(case) + planes + 500,
                                       saturate=name == "saturated")
    dh_n, dc_n = seeds(lyr, n * b, HID, seed=CASES.index(case))
    got, ktape, _ = lstm16_run(xo, s, h0, c0, ws, lyr, planes, d_top, dh_n, dc_n)
    ref = state_gradients(xo, s, h0, c0, ws, lyr, planes, ktape, d_top, dh_n, dc_n)
    errs = grad_errors(got, ref)
    unseeded, _, _ = lstm16_run(xo, s, h0, c0, ws, lyr, planes, d_top, None, None)
    control = max(grad_errors(unseeded, ref).values())
    print(f"lstm16 extras {name} P={planes}: worst {max(errs.values()):.2e} ({max(errs, key=errs.get)}), "
          f"d_xo {errs['d_xo']:.2e} dh0 {errs['dh0']:.2e} dc0 {errs['dc0']:.2e}; control (no seeds) {control:.2e}")
    w_bar = 2e-4 if (name == "saturated" and planes == 2) else GRAD_TOL
    assert max(errs[k] for k in ("d_xo", "d_s", "dh0", "dc0")) <= GRAD_TOL, errs
    assert max(v for k, v in errs.items() if k.startswith("param")) <= w_bar, errs
    assert control > w_bar, f"dropping the seeds stays within the bar ({control:.2e})"


# ======================================================================================================================
# exact-fp32 kernels
# ======================================================================================================================
@pytest.mark.parametrize("case", EXACT_CASES, ids=[c[0] for c in EXACT_CASES])
def test_exact_input_and_state_gradients(case):
    name, hid, lyr, t, c, n, b, state = case
    xo, s, h0, c0, ws, d_top = (None if v is None else v.to(DEV) if torch.is_tensor(v) else [w.to(DEV) for w in v]
                                for v in lstm_inputs(n, b, t, lyr, c, hid, state, seed=700 + EXACT_CASES.index(case)))
    dh_n, dc_n = seeds(lyr, n * b, hid, seed=40 + EXACT_CASES.index(case))
    got, ktape = exact_run(xo, s, h0, c0, ws, lyr, hid, d_top, dh_n, dc_n)
    ref = state_gradients(xo, s, h0, c0, ws, lyr, 2, ktape, d_top, dh_n, dc_n)
    errs = grad_errors(got, ref)
    unseeded, _ = exact_run(xo, s, h0, c0, ws, lyr, hid, d_top, None, None)
    control = max(grad_errors(unseeded, ref).values())
    print(f"lstm extras {name}: worst {max(errs.values()):.2e} ({max(errs, key=errs.get)}); control {control:.2e}")
    assert max(errs.values()) <= GRAD_TOL, errs
    assert control > GRAD_TOL, control


@pytest.mark.parametrize("state", [False, True])
def test_tensor_core_and_exact_extras_agree(state):
    """H = 64, two planes: the two kernel families give the same d_xo, dh0, dc0 and weight gradients."""
    n, b, t, lyr, c = 6, 30, 7, 3, 2
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n, b, t, lyr, c, state, seed=77)
    dh_n, dc_n = seeds(lyr, n * b, HID, seed=78)
    tc, _, _ = lstm16_run(xo, s, h0, c0, ws, lyr, 2, d_top, dh_n, dc_n)
    ex, _ = exact_run(xo, s, h0, c0, ws, lyr, HID, d_top, dh_n, dc_n)
    errs = grad_errors(tc, ex)
    print(f"tensor cores vs exact (state={state}): worst {max(errs.values()):.2e}")
    assert max(errs.values()) <= GRAD_TOL, errs


# ======================================================================================================================
# the extended entry points with every extra NULL are the old ones
# ======================================================================================================================
class _ViaEx:
    """``ops.L`` whose two backward entry points go through the _ex entry points with every extra NULL."""

    def __init__(self, real):
        self.real = real

    def __getattr__(self, name):
        return getattr(self.real, name)

    def stmgcn_lstm16_bwd(self, *a):
        return self.real.stmgcn_lstm16_bwd_ex(*a[:-1], None, None, None, None, None, a[-1])

    def stmgcn_lstm_bwd(self, *a):
        return self.real.stmgcn_lstm_bwd_ex(*a[:-1], None, None, None, None, None, a[-1])


def _backward_outputs(run):
    torch.cuda.synchronize()
    n0 = lib().stmgcn_launch_count()
    d_s, grads = run()
    torch.cuda.synchronize()
    return [d_s] + list(grads), lib().stmgcn_launch_count() - n0


# How the backward kernels write each output decides what two runs can be asked to agree on:
# * sums of atomics, whose order changes from run to run: d_s (atomicAdd in lstm16_bwd_kernel and in lstm.cu's pointwise
#   kernel, there through a shared-memory partial), the weight gradients (red.add into per-CTA slices in lstm16.cu,
#   atomicAdd in the reduce GEMM of gemm_tall.cuh and for lstm.cu's layer-0 W_ih) and the bias gradients (atomicAdd);
# * plain stores, each element written once from values computed in a fixed order: d_xo (layer 0's dx * s), dh0 / dc0
#   (copies of dh_rec / dc after the step at t = 0, which the data GEMM and the pointwise kernels store).
_PLAIN_STORES = ("d_xo", "dh0", "dc0")


def _path_runs(path, seeded):
    """(forward + backward closures) of the five-region, T = 7, L = 3 case with an initial state: ``old()`` through the
    plain backward entry point, ``ex()`` through the _ex entry point with every extra wanted (and the seeds if
    ``seeded``)."""
    from stmgcn_b200 import ops
    n, b, t, lyr, c = 5, 60, 7, 3, 2
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n, b, t, lyr, c, True, seed=9)
    dh_n, dc_n = seeds(lyr, n * b, HID, seed=10) if seeded else (None, None)
    if path == "tc":
        _, _, _, tape = ops._lstm16_forward(xo, s, h0, c0, lyr, True, ws, 2, True)
        old = lambda: ops._lstm16_backward(xo, s, tape, lyr, 2, d_top)      # noqa: E731
        ex = lambda: ops._lstm16_backward_ex(xo, s, tape, lyr, 2, d_top, dh_n, dc_n, (True, True, True))      # noqa: E731
    else:
        def fresh_tape():       # the exact backward eats its tape
            return ops._exact_forward(xo, s, h0, c0, lyr, HID, True, ws, True)[3]

        old = lambda: ops._exact_backward(xo, s, fresh_tape(), lyr, HID, d_top)      # noqa: E731
        ex = lambda: ops._exact_backward_ex(xo, s, fresh_tape(), lyr, HID, d_top, dh_n, dc_n, (True, True, True))  # noqa: E731
    return old, ex


@pytest.mark.parametrize("path", ["tc", "exact"])
def test_extended_entry_points_with_null_extras_equal_the_old_ones(path, monkeypatch):
    """Every output of the old entry points -- d_s and the weight and bias gradients -- is a sum of atomics (see
    _PLAIN_STORES), so the _ex entry points with every extra NULL must give them within the gradient bar, in the same
    number of launches."""
    from stmgcn_b200 import ops
    run, _ = _path_runs(path, seeded=False)
    old, n_old = _backward_outputs(run)
    monkeypatch.setattr(ops, "L", _ViaEx(ops.L))
    new, n_new = _backward_outputs(run)
    assert n_new == n_old
    for i, (a, o) in enumerate(zip(new, old)):
        assert rel_err(a, o) <= GRAD_TOL, f"{path} output {i}: {rel_err(a, o):.2e}"


@pytest.mark.parametrize("path", ["tc", "exact"])
def test_extended_entry_points_store_the_input_and_state_gradients_reproducibly(path):
    """Two runs of the _ex entry point with the seeds and every extra wanted give the plain-store outputs d_xo, dh0 and
    dc0 bit for bit."""
    _, ex = _path_runs(path, seeded=True)
    runs = []
    for _ in range(2):
        _, _, extras = ex()
        torch.cuda.synchronize()
        runs.append(dict(zip(("d_xo", "dh0", "dc0"), (v.clone() for v in extras))))
    for k in _PLAIN_STORES:
        assert torch.equal(runs[0][k], runs[1][k]), f"{path} {k}: two runs differ ({rel_err(runs[0][k], runs[1][k]):.1e})"


# ======================================================================================================================
# memory contract of the new entry points (harness of test_gpu_abi_contract.py)
# ======================================================================================================================
@pytest.mark.parametrize("c,which", [(1, ("xt",)), (3, ("xo", "xt")), (2, ("xo",))])
def test_obs_grad_keeps_the_memory_contract(c, which):
    drive(obs_grad_calls(c, which), run_contract)


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("shape", [(1, 1, 3, 2, 1, False), (5, 60, 5, 4, 3, True), (3, 43, 4, 1, 4, False)],
                         ids=["one_row", "c3_l4_state", "l1_c4"])
def test_tensor_core_extended_backward_keeps_the_memory_contract(shape, planes):
    drive(lstm16_ex_calls(*shape, planes), run_contract)


@pytest.mark.parametrize("state", [False, True])
def test_exact_extended_backward_keeps_the_memory_contract(state):
    drive(lstm_ex_calls(7, 5, state), run_contract)


@pytest.mark.parametrize("family", ["obs_grad", "lstm16_bwd_ex", "lstm_bwd_ex"])
def test_new_entry_points_replay_from_a_cuda_graph(family):
    calls = {"obs_grad": lambda: obs_grad_calls(3, ("xo", "xt")),
             "lstm16_bwd_ex": lambda: lstm16_ex_calls(5, 60, 5, 4, 3, True, 2),
             "lstm_bwd_ex": lambda: lstm_ex_calls(7, 5, True)}[family]
    drive(calls(), run_captured)


def test_new_entry_points_reject_bad_calls_without_launching():
    gen = torch.Generator().manual_seed(0)
    bufs = [Buf("in", torch.randn(1 << 16, generator=gen)) for _ in range(4)]
    a, b, c, d = (x.p for x in bufs)
    calls = {"obs_grad: n = 0": lambda: lib().stmgcn_obs_grad(a, b, c, 2, 3, 0, 1, None),
             "lstm16_bwd_ex: T = 65": lambda: lib().stmgcn_lstm16_bwd_ex(
                 65, 2, 100, 1, 4, 2, *([a, b, c, d] * 5)[:18], a, b, c, d, a, None),
             "lstm_bwd_ex: H = 6": lambda: lib().stmgcn_lstm_bwd_ex(
                 3, 2, 8, 6, 1, 2, *([a, b, c, d] * 5)[:17], a, b, c, d, a, None)}
    for what, call in calls.items():
        torch.cuda.synchronize()
        n0 = lib().stmgcn_launch_count()
        rc = call()
        torch.cuda.synchronize()
        assert rc < 0, f"{what}: rc={rc}"
        assert lib().stmgcn_launch_count() == n0, what
        for i, x in enumerate(bufs):
            assert x.guards_intact() and torch.equal(bits(x.t), bits(x.init)), f"{what}: buffer {i} changed"


# ======================================================================================================================
# modules
# ======================================================================================================================
def _golden():
    return np.load(f"{GOLDEN}/inputgrad_ref.npz")


def _model_params(blob, prefix):
    return {k[len(prefix) + 6:]: torch.from_numpy(blob[k]) for k in blob.files if k.startswith(prefix + "param.")}


def test_st_mgcn_obs_gradient_matches_the_reference():
    import STMGCN
    blob = _golden()
    n, m, k, t, b, c, hid, layers, gcn_hid = [int(v) for v in blob["st.meta"]]
    model = STMGCN.ST_MGCN(M=m, seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=layers,
                           gcn_hidden_dim=gcn_hid, sta_kernel_config={"kernel_type": "chebyshev", "K": k},
                           gconv_use_bias=True, gconv_activation=nn.ReLU).to(DEV)
    model.load_state_dict(_model_params(blob, "st."))
    x = torch.from_numpy(blob["st.x"]).to(DEV).requires_grad_(True)
    sups = [torch.from_numpy(blob[f"st.supports.{g}"]).to(DEV) for g in range(m)]
    out = model(obs_seq=x, sta_adj_list=sups)
    nn.MSELoss()(out, torch.from_numpy(blob["st.y"]).to(DEV)).backward()
    errs = {"out": rel_err(out, torch.from_numpy(blob["st.out"])),
            "d obs": rel_err(x.grad, torch.from_numpy(blob["st.grad_obs"]))}
    errs.update({key: rel_err(p.grad, torch.from_numpy(blob["st.grad." + key])) for key, p in model.named_parameters()})
    print(f"ST_MGCN vs reference: d obs {errs['d obs']:.2e}, worst {max(errs.values()):.2e}")
    assert max(errs.values()) <= TOL, errs


def test_cg_lstm_obs_and_state_gradients_match_the_reference():
    import STMGCN
    blob = _golden()
    n, k, t, b, c, hid, layers = [int(v) for v in blob["cg.meta"]]
    model = STMGCN.CG_LSTM(seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=layers, K=k + 1,
                           gconv_use_bias=True, gconv_activation=nn.ReLU).to(DEV)
    model.load_state_dict(_model_params(blob, "cg."))
    g = lambda key: torch.from_numpy(blob["cg." + key]).to(DEV)      # noqa: E731
    x, h0, c0 = (g(key).requires_grad_(True) for key in ("x", "h0", "c0"))
    out, (h_n, c_n) = model(g("supports"), x, (h0, c0))
    loss = nn.MSELoss()(out, g("y")) + (h_n * g("r1")).sum() + (c_n * g("r2")).sum()
    loss.backward()
    errs = {"h_n": rel_err(h_n, g("h_n")), "c_n": rel_err(c_n, g("c_n"))}
    errs.update({f"d {v}": rel_err(t_.grad, g("grad_" + v)) for v, t_ in (("obs", x), ("h0", h0), ("c0", c0))})
    errs.update({key: rel_err(p.grad, g("grad." + key)) for key, p in model.named_parameters()})
    print(f"CG_LSTM vs reference: d obs {errs['d obs']:.2e}, d h0 {errs['d h0']:.2e}, d c0 {errs['d c0']:.2e}, "
          f"worst {max(errs.values()):.2e}")
    assert max(errs.values()) <= TOL, errs


@pytest.mark.parametrize("kind", ["localpool", "c3", "tanh", "bf16"])
def test_st_mgcn_obs_gradient_matches_the_dense_oracle(kind, monkeypatch):
    """localpool supports (generic stacks), C = 3, an activation the kernels do not fuse (torch applies it), and the
    one-plane bf16 mode (without the GCN activation) against the fp64 reference of that mode forced with the kernels'
    own values at every rounding point (test_gpu_bf16_mode.py), all at 1e-4 (bf16 mode measured on an H100: 1.1e-5,
    d obs)."""
    from stmgcn_b200 import ops
    if kind == "bf16":
        monkeypatch.setattr(ops, "_PLANES", 1)
        monkeypatch.setattr(ops, "_LSTM_PATH", "tc")
    c = 3 if kind == "c3" else 1
    act = {"tanh": "tanh", "bf16": "none"}.get(kind, "relu")
    model, sups, n, t = small_model(2, c, "localpool" if kind == "localpool" else "chebyshev", act, seed=5)
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(4, t, n, c, generator=gen)
    y = torch.randn(4, n, c, generator=gen)
    if kind == "bf16":
        params = {k: v.detach().clone() for k, v in model.state_dict().items()}
        picks = list(range(x.shape[0]))
        run = gpu_run(model, [s.to(DEV) for s in sups], x, y, picks, want_obs=True)
        chains = [[O.laplacian_csr_from_supports(s)] for s in sups]
        step, errs = forced_errors(run, params, chains, sups[0].shape[0], x, y, picks, relu=False, want_obs=True)
        errs.update(step)
    else:
        x, y = x.to(DEV).requires_grad_(True), y.to(DEV)
        out = model(obs_seq=x, sta_adj_list=[s.to(DEV) for s in sups])
        nn.MSELoss()(out, y).backward()
        d_obs, d_params = dense_grads(model, sups, x, y, act)
        errs = {"d obs": rel_err(x.grad, d_obs)}
        errs.update({k: rel_err(p.grad, d_params[k]) for k, p in model.named_parameters()})
    print(f"ST_MGCN {kind} vs {'forced bf16-mode' if kind == 'bf16' else 'dense'} oracle: d obs {errs['d obs']:.2e}, "
          f"worst {max(errs.values()):.2e}")
    assert max(errs.values()) <= TOL, errs


def test_two_step_rollout_matches_the_dense_oracle():
    """Step 1's prediction is appended to the window of step 2; the loss is on both predictions."""
    model, sups, n, t = small_model(2, 1, "chebyshev", "relu", seed=8)
    gen = torch.Generator().manual_seed(9)
    x = torch.randn(3, t, n, 1, generator=gen).to(DEV).requires_grad_(True)
    y1, y2 = (torch.randn(3, n, 1, generator=gen).to(DEV) for _ in range(2))
    sd = [s.to(DEV) for s in sups]

    def rollout(fwd, x_):
        p1 = fwd(x_)
        p2 = fwd(torch.cat([x_[:, 1:], p1[:, None]], dim=1))
        return torch.mean((p1 - y1.to(p1)) ** 2) + torch.mean((p2 - y2.to(p2)) ** 2)

    rollout(lambda v: model(obs_seq=v, sta_adj_list=sd), x).backward()
    params = {k: v.detach().double().cpu().requires_grad_(True) for k, v in model.state_dict().items()}
    xd = x.detach().double().cpu().requires_grad_(True)
    loss = rollout(lambda v: O.dense_st_mgcn(params, v, [s.double() for s in sups]), xd)
    g = torch.autograd.grad(loss, [xd] + list(params.values()))
    errs = {"d obs": rel_err(x.grad, g[0])}
    errs.update({k: rel_err(p.grad, r) for (k, p), r in zip(model.named_parameters(), g[1:])})
    print(f"two-step rollout: d obs {errs['d obs']:.2e}, worst {max(errs.values()):.2e}")
    assert max(errs.values()) <= TOL, errs


@pytest.mark.parametrize("path", ["tc", "fma"])
def test_parameter_gradients_do_not_depend_on_input_grads(path, monkeypatch):
    """The same parameter gradients (5e-5) whether obs / h0 / c0 require grad or not."""
    from stmgcn_b200 import ops
    import STMGCN
    monkeypatch.setattr(ops, "_LSTM_PATH", path)
    n, t, b, c, hid, layers = 23, 6, 4, 2, 64, 3
    torch.manual_seed(3)
    model = STMGCN.CG_LSTM(seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=layers, K=3,
                           gconv_use_bias=True).to(DEV)
    gen = torch.Generator().manual_seed(4)
    adj = (torch.rand(n, n, generator=gen) < 0.3).float()
    sup = O.chebyshev_supports_dense(adj.double(), 2).float().to(DEV)
    x = torch.randn(b, t, n, c, generator=gen).to(DEV)
    h0, c0 = (0.3 * torch.randn(layers, b * n, hid, generator=gen)).to(DEV), torch.randn(layers, b * n, hid, generator=gen).to(DEV)
    y = torch.randn(b, n, hid, generator=gen).to(DEV)
    runs = []
    for grad in (False, True):
        model.zero_grad()
        xs, hs, cs = (v.clone().requires_grad_(grad) for v in (x, h0, c0))
        out, _ = model(sup, xs, (hs, cs))
        nn.MSELoss()(out, y).backward()
        runs.append({k: p.grad.clone() for k, p in model.named_parameters()})
        if grad:
            assert xs.grad is not None and hs.grad is not None and cs.grad is not None
    errs = {k: rel_err(runs[1][k], runs[0][k]) for k in runs[0]}
    assert max(errs.values()) <= GRAD_TOL, errs


# ======================================================================================================================
# full size
# ======================================================================================================================
def test_obs_gradient_at_cfg3_size_on_every_window():
    """cfg3 (4096 regions, 3 graphs, K = 3, T = 12, batch 64, C = 1), smooth model, every window with its true target:
    d obs against the fp64 reference (tests/full_batch.py), held to the bar in max-norm, per window and per time step
    (``per_step.worst_step`` along T), with every parameter gradient and every window's output."""
    import full_batch
    from stmgcn_b200 import synth
    w = synth.WORKLOADS["cfg3"]
    model, sups, laps, params, x, y = cheb_workload(w, 64, relu=False)
    errs = full_batch.run("cfg3 d obs", model, sups, params, [[lap] for lap in laps], w.n_supports, x, y, relu=False,
                          window_chunk=CHUNK["cfg3"], want_obs=True)
    full_batch.assert_within(errs, TOL, what="cfg3 d obs")
