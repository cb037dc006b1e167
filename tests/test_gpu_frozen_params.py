"""Frozen parameters: a backward that is asked for no weight gradient computes none.

Model level: seven freeze patterns on both tensor-core plane modes and the exact-fp32 path, for Chebyshev and sparse
random-walk-diffusion supports, plus one cfg3-size case.  Frozen parameters end with ``.grad is None``, and every
requested gradient equals the all-trainable backward's within the spread of two all-trainable runs (the LSTM's d_s and
the weight gradients are sums of atomics, so two runs of the same backward differ in their last bits; the bound is four
times that spread, and at least 1e-5).

Entry-point level (the harness of test_gpu_abi_contract.py): with NULL weight outputs the per-row outputs are
bit-identical to the full call's, poisoned workspaces and guard bands show that nothing else is written, the launch
count drops by exactly the skipped launches, mixed NULL outputs are rejected without a launch, and the calls replay
from a CUDA graph.
"""
import math

import pytest
import torch
from torch import nn

import stmgcn_oracle as O
from abi_harness import (LSTM16_CASES, Buf, Call, bits, drive, fuse_calls, gate_calls, lstm16_calls, lstm16_ex_calls,
                         lstm_calls, lstm_ex_calls, proj_calls, run_captured, run_contract, run_once)
from helpers import DEV, GRAD_TOL, lib, rel_err
from model_cases import cheb_workload

pytestmark = pytest.mark.gpu


# ======================================================================================================================
# entry points
# ======================================================================================================================
class Null:
    """A NULL pointer in a Call's buffer dict: the launch lambdas read ``bufs[name].p`` at call time."""
    role, p, exact, finite = "null", None, True, True

    def prepare(self, mode, seed):
        return []

    def unchanged(self, snap):
        return True

    def guards_intact(self):
        return True


def _blocked_out(buf, rows):
    """A tile-blocked workspace the backward leaves holding per-row values, checked as an output (its first ``rows``)."""
    from stmgcn_b200 import ops
    return Buf("out", shape=tuple(buf.t.shape), part=lambda v: ops.from_blocked(v, rows))


def _lstm16_saved(call):
    return call.launches // 2                      # one slice-sum launch per layer


def _lstm_saved(call):
    return _LSTM_LAYERS                            # one reduce GEMM per layer


_LSTM_LAYERS = 3                                   # lstm_calls / lstm_ex_calls: L = 3


def _frozen_variant(call, null, keep=()):
    """The call with the buffers ``null`` passed as NULL and the buffers ``keep`` given but required untouched."""
    bufs = call.bufs
    for k in null:
        bufs[k] = Null()
    for k in keep:
        bufs[k] = Buf("keep", shape=tuple(bufs[k].t.shape), dtype=bufs[k].t.dtype)
    return bufs


def _lstm16_rows(call):
    rows = call.bufs["xo"].t.shape[0]
    for k in ("dh_rec", "dc", "dx_work"):
        if k in call.bufs:
            call.bufs[k] = _blocked_out(call.bufs[k], rows)


def _exact_rows(call):
    for k in ("dh_rec", "dc", "dx_work"):
        call.bufs[k] = Buf("out", shape=tuple(call.bufs[k].t.shape))


# name -> (weight outputs, other weight-only buffers, per-row preparation, launches saved)
ENTRIES = {
    "lstm16_bwd": (("grads",), ("dw_scratch", "dbp"), _lstm16_rows, _lstm16_saved),
    "lstm16_bwd_ex": (("grads",), ("dw_scratch", "dbp"), _lstm16_rows, _lstm16_saved),
    "lstm_bwd": (("dwx", "dwp", "dbp"), (), _exact_rows, _lstm_saved),
    "lstm_bwd_ex": (("dwx", "dwp", "dbp"), (), _exact_rows, _lstm_saved),
    "gate_bwd": (("d_fcw", "d_fcb"), (), None, lambda c: 0),
    "fuse_out_bwd": (("d_fcw", "d_fcb"), (), None, lambda c: 0),
}


def _frozen_driver(which, keep_ws, runner=run_contract, proj_saved=None):
    """A drive runner: the calls before the backward ``which`` run clean; the backward runs in full (contract), then
    with its weight outputs NULL (and, with ``keep_ws``, its weight-only workspaces given but required untouched):
    the contract again, the per-row outputs bit-identical to the full call's, the launch count lower by exactly the
    skipped launches."""
    def run(call):
        if call.name != which:
            return run_once(call, "clean")
        if which == "proj_bwd":
            weights, ws_only, rows_prep, saved = ("dw",), (), None, lambda c: proj_saved
        else:
            weights, ws_only, rows_prep, saved = ENTRIES[which]
        if rows_prep is not None:
            rows_prep(call)
        full = run_contract(call)
        n_saved = saved(call)
        _frozen_variant(call, weights + (() if keep_ws else ws_only), ws_only if keep_ws else ())
        frozen = Call(call.name + " (NULL weight outputs)", call.bufs, call.launch, None, call.launches - n_saved)
        got = runner(frozen)
        for k, v in got.items():
            b = call.bufs[k]
            if b.role == "acc" or not b.exact:       # d_s, the bias gradient of the projection: sums of atomics
                err = rel_err(v, full[k])
                assert err <= GRAD_TOL, f"{frozen.name}: {k} is {err:.2e} off the full call"
            else:
                assert torch.equal(bits(v), bits(full[k])), f"{frozen.name}: {k} differs from the full call"
        return full
    return run


@pytest.mark.parametrize("keep_ws", [False, True], ids=["ws_null", "ws_untouched"])
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", ["one_row", "l1_no_dx_work", "c3_l4_state", "waves_b37_state"])
def test_tensor_core_lstm_backward_without_weight_gradients(case, planes, keep_ws):
    spec = next(c for c in LSTM16_CASES if c[0] == case)
    drive(lstm16_calls(spec, planes), _frozen_driver("lstm16_bwd", keep_ws))


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("shape", [(1, 1, 3, 2, 1, False), (5, 60, 5, 4, 3, True), (3, 43, 4, 1, 4, False)],
                         ids=["one_row", "c3_l4_state", "l1_c4"])
def test_tensor_core_extended_backward_without_weight_gradients(shape, planes):
    """dh0, dc0, d_xo and the seeded state: bit-identical to the full call's."""
    drive(lstm16_ex_calls(*shape, planes), _frozen_driver("lstm16_bwd_ex", False))


@pytest.mark.parametrize("state", [False, True])
def test_exact_lstm_backward_without_weight_gradients(state):
    n, b_sz = (7, 5) if state else (61, 5)
    drive(lstm_calls(n, b_sz, state), _frozen_driver("lstm_bwd", False))
    drive(lstm_ex_calls(7, 5, state), _frozen_driver("lstm_bwd_ex", False))


# (name, ks, p, q, regions N, batch B, gap, weight images, broadcast dOut, ReLU, bias)
PROJ = [("tc_ks1", 1, 64, 64, 3, 43, 0, True, False, True, True),
        ("tc_ks5", 5, 64, 64, 40, 37, 0, True, False, False, True),
        ("tc_ks8_nobias", 8, 64, 64, 3, 43, 36, True, False, True, False),
        ("tc_odd_gap_ffma", 3, 64, 64, 3, 43, 7, True, False, True, True),
        ("ffma_pool", 4, 12, 12, 33, 5, 0, False, True, True, True),
        ("ffma_p64_q32", 2, 64, 32, 43, 3, 4, False, False, False, False)]


@pytest.mark.parametrize("case", PROJ, ids=[c[0] for c in PROJ])
def test_projection_backward_without_weight_gradient(case):
    """No dW launch on either family: the tensor-core backward keeps its row launches (two beyond 4 supports), the
    FFMA backward its dZ and U launches."""
    _, ks, p, q, n, b_sz, gap, tc, bcast, relu, bias = case
    on_tc = tc and not bcast and gap % 4 == 0
    saved = (ks + 1) // 2 if on_tc else 1
    drive(proj_calls(ks, p, q, n, b_sz, gap, tc, bcast, relu, bias, seed=300 + PROJ.index(case)),
           _frozen_driver("proj_bwd", False, proj_saved=saved))


@pytest.mark.parametrize("t", [12, 300])
def test_context_gate_backward_without_fc_gradients(t):
    drive(gate_calls(t, 5), _frozen_driver("gate_bwd", False))


@pytest.mark.parametrize("c", [1, 40])
def test_fuse_out_backward_without_fc_gradients(c):
    drive(fuse_calls(3, c), _frozen_driver("fuse_out_bwd", False))


CAPTURED = {
    "tensor_core_lstm": (lambda: lstm16_calls(("c3_l4_state", 5, 60, 5, 4, 3, True), 2), "lstm16_bwd", None),
    "tensor_core_lstm_ex": (lambda: lstm16_ex_calls(5, 60, 5, 4, 3, True, 1), "lstm16_bwd_ex", None),
    "exact_lstm_ex": (lambda: lstm_ex_calls(7, 5, True), "lstm_bwd_ex", None),
    "projection_tensor_cores": (lambda: proj_calls(5, 64, 64, 40, 37, 0, True, False, True, True, seed=1), "proj_bwd", 3),
    "context_gate": (lambda: gate_calls(12, 5), "gate_bwd", None),
    "fuse_out": (lambda: fuse_calls(3, 40), "fuse_out_bwd", None),
}


@pytest.mark.parametrize("family", list(CAPTURED))
def test_backward_without_weight_gradients_replays_from_a_cuda_graph(family):
    """The NULL-weight call eagerly on a side stream, then captured and replayed (test_gpu_abi_contract.run_captured);
    both equal the full call's per-row outputs."""
    calls, which, saved = CAPTURED[family]
    drive(calls(), _frozen_driver(which, False, runner=run_captured, proj_saved=saved))


# (what, call(lib, a, b, c, d, e, f)): one NULL weight output where its partner is given, or nothing to compute
REJECTS = [
    ("lstm16_bwd: grads without dw_scratch", lambda L, a, b, c, d, e, f: L.stmgcn_lstm16_bwd(
        5, 2, 100, 1, 4, 2, a, b, c, d, e, None, None, f, a, b, c, d, e, None, a, b, c, d, None)),
    ("lstm16_bwd_ex: grads without dbp", lambda L, a, b, c, d, e, f: L.stmgcn_lstm16_bwd_ex(
        5, 2, 100, 1, 4, 2, a, b, c, d, e, None, None, f, a, b, c, d, e, f, None, b, c, d, None, None, None, None, None,
        None)),
    ("lstm_bwd: dwx NULL, dwp and dbp given", lambda L, a, b, c, d, e, f: L.stmgcn_lstm_bwd(
        3, 2, 8, 8, 1, 2, a, b, c, d, None, None, e, f, a, b, c, d, e, f, None, b, c, None)),
    ("lstm_bwd: dbp NULL", lambda L, a, b, c, d, e, f: L.stmgcn_lstm_bwd(
        3, 2, 8, 8, 1, 2, a, b, c, d, None, None, e, f, a, b, c, d, e, f, a, b, None, None)),
    ("lstm_bwd_ex: dwp NULL", lambda L, a, b, c, d, e, f: L.stmgcn_lstm_bwd_ex(
        3, 2, 8, 8, 1, 2, a, b, c, d, None, None, e, f, a, b, c, d, e, f, a, None, c, None, None, None, None, None, None)),
    ("proj_bwd: dw, dbias and u all NULL", lambda L, a, b, c, d, e, f: L.stmgcn_proj_bwd(
        a, 768, 1, 64, 12, b, 12, 1, c, d, None, 1.0, 4, e, None, None, None, 0, None, None)),
    ("gate_bwd: d_fcw NULL, d_fcb given", lambda L, a, b, c, d, e, f: L.stmgcn_gate_bwd(
        a, b, c, d, 2, 12, e, None, f, a, None)),
    ("gate_bwd: d_fcb NULL, d_fcw given", lambda L, a, b, c, d, e, f: L.stmgcn_gate_bwd(
        a, b, c, d, 2, 12, e, f, None, a, None)),
    ("fuse_out_bwd: d_fcb NULL, d_fcw given", lambda L, a, b, c, d, e, f: L.stmgcn_fuse_out_bwd(
        a, b, 4, 2, 8, 2, c, d, e, None, None)),
    ("fuse_out_bwd: d_fcw NULL, d_fcb given", lambda L, a, b, c, d, e, f: L.stmgcn_fuse_out_bwd(
        a, b, 4, 2, 8, 2, c, d, None, f, None)),
]


@pytest.mark.parametrize("case", REJECTS, ids=[r[0] for r in REJECTS])
def test_mixed_null_weight_outputs_are_rejected_without_a_launch(case):
    what, call = case
    gen = torch.Generator().manual_seed(0)
    bufs = [Buf("in", torch.randn(1 << 16, generator=gen)) for _ in range(6)]
    torch.cuda.synchronize()
    n0 = lib().stmgcn_launch_count()
    rc = call(lib(), *(x.p for x in bufs))
    torch.cuda.synchronize()
    assert rc < 0, f"{what}: rc={rc}"
    assert lib().stmgcn_last_error(), f"{what}: no message"
    assert lib().stmgcn_launch_count() == n0, f"{what}: a kernel was launched"
    for i, x in enumerate(bufs):
        assert x.guards_intact() and torch.equal(bits(x.t), bits(x.init)), f"{what}: buffer {i} changed"


# ======================================================================================================================
# modules
# ======================================================================================================================
MODES = {"tc_p2": ("tc", 2), "tc_p1": ("tc", 1), "fma": ("fma", 2)}
N, T, B, M, LAYERS, HID = 19, 5, 4, 2, 2, 64


def _set_mode(monkeypatch, mode):
    from stmgcn_b200 import ops
    path, planes = MODES[mode]
    monkeypatch.setattr(ops, "_LSTM_PATH", path)
    monkeypatch.setattr(ops, "_PLANES", planes)


def _supports(kernel, seed):
    import GCN
    gen = torch.Generator().manual_seed(seed)
    adjs = [(torch.rand(N, N, generator=gen) < 0.3).float() * (0.5 + torch.rand(N, N, generator=gen)) for _ in range(M)]
    if kernel == "chebyshev":
        return [O.chebyshev_supports_dense(a.double(), 2).float().to(DEV) for a in adjs], 2
    pre = GCN.Adj_Preprocessor("random_walk_diffusion", 1)
    return [pre.process_sparse(a).to(DEV) for a in adjs], 1


def _st_model(kernel, k):
    import STMGCN
    torch.manual_seed(11)
    # gcn_hidden_dim = H = 64: the spatial projections run on the tensor cores on the tc path.  No GCN activation: a ReLU
    # mask that flips between two forwards (the forward's pooling sums with atomics) would move a gradient by more than
    # the run-to-run spread measured here (the ReLU backward with NULL weight outputs is covered by the entry-point tests)
    return STMGCN.ST_MGCN(M=M, seq_len=T, n_nodes=N, input_dim=1, lstm_hidden_dim=HID, lstm_num_layers=LAYERS,
                          gcn_hidden_dim=64, sta_kernel_config={"kernel_type": kernel, "K": k}, gconv_use_bias=True,
                          gconv_activation=None).to(DEV)


def _gcns(model):
    return [g for r in model.rnn_list for g in [r.gconv_temporal_feats]] + list(model.gcn_list)


# pattern -> (frozen-parameter predicate on (model, name, param), obs requires grad)
def _is(mods):
    return lambda model, p: any(p is q for mod in mods(model) for q in mod.parameters())


PATTERNS = {
    "model_frozen_obs_grad": (lambda model, p: True, True),
    "lstm_frozen": (_is(lambda m: [r.lstm for r in m.rnn_list]), False),
    "spatial_gcns_frozen": (_is(lambda m: list(m.gcn_list)), False),
    "gate_fc_and_temporal_gcn_frozen": (_is(lambda m: [r.fc for r in m.rnn_list] +
                                            [r.gconv_temporal_feats for r in m.rnn_list]), False),
    "gcn_w_frozen_b_trainable": (lambda model, p: any(p is g.W for g in _gcns(model)), False),
    "output_fc_frozen": (_is(lambda m: [m.fc]), False),
}


def _step(model, frozen, leaves, run):
    """One backward with the parameters ``frozen`` not requiring grad; returns {name: grad} of every requested tensor
    (trainable parameters and the input leaves) and the names of the frozen ones."""
    named = dict(model.named_parameters())
    for name, p in named.items():
        p.requires_grad_(name not in frozen)
        p.grad = None
    xs = {k: v.detach().clone().requires_grad_(True) for k, v in leaves.items()}
    run(xs).backward()
    for name in frozen:
        assert named[name].grad is None, f"frozen {name} has a gradient"
    got = {k: p.grad.clone() for k, p in named.items() if k not in frozen}
    got.update({"leaf " + k: v.grad.clone() for k, v in xs.items()})
    for p in named.values():
        p.requires_grad_(True)
    return got


def _check_pattern(model, frozen, leaves, run, what):
    base = [_step(model, set(), leaves, run) for _ in range(2)]
    got = _step(model, frozen, leaves, run)
    assert set(got) == set(base[0]) - set(frozen), what
    errs = {}
    for k, g in got.items():
        spread = rel_err(base[1][k], base[0][k])
        err = rel_err(g, base[0][k])
        # within the atomics' run-to-run spread (x4: two runs are a small sample of it), and never further than fp32
        # summation-order noise (1e-5, a fifth of the 5e-5 gradient bar) where the two runs happen to agree bit for bit
        bound = max(4 * spread, 1e-5)
        errs[k] = (err, spread)
        assert err <= bound, f"{what}: {k} is {err:.2e} off the all-trainable backward (spread {spread:.2e})"
    return errs


@pytest.mark.parametrize("pattern", list(PATTERNS))
@pytest.mark.parametrize("kernel", ["chebyshev", "random_walk_diffusion"])
@pytest.mark.parametrize("mode", list(MODES))
def test_st_mgcn_freeze_pattern(mode, kernel, pattern, monkeypatch):
    _set_mode(monkeypatch, mode)
    sups, k = _supports(kernel, seed=5)
    model = _st_model(kernel, k)
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(B, T, N, 1, generator=gen).to(DEV)
    y = torch.randn(B, N, 1, generator=gen).to(DEV)
    pred, obs_grad = PATTERNS[pattern]
    frozen = {name for name, p in model.named_parameters() if pred(model, p)}
    assert frozen
    leaves = {"obs": x} if obs_grad else {}

    def run(xs):
        return nn.MSELoss()(model(obs_seq=xs.get("obs", x), sta_adj_list=sups), y)

    _check_pattern(model, frozen, leaves, run, f"{mode} {kernel} {pattern}")


@pytest.mark.parametrize("kernel", ["chebyshev", "random_walk_diffusion"])
@pytest.mark.parametrize("mode", list(MODES))
def test_cg_lstm_frozen_with_state_gradients(mode, kernel, monkeypatch):
    """CG_LSTM frozen, the gradients of h0 and c0 wanted (learned initial states on a fixed model)."""
    _set_mode(monkeypatch, mode)
    sups, k = _supports(kernel, seed=7)
    model = _st_model(kernel, k).rnn_list[0]
    gen = torch.Generator().manual_seed(8)
    x = torch.randn(B, T, N, 1, generator=gen).to(DEV)
    h0, c0 = (0.3 * torch.randn(LAYERS, B * N, HID, generator=gen)).to(DEV), torch.randn(LAYERS, B * N, HID, generator=gen).to(DEV)
    y, r = torch.randn(B, N, HID, generator=gen).to(DEV), torch.randn(LAYERS, B * N, HID, generator=gen).to(DEV)

    def run(xs):
        out, (h_n, c_n) = model(sups[0], x, (xs["h0"], xs["c0"]))
        return nn.MSELoss()(out, y) + (h_n * r).sum() * 1e-3 + (c_n * r).sum() * 1e-3

    frozen = {name for name, _ in model.named_parameters()}
    _check_pattern(model, frozen, {"h0": h0, "c0": c0}, run, f"{mode} {kernel} CG_LSTM frozen")


@pytest.mark.parametrize("pattern", ["lstm_frozen", "model_frozen_obs_grad"])
def test_freeze_pattern_at_cfg3_size(pattern):
    """cfg3 (4096 regions, 3 graphs, K = 3, T = 12, C = 1) at batch 16 on the default path, without the GCN activation
    (with it, cfg3's obs gradient is vanishing and a flipped ReLU mask moves it by up to 6e-2 between two all-trainable
    runs, measured on an H100)."""
    from stmgcn_b200 import synth
    model, sups, _, _, x, y = cheb_workload(synth.WORKLOADS["cfg3"], 16, relu=False)
    xd, yd = x.to(DEV), y.to(DEV)
    pred, obs_grad = PATTERNS[pattern]
    frozen = {name for name, p in model.named_parameters() if pred(model, p)}
    leaves = {"obs": xd} if obs_grad else {}

    def run(xs):
        return nn.MSELoss()(model(obs_seq=xs.get("obs", xd), sta_adj_list=sups), yd)

    errs = _check_pattern(model, frozen, leaves, run, f"cfg3 {pattern}")
    print(f"cfg3 {pattern}: worst {max(e for e, _ in errs.values()):.2e} against the all-trainable backward")


@pytest.mark.parametrize("mode", list(MODES))
def test_launch_count_drops_by_the_skipped_launches(mode, monkeypatch):
    """Per graph branch: LSTM frozen saves one launch per layer (the slice sum of the tensor-core backward, the reduce
    GEMM of the exact one); every GCN's W frozen saves the projection's dW launches: one per pair of supports on the
    tensor cores (the spatial GCN on the tc path, H = 64), one FFMA dW otherwise (the temporal GCN, and everything on
    the fma path)."""
    _set_mode(monkeypatch, mode)
    sups, k = _supports("chebyshev", seed=5)
    model = _st_model("chebyshev", k)
    ks = model.sta_K
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(B, T, N, 1, generator=gen).to(DEV)
    y = torch.randn(B, N, 1, generator=gen).to(DEV)

    def backward_launches(pattern):
        frozen = set() if pattern is None else {n for n, p in model.named_parameters() if PATTERNS[pattern][0](model, p)}
        for name, p in model.named_parameters():
            p.requires_grad_(name not in frozen)
            p.grad = None
        loss = nn.MSELoss()(model(obs_seq=x, sta_adj_list=sups), y)
        torch.cuda.synchronize()
        n0 = lib().stmgcn_launch_count()
        loss.backward()
        torch.cuda.synchronize()
        return lib().stmgcn_launch_count() - n0

    full = backward_launches(None)
    assert full - backward_launches("lstm_frozen") == M * LAYERS
    spatial_dw = math.ceil(ks / 2) if MODES[mode][0] == "tc" else 1
    assert full - backward_launches("gcn_w_frozen_b_trainable") == M * (spatial_dw + 1)
    for p in model.parameters():
        p.requires_grad_(True)


def test_fine_tuning_with_the_lstms_frozen():
    """A few Adam steps on a new target with the shared LSTMs frozen: the loss falls, the LSTM weights stay bit-unchanged."""
    sups, k = _supports("chebyshev", seed=9)
    model = _st_model("chebyshev", k)
    gen = torch.Generator().manual_seed(10)
    x = torch.randn(B, T, N, 1, generator=gen).to(DEV)
    # the target: a model with the same LSTMs and everything else moved, which the trainable part can reach
    teacher = _st_model("chebyshev", k)
    with torch.no_grad():
        for n, p in teacher.named_parameters():
            if ".lstm." not in n:
                p.add_(0.2 * torch.randn(p.shape, generator=gen).to(DEV))
        y = teacher(obs_seq=x, sta_adj_list=sups)
    lstm = {n: p.detach().clone() for n, p in model.named_parameters() if ".lstm." in n}
    assert len(lstm) == M * LAYERS * 4
    for n, p in model.named_parameters():
        p.requires_grad_(n not in lstm)
    opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=3e-3)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        loss = nn.MSELoss()(model(obs_seq=x, sta_adj_list=sups), y)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    print("fine-tuning losses:", " ".join(f"{v:.4f}" for v in losses))
    assert losses[-1] < 0.8 * losses[0], losses
    for n, p in model.named_parameters():
        if n in lstm:
            assert p.grad is None and torch.equal(bits(p.detach()), bits(lstm[n])), f"{n} changed"
