"""Gradients of learnable support values on the H100: the CSR SDDMM entry point against fp64 (widths, term counts, +=,
guard bands, bit-identical reruns, NaN tracing), the graph convolutions' d vals against dense fp64 autograd for every
support kind and both projection families, the model (shared handles, branch streams, both LSTM families, the
bf16-arithmetic mode, the benchmarked size), training through ``process_sparse`` under a fused optimizer, and the frozen
path unchanged."""
import pytest
import torch
from torch import nn

import support_grad_cases as S
from helpers import DEV, GRAD_TOL, TOL, assert_close, build_model, rel_err
from kernel_cases import handmade_csr

pytestmark = pytest.mark.gpu


def _rand(shape, seed, device=DEV):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(device)


# ======================================================================================================================
# the entry point
# ======================================================================================================================
def _sddmm(n, rp, ci, terms, dvals, rnd=False, nnz=None):
    from stmgcn_b200 import _lib, ops
    f_total = terms[0][0].numel() // n
    nnz = ci.numel() if nnz is None else nnz
    tiles = ops.sddmm_tiles(f_total)
    work = torch.full((tiles * nnz,), float("nan"), device=DEV) if tiles > 1 else None
    rc = _lib.lib.stmgcn_csr_sddmm(n, rp.data_ptr(), ci.data_ptr(), nnz, len(terms),
                                   _lib.ptr_array([t[0].data_ptr() for t in terms]),
                                   _lib.ptr_array([t[1].data_ptr() for t in terms]),
                                   _lib.float_array([t[2] for t in terms]), int(rnd), f_total,
                                   None if work is None else work.data_ptr(), 0 if work is None else work.numel(),
                                   dvals.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "csr_sddmm")


def _ref(rows, cols, terms, rnd=False):
    out = 0.0
    for a, b, c in terms:
        b64 = b.double()
        if rnd:
            b64 = b.to(torch.bfloat16).double()
        out = out + c * (a.double().reshape(a.shape[0], -1)[rows] * b64.reshape(b.shape[0], -1)[cols]).sum(1)
    return out


@pytest.mark.parametrize("f_total", [1, 3, 4, 8, 768, 4096])
@pytest.mark.parametrize("nterms", [1, 2, 3, 5, 8])
def test_sddmm_against_fp64_with_accumulate_and_guards(f_total, nterms):
    n = 70
    rp, ci, _ = (t.to(DEV) for t in handmade_csr(n, 3 + nterms))
    rows, cols = S.coo_of(rp, ci)
    nnz = ci.numel()
    terms = [(_rand((n, f_total), 10 * nterms + t), _rand((n, f_total), 10 * nterms + t + 100), 1.0 if t == 0 else 2.0)
             for t in range(nterms)]
    guard = 64
    buf = torch.full((nnz + 2 * guard,), float("nan"), device=DEV)
    v0 = _rand((nnz,), 7)
    buf[guard:guard + nnz] = v0
    dvals = buf[guard:guard + nnz]
    _sddmm(n, rp, ci, terms, dvals)
    torch.cuda.synchronize()
    assert torch.isnan(buf[:guard]).all() and torch.isnan(buf[guard + nnz:]).all()
    assert rel_err(dvals - v0, _ref(rows, cols, terms)) <= 5e-6
    # bit-identical rerun
    again = v0.clone()
    _sddmm(n, rp, ci, terms, again)
    assert torch.equal(again, dvals)
    # bf16 rounding of B (any width: the kernel rounds on load)
    r = torch.zeros(nnz, device=DEV)
    _sddmm(n, rp, ci, terms, r, rnd=True)
    assert rel_err(r, _ref(rows, cols, terms, rnd=True)) <= 5e-6


def test_sddmm_nan_tracer():
    """A NaN in row i of A reaches exactly row i's entries; a NaN in row j of B exactly the entries in column j."""
    n, f = 60, 256
    rp, ci, _ = (t.to(DEV) for t in handmade_csr(n, 4))
    rows, cols = S.coo_of(rp, ci)
    for which, idx in (("a", 0), ("a", 13), ("b", 1), ("b", 22)):
        a, b = _rand((n, f), 1), _rand((n, f), 2)
        (a if which == "a" else b)[idx, 77] = float("nan")
        d = torch.zeros(ci.numel(), device=DEV)
        _sddmm(n, rp, ci, [(a, b, 1.0)], d)
        want = (rows == idx) if which == "a" else (cols == idx)
        assert torch.equal(torch.isnan(d), want), (which, idx)


# ======================================================================================================================
# the graph convolutions
# ======================================================================================================================
def _handle(kind, n, seed):
    import GCN
    from stmgcn_b200 import synth
    from stmgcn_b200.graph import ChebSupports, SparseSupports
    if kind == "chebyshev":
        h = GCN.Adj_Preprocessor("chebyshev", 3).process_sparse(synth.make_adjacency(n, seed, 0.3))
    elif kind == "diffusion":
        h = GCN.Adj_Preprocessor("random_walk_diffusion", 2).process_sparse(S.directed_graph(n, seed).float())
    elif kind == "localpool":
        h = GCN.Adj_Preprocessor("localpool", 1).process_sparse(synth.make_adjacency(n, seed, 0.3))
    elif kind == "handmade_cheb":
        h = ChebSupports(n, 4, *handmade_csr(n, seed))
    else:                   # hand-made generic stack of three supports
        h = SparseSupports("generic", n, 3, [handmade_csr(n, seed + k) for k in range(3)])
    h = h.to(DEV)
    h.mats = [(rp, ci, v.detach().clone().requires_grad_(True)) for rp, ci, v in h.mats]
    return h


KINDS = ["chebyshev", "diffusion", "localpool", "handmade_cheb", "handmade_generic"]


@pytest.mark.parametrize("path", ["tc", "fma"])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("fn", ["spatial", "temporal"])
def test_gcn_value_grads_against_dense_fp64(monkeypatch, fn, kind, path):
    import stmgcn_oracle as O
    from stmgcn_b200 import _lib, ops
    monkeypatch.setattr(ops, "_LSTM_PATH", path)
    n, b = 37, 3
    h = _handle(kind, n, 5)
    sset = h.support_set()
    p = q = 64 if fn == "spatial" else 12
    x = _rand((n, b, p), 1)
    w = (_rand((h.ks * p, q), 2) / p ** 0.5).requires_grad_(True)
    bias = _rand((q,), 3).requires_grad_(True)
    r = _rand((n, b, q) if fn == "spatial" else (b, q), 4)
    if fn == "spatial":
        out = ops.ChebGCN.apply(x, w, bias, sset, _lib.ACT_RELU, *sset.grad_values())
    else:
        out = ops.TemporalPool.apply(x, w, bias, sset, _lib.ACT_RELU, *sset.grad_values())
    (out * r).sum().backward()
    leaves = [v.detach().double().clone().requires_grad_(True) for _, _, v in h.mats]
    stack = S.handle_stack(h, leaves, DEV)
    x64 = x.double().permute(1, 0, 2)
    g = O.dense_gcn(stack, x64, w.detach().double(), bias.detach().double(), True)     # (B, N, q)
    ref = (g * r.double().permute(1, 0, 2)).sum() if fn == "spatial" else ((x64 + g).sum(1) * r.double()).sum()
    ref.backward()
    for (_, _, v), leaf in zip(h.mats, leaves):
        assert v.grad is not None and v.grad.shape == v.shape
        assert_close(v.grad.cpu(), leaf.grad.cpu(), f"{fn} {kind} d vals", TOL)


# ======================================================================================================================
# the model
# ======================================================================================================================
META = dict(n=24, m=3, k=2, t=4, b=3, c=1, hid=64, layers=2, gcn_hid=64)


def _model_case(kernel_type="chebyshev", seed=0):
    import GCN
    from stmgcn_b200 import synth
    meta = dict(META, kernel_type=kernel_type, k=1 if kernel_type == "localpool" else META["k"])
    torch.manual_seed(seed)
    model = build_model(meta, DEV)
    pre = GCN.Adj_Preprocessor(kernel_type, meta["k"])
    adjs = [S.directed_graph(meta["n"], 3 + g).float() if kernel_type == "random_walk_diffusion"
            else synth.make_adjacency(meta["n"], g, 0.3) for g in range(2)]
    handles = []
    for a in adjs:
        h = pre.process_sparse(a).to(DEV)
        h.mats = [(rp, ci, nn.Parameter(v.detach().clone())) for rp, ci, v in h.mats]
        handles.append(h)
    x = _rand((meta["b"], meta["t"], meta["n"], meta["c"]), 11)
    y = _rand((meta["b"], meta["n"], meta["c"]), 12)
    return meta, model, handles, x, y


def _check_model(model, handles, branch_handle, x, y, what, tol=TOL, relu=True):
    x = x.clone().requires_grad_(True)
    with S.record_relu_masks() as rec:
        out = model(obs_seq=x, sta_adj_list=[handles[i] for i in branch_handle])
    loss = nn.MSELoss()(out, y)
    loss.backward()
    params = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    l_ref, g_ref, d_obs, d_vals = S.model_reference(params, x.detach().cpu(), y.cpu(), handles, branch_handle, relu,
                                                    masks=rec.masks if relu else None)
    assert abs(loss.item() - l_ref) <= tol * abs(l_ref)
    for name, prm in model.named_parameters():
        assert_close(prm.grad.cpu(), g_ref[name], f"{what} {name}", tol)
    assert_close(x.grad.cpu(), d_obs, f"{what} d obs", tol)
    worst = 0.0
    for h, dv in zip(handles, d_vals):
        for (_, _, v), want in zip(h.mats, dv):
            worst = max(worst, assert_close(v.grad.cpu(), want, f"{what} d vals", tol))
    return worst


@pytest.mark.parametrize("path", ["tc", "fma"])
@pytest.mark.parametrize("streams", ["1", "0"])
@pytest.mark.parametrize("kernel_type", ["chebyshev", "random_walk_diffusion", "localpool"])
def test_st_mgcn_shared_handle_against_fp64(monkeypatch, path, streams, kernel_type):
    """M = 3, the first handle feeds two branches: d vals, every parameter gradient and d obs within 1e-4."""
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_LSTM_PATH", path)
    monkeypatch.setenv("STMGCN_GRAPH_STREAMS", streams)
    meta, model, handles, x, y = _model_case(kernel_type)
    _check_model(model, handles, [0, 1, 0], x, y, f"{kernel_type} {path} streams={streams}")


def test_st_mgcn_with_frozen_model_and_d_obs_only_values_learn():
    meta, model, handles, x, y = _model_case("chebyshev", 1)
    for prm in model.parameters():
        prm.requires_grad_(False)
    out = model(obs_seq=x, sta_adj_list=[handles[0], handles[1], handles[1]])
    nn.MSELoss()(out, y).backward()
    params = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    _, _, _, d_vals = S.model_reference(params, x.cpu(), y.cpu(), handles, [0, 1, 1])
    for h, dv in zip(handles, d_vals):
        assert_close(h.mats[0][2].grad.cpu(), dv[0], "frozen model d vals")
    assert all(p.grad is None for p in model.parameters())


@pytest.mark.parametrize("path", ["tc", "fma"])
def test_cg_lstm_value_grads_and_state_grads(monkeypatch, path):
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_LSTM_PATH", path)
    import STMGCN
    meta, _, handles, x, y = _model_case("random_walk_diffusion", 2)
    torch.manual_seed(3)
    m = STMGCN.CG_LSTM(seq_len=meta["t"], n_nodes=meta["n"], input_dim=1, lstm_hidden_dim=64, lstm_num_layers=2, K=5,
                       gconv_use_bias=True).to(DEV)
    h0 = (_rand((2, meta["b"] * meta["n"], 64), 5) * 0.1).requires_grad_(True)
    c0 = (_rand((2, meta["b"] * meta["n"], 64), 6) * 0.1).requires_grad_(True)
    out, (hn, cn) = m(handles[0], x, (h0, c0))
    r = _rand(tuple(out.shape), 7)
    ((out * r).sum() + hn.sum() + cn.square().sum()).backward()
    import stmgcn_oracle as O
    p64 = {"rnn_list.0." + k: v.detach().double().cpu().requires_grad_(True) for k, v in m.state_dict().items()}
    leaves = [v.detach().double().cpu().requires_grad_(True) for _, _, v in handles[0].mats]
    h64 = [t.detach().double().cpu().requires_grad_(True) for t in (h0, c0)]
    stack = S.handle_stack(handles[0], [leaf.to(DEV) for leaf in leaves], DEV).cpu()
    o64, (hn64, cn64) = O.dense_cg_lstm(stack, x.double().cpu(), p64, "rnn_list.0.", hidden=tuple(h64))
    ((o64 * r.double().cpu()).sum() + hn64.sum() + cn64.square().sum()).backward()
    for (_, _, v), leaf in zip(handles[0].mats, leaves):
        assert_close(v.grad.cpu(), leaf.grad, "CG_LSTM d vals")
    assert_close(h0.grad.cpu(), h64[0].grad, "dh0")
    assert_close(c0.grad.cpu(), h64[1].grad, "dc0")
    for k, prm in m.named_parameters():
        assert_close(prm.grad.cpu(), p64["rnn_list.0." + k].grad, f"CG_LSTM {k}")


def test_bf16_mode_value_grads(monkeypatch):
    """Single-plane bf16 arithmetic: the spatial SDDMM multiplies by bf16(T_{k-1}), the operand its forward gathered.
    GCN level: d vals within 1e-4 of a reference that rounds where the kernels round, and an SDDMM reading fp32 T_{k-1}
    misses that reference."""
    from stmgcn_b200 import _lib, ops
    monkeypatch.setattr(ops, "_PLANES", 1)
    # GCN level, forced reference: T_k = 2 X r(T_{k-1}) - T_{k-2}, r = bf16 rounding with an identity gradient
    n, b = 37, 4
    h = _handle("chebyshev", n, 6)
    sset = h.support_set()
    x = _rand((n, b, 64), 1)
    w = _rand((4 * 64, 64), 2) / 8.0
    r = _rand((n, b, 64), 3)
    out = ops.ChebGCN.apply(x, w, None, sset, _lib.ACT_NONE, *sset.grad_values())
    (out * r).sum().backward()
    got = h.mats[0][2].grad

    def forced(fp32_b):
        leaf = h.mats[0][2].detach().double().clone().requires_grad_(True)
        rows, cols = S.coo_of(h.mats[0][0], h.mats[0][1])
        xm = S.dense_matrix(n, rows, cols, leaf)
        rnd = lambda v: v + (v.float().to(torch.bfloat16).double() - v).detach()

        def mul(t):
            if fp32_b:          # the value of the rounded product, the gradient of the unrounded one
                return (xm @ rnd(t)).detach() + xm @ t - (xm @ t).detach()
            return xm @ rnd(t)
        t = [x.double().reshape(n, -1)]
        t.append(mul(t[0]))
        for _ in range(2, 4):
            t.append(2.0 * mul(t[-1]) - t[-2])
        z = sum(tk.reshape(n, b, 64) @ w.double()[64 * k:64 * (k + 1)] for k, tk in enumerate(t))
        (z * r.double()).sum().backward()
        return leaf.grad

    assert_close(got.cpu(), forced(False).cpu(), "bf16 mode GCN d vals (forced reference)", TOL)
    assert rel_err(got, forced(True)) > TOL             # negative control: fp32 T_{k-1} in the SDDMM


@pytest.mark.parametrize("streams", ["1", "0"])
def test_bf16_mode_model_value_grads_against_forced_and_unrounded(monkeypatch, streams):
    """ST_MGCN (M = 3, one handle on two branches) in the bf16-arithmetic mode: d vals, the loss, every parameter
    gradient and d obs within 1e-4 of the fp64 reference that rounds where the kernels round, forced with the step's own
    values at every rounding point and its ReLU masks; d vals within 2e-2 of the unrounded reference at the same masks."""
    from full_batch import gpu_step
    from model_cases import FullBatchRecorder
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_PLANES", 1)
    monkeypatch.setenv("STMGCN_GRAPH_STREAMS", streams)
    meta, model, handles, x, y = _model_case("chebyshev", 4)
    branch = [0, 1, 0]
    sups = [handles[i] for i in branch]
    with FullBatchRecorder() as rec:
        got = gpu_step(model, sups, x.clone(), y, want_obs=True)
    rec.check_intact()
    tapes = rec.take_tapes()
    params = {k: v.detach() for k, v in model.state_dict().items()}
    ref = S.ForcedValueReference(params, handles, branch, relu_masks=got["masks"], device=DEV)
    loss, grads, d_obs, d_vals = ref.value_grads(x, y, tapes)
    assert abs(got["loss"] - loss) <= TOL * abs(loss)
    for name, g in got["grads"].items():
        assert_close(g.cpu(), grads[name].cpu(), f"bf16 mode (forced) {name}")
    assert_close(got["d_obs"].cpu(), d_obs.cpu(), "bf16 mode (forced) d obs")
    unrounded = S.ForcedValueReference(params, handles, branch, rounding=False, relu_masks=got["masks"], device=DEV)
    d_vals_u = unrounded.value_grads(x, y)[3]
    for h, dv, du in zip(handles, d_vals, d_vals_u):
        assert_close(h.mats[0][2].grad.cpu(), dv[0].cpu(), "bf16 mode (forced) d vals")
        err = assert_close(h.mats[0][2].grad.cpu(), du[0].cpu(), "bf16 mode (unrounded) d vals", 2e-2)
        print(f"[bf16 mode support grads] d vals against the unrounded reference {err:.3e}")


@pytest.mark.parametrize("handle", [False, True])
def test_bf16_mode_runs_chebyshev_order_zero(monkeypatch, handle):
    """K = 0 (one support, T_0 = I, no graph) in the bf16-arithmetic mode: forward and backward run and match fp64."""
    import GCN
    import stmgcn_oracle as O
    from stmgcn_b200 import ops, synth
    monkeypatch.setattr(ops, "_PLANES", 1)
    meta = dict(META, k=0, m=1)
    torch.manual_seed(8)
    model = build_model(meta, DEV)
    a = synth.make_adjacency(meta["n"], 0, 0.3)
    pre = GCN.Adj_Preprocessor("chebyshev", 0)
    sup = (pre.process_sparse(a) if handle else pre.process(a)).to(DEV)
    x = _rand((meta["b"], meta["t"], meta["n"], meta["c"]), 13)
    y = _rand((meta["b"], meta["n"], meta["c"]), 14)
    out = model(obs_seq=x, sta_adj_list=[sup])
    nn.MSELoss()(out, y).backward()
    params = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    ref = O.dense_st_mgcn(params, x.double().cpu(), [torch.eye(meta["n"], dtype=torch.float64)[None]])
    assert_close(out.detach().cpu(), ref, "K = 0 bf16 mode output", 2e-2)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())


# ======================================================================================================================
# training, the frozen path, the captured step
# ======================================================================================================================
def test_training_through_process_sparse_under_fused_adam():
    """Learnable edge weights rebuilt by process_sparse every step, Adam(fused=True) on them and the model: after each
    step the output and the gradients match fp64 at the weights read back."""
    import GCN
    import stmgcn_oracle as O
    from stmgcn_b200 import synth
    meta, model, _, x, y = _model_case("chebyshev", 5)
    pre = GCN.Adj_Preprocessor("chebyshev", meta["k"])
    adjs = [synth.make_adjacency(meta["n"], g, 0.3).to(DEV) for g in range(3)]
    weights = [nn.Parameter(a.to_sparse_coo().coalesce().values().clone()) for a in adjs]
    idx = [a.to_sparse_coo().coalesce().indices() for a in adjs]
    opt = torch.optim.Adam(list(model.parameters()) + weights, lr=1e-2, fused=True)
    for step in range(3):
        opt.zero_grad()
        hs = [pre.process_sparse(torch.sparse_coo_tensor(i, wv, a.shape)) for i, wv, a in zip(idx, weights, adjs)]
        out = model(obs_seq=x, sta_adj_list=hs)
        loss = nn.MSELoss()(out, y)
        loss.backward()
        # fp64 at the weights as they are now (read back): dense process() on the dense adjacency built from them
        w64 = [wv.detach().double().cpu().clone().requires_grad_(True) for wv in weights]
        stacks = [pre.process(S.dense_matrix(meta["n"], i[0].cpu(), i[1].cpu(), wv)) for i, wv in zip(idx, w64)]
        params = {k: v.detach().cpu() for k, v in model.state_dict().items()}
        leaves = {k: v.double().requires_grad_(True) for k, v in params.items()}
        out64 = O.dense_st_mgcn(leaves, x.double().cpu(), stacks)
        ((out64 - y.double().cpu()) ** 2).mean().backward()
        assert_close(out.detach().cpu(), out64.detach(), f"step {step} output")
        for wv, w6 in zip(weights, w64):
            assert_close(wv.grad.cpu(), w6.grad, f"step {step} d edge weights")
        for k, prm in model.named_parameters():
            assert_close(prm.grad.cpu(), leaves[k].grad, f"step {step} {k}")
        opt.step()


def test_frozen_handles_launch_the_same_and_agree_within_the_atomic_spread():
    """No value requires grad: two runs on fixed handles launch the same kernels and agree within the last bits of the
    kernels' float-atomic sums (CHEB_LAUNCHES pins the launch count against the parent); learnable handles compute the
    same results within that spread and launch more (their backward's SDDMM and adjoint)."""
    from stmgcn_b200 import _lib
    from stmgcn_b200.graph import SparseSupports
    meta, model, handles, x, y = _model_case("chebyshev", 6)

    def run(hs):
        model.zero_grad()
        before = _lib.launch_count()
        out = model(obs_seq=x, sta_adj_list=[hs[0], hs[1], hs[0]])
        nn.MSELoss()(out, y).backward()
        torch.cuda.synchronize()
        return _lib.launch_count() - before, out.detach().clone(), [p.grad.clone() for p in model.parameters()]

    runs = [run([SparseSupports(h.mode, h.n, h.ks, [(rp, ci, v.detach().clone()) for rp, ci, v in h.mats])
                 for h in handles]) for _ in range(2)]
    assert runs[0][0] == runs[1][0]
    # two runs of the fixed handles differ only in the order of the kernels' float-atomic sums (the temporal pooling,
    # the backward's reductions): up to 1.5e-5 measured on an H100, so both comparisons use the suite's gradient bar
    spread = max([rel_err(runs[0][1], runs[1][1])] + [rel_err(a, b) for a, b in zip(runs[0][2], runs[1][2])])
    assert spread <= GRAD_TOL
    learn = run(handles)
    assert rel_err(learn[1], runs[0][1]) <= GRAD_TOL
    for a, b in zip(learn[2], runs[0][2]):
        assert rel_err(a, b) <= GRAD_TOL
    assert learn[0] > runs[0][0]


def test_graphed_step_refuses_learnable_handles():
    from stmgcn_b200.graphs import GraphedStep
    meta, model, handles, x, y = _model_case("chebyshev", 7)
    with pytest.raises(ValueError, match="require grad"):
        GraphedStep(model, nn.MSELoss(), x, y, [handles[0], handles[1], handles[0]])


# ======================================================================================================================
# the benchmarked size
# ======================================================================================================================
def test_fullsize_value_grads_every_window(monkeypatch):
    """cfg3 shapes (4096 regions, three learnable Chebyshev handles, K = 3, T = 12, 64 windows), every window carrying
    gradient: d vals within 1e-4 of fp64 evaluated in chunks of windows, the reference taking the step's own ReLU masks
    (a pre-activation within rounding distance of the kink must take the same branch in both); the worst is printed."""
    import GCN
    import STMGCN
    from stmgcn_b200 import synth
    w = synth.WORKLOADS["cfg3"]
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(**synth.model_kwargs(w)).to(DEV)
    pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
    handles = []
    for a in synth.make_adjacency_list(w):
        h = pre.process_sparse(a).to(DEV)
        h.mats = [(rp, ci, nn.Parameter(v.detach().clone())) for rp, ci, v in h.mats]
        handles.append(h)
    x, y = (t.to(DEV) for t in synth.make_inputs(w, seed=0))
    with S.record_relu_masks() as rec:
        out = model(obs_seq=x, sta_adj_list=handles)
    nn.MSELoss()(out, y).backward()
    params = {k: v.detach() for k, v in model.state_dict().items()}
    _, _, _, d_vals = S.model_reference(params, x, y, handles, list(range(len(handles))), device=DEV, window_chunk=8,
                                        masks=rec.masks)
    worst = 0.0
    for h, dv in zip(handles, d_vals):
        worst = max(worst, assert_close(h.mats[0][2].grad.cpu(), dv[0].cpu(), "cfg3 d vals"))
    print(f"[cfg3 support grads] worst d vals error {worst:.3e} over {x.shape[0]} windows")
