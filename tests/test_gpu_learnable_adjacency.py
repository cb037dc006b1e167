"""Learnable adjacencies on the H100: the normalisation entry points against the fp64 restatement for every kind (at
lambda_max = 2 and not), bit-identical reruns, NaN tracing, the C-ABI contract, the model with three learnable graphs
under ``Adam(fused=True)`` against dense fp64, agreement with ``process_sparse`` rebuilt per step, no host
synchronisation, and ``GraphedStep`` replays at the optimizer's weights."""
import pytest
import torch
from torch import nn

import learnable_adjacency_cases as LA
import support_grad_cases as S
from abi_harness import drive, run_captured, run_contract
from helpers import DEV, GRAD_TOL, TOL, build_model, rel_err

pytestmark = pytest.mark.gpu

ORDERS = {"chebyshev": 3, "localpool": 1, "random_walk_diffusion": 2}


def _adj(kind, a, lam=2.0, order=None):
    import GCN
    return GCN.Adj_Preprocessor(kind, ORDERS[kind] if order is None else order, lambda_max=lam).process_learnable(a).to(DEV)


def _values(adj):
    from stmgcn_b200 import ops
    return ops.AdjNorm.apply(adj.weight, adj.kind, adj.scale, *adj.pattern())


def _flat(v):
    return torch.cat(list(v)) if isinstance(v, tuple) else v


GRAPHS = {"sym37": dict(n=37, directed=False), "directed61": dict(n=61, directed=True),
          "hubs1000": dict(n=1000, directed=True, density=0.01)}


# ======================================================================================================================
# the entry points
# ======================================================================================================================
@pytest.mark.parametrize("graph", list(GRAPHS))
@pytest.mark.parametrize("lam", [2.0, 1.37])
@pytest.mark.parametrize("kind", LA.KINDS)
def test_normalisation_and_gradient_against_fp64(kind, lam, graph):
    g = GRAPHS[graph]
    # a sink (an empty row of a directed graph) has D^-1/2 = inf: Inf values in its column, in fp64 as here (traced below)
    a = LA.graph(g["n"], 11, directed=g["directed"], density=g.get("density", 0.25),
                 isolated=kind == "random_walk_diffusion" or not g["directed"]).float()
    adj = _adj(kind, a, lam)
    vals = _values(adj)
    w64 = adj.weight.detach().double().cpu().requires_grad_(True)
    ref = LA.module_values64(adj, w64)
    assert rel_err(_flat(vals), _flat(ref)) <= 2e-6
    gen = torch.Generator().manual_seed(3)
    gs = tuple(torch.randn(v.shape, generator=gen) for v in (ref if isinstance(ref, tuple) else (ref,)))
    (dw,) = torch.autograd.grad(vals, adj.weight, tuple(x.to(DEV) for x in gs) if len(gs) > 1 else gs[0].to(DEV))
    (dw64,) = torch.autograd.grad(ref, w64, tuple(x.double() for x in gs) if len(gs) > 1 else gs[0].double())
    assert rel_err(dw, dw64) <= 1e-5
    # two runs, bit for bit
    vals2 = _values(adj)
    (dw2,) = torch.autograd.grad(vals2, adj.weight, tuple(x.to(DEV) for x in gs) if len(gs) > 1 else gs[0].to(DEV))
    assert torch.equal(_flat(vals2), _flat(vals)) and torch.equal(dw2, dw)


@pytest.mark.parametrize("kind", LA.KINDS)
def test_nan_weight_is_non_finite_exactly_where_fp64_is(kind):
    a = LA.graph(53, 5, directed=kind == "random_walk_diffusion").float()
    adj = _adj(kind, a, 1.5)
    gen = torch.Generator().manual_seed(9)
    n_out = 2 if kind == "random_walk_diffusion" else 1
    gs = [torch.randn(adj.colidx.numel(), generator=gen) for _ in range(n_out)]

    def run(w):
        with torch.no_grad():
            adj.weight.copy_(w)
        v = _values(adj)
        (d,) = torch.autograd.grad(v, adj.weight, tuple(x.to(DEV) for x in gs) if n_out > 1 else gs[0].to(DEV))
        return _flat(v).cpu(), d.cpu()

    w0 = adj.weight.detach().clone()
    clean_v, clean_d = run(w0)
    for e in (0, 7, int(w0.numel()) - 1):
        w = w0.clone()
        w[e] = float("nan")
        v, d = run(w)
        w64 = w.double().cpu().requires_grad_(True)
        ref = LA.module_values64(adj, w64)
        (d64,) = torch.autograd.grad(ref, w64, tuple(x.double() for x in gs) if n_out > 1 else gs[0].double())
        for got, want, clean, what in ((v, _flat(ref).detach(), clean_v, "values"), (d, d64, clean_d, "d w")):
            bad = ~torch.isfinite(got)
            assert torch.equal(bad, ~torch.isfinite(want)), f"{kind} NaN at {e}: {what} non-finite elsewhere than fp64"
            assert torch.equal(got[~bad], clean[~bad]), f"{kind} NaN at {e}: {what} finite entries moved"
            assert bad.any()


def _norm_calls(kind, lam):
    """stmgcn_adj_norm_fwd then stmgcn_adj_norm_bwd on guarded buffers, workspaces poisoned, against fp64."""
    from abi_harness import Buf, Call
    from helpers import lib
    from stmgcn_b200 import ops
    a = LA.graph(45, 2, directed=kind == "random_walk_diffusion").float()
    adj = _adj(kind, a, lam)
    n, nnz, nnz_w = adj.n, adj.colidx.numel(), adj.weight.numel()
    diff = kind == "random_walk_diffusion"
    ig = 0x7FA5A5A5
    pat = {k: Buf("in", t, guard=ig) for k, t in zip(("rowptr", "colidx", "rowptr_t", "colidx_t", "perm_t", "widx"),
                                                      adj.pattern()) if t is not None}
    w = adj.weight.detach().clone()
    w64 = w.double().cpu().requires_grad_(True)
    ref = LA.module_values64(adj, w64)
    opt = lambda b, k: b[k].p if k in b else None      # noqa: E731

    def head(b):
        return (ops.NORM_KINDS[kind], n, b["rowptr"].p, b["colidx"].p, b["rowptr_t"].p, b["colidx_t"].p, b["perm_t"].p,
                nnz, opt(b, "widx"), b["w"].p, nnz_w, adj.scale)

    b = dict(pat, w=Buf("in", w), work=Buf("ws", shape=(2 * n,)), vals=Buf("out", shape=(nnz,)))
    if diff:
        b["vals_t"] = Buf("out", shape=(nnz,))

    def ref_fwd(res):
        got = torch.cat([res["vals_t"], res["vals"]]) if diff else res["vals"]
        assert rel_err(got, _flat(ref)) <= 2e-6, f"adj_norm_fwd {kind}"

    yield Call("adj_norm_fwd", b, lambda st: lib().stmgcn_adj_norm_fwd(
        *head(b), b["work"].p, 2 * n, b["vals"].p, opt(b, "vals_t"), st), ref_fwd, 2)
    gen = torch.Generator().manual_seed(4)
    g = [torch.randn(nnz, generator=gen) for _ in range(2 if diff else 1)]
    c = dict(pat, w=Buf("in", w), dvals=Buf("in", g[-1]), work=Buf("ws", shape=(3 * n + nnz,)),
             dw=Buf("out", shape=(nnz_w,)))
    if diff:
        c["dvals_t"] = Buf("in", g[0])

    def ref_bwd(res):
        (d64,) = torch.autograd.grad(ref, w64, tuple(x.double() for x in g) if diff else g[0].double(), retain_graph=True)
        assert rel_err(res["dw"], d64) <= 1e-5, f"adj_norm_bwd {kind}"

    yield Call("adj_norm_bwd", c, lambda st: lib().stmgcn_adj_norm_bwd(
        *head(c), c["dvals"].p, opt(c, "dvals_t"), c["work"].p, 3 * n + nnz, c["dw"].p, st), ref_bwd, 3)


@pytest.mark.parametrize("lam", [2.0, 1.4])
@pytest.mark.parametrize("kind", LA.KINDS)
def test_adj_norm_abi_contract(kind, lam):
    drive(_norm_calls(kind, lam), run_contract)
    drive(_norm_calls(kind, lam), run_captured)


# ======================================================================================================================
# the model
# ======================================================================================================================
META = dict(n=24, m=3, k=2, t=4, b=3, c=1, hid=64, layers=2, gcn_hid=64)


def _model_case(kind, seed=0, lam=1.6):
    meta = dict(META, kernel_type=kind, k=1 if kind == "localpool" else META["k"])
    torch.manual_seed(seed)
    model = build_model(meta, DEV)
    a = [LA.graph(meta["n"], 20 + g, directed=kind == "random_walk_diffusion", density=0.3).float() for g in range(2)]
    adjs = [_adj(kind, x, lam, meta["k"]) for x in a]
    gen = torch.Generator().manual_seed(seed + 11)
    x = torch.randn(meta["b"], meta["t"], meta["n"], meta["c"], generator=gen).to(DEV)
    y = torch.randn(meta["b"], meta["n"], meta["c"], generator=gen).to(DEV)
    return meta, model, adjs, x, y


def _reference(model, adjs, branch, x, y, masks):
    import stmgcn_oracle as O
    params = {k: v.detach().double().cpu().requires_grad_(True) for k, v in model.state_dict().items()}
    ws = [a.weight.detach().double().cpu().requires_grad_(True) for a in adjs]
    stacks = [LA.module_stack64(a, w) for a, w in zip(adjs, ws)]
    out = O.dense_st_mgcn(params, x.double().cpu(), [stacks[i] for i in branch], True, masks=[m.cpu() for m in masks])
    loss = ((out - y.double().cpu()) ** 2).mean()
    loss.backward()
    return out.detach(), loss.item(), {k: v.grad for k, v in params.items()}, [w.grad for w in ws]


def _check_step(model, adjs, branch, x, y, what, tol=TOL):
    model.zero_grad(set_to_none=False)
    for a in adjs:
        a.weight.grad = None
    with S.record_relu_masks() as rec:
        out = model(obs_seq=x, sta_adj_list=[adjs[i] for i in branch])
    loss = nn.MSELoss()(out, y)
    loss.backward()
    o_ref, l_ref, g_ref, dw_ref = _reference(model, adjs, branch, x, y, rec.masks)
    assert rel_err(out, o_ref) <= tol, f"{what} output"
    assert abs(loss.item() - l_ref) <= tol * abs(l_ref), what
    for name, prm in model.named_parameters():
        assert rel_err(prm.grad, g_ref[name]) <= tol, f"{what} {name}"
    for i, a in enumerate(adjs):
        assert rel_err(a.weight.grad, dw_ref[i]) <= tol, f"{what} d weight {i}"


@pytest.mark.parametrize("path", ["tc", "fma"])
@pytest.mark.parametrize("streams", ["1", "0"])
@pytest.mark.parametrize("kind", LA.KINDS)
def test_st_mgcn_three_learnable_graphs_under_fused_adam(monkeypatch, path, streams, kind):
    """M = 3 on two modules (the first feeds two branches), three Adam(fused=True) steps: output, every parameter
    gradient and d weight within 1e-4 of dense fp64 at the current weights."""
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_LSTM_PATH", path)
    monkeypatch.setenv("STMGCN_GRAPH_STREAMS", streams)
    _, model, adjs, x, y = _model_case(kind)
    opt = torch.optim.Adam(list(model.parameters()) + [p for a in adjs for p in a.parameters()], lr=1e-2, fused=True)
    w_init = adjs[0].weight.detach().clone()
    for step in range(3):
        _check_step(model, adjs, [0, 0, 1], x, y, f"{kind} path={path} streams={streams} step {step}")
        opt.step()
    assert not torch.equal(adjs[0].weight.detach(), w_init), "the optimizer moved no edge weight"


def test_zero_sum_degrees_with_stored_entries_are_nan_as_in_fp64():
    """Diffusion with a column and a row of stored zeros: the kernels' values and d w are non-finite exactly where the
    fp64 restatement is (torch's ``0 * -inf`` in the degree term), and within the bars elsewhere."""
    adj = _adj("random_walk_diffusion", LA.zero_sum_graph())
    vals = _values(adj)
    w64 = adj.weight.detach().double().cpu().requires_grad_(True)
    ref = LA.module_values64(adj, w64)
    gen = torch.Generator().manual_seed(6)
    gs = tuple(torch.randn(v.shape, generator=gen) for v in ref)
    (dw,) = torch.autograd.grad(vals, adj.weight, tuple(x.to(DEV) for x in gs))
    (dw64,) = torch.autograd.grad(ref, w64, tuple(x.double() for x in gs))
    for got, want, bar in ((_flat(vals), _flat(ref).detach(), 2e-6), (dw, dw64, 1e-5)):
        bad = ~torch.isfinite(want)
        assert torch.equal(~torch.isfinite(got.cpu()), bad)
        assert rel_err(got.cpu()[~bad], want[~bad]) <= bar
    assert bool(torch.isnan(dw64).any())


@pytest.mark.parametrize("streams", ["1", "0"])
@pytest.mark.parametrize("kind", ["chebyshev", "random_walk_diffusion"])
def test_bf16_mode_model_against_forced_reference(monkeypatch, kind, streams):
    """ST_MGCN (M = 3, one module on two branches) in the bf16-arithmetic mode: the loss, the output, every parameter
    gradient and d weight within 1e-4 of the fp64 reference that rounds where the kernels round, forced with the step's
    own values and ReLU masks.  The reference's d vals of the supports' values are carried to d weight through the fp64
    restatement of the normalisation.  (Chebyshev-chain kinds: the bf16 gathers run on the recurrence chains only.)"""
    from full_batch import gpu_step
    from model_cases import FullBatchRecorder
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_PLANES", 1)
    monkeypatch.setenv("STMGCN_GRAPH_STREAMS", streams)
    _, model, adjs, x, y = _model_case(kind, seed=4)
    branch = [0, 1, 0]
    for a in adjs:
        a.weight.grad = None
    with FullBatchRecorder() as rec:
        got = gpu_step(model, [adjs[i] for i in branch], x.clone(), y, want_obs=True)
    rec.check_intact()
    tapes = rec.take_tapes()
    params = {k: v.detach() for k, v in model.state_dict().items()}
    handles = [a.supports() for a in adjs]               # the values the kernels multiplied by
    ref = S.ForcedValueReference(params, handles, branch, relu_masks=got["masks"], device=DEV)
    loss, grads, d_obs, d_vals = ref.value_grads(x, y, tapes)
    assert abs(got["loss"] - loss) <= TOL * abs(loss)
    for name, g in got["grads"].items():
        assert rel_err(g, grads[name]) <= TOL, f"bf16 mode (forced) {kind} {name}"
    assert rel_err(got["d_obs"], d_obs) <= TOL, f"bf16 mode (forced) {kind} d obs"
    for a, dv in zip(adjs, d_vals):
        w64 = a.weight.detach().double().cpu().requires_grad_(True)
        v64 = LA.module_values64(a, w64)
        v64 = v64 if isinstance(v64, tuple) else (v64,)
        (dw64,) = torch.autograd.grad(v64, w64, tuple(d.double().cpu() for d in dv))
        assert rel_err(a.weight.grad, dw64) <= TOL, f"bf16 mode (forced) {kind} d weight"


@pytest.mark.parametrize("kind", LA.KINDS)
def test_module_agrees_with_process_sparse_rebuilt_per_step(kind):
    import GCN
    _, model, adjs, x, y = _model_case(kind, seed=3)
    pre = GCN.Adj_Preprocessor(kind, 1 if kind == "localpool" else META["k"], lambda_max=1.6)

    def run(sups_fn, weights):
        model.zero_grad(set_to_none=False)
        for w in weights:
            w.grad = None
        loss = nn.MSELoss()(model(obs_seq=x, sta_adj_list=sups_fn()), y)
        loss.backward()
        return loss.item(), {k: p.grad.clone() for k, p in model.named_parameters()}, [w.grad.clone() for w in weights]

    ws = [nn.Parameter(a.weight.detach().clone()) for a in adjs]
    idx = [torch.stack(a.edges()) for a in adjs]
    l1, g1, d1 = run(lambda: [adjs[i] for i in (0, 1, 0)], [a.weight for a in adjs])
    l2, g2, d2 = run(lambda: [pre.process_sparse(torch.sparse_coo_tensor(idx[i], ws[i], (a.n, a.n)))
                              for i, a in zip((0, 1, 0), [adjs[0], adjs[1], adjs[0]])], ws)
    assert abs(l1 - l2) <= GRAD_TOL * abs(l2)
    for k in g1:
        assert rel_err(g1[k], g2[k]) <= GRAD_TOL, k
    for a, b in zip(d1, d2):
        assert rel_err(a, b) <= GRAD_TOL


@pytest.mark.parametrize("kind", LA.KINDS)
def test_forward_and_backward_never_synchronise(kind):
    adj = _adj(kind, LA.graph(300, 6, directed=True, density=0.05).float(), 1.5)
    sset = adj()                         # the first call converts the structure (one check, with a host sync)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sset = adj()
        (d,) = torch.autograd.grad(sum(v.sum() for v in sset.values), adj.weight)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert d.shape == adj.weight.shape


def test_graphed_step_replays_match_eager_at_the_optimizers_weights():
    from stmgcn_b200.graphs import GraphedStep
    _, model, adjs, x, y = _model_case("chebyshev", seed=5)
    sups = [adjs[0], adjs[1], adjs[0]]
    crit = nn.MSELoss()
    opt = torch.optim.Adam(list(model.parameters()) + [p for a in adjs for p in a.parameters()], lr=1e-2, fused=True)
    step = GraphedStep(model, crit, x, y, sups)
    assert {id(p) for p in step.bucket.params} >= {id(a.weight) for a in adjs}
    for i in range(3):
        loss = step(x, y).item()
        replay = step.bucket.flat.clone()
        step.bucket.zero_()
        eager = crit(model(obs_seq=x, sta_adj_list=sups), y)
        eager.backward()
        assert abs(loss - eager.item()) <= GRAD_TOL * abs(eager.item()), f"step {i}"
        assert rel_err(replay, step.bucket.flat) <= GRAD_TOL, f"step {i}"
        assert adjs[0].weight.grad.abs().max() > 0
        opt.step()
    # the short last batch runs eagerly
    short = step(x[:2], y[:2]).item()
    step.bucket.zero_()
    want = crit(model(obs_seq=x[:2], sta_adj_list=sups), y[:2]).item()
    assert abs(short - want) <= GRAD_TOL * abs(want)
