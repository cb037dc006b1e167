"""The graph convolutions against fp64 for every way supports reach the kernels, and the support contract of the handles
and of captured steps.

* A. every support route -- dense ``process`` stack (Chebyshev), dense ``localpool``, a hand-made non-polynomial dense
  stack, a dense ``2K+1`` diffusion stack, a ``ChebSupports`` handle, a two-chain diffusion handle, a generic
  ``SparseSupports`` from hand-made CSR, K = 0 -- through ``ops.build_stack`` / ``ops.adjoint_stack_`` and the ``GCN``
  module, with the tensor-core (p = q = 64) and the FFMA (p = q = 12) projection, against fp64 dense references built
  from the stack as the caller holds it, and the adjoint identity <stack(X), U> = <X, adjoint(U)>;
* B. hand-made CSR at the edges of the SpMM's gather loop (degrees 0..9, hub rows and columns, shuffled columns,
  repeated entries, stored +-0), alone and in ``ST_MGCN`` against the fp64 sparse oracles;
* C. a malformed CSR raises ``ValueError`` before any kernel launches;
* D. in-place edits of dense stacks and of handles are seen by the forward and the backward alike; negative control:
  the handles' behaviour before they copied their CSR and rebuilt on a version change;
* E. ``graphs.GraphedStep`` holds the support sets it captured and refuses to replay after a support edit;
* F. the Chebyshev classifier's tolerance: results on a stack just inside it are still those of the stack as given.

Bars: SpMM-level results (``build_stack`` slices, ``adjoint_stack_``) 1e-5, the GCN module 2e-5 forward / 5e-5 gradients
(the kernel bars of ``test_gpu_exact_kernels.py``), models 1e-4 (``helpers.TOL``), all max-norm relative.  The adjoint
identity's residual is held relative to sum_k <|S_k| |X|, |U_k|> at ``ADJ_TOL``.

Measured on an H100 80GB HBM3 (700 W): SpMM-level errors at most 4.2e-7 (diffusion_dense), GCN module 3.1e-6 forward and
1.2e-6 gradients (the 3xTF32 projection; 4.2e-7 / 2.8e-7 with FFMA), models at most 1.8e-6, a captured step 8.7e-6; the
adjoint identity's residual at most 9.3e-10 over every route and edit, while a handle whose backward kept the
pre-edit matrix left 6.9e-4 .. 7.4e-3 (gradients 0.54 .. 1.6 off).
"""
import gc
import weakref

import numpy as np
import pytest
import torch
from torch import nn

import diffusion_oracle as D
import stmgcn_oracle as O
from helpers import DEV, FWD_TOL, GRAD_TOL, TOL, rel_err
from kernel_cases import MALFORMED, handmade_csr, malformed, scipy_of

pytestmark = pytest.mark.gpu
SPMM_TOL = 1e-5
ADJ_TOL = 1e-8           # 10x the largest residual measured (9.3e-10); a forward and backward of different matrices: >= 6.9e-4
N_ROUTE, B_ROUTE = 200, 3


def dense64(sup):
    """The fp64 dense stack of ``sup`` as it is now: a dense stack's values, or the matrices a handle stores now (its
    chains' polynomials, or its generic supports), repeated entries summed."""
    from stmgcn_b200.graph import SparseSupports
    if not isinstance(sup, SparseSupports):
        return sup.detach().double().cpu()
    mats = [scipy_of(*m, sup.n) for m in sup.mats]
    if sup.mode == "generic":
        return torch.from_numpy(np.stack([m.toarray() for m in mats]))
    if sup.ks == 1:
        return torch.eye(sup.n, dtype=torch.float64)[None]
    return O.chain_stack_dense([torch.from_numpy(m.toarray()) for m in mats], (sup.ks - 1) // len(mats))


ROUTES = {  # name: (mode, number of graphs of the support set)
    "cheb_dense": ("cheb", 1), "localpool_dense": ("generic", 1), "handmade_dense": ("generic", 3),
    "diffusion_dense": ("generic", 5), "cheb_handle": ("cheb", 1), "diffusion_handle": ("cheb", 2),
    "generic_handle": ("generic", 3), "k0": ("cheb", 0)}


def route_supports(name, n=N_ROUTE):
    """The support stack of one route, on the device."""
    import GCN
    from stmgcn_b200 import synth
    from stmgcn_b200.graph import SparseSupports
    adj, dadj = synth.make_adjacency(n, 0, 0.05), synth.make_directed_adjacency(n, 0, 0.05)
    if name == "cheb_dense":
        return GCN.Adj_Preprocessor("chebyshev", 3).process(adj).to(DEV)
    if name == "localpool_dense":
        return GCN.Adj_Preprocessor("localpool", 1).process(adj).to(DEV)
    if name == "handmade_dense":
        return torch.stack([torch.from_numpy(scipy_of(*handmade_csr(n, s), n).toarray()).float()
                            for s in (1, 2, 3)]).to(DEV)
    if name == "diffusion_dense":
        return D.diffusion_supports_dense(dadj, 2).to(DEV)
    if name == "cheb_handle":
        return GCN.Adj_Preprocessor("chebyshev", 3).process_sparse(adj).to(DEV)
    if name == "diffusion_handle":
        return GCN.Adj_Preprocessor("random_walk_diffusion", 2).process_sparse(dadj).to(DEV)
    if name == "generic_handle":
        return SparseSupports("generic", n, 3, [handmade_csr(n, s) for s in (11, 12, 13)]).to(DEV)
    if name == "k0":
        return GCN.Adj_Preprocessor("chebyshev", 0).process(adj).to(DEV)
    raise KeyError(name)


def stack_and_adjoint(sset, s64, x, u):
    """``ops.build_stack`` and ``ops.adjoint_stack_`` on (x, u) against fp64: (errors, adjoint-identity residual)."""
    from stmgcn_b200 import ops
    ks, n = s64.shape[0], s64.shape[1]
    stack = ops.build_stack(sset, x)
    dx = ops.adjoint_stack_(sset, u.clone())
    torch.cuda.synchronize()
    x64, u64 = x.double().cpu().reshape(n, -1), u.double().cpu().reshape(ks, n, -1)
    st64, dx64 = stack.double().cpu().reshape(ks, n, -1), dx.double().cpu().reshape(n, -1)
    errs = {f"S_{k} X": rel_err(st64[k], s64[k] @ x64) for k in range(ks)}
    errs["adjoint"] = rel_err(dx64, sum(s64[k].t() @ u64[k] for k in range(ks)))
    lhs = float((st64 * u64).sum())
    rhs = float((x64 * dx64).sum())
    scale = float(sum(((s64[k].abs() @ x64.abs()) * u64[k].abs()).sum() for k in range(ks)))
    return errs, abs(lhs - rhs) / scale


def gcn_vs_fp64(sup, s64, p, seed, relu=True):
    """The ``GCN`` module (K = Ks supports, p -> p) on ``sup``: (forward error, {dX, dW, db: error}) against
    ``O.dense_gcn`` on ``s64`` in fp64, with the kernel's ReLU mask."""
    import GCN
    ks, n = s64.shape[0], s64.shape[1]
    torch.manual_seed(seed)
    layer = GCN.GCN(K=ks, input_dim=p, hidden_dim=p, activation=nn.ReLU if relu else None).to(DEV)
    with torch.no_grad():
        layer.b.uniform_(-0.1, 0.1)
    gen = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(B_ROUTE, n, p, generator=gen)
    probe = torch.randn(B_ROUTE, n, p, generator=gen)
    xd = x.to(DEV).requires_grad_(True)
    out = layer(sup, xd)
    (out * probe.to(DEV)).sum().backward()
    torch.cuda.synchronize()
    x64 = x.double().requires_grad_(True)
    w64 = layer.W.detach().double().cpu().requires_grad_(True)
    b64 = layer.b.detach().double().cpu().requires_grad_(True)
    z = O.dense_gcn(s64, x64, w64, b64, relu=False)
    mask = (out.detach().cpu() > 0).double() if relu else 1.0
    ref = z * mask
    grads = torch.autograd.grad((ref * probe.double()).sum(), [x64, w64, b64])
    gerrs = {"dX": rel_err(xd.grad, grads[0]), "dW": rel_err(layer.W.grad, grads[1]), "db": rel_err(layer.b.grad, grads[2])}
    return rel_err(out, ref), gerrs


# ======================================================================================================================
# A. every support route
# ======================================================================================================================
@pytest.mark.parametrize("p", [64, 12])
@pytest.mark.parametrize("name", sorted(ROUTES))
def test_every_support_route_matches_fp64(name, p):
    """The route's support set has the expected mode and graphs; build_stack's every slice and adjoint_stack_ at 1e-5,
    the adjoint identity at ADJ_TOL, the GCN module's output at 2e-5 and dX / dW / db at 5e-5."""
    from stmgcn_b200.graph import supports_from_dense
    sup = route_supports(name)
    mode, n_graphs = ROUTES[name]
    sset = supports_from_dense(sup)
    assert (sset.mode, len(sset.graphs)) == (mode, n_graphs)
    s64 = dense64(sup)
    ks = s64.shape[0]
    gen = torch.Generator().manual_seed(p)
    x = torch.randn(N_ROUTE, B_ROUTE, p, generator=gen).to(DEV)
    u = torch.randn(ks, N_ROUTE, B_ROUTE, p, generator=gen).to(DEV)
    errs, resid = stack_and_adjoint(sset, s64, x, u)
    out_err, gerrs = gcn_vs_fp64(sup, s64, p, seed=7 * p + ks)
    worst = max(errs, key=errs.get)
    print(f"route {name} p={p}: worst SpMM-level {errs[worst]:.2e} ({worst}), adjoint identity {resid:.2e}, "
          f"GCN out {out_err:.2e}, " + ", ".join(f"{k} {v:.2e}" for k, v in gerrs.items()))
    assert errs[worst] <= SPMM_TOL, errs
    assert resid <= ADJ_TOL, resid
    assert out_err <= FWD_TOL, out_err
    assert max(gerrs.values()) <= GRAD_TOL, gerrs


# ======================================================================================================================
# B. hand-made CSR at the edges of the gather loop
# ======================================================================================================================
@pytest.mark.parametrize("f", [40, 7])
@pytest.mark.parametrize("transpose", [False, True])
def test_spmm_on_handmade_csr_matches_scipy(transpose, f):
    """``ops.spmm_step`` with the CSR (A X) and the CSR^T (A^T U) of a hand-made matrix (degrees 0..9, a hub row and a
    hub column, shuffled columns, repeated entries, stored +-0): f = 40 the float4 kernel, f = 7 the scalar one, against
    scipy in fp64 at 1e-5; rows without entries, if any, are exactly 0."""
    from stmgcn_b200 import ops
    from stmgcn_b200.graph import GraphHandle
    n = 300
    rp, ci, v = handmade_csr(n, 5)
    a = scipy_of(rp, ci, v, n)
    g = GraphHandle.from_csr(n, rp.to(DEV), ci.to(DEV), v.to(DEV))
    x = torch.randn(n, f, generator=torch.Generator().manual_seed(f)).to(DEV)
    y = torch.full_like(x, float("nan"))
    ops.spmm_step(g, transpose, 1.0, x, 0.0, None, 0.0, None, y)
    torch.cuda.synchronize()
    op = a.T.tocsr() if transpose else a
    ref = op @ x.double().cpu().numpy()
    err = O.max_rel_err(y.double().cpu().numpy(), ref)
    empty = np.flatnonzero(np.diff(op.indptr) == 0)
    print(f"hand-made CSR transpose={transpose} f={f}: {err:.2e}, {len(empty)} empty rows")
    assert bool((y[torch.from_numpy(empty).to(DEV)] == 0).all())
    assert err <= SPMM_TOL, err


def _model(ks, n, relu=True, hid=32, gcn_hid=16, m=1, t=6):
    import STMGCN
    meta = dict(n=n, m=m, t=t, b=3, c=1, hid=hid, layers=2, gcn_hid=gcn_hid)
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(M=m, seq_len=t, n_nodes=n, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=2,
                           gcn_hidden_dim=gcn_hid, sta_kernel_config={"kernel_type": "chebyshev", "K": ks - 1},
                           gconv_use_bias=True, gconv_activation=nn.ReLU if relu else None)
    params = O.init_params(m, t, 1, hid, 2, gcn_hid, ks, seed=ks + n)
    model.load_state_dict(params)
    gen = torch.Generator().manual_seed(n)
    x = torch.randn(meta["b"], t, n, 1, generator=gen)
    y = torch.randn(meta["b"], n, 1, generator=gen)
    return model.to(DEV), params, x, y


@pytest.mark.parametrize("kind", ["chebyshev", "two_chains"])
def test_model_on_handmade_csr_matches_sparse_oracle(kind):
    """ST_MGCN (two graphs) on handles made from hand-made CSR -- a ``ChebSupports`` (K = 2) or a two-chain
    ``SparseSupports`` (2K+1 = 5) -- forward, loss and every gradient against ``O.SparseOracle`` / ``D.ChainOracle``
    in fp64 at 1e-4."""
    from stmgcn_b200.graph import ChebSupports, SparseSupports
    n = 150
    if kind == "chebyshev":
        ks = 3
        sups = [ChebSupports(n, ks, *handmade_csr(n, 20 + g)) for g in range(2)]
    else:
        ks = 5
        sups = [SparseSupports("cheb", n, ks, [handmade_csr(n, 30 + g), handmade_csr(n, 40 + g, hub_row=5, hub_col=7)])
                for g in range(2)]
    chains = [[scipy_of(*m, n) for m in s.mats] for s in sups]
    model, params, x, y = _model(ks, n, m=2)
    out = model(obs_seq=x.to(DEV), sta_adj_list=[s.to(DEV) for s in sups])
    loss = nn.MSELoss()(out, y.to(DEV))
    loss.backward()
    orc = D.ChainOracle({k: v.numpy() for k, v in params.items()}, chains, ks, dtype=np.float64)
    o_ref, l_ref, g_ref = orc.loss_and_grads(x.numpy(), y.numpy())
    errs = {"out": O.max_rel_err(out.detach().cpu().numpy(), o_ref)}
    errs.update({k: O.max_rel_err(p.grad.cpu().numpy(), g_ref[k]) for k, p in model.named_parameters()})
    worst = max(errs, key=errs.get)
    print(f"hand-made CSR model ({kind}): forward {errs['out']:.2e}, worst {errs[worst]:.2e} ({worst})")
    assert errs[worst] <= TOL, errs
    assert abs(loss.item() - l_ref) <= 1e-5 * max(1.0, abs(l_ref))


# ======================================================================================================================
# C. a malformed CSR never reaches a kernel
# ======================================================================================================================
@pytest.mark.parametrize("case", [c for c in MALFORMED if c != "dtype"] + ["mixed_devices"])
def test_malformed_handle_raises_before_any_launch(case):
    """A ``ChebSupports`` with a malformed CSR: ``support_set()`` and a model forward raise ``ValueError`` naming the
    fault, and the library's launch count is unchanged (nothing ran, the CSR never reached a kernel).  (A dtype fault
    cannot reach here: the handle converts its tensors to int32 / float32.)"""
    from stmgcn_b200 import _lib
    from stmgcn_b200.graph import ChebSupports
    if case == "mixed_devices":
        n, msg = 40, "mixed devices"
        rp, ci, v = handmade_csr(n, 7)
        bad = ChebSupports(n, 3, rp.to(DEV), ci.to(DEV), v)
    else:
        n, rp, ci, v, msg = malformed(case)
        bad = ChebSupports(n, 3, rp.to(DEV), ci.to(DEV), v.to(DEV))
    model, _, x, _ = _model(3, n)
    xd = x.to(DEV)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match=msg):
        bad.support_set()
    with pytest.raises(ValueError, match=msg):
        model(obs_seq=xd, sta_adj_list=[bad])
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0


# ======================================================================================================================
# D. in-place edits are seen by both directions
# ======================================================================================================================
EDITS = {   # name: (support route, the edit)
    "dense_mul": ("cheb_dense", lambda s: s.mul_(0.5)),
    "dense_zero_slice": ("cheb_dense", lambda s: s[2].zero_()),                 # cheb -> generic
    "cheb_vals_mul": ("cheb_handle", lambda s: s.vals.mul_(0.5)),
    "cheb_vals_setitem": ("cheb_handle", lambda s: s.vals.__setitem__(slice(None, None, 3), -0.3)),
    "cheb_vals_copy": ("cheb_handle", lambda s: s.vals.copy_(torch.flip(s.vals, [0]))),
    "diffusion_second_chain": ("diffusion_handle", lambda s: s.mats[1][2].mul_(-0.7)),
}
HANDLE_EDITS = [k for k, (r, _) in EDITS.items() if r.endswith("handle")]
N_EDIT = 60


def dense_reference(params, sups64, x, y):
    """Loss, output and every parameter gradient plus d obs of ST_MGCN on the dense fp64 stacks ``sups64``."""
    leaves = {k: v.detach().double().clone().requires_grad_(True) for k, v in params.items()}
    obs = x.double().requires_grad_(True)
    out = O.dense_st_mgcn(leaves, obs, sups64)
    loss = torch.mean((out - y.double()) ** 2)
    grads = torch.autograd.grad(loss, list(leaves.values()) + [obs])
    g = dict(zip(list(leaves) + ["d obs"], grads))
    return out.detach(), loss.item(), g


def model_errors(model, sup, params, x, y):
    """One forward + backward of ``model`` on ``sup`` against :func:`dense_reference` on the stack as it is now."""
    model.zero_grad(set_to_none=True)
    xd = x.to(DEV).requires_grad_(True)
    out = model(obs_seq=xd, sta_adj_list=[sup])
    loss = nn.MSELoss()(out, y.to(DEV))
    loss.backward()
    o_ref, l_ref, g_ref = dense_reference(params, [dense64(sup)], x, y)
    errs = {"out": rel_err(out, o_ref), "d obs": rel_err(xd.grad, g_ref["d obs"])}
    errs.update({k: rel_err(p.grad, g_ref[k]) for k, p in model.named_parameters()})
    return errs


def _edit_case(edit):
    route, fn = EDITS[edit]
    sup = route_supports(route, N_EDIT)
    model, params, x, y = _model(dense64(sup).shape[0], N_EDIT)
    return sup, fn, model, params, x, y


def _identity_residual(sup, seed):
    from stmgcn_b200.graph import supports_from_dense
    s64 = dense64(sup)
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(N_EDIT, 2, 16, generator=gen).to(DEV)
    u = torch.randn(s64.shape[0], N_EDIT, 2, 16, generator=gen).to(DEV)
    return stack_and_adjoint(supports_from_dense(sup), s64, x, u)


@pytest.mark.parametrize("edit", sorted(EDITS))
def test_in_place_edit_is_seen_by_forward_and_backward(edit):
    """A forward and backward, then one in-place edit of the supports, then a forward and backward again: output, every
    parameter gradient and d obs at 1e-4 of the fp64 model on the edited stack, and the SpMM-level stack, adjoint and
    adjoint identity on the edited support set at their bars."""
    sup, fn, model, params, x, y = _edit_case(edit)
    before = dense64(sup)
    errs0 = model_errors(model, sup, params, x, y)
    with torch.no_grad():
        fn(sup)
    after = dense64(sup)
    assert float((after - before).abs().max()) > 0.1 * float(before.abs().max()), "the edit changed nothing"
    errs = model_errors(model, sup, params, x, y)
    spmm, resid = _identity_residual(sup, 3)
    worst = max(errs, key=errs.get)
    print(f"edit {edit}: before the edit worst {max(errs0.values()):.2e}; after: forward {errs['out']:.2e}, worst "
          f"{errs[worst]:.2e} ({worst}), SpMM-level {max(spmm.values()):.2e}, adjoint identity {resid:.2e}")
    assert max(errs0.values()) <= TOL, errs0
    assert errs[worst] <= TOL, errs
    assert max(spmm.values()) <= SPMM_TOL and resid <= ADJ_TOL, (spmm, resid)


@pytest.mark.parametrize("edit", HANDLE_EDITS)
def test_negative_control_handles_that_alias_and_never_rebuild(edit, monkeypatch):
    """The handles as they were before this contract: the forward CSR is the caller's ``vals`` tensor itself (the CSR^T
    a copy) and the support set is built once.  After the edit the forward still matches the edited stack, but the
    gradients and the adjoint identity must land outside their bars."""
    from stmgcn_b200 import graph
    real = graph.csr_from_coo

    def aliasing(n, rows, cols, vals):
        rp, ci, _ = real(n, rows, cols, vals)
        return rp, ci, vals.to(torch.float32).contiguous()

    monkeypatch.setattr(graph, "csr_from_coo", aliasing)
    monkeypatch.setattr(graph.SparseSupports, "version", lambda self: ())
    sup, fn, model, params, x, y = _edit_case(edit)
    model_errors(model, sup, params, x, y)
    with torch.no_grad():
        fn(sup)
    errs = model_errors(model, sup, params, x, y)
    _, resid = _identity_residual(sup, 3)
    grads = {k: v for k, v in errs.items() if k != "out"}
    worst = max(grads, key=grads.get)
    print(f"control {edit}: forward {errs['out']:.2e}, worst gradient {grads[worst]:.2e} ({worst}), adjoint identity "
          f"{resid:.2e}")
    assert errs["out"] <= TOL
    assert grads[worst] > TOL and resid > ADJ_TOL, (grads, resid)


# ======================================================================================================================
# E. captured steps and support edits
# ======================================================================================================================
def _graphed(n=N_EDIT):
    """A two-graph model (H = G = 64: the tensor-core kernels) on a dense stack and a ChebSupports handle, and its
    captured step."""
    from stmgcn_b200 import dp, graphs
    sups = [route_supports("cheb_dense", n), route_supports("cheb_handle", n)]
    model, params, x, y = _model(4, n, hid=64, gcn_hid=64, m=2)
    gstep = graphs.GraphedStep(model, nn.MSELoss(), x.to(DEV), y.to(DEV), sups, bucket=dp.GradBucket(model))
    return sups, model, params, x, y, gstep


def test_graphed_step_holds_its_support_sets_and_matches_fp64():
    """After ``graph.clear_cache()`` and 40 unrelated conversions (more than the cache holds), the support sets the step
    captured are still alive -- checked with weak references before any replay, since a replay would read their CSR --
    and a replay on a new batch matches the fp64 model: loss, output and every gradient at 1e-4."""
    from stmgcn_b200 import graph, synth
    sups, model, params, x, y, gstep = _graphed()
    captured = [graph.supports_from_dense(s) for s in sups]
    assert all(a is b for a, b in zip(captured, gstep.support_sets))
    refs = [weakref.ref(s) for s in captured]
    del captured
    graph.clear_cache()
    for i in range(40):
        graph.supports_from_dense(torch.stack([torch.eye(16), synth.make_adjacency(16, i, 0.2) * 0.1]).to(DEV))
    gc.collect()
    alive = [r() is not None for r in refs]
    assert all(alive), f"captured support sets were freed: {alive}; a replay would read freed CSR"
    gen = torch.Generator().manual_seed(99)
    x2, y2 = torch.randn(x.shape, generator=gen), torch.randn(y.shape, generator=gen)
    loss = gstep(x2.to(DEV), y2.to(DEV))
    torch.cuda.synchronize()
    o_ref, l_ref, g_ref = dense_reference(params, [dense64(s) for s in sups], x2, y2)
    errs = {"out": rel_err(gstep.out, o_ref), "loss": abs(loss.item() - l_ref) / abs(l_ref)}
    errs.update({k: rel_err(p.grad, g_ref[k]) for k, p in model.named_parameters()})
    worst = max(errs, key=errs.get)
    print(f"graphed step after clear_cache + 40 conversions: worst {errs[worst]:.2e} ({worst})")
    assert errs[worst] <= TOL, errs


@pytest.mark.parametrize("batch", ["full", "short"])
@pytest.mark.parametrize("which", ["dense", "handle"])
def test_graphed_step_refuses_to_replay_after_a_support_edit(which, batch):
    """After an in-place edit of either support, a call of the captured step -- a replay, or the eager path of a short
    batch -- raises ``RuntimeError``; nothing runs: the gradient buffer keeps its sentinel and no kernel launches."""
    from stmgcn_b200 import _lib
    sups, model, params, x, y, gstep = _graphed()
    gstep(x.to(DEV), y.to(DEV))
    with torch.no_grad():
        if which == "dense":
            sups[0].mul_(0.5)
        else:
            sups[1].vals.mul_(0.5)
    bucket = gstep.bucket
    bucket.flat.fill_(float("nan"))
    xs, ys = (x, y) if batch == "full" else (x[:2].contiguous(), y[:2].contiguous())
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(RuntimeError, match="edited after the step was captured"):
        gstep(xs.to(DEV), ys.to(DEV))
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
    assert bool(bucket.flat.isnan().all()), "the step ran although a support was edited"


# ======================================================================================================================
# F. the Chebyshev classifier's tolerance
# ======================================================================================================================
@pytest.mark.parametrize("factor", [0.1, 10.0])
def test_gcn_on_a_stack_at_the_classifier_tolerance_matches_the_stack_as_given(factor):
    """A ``process`` stack (K = 3) with its last slice scaled by 1 + factor * 5e-5 (the classifier's tolerance): at 10x it
    goes generic, at 0.1x it is taken as Chebyshev -- the recurrence then applies the unscaled T_3 -- and the GCN
    module's output and gradients must still be within 1e-4 of fp64 on the stack as given."""
    from stmgcn_b200.graph import supports_from_dense
    sup = route_supports("cheb_dense")
    with torch.no_grad():
        sup[3].mul_(1.0 + factor * 5e-5)
    mode = supports_from_dense(sup).mode
    assert mode == ("cheb" if factor < 1 else "generic")
    out_err, gerrs = gcn_vs_fp64(sup, dense64(sup), 64, seed=3)
    print(f"stack scaled at {factor}x the classifier tolerance ({mode}): out {out_err:.2e}, "
          + ", ".join(f"{k} {v:.2e}" for k, v in gerrs.items()))
    assert out_err <= TOL and max(gerrs.values()) <= TOL, (out_err, gerrs)
