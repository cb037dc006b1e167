"""Learnable adjacencies without a GPU: the fp64 restatement of the normalisation against dense torch autograd and
against ``process_sparse``, the pattern build (self-loops, empty rows, directed graphs, stored zeros), the module's
surface and ``state_dict``, the C entry points' argument and overlap checks, ``GradBucket`` over several modules (with a
world-size-2 gloo run) and ``GraphedStep``'s refusal of a bucket without the module's parameters."""
import ctypes
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from torch import nn

import learnable_adjacency_cases as LA
import support_grad_cases as S

ORDERS = {"chebyshev": 3, "localpool": 1, "random_walk_diffusion": 2}


def _module(kind, a, lam="reference"):
    import GCN
    return GCN.Adj_Preprocessor(kind, ORDERS[kind], lambda_max=lam).process_learnable(a)


# ======================================================================================================================
# the restatement
# ======================================================================================================================
@pytest.mark.parametrize("lam", [2.0, 1.37])
@pytest.mark.parametrize("directed", [False, True])
@pytest.mark.parametrize("kind", LA.KINDS)
def test_restatement_and_gradient_match_dense_autograd(kind, directed, lam):
    """Values and d w of the sparse fp64 restatement equal those of the dense preprocessing, on the stored pattern."""
    n = 23
    symmetric = kind != "random_walk_diffusion"
    # a zero degree makes the dense D^-1/2 A D^-1/2 NaN over a whole row and column: symmetric kinds without one
    a = LA.graph(n, 4, directed=directed, isolated=not symmetric)
    adj = _module(kind, a.float(), lam)
    assert adj.scale == pytest.approx(2.0 / lam if kind == "chebyshev" else 2.0 / adj.lambda_max)
    w0 = adj.weight.detach().double()
    rows, cols = adj.edges()
    w_s = w0.clone().requires_grad_(True)
    stack_s = LA.module_stack64(adj, w_s)
    w_d = w0.clone().requires_grad_(True)
    stack_d = LA.dense_reference_stack(kind, ORDERS[kind], LA.dense_of(n, rows, cols, w_d), lam)
    assert stack_s.shape == stack_d.shape == (adj.ks, n, n)
    torch.testing.assert_close(stack_s, stack_d, rtol=1e-12, atol=1e-12)
    r = torch.randn(stack_s.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    (g_s,) = torch.autograd.grad((stack_s * r).sum(), w_s)
    (g_d,) = torch.autograd.grad((stack_d * r).sum(), w_d)
    torch.testing.assert_close(g_s, g_d, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("kind", LA.KINDS)
def test_restatement_matches_process_sparse_with_isolated_rows(kind):
    """On a graph with an isolated region, self-loops and a hub, the module's supports at its initial weights are the
    ones ``process_sparse`` builds, and so are their gradients."""
    import GCN
    n = 29
    a = LA.graph(n, 7, directed=kind == "random_walk_diffusion").float()
    pre = GCN.Adj_Preprocessor(kind, ORDERS[kind], lambda_max=1.6)
    adj = pre.process_learnable(a)
    a_leaf = a.clone().requires_grad_(True)
    h = pre.process_sparse(a_leaf)
    w = adj.weight.detach().double().requires_grad_(True)
    v = LA.module_values64(adj, w)
    prow, pcol, _, perm_t = LA.pattern_of(adj)
    mats = ([LA.dense_of(n, pcol[perm_t], prow[perm_t], v[0]), LA.dense_of(n, prow, pcol, v[1])]
            if kind == "random_walk_diffusion" else [LA.dense_of(n, prow, pcol, v)])
    want = h.matrices_dense()
    for got, ref in zip(mats, want):
        torch.testing.assert_close(got.float(), ref, rtol=2e-6, atol=2e-6)
    # d w: the same dense loss through both
    r = [torch.randn(n, n, generator=torch.Generator().manual_seed(5 + i)) for i in range(len(mats))]
    (g,) = torch.autograd.grad(sum((m * ri.double()).sum() for m, ri in zip(mats, r)), w)
    dense_h = [S.dense_matrix(n, *S.coo_of(rp, ci), vv) for rp, ci, vv in h.mats]
    sum((m * ri).sum() for m, ri in zip(dense_h, r)).backward()
    torch.testing.assert_close(g.float(), a_leaf.grad[adj.edges()], rtol=1e-5, atol=1e-5)


def test_zero_sum_degrees_with_stored_entries_give_torchs_nan():
    """Diffusion: where a row or column has stored entries that sum to zero, d w is NaN in the restatement as in
    ``process_sparse``'s autograd (``0 * -inf`` through the masked reciprocal), and finite elsewhere, equal to it."""
    import GCN
    coo = LA.zero_sum_graph()
    pre = GCN.Adj_Preprocessor("random_walk_diffusion", 2)
    adj = pre.process_learnable(coo)
    leaf = coo.values().clone().requires_grad_(True)
    h = pre.process_sparse(torch.sparse_coo_tensor(coo.indices(), leaf, (6, 6)))
    gen = torch.Generator().manual_seed(2)
    r = [torch.randn(6, 6, generator=gen) for _ in range(2)]
    sum((S.dense_matrix(6, *S.coo_of(rp, ci), v) * ri).sum() for (rp, ci, v), ri in zip(h.mats, r)).backward()
    w = adj.weight.detach().double().requires_grad_(True)
    vf, vb = LA.module_values64(adj, w)
    prow, pcol, _, perm_t = LA.pattern_of(adj)
    mats = [LA.dense_of(6, pcol[perm_t], prow[perm_t], vf), LA.dense_of(6, prow, pcol, vb)]
    (g,) = torch.autograd.grad(sum((m * ri.double()).sum() for m, ri in zip(mats, r)), w)
    rows, cols = adj.edges()
    want_nan = (cols == 2) | (rows == 4)
    assert torch.equal(torch.isnan(g), want_nan) and torch.equal(torch.isnan(leaf.grad), want_nan)
    torch.testing.assert_close(g[~want_nan].float(), leaf.grad[~want_nan], rtol=1e-5, atol=1e-6)


# ======================================================================================================================
# the pattern and the module
# ======================================================================================================================
def test_pattern_adds_diagonal_slots_only_where_a_kind_needs_them():
    n = 9
    a = torch.zeros(n, n)
    a[0, 1] = a[1, 0] = 1.0
    a[3, 3] = 2.0                      # a stored self-loop
    a[4, 5] = 0.5                      # directed
    # rows 2, 6, 7, 8 are empty
    for kind, lam, added in (("chebyshev", "reference", False), ("chebyshev", 1.5, True), ("localpool", "reference", True),
                             ("random_walk_diffusion", "reference", False)):
        adj = _module(kind, a, lam)
        prow, pcol, widx, perm_t = LA.pattern_of(adj)
        assert adj.weight.numel() == 4
        rows, cols = adj.edges()
        assert torch.equal(rows, torch.tensor([0, 1, 3, 4])) and torch.equal(cols, torch.tensor([1, 0, 3, 5]))
        keys = prow * n + pcol
        assert bool((keys[1:] > keys[:-1]).all()), "CSR order, no repeat"
        if added:
            assert adj.widx is not None
            diag = set((prow[prow == pcol]).tolist())
            assert diag == set(range(n)), "every row has a diagonal slot"
            assert int((widx == -1).sum()) == n - 1          # every row but 3, which stores its own
            assert widx[(prow == 3) & (pcol == 3)].item() == 2
            assert sorted(widx[widx >= 0].tolist()) == [0, 1, 2, 3]
        else:
            assert adj.widx is None and prow.numel() == 4
        # CSR^T: column-major order, perm_t into the CSR
        assert torch.equal(adj.colidx_t.long().cpu(), prow[perm_t])
        kt = pcol[perm_t] * n + prow[perm_t]
        assert bool((kt[1:] > kt[:-1]).all())


def test_sparse_inputs_keep_stored_zeros_and_match_dense_otherwise():
    n = 6
    idx = torch.tensor([[0, 1, 1, 2, 4], [1, 0, 2, 1, 4]])
    vals = torch.tensor([1.0, 1.0, 0.0, 0.0, 3.0])          # (1,2) and (2,1) stored zeros
    coo = torch.sparse_coo_tensor(idx, vals, (n, n))
    adj = _module("localpool", coo)
    assert adj.weight.numel() == 5 and torch.equal(adj.weight.detach(), vals)
    csr = _module("localpool", coo.to_sparse_csr())
    assert all(torch.equal(u, v) for u, v in zip(csr.edges(), adj.edges()))
    dense = _module("localpool", coo.to_dense())
    assert dense.weight.numel() == 3                          # a dense adjacency's zeros are no edges


def test_module_surface_state_dict_and_read_back():
    import GCN
    n = 12
    a = LA.graph(n, 3).float()
    adj = _module("chebyshev", a, 1.8)
    assert adj.shape == (4, n, n) and len(adj) == 4 and adj.device == torch.device("cpu")
    assert [name for name, _ in adj.named_parameters()] == ["weight"]
    assert adj.to("cpu") is adj
    back = adj.learned_adjacency()
    assert back.is_sparse and torch.equal(back.to_dense(), a)
    with torch.no_grad():
        adj.weight.mul_(1.5)
    other = _module("chebyshev", a, 1.8)
    other.load_state_dict(adj.state_dict())
    assert torch.equal(other.weight, adj.weight)
    assert torch.equal(other.learned_adjacency().to_dense(), a * 1.5)
    with pytest.raises(ValueError, match="at most 8 supports"):
        GCN.Adj_Preprocessor("random_walk_diffusion", 4).process_learnable(a)
    from stmgcn_b200.graph import LearnableAdjacency
    with pytest.raises(ValueError, match="at most 8 supports"):
        LearnableAdjacency("random_walk_diffusion", 4, a)
    assert set(adj.state_dict()) == {"weight", "rowptr", "colidx", "rowptr_t", "colidx_t", "perm_t", "widx"}
    with pytest.raises(RuntimeError, match="CUDA device"):
        adj.support_set()


def test_power_lambda_is_evaluated_once_and_held():
    import GCN
    a = LA.graph(15, 9).float()
    pre = GCN.Adj_Preprocessor("chebyshev", 2, lambda_max="power")
    adj = pre.process_learnable(a)
    h = pre.process_sparse(a)
    lam = 2.0 / adj.scale
    assert adj.lambda_max == pytest.approx(lam) and 1.0 < lam <= 2.0 + 1e-6
    # the same rescaled Laplacian as process_sparse's (which estimates lambda_max the same way)
    w = adj.weight.detach().double()
    prow, pcol, _, _ = LA.pattern_of(adj)
    got = LA.dense_of(15, prow, pcol, LA.module_values64(adj, w))
    torch.testing.assert_close(got.float(), h.matrices_dense()[0], rtol=2e-6, atol=2e-6)


# ======================================================================================================================
# the C entry points' checks
# ======================================================================================================================
def test_adj_norm_entries_reject_bad_arguments_before_any_launch():
    from stmgcn_b200 import _lib
    lib = _lib.lib
    p = ctypes.c_void_p
    fake = 0x100000          # never dereferenced: every call below fails its checks first
    before = _lib.launch_count()
    n, nnz = 10, 40
    # ranges: rowptr @0, colidx @4096, rowptr_t @8192, colidx_t @12288, perm_t @16384, widx @20480, w @24576,
    # work @32768, vals @65536, vals_t @69632 (all disjoint; each spans at most 4 * (3n + nnz) bytes)
    at = dict(rowptr=0, colidx=4096, rowptr_t=8192, colidx_t=12288, perm_t=16384, widx=20480, w=24576, work=32768,
              vals=65536, vals_t=69632, dvals=73728, dvals_t=77824, dw=81920)

    def fwd(kind=2, n=n, nnz=nnz, nnz_w=nnz, scale=1.0, work_count=2 * n, **over):
        ptr = {k: (None if over.get(k, 0) is None else fake + over.get(k, v)) for k, v in at.items()}
        if "widx" not in over:
            ptr["widx"] = None
        return lib.stmgcn_adj_norm_fwd(kind, n, p(ptr["rowptr"]), p(ptr["colidx"]), p(ptr["rowptr_t"]),
                                       p(ptr["colidx_t"]), p(ptr["perm_t"]), nnz, p(ptr["widx"]), p(ptr["w"]), nnz_w,
                                       scale, p(ptr["work"]), work_count, p(ptr["vals"]), p(ptr["vals_t"]), None)

    def bwd(kind=2, n=n, nnz=nnz, nnz_w=nnz, scale=1.0, work_count=3 * n + nnz, **over):
        ptr = {k: (None if over.get(k, 0) is None else fake + over.get(k, v)) for k, v in at.items()}
        if "widx" not in over:
            ptr["widx"] = None
        return lib.stmgcn_adj_norm_bwd(kind, n, p(ptr["rowptr"]), p(ptr["colidx"]), p(ptr["rowptr_t"]),
                                       p(ptr["colidx_t"]), p(ptr["perm_t"]), nnz, p(ptr["widx"]), p(ptr["w"]), nnz_w,
                                       scale, p(ptr["dvals"]), p(ptr["dvals_t"]), p(ptr["work"]), work_count,
                                       p(ptr["dw"]), None)

    fwd_cases = [
        (dict(kind=3), "kind=3"), (dict(kind=-1), "kind=-1"), (dict(n=0), "n=0"), (dict(nnz=-1), "nnz=-1"),
        (dict(nnz_w=nnz - 1), "equal to it without widx"), (dict(nnz_w=nnz + 1, widx=at["widx"]), "nnz_w"),
        (dict(rowptr=None), "null rowptr"), (dict(rowptr_t=None), "null rowptr"), (dict(colidx=None), "null colidx"),
        (dict(perm_t=None), "null colidx"), (dict(w=None), "null w"), (dict(vals=None), "null vals"),
        (dict(vals_t=None), "null vals"), (dict(kind=1), "diffusion kind only"),
        (dict(kind=0, scale=float("inf"), vals_t=None), "finite"), (dict(kind=0, scale=float("nan"), vals_t=None), "finite"),
        (dict(work=None), "workspace"), (dict(work_count=2 * n - 1), "workspace"),
        (dict(vals=at["w"] + 4), "overlaps input"), (dict(vals_t=at["vals"] + 156), "outputs"),
        (dict(work=at["perm_t"] + 100), "overlaps input"), (dict(work=at["vals"] - 4), "outputs"),
        (dict(vals=at["rowptr"] + 40), "overlaps input"), (dict(widx=at["vals"] + 8), "overlaps input"),
    ]
    for over, msg in fwd_cases:
        rc = fwd(**over)
        assert rc < 0, (over, rc)
        assert msg in lib.stmgcn_last_error().decode(), (over, lib.stmgcn_last_error())
    bwd_cases = [
        (dict(kind=5), "kind=5"), (dict(dvals=None), "null dvals"), (dict(dvals_t=None), "null dvals"),
        (dict(dw=None), "null dvals"), (dict(kind=0, scale=1.0), "diffusion kind only"),
        (dict(work_count=3 * n + nnz - 1), "workspace"), (dict(dw=at["dvals"] + 8), "overlaps input"),
        (dict(dw=at["work"] + 4 * (3 * n + nnz) - 4), "outputs"), (dict(work=at["dvals_t"] + 40), "overlaps input"),
        (dict(dw=at["w"]), "overlaps input"),
    ]
    for over, msg in bwd_cases:
        rc = bwd(**over)
        assert rc < 0, (over, rc)
        assert msg in lib.stmgcn_last_error().decode(), (over, lib.stmgcn_last_error())
    # nothing to compute: accepted without enqueuing anything
    assert fwd(nnz=0, nnz_w=0) == 0
    assert bwd(nnz_w=0, widx=at["widx"]) == 0
    assert _lib.launch_count() == before, "a rejected (or empty) call launched a kernel"


# ======================================================================================================================
# the bucket and the captured step
# ======================================================================================================================
def test_grad_bucket_takes_several_modules_once_each():
    from stmgcn_b200.dp import GradBucket
    m1, m2 = nn.Linear(3, 2), nn.Linear(2, 2)
    m2.bias.requires_grad_(False)
    adj = _module("localpool", LA.graph(8, 1).float())
    b = GradBucket(m1, adj, m2, m1)
    assert [id(p) for p in b.params] == [id(m1.weight), id(m1.bias), id(adj.weight), id(m2.weight)]
    assert b.flat.numel() == 6 + 2 + adj.weight.numel() + 4
    assert adj.weight.grad.data_ptr() == b.flat.data_ptr() + 8 * 4
    adj.weight.grad = None
    assert b.rebind_() == 1
    with pytest.raises(ValueError, match="one dtype and device"):
        GradBucket(m1, nn.Linear(2, 2).double())


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, out):
    import GCN
    from stmgcn_b200.dp import GradBucket
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.manual_seed(0)
        model = nn.Linear(4, 1)
        adj = GCN.Adj_Preprocessor("chebyshev", 2).process_learnable(LA.graph(10, 2).float())
        opt = torch.optim.SGD(list(model.parameters()) + list(adj.parameters()), lr=0.1)
        bucket = GradBucket(model, adj)
        bucket.zero_()
        # a rank-dependent loss through the edge weights and the model
        x = torch.full((3, 4), float(rank + 1))
        loss = (model(x).sum() + (adj.weight * (rank + 1.0) * torch.arange(adj.weight.numel())).sum())
        loss.backward()
        bucket.all_reduce_mean_()
        torch.save(dict(grad=adj.weight.grad.clone(), mgrad=model.weight.grad.clone()), f"{out}.{rank}.grad")
        opt.step()
        torch.save(dict(w=adj.weight.detach().clone(), mw=model.weight.detach().clone()), f"{out}.{rank}.step")
    finally:
        dist.destroy_process_group()


def test_grad_bucket_averages_edge_weights_over_two_gloo_ranks(tmp_path):
    out = str(tmp_path / "r")
    mp.spawn(_dp_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    g = [torch.load(f"{out}.{r}.grad") for r in range(2)]
    s = [torch.load(f"{out}.{r}.step") for r in range(2)]
    nnz = g[0]["grad"].numel()
    want = 1.5 * torch.arange(nnz, dtype=torch.float32)          # mean of (rank + 1) * e over ranks 0, 1
    for r in range(2):
        torch.testing.assert_close(g[r]["grad"], want)
    assert torch.equal(g[0]["mgrad"], g[1]["mgrad"])
    assert torch.equal(s[0]["w"], s[1]["w"]) and torch.equal(s[0]["mw"], s[1]["mw"]), "replicas differ after a step"


def test_graphed_step_refuses_a_bucket_without_the_modules_parameters():
    from stmgcn_b200.dp import GradBucket
    from stmgcn_b200.graphs import GraphedStep
    model = nn.Linear(2, 2)
    adj = _module("localpool", LA.graph(8, 1).float())
    with pytest.raises(ValueError, match=r"lacks the parameters of the learnable adjacencies \[1\]"):
        GraphedStep(model, nn.MSELoss(), torch.zeros(1), torch.zeros(1), [torch.zeros(1, 8, 8), adj],
                    bucket=GradBucket(model))
