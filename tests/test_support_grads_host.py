"""Gradients of learnable support values, on the host: the sparse fp64 formula the SDDMM kernel implements against
dense fp64 autograd (Chebyshev chains, two-chain diffusion, localpool, hand-made CSR), ``process_sparse`` carrying the
gradient to dense and COO adjacencies, the plumbing of ``ops`` (segments, coefficients, chains) with the launches
replaced by fp64 torch, structure caching with the value refresh, and the argument checks of ``stmgcn_csr_sddmm``."""
import ctypes

import pytest
import torch

import support_grad_cases as S
from helpers import assert_close, rel_err


def _lap_csr(n, seed):
    """Entries (rows, cols, vals fp64) of the rescaled Laplacian of a random symmetric graph (self-loops of L~ kept)."""
    import GCN
    from stmgcn_b200 import synth
    h = GCN.Adj_Preprocessor("chebyshev", 1).process_sparse(synth.make_adjacency(n, seed, 0.3))
    rows, cols = S.coo_of(h.rowptr, h.colidx)
    return rows, cols, h.vals.double()


def _dense_dvals(n, rows, cols, vals, x, rs, order):
    """d vals of sum_k <R_k, T_k(X) x> by dense autograd on X built from a leaf of the values."""
    leaf = vals.clone().requires_grad_(True)
    polys = S.dense_chain(S.dense_matrix(n, rows, cols, leaf), order)
    loss = sum((r * torch.einsum("ij,jf->if", p, x)).sum() for r, p in zip(rs, polys))
    loss.backward()
    return leaf.grad


def _rand(shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


@pytest.mark.parametrize("order", [1, 2, 3, 4, 5, 6, 7])
def test_chebyshev_formula_equals_dense_autograd(order):
    n = 29
    rows, cols, vals = _lap_csr(n, order)
    x = _rand((n, 6), 1)
    rs = [_rand((n, 6), 10 + k) for k in range(order + 1)]
    got = S.dvals_formula(rows, cols, vals, x, rs)
    assert_close(got.numpy(), _dense_dvals(n, rows, cols, vals, x, rs, order).numpy(), f"cheb K={order}", 1e-12)


@pytest.mark.parametrize("order", [1, 2, 3])
def test_diffusion_formula_equals_dense_autograd(order):
    """Two chains (P_f^T, P_b^T of a directed graph with a sink, a source and an isolated region) sharing T_0."""
    import GCN
    n = 23
    a = S.directed_graph(n, 4 + order)
    h = GCN.Adj_Preprocessor("random_walk_diffusion", order).process_sparse(a.float())
    x = _rand((n, 5), 2)
    for c, (rp, ci, v) in enumerate(h.mats):
        rows, cols = S.coo_of(rp, ci)
        rs = [_rand((n, 5), 20 + 7 * c + k) for k in range(order + 1)]
        got = S.dvals_formula(rows, cols, v.double(), x, rs)
        assert_close(got.numpy(), _dense_dvals(n, rows, cols, v.double(), x, rs, order).numpy(),
                     f"diffusion chain {c}", 1e-12)


def test_localpool_and_handmade_generic_formula_equal_dense_autograd():
    """Generic supports S = A x: d vals[e] = <U[i], x[j]>; hand-made CSR with repeats, unsorted columns, stored zeros
    and empty rows (every repeat gets the full dL/dA[i, j], every stored zero its gradient)."""
    import GCN
    from stmgcn_b200 import synth
    n = 40
    lp = GCN.Adj_Preprocessor("localpool", 1).process_sparse(synth.make_adjacency(n, 3, 0.2))
    cases = [lp.mats[0], S.handmade(n, 5)]
    for rp, ci, v in cases:
        rows, cols = S.coo_of(rp, ci)
        x, u = _rand((n, 7), 3), _rand((n, 7), 4)
        got = (u[rows] * x[cols]).sum(1)
        leaf = v.double().clone().requires_grad_(True)
        (u * (S.dense_matrix(n, rows, cols, leaf) @ x)).sum().backward()
        assert_close(got.numpy(), leaf.grad.numpy(), "generic", 1e-12)
        # the repeats: equal gradients at every copy of one (i, j)
        key = rows * n + cols
        for k in key.unique():
            sel = (key == k).nonzero().flatten()
            assert bool((leaf.grad[sel] == leaf.grad[sel[0]]).all())


@pytest.mark.parametrize("order", [1, 3, 5])
def test_handmade_chain_formula_equals_dense_autograd(order):
    n = 40
    rp, ci, v = S.handmade(n, 9)
    rows, cols = S.coo_of(rp, ci)
    x = _rand((n, 3), 5)
    rs = [_rand((n, 3), 30 + k) for k in range(order + 1)]
    got = S.dvals_formula(rows, cols, v.double(), x, rs)
    assert_close(got.numpy(), _dense_dvals(n, rows, cols, v.double(), x, rs, order).numpy(), "hand-made chain", 1e-12)


def test_negative_controls_fail():
    """c_k = 1 for k >= 2, and a directed graph's transposed pattern, each miss dense autograd by far."""
    import GCN
    n, order = 23, 3
    rows, cols, vals = _lap_csr(n, 2)
    x = _rand((n, 4), 6)
    rs = [_rand((n, 4), 40 + k) for k in range(order + 1)]
    want = _dense_dvals(n, rows, cols, vals, x, rs, order)
    assert rel_err(S.dvals_formula(rows, cols, vals, x, rs, coefs=[1.0] * order), want) > 1e-2
    h = GCN.Adj_Preprocessor("random_walk_diffusion", 2).process_sparse(S.directed_graph(n, 3).float())
    rows, cols = S.coo_of(*h.mats[0][:2])
    v = h.mats[0][2].double()
    rs = [_rand((n, 4), 50 + k) for k in range(3)]
    want = _dense_dvals(n, rows, cols, v, x, rs, 2)
    assert rel_err(S.dvals_formula(rows, cols, v, x, rs), want) <= 1e-12
    assert rel_err(S.dvals_formula(rows, cols, v, x, rs, pattern=(cols, rows)), want) > 1e-2


# ---- process_sparse -------------------------------------------------------------------------------------------------
def _dense_pattern_grads(kernel_type, a64, rs):
    """Gradient at adj of sum_m <R_m, M_m(adj)> with the dense matrices of process() (fp64)."""
    import GCN
    leaf = a64.clone().requires_grad_(True)
    pre = GCN.Adj_Preprocessor(kernel_type, 1)
    if kernel_type == "random_walk_diffusion":
        d_in = leaf.sum(0).pow(-1)
        d_in = torch.where(torch.isinf(d_in), torch.zeros_like(d_in), d_in)
        mats = [pre.process(leaf)[1], leaf * d_in[None, :]]          # P_f^T, P_b^T = A D_in^-1
    else:
        mats = [pre.process(leaf)[1 if kernel_type == "chebyshev" else 0]]
    sum(((r * m).sum() for r, m in zip(rs, mats))).backward()
    return leaf.grad


@pytest.mark.parametrize("layout", ["dense", "coo"])
@pytest.mark.parametrize("kernel_type", ["chebyshev", "localpool", "random_walk_diffusion"])
def test_process_sparse_carries_the_gradient_to_the_adjacency(kernel_type, layout):
    import GCN
    from stmgcn_b200 import synth
    n = 31
    if kernel_type == "random_walk_diffusion":
        a = S.directed_graph(n, 8)
    else:
        a = synth.make_adjacency(n, 1, 0.25).double() * (0.5 + torch.rand(n, n, generator=torch.Generator().manual_seed(1),
                                                                           dtype=torch.float64))
        a = 0.5 * (a + a.t())
    pre = GCN.Adj_Preprocessor(kernel_type, 1)
    if layout == "dense":
        leaf = a.float().clone().requires_grad_(True)
        h = pre.process_sparse(leaf)
    else:
        coo = a.float().to_sparse_coo().coalesce()
        leaf = coo.values().clone().requires_grad_(True)
        h = pre.process_sparse(torch.sparse_coo_tensor(coo.indices(), leaf, coo.shape))
    assert h.requires_grad
    rs = [_rand((n, n), 60 + m) for m in range(len(h.mats))]
    loss = 0.0
    for (rp, ci, v), r in zip(h.mats, rs):
        rows, cols = S.coo_of(rp, ci)
        loss = loss + (v.double() * r[rows, cols]).sum()
    loss.backward()
    want = _dense_pattern_grads(kernel_type, a, rs)
    got = leaf.grad.double() if layout == "dense" else torch.sparse_coo_tensor(coo.indices(), leaf.grad, coo.shape).to_dense().double()
    on = a != 0
    assert_close(got[on].numpy(), want[on].numpy(), f"{kernel_type} d adj ({layout})", 1e-5)
    assert float(got[~on].abs().max()) == 0.0           # the gradient lives on the stored pattern


def test_process_sparse_without_grad_keeps_detached_values():
    import GCN
    from stmgcn_b200 import synth
    for kt in ("chebyshev", "localpool", "random_walk_diffusion"):
        h = GCN.Adj_Preprocessor(kt, 1).process_sparse(synth.make_adjacency(20, 0, 0.3))
        assert not h.requires_grad and all(v.grad_fn is None and v.is_leaf for _, _, v in h.mats)


# ---- the plumbing of ops, launches replaced by fp64 torch -------------------------------------------------------------
class _Graph:
    """A CSR stand-in for GraphHandle: entries (rows, cols, vals) fp64."""

    def __init__(self, n, rows, cols, vals):
        self.n, self.nnz, self.rows, self.cols, self.vals = n, rows.numel(), rows, cols, vals


def _fake_launches(monkeypatch):
    from stmgcn_b200 import ops

    def spmm_step(g, transpose, alpha, x, beta, z, gamma, u, y):
        r = alpha * S.spmm(g.rows, g.cols, g.vals, x, transpose)
        if z is not None:
            r = r + beta * z
        if u is not None:
            r = r + gamma * u
        y.copy_(r)

    def csr_sddmm_(g, terms, dvals, round_b16=False):
        assert not round_b16
        for a, b, c in terms:
            dvals += c * (a.reshape(g.n, -1)[g.rows] * b.reshape(g.n, -1)[g.cols]).sum(1)

    monkeypatch.setattr(ops, "spmm_step", spmm_step)
    monkeypatch.setattr(ops, "csr_sddmm_", csr_sddmm_)
    return ops


@pytest.mark.parametrize("chains,order", [(1, 1), (1, 3), (1, 7), (2, 1), (2, 3)])
@pytest.mark.parametrize("need_dx", [True, False])
def test_ops_value_grads_equal_dense_autograd(monkeypatch, chains, order, need_dx):
    """cheb_stack_ / adjoint_stack_ / support_value_grads on fp64 with each chain's segments: d vals of
    sum_k <U_k, S_k> against dense autograd, with and without dX."""
    from stmgcn_b200.graph import SupportSet
    ops = _fake_launches(monkeypatch)
    n, f = 19, 6
    graphs = []
    for c in range(chains):
        rp, ci, v = S.handmade(n, 11 + c)
        rows, cols = S.coo_of(rp, ci)
        graphs.append(_Graph(n, rows, cols, v.double()))
    ks = chains * order + 1
    sset = SupportSet("cheb", n, ks, graphs, torch.device("cpu"))
    s = torch.zeros((ks, n, f), dtype=torch.float64)
    s[0] = _rand((n, f), 1)
    ops.cheb_stack_(sset, s)
    us = torch.stack([_rand((n, f), 70 + k) for k in range(ks)])
    u = us.clone()
    dx = ops.adjoint_stack_(sset, u, need_dx)
    got = ops.support_value_grads(sset, s, u, None, False, [True] * chains)
    leaves = [g.vals.clone().requires_grad_(True) for g in graphs]
    x_leaf = s[0].clone().requires_grad_(True)
    terms = [x_leaf]
    for g, leaf in zip(graphs, leaves):
        polys = S.dense_chain(S.dense_matrix(n, g.rows, g.cols, leaf), order)
        terms += [p @ x_leaf for p in polys[1:]]
    sum((uk * t).sum() for uk, t in zip(us, terms)).backward()
    for c in range(chains):
        assert_close(got[c].numpy(), leaves[c].grad.numpy(), f"chain {c}", 1e-6)          # d vals is fp32
    if need_dx:
        assert_close(dx.numpy(), x_leaf.grad.numpy(), "dX", 1e-11)
    else:
        assert dx is None and torch.equal(u[0], us[0])          # the step into U_0 was skipped


def test_ops_generic_value_grads(monkeypatch):
    from stmgcn_b200.graph import SupportSet
    ops = _fake_launches(monkeypatch)
    n, f = 21, 5
    graphs = []
    for k in range(3):
        rp, ci, v = S.handmade(n, 20 + k)
        graphs.append(_Graph(n, *S.coo_of(rp, ci), v.double()))
    sset = SupportSet("generic", n, 3, graphs, torch.device("cpu"))
    x = _rand((n, f), 2)
    u = torch.stack([_rand((n, f), 80 + k) for k in range(3)])
    got = ops.support_value_grads(sset, None, u, x, False, [True, False, True])
    assert got[1] is None
    for k in (0, 2):
        leaf = graphs[k].vals.clone().requires_grad_(True)
        (u[k] * (S.dense_matrix(n, graphs[k].rows, graphs[k].cols, leaf) @ x)).sum().backward()
        assert_close(got[k].numpy(), leaf.grad.numpy(), f"generic {k}", 1e-6)


# ---- structure caching and the value refresh --------------------------------------------------------------------------
def test_learnable_handle_caches_structure_and_refreshes_values(monkeypatch):
    """The CSR / CSR^T indices and the transpose's permutation are built once; the values are copied again at every
    call, also after a write that bypasses the version counter (``.data``, as fused optimizers write)."""
    from stmgcn_b200 import graph as G
    monkeypatch.setattr(G.SparseSupports, "is_cuda", property(lambda self: True))
    builds = []
    orig = G.GraphHandle.from_csr.__func__
    monkeypatch.setattr(G.GraphHandle, "from_csr", classmethod(lambda cls, *a: builds.append(1) or orig(cls, *a)))
    n = 30
    rp, ci, v = S.handmade(n, 3)
    vals = torch.nn.Parameter(v.clone())
    h = G.ChebSupports(n, 4, rp, ci, vals)
    assert h.requires_grad and h.vals is vals
    s1 = h.support_set()
    assert s1.grad_values() == (vals,)
    s2 = h.support_set()
    assert len(builds) == 1 and s1 is not s2
    (rp1, ci1, v1), (rpt1, cit1, vt1) = s1.graphs[0].export(False), s1.graphs[0].export(True)
    (rp2, ci2, v2), (rpt2, cit2, vt2) = s2.graphs[0].export(False), s2.graphs[0].export(True)
    assert rp1 is rp2 and ci1 is ci2 and rpt1 is rpt2 and cit1 is cit2 and v1 is not v2
    ver = vals._version
    vals.data.mul_(3.0)
    assert vals._version == ver                          # no version bump ...
    s3 = h.support_set()
    assert len(builds) == 1
    assert torch.equal(s3.graphs[0].export(False)[2], vals.detach())        # ... and yet the new values
    assert torch.equal(v1, v.float())                   # an earlier forward's copy is its own
    # the transpose's values follow the permutation of the CSR^T
    ref = G.GraphHandle.from_csr(n, rp, ci, vals.detach())
    assert torch.equal(s3.graphs[0].export(True)[2], ref.export(True)[2])
    # an edit of the structure rebuilds it
    ci.add_(0)
    h.support_set()
    assert len(builds) == 3
    # frozen values: the cached support set of before, no values carried
    vals.requires_grad_(False)
    f1 = h.support_set()
    assert f1 is h.support_set() and f1.grad_values() == () and f1.values is None


def test_graphed_step_refuses_learnable_supports_before_any_warmup():
    from stmgcn_b200.graph import ChebSupports
    from stmgcn_b200.graphs import GraphedStep
    rp, ci, v = S.handmade(10, 1)
    h = ChebSupports(10, 3, rp, ci, v.clone().requires_grad_(True))

    class _Model:                                       # never called: the refusal comes first
        def __call__(self, **_):
            raise AssertionError("warm-up ran")

    with pytest.raises(ValueError, match="require grad"):
        GraphedStep(_Model(), None, torch.zeros(1), torch.zeros(1), [h], bucket=object())


# ---- the C entry point's argument checks --------------------------------------------------------------------------------
def test_csr_sddmm_rejects_bad_arguments_before_any_launch():
    from stmgcn_b200 import _lib
    lib = _lib.lib
    p = ctypes.c_void_p
    fake = 0x10000          # never dereferenced: every call below fails its checks first
    before = _lib.launch_count()

    def call(n=4, rowptr=fake, colidx=fake, nnz=10, nterms=1, a=(fake,), b=(fake,), coef=(1.0,), rnd=0, f_total=8,
             work=0, work_count=0, dvals=fake + 4096):
        return lib.stmgcn_csr_sddmm(n, p(rowptr), p(colidx), nnz, nterms, _lib.ptr_array(list(a)),
                                    _lib.ptr_array(list(b)), _lib.float_array(list(coef)), rnd, f_total, p(work),
                                    work_count, p(dvals), None)

    cases = [
        (dict(rowptr=0), "null pointer"),
        (dict(n=0), "n=0"),
        (dict(nnz=-1), "nnz=-1"),
        (dict(colidx=0), "colidx / dvals null"),
        (dict(dvals=0), "colidx / dvals null"),
        (dict(nterms=0), "nterms=0"),
        (dict(nterms=9, a=(fake,) * 9, b=(fake,) * 9, coef=(1.0,) * 9), "nterms=9"),
        (dict(f_total=0), "f_total=0"),
        (dict(rnd=2), "round_b_bf16=2"),
        (dict(a=(0,)), "null operand of term 0"),
        (dict(b=(fake + 4,)), "16-byte aligned"),
        (dict(a=(fake + 4096,)), "must not overlap"),
        (dict(b=(fake + 4096 - 16,)), "must not overlap"),           # overlaps dvals at another offset
        (dict(f_total=256, work=fake + 8192, work_count=10 * 2, b=(fake + 8192 + 64,)), "must not overlap"),
        (dict(f_total=256), "workspace"),
        (dict(f_total=256, work=fake + 8192, work_count=19), "workspace"),
        (dict(f_total=33, work=fake + 4096), "workspace"),
    ]
    for kw, msg in cases:
        rc = call(**kw)
        assert rc < 0, kw
        assert msg.encode() in lib.stmgcn_last_error(), (kw, lib.stmgcn_last_error())
    assert _lib.launch_count() == before


def test_forced_value_reference_equals_the_dense_restatement():
    """The value-differentiable BF16ModeReference (rounding off, no masks, no tapes) and the dense fp64 restatement give
    the same loss, parameter gradients, d obs and d vals (two handles, one on two branches)."""
    import GCN
    import stmgcn_oracle as O
    from stmgcn_b200 import synth
    n, order = 14, 2
    pre = GCN.Adj_Preprocessor("chebyshev", order)
    handles = [pre.process_sparse(synth.make_adjacency(n, g, 0.3)) for g in range(2)]
    params = O.init_params(3, 4, 1, 8, 2, 6, order + 1, seed=3)
    gen = torch.Generator().manual_seed(4)
    x, y = torch.randn(2, 4, n, 1, generator=gen), torch.randn(2, n, 1, generator=gen)
    branch = [0, 1, 0]
    loss, grads, d_obs, d_vals = S.ForcedValueReference(params, handles, branch, rounding=False).value_grads(x, y)
    l_d, g_d, o_d, v_d = S.model_reference(params, x, y, handles, branch)
    assert abs(loss - l_d) <= 1e-12 * abs(l_d)
    for k in g_d:
        assert_close(grads[k].numpy(), g_d[k].numpy(), k, 1e-10)
    assert_close(d_obs.numpy(), o_d.numpy(), "d obs", 1e-10)
    for a, b in zip(d_vals, v_d):
        assert_close(a[0].numpy(), b[0].numpy(), "d vals", 1e-10)
