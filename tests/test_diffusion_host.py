"""``kernel_type='random_walk_diffusion'`` on the host: the sparse supports of ``Adj_Preprocessor.process_sparse``
against the reference's recipe, the handle's tensor surface, the support limit, the chain plumbing of the stack and its
adjoint (launch for launch), ``localpool``'s sparse supports, and the chain-extended oracle against the reference's
golden vectors (``tests/golden/diffusion_ref.npz``, ``oracle/make_diffusion_golden.py``)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch
from torch import nn

import diffusion_oracle as D
import stmgcn_oracle as O
from helpers import assert_close


def _directed(n, seed, density=0.15):
    """Weighted directed graph with two sinks, two sources and an isolated region."""
    gen = torch.Generator().manual_seed(seed)
    a = (torch.rand(n, n, generator=gen) < density).double() * (0.5 + torch.rand(n, n, generator=gen, dtype=torch.float64))
    a.fill_diagonal_(0.0)
    a[[0, 3], :] = 0.0          # sinks
    a[:, [1, 4]] = 0.0          # sources
    a[2, :] = 0.0
    a[:, 2] = 0.0               # isolated
    return a


def _stack_from_handle(h):
    """fp64 dense (Ks, N, N) stack of a diffusion handle: T_k of each stored chain matrix, computed with scipy."""
    mats = [sp.csr_matrix(m.double().numpy()) for m in h.matrices_dense()]
    order = (h.ks - 1) // len(mats)
    eye = sp.identity(h.n, format="csr", dtype=np.float64)
    out = [eye]
    for x in mats:
        terms = [eye, x]
        for _ in range(2, order + 1):
            terms.append(2.0 * (x @ terms[-1]) - terms[-2])
        out += terms[1:order + 1]
    return np.stack([t.toarray() for t in out])


@pytest.mark.parametrize("order", [0, 1, 2, 3])
@pytest.mark.parametrize("layout", ["dense", "sparse"])
def test_diffusion_process_sparse_equals_reference_recipe(order, layout):
    import GCN
    a = _directed(33, 10 + order)
    pre = GCN.Adj_Preprocessor("random_walk_diffusion", order)
    h = pre.process_sparse(a.float() if layout == "dense" else a.float().to_sparse_coo())
    assert len(h) == 2 * order + 1 and tuple(h.shape) == (2 * order + 1, 33, 33)
    assert all(bool(torch.isfinite(v).all()) for _, _, v in h.mats)
    got = _stack_from_handle(h)
    want = D.diffusion_supports_dense(a, order).numpy()
    assert np.isfinite(want).all()
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()
    # the sink's and the source's rows / columns: d_inv = 0, no NaN, nothing diffuses out of a sink (P_f^T column 0)
    pf_t, pb_t = (m.double() for m in h.matrices_dense())
    assert float(pf_t[:, 0].abs().sum()) == 0.0 and float(pb_t[:, 1].abs().sum()) == 0.0


def test_diffusion_supports_of_the_golden_graphs():
    """The golden fixture's supports (built by the reference's own functions) equal the oracle's restatement and the
    handle's chains."""
    import GCN
    meta, _, _, supports, adjs, _ = D.load_golden()
    for a, s in zip(adjs, supports):
        assert_close(D.diffusion_supports_dense(a, meta["k"]).numpy(), s.numpy(), "dense diffusion supports", 1e-6)
        h = GCN.Adj_Preprocessor("random_walk_diffusion", meta["k"]).process_sparse(a)
        assert_close(_stack_from_handle(h), s.numpy(), "sparse diffusion supports", 1e-6)


def test_diffusion_handle_surface():
    import GCN
    import STMGCN
    from stmgcn_b200.graph import SparseSupports, supports_from_dense
    a = _directed(20, 3).float()
    for order in range(4):
        h = GCN.Adj_Preprocessor("random_walk_diffusion", order).process_sparse(a)
        assert isinstance(h, SparseSupports) and h.mode == "cheb" and len(h.mats) == 2
        cfg = {"kernel_type": "random_walk_diffusion", "K": order}
        assert len(h) == h.shape[0] == STMGCN.ST_MGCN.get_support_K(cfg)
        assert h.device == torch.device("cpu") and not h.is_cuda
        assert h.to("cpu") is h
    with pytest.raises(RuntimeError, match="CUDA"):
        supports_from_dense(h)                     # a CPU handle is refused before any kernel


def test_diffusion_rejects_more_than_eight_supports():
    import GCN
    pre = GCN.Adj_Preprocessor("random_walk_diffusion", 4)
    with pytest.raises(ValueError, match="8 supports"):
        pre.process_sparse(_directed(10, 1).float())
    assert pre.process(_directed(10, 1).float()).shape[0] == 5       # process() keeps the reference's K+1 stack


def test_localpool_process_sparse_equals_process():
    import GCN
    from stmgcn_b200 import synth
    pre = GCN.Adj_Preprocessor("localpool", 1)
    for g in range(3):
        a = synth.make_adjacency(45, g, 0.2)
        h = pre.process_sparse(a)
        assert h.mode == "generic" and len(h) == 1 and tuple(h.shape) == (1, 45, 45)
        assert_close(h.matrices_dense()[0].numpy(), pre.process(a)[0].numpy(), "localpool sparse", 1e-6)
    # weighted, asymmetric, given as sparse COO
    a = synth.make_adjacency(30, 0, 0.3) * (0.5 + torch.rand(30, 30, generator=torch.Generator().manual_seed(2)))
    h = pre.process_sparse(a.to_sparse_coo())
    assert_close(h.matrices_dense()[0].numpy(), pre.process(a)[0].numpy(), "localpool sparse (weighted)", 1e-6)


class _Graph:
    """A stand-in support matrix (compared by identity)."""
    n = 4


class _Recorder:
    """Stands in for the SpMM / bf16-copy launches of ops.py: records (entry point, matrix, transpose, scalars, operand
    names) for each call."""

    def __init__(self, names):
        self.calls, self.names = [], names

    def name(self, t):
        return None if t is None else self.names.get(t.data_ptr(), "tmp")

    def spmm_step(self, g, transpose, alpha, x, beta, z, gamma, u, y):
        self.calls.append(("spmm", g, transpose, alpha, self.name(x), beta, self.name(z), gamma, self.name(u),
                           self.name(y)))

    def spmm_step16(self, g, transpose, alpha, x16, beta, z, gamma, u, y, y16):
        self.calls.append(("spmm16", g, transpose, alpha, beta, self.name(z), gamma, self.name(u), self.name(y),
                           y16 is not None))

    def to_bf16(self, x):
        self.calls.append(("to_bf16", self.name(x)))
        return torch.empty(x.shape, dtype=torch.bfloat16)


def _record(monkeypatch, sset, ks, planes, gather16):
    from stmgcn_b200 import ops
    s = torch.zeros((ks, 4, 2, 8))
    rec = _Recorder({s[k].data_ptr(): f"s{k}" for k in range(ks)})
    for fn in ("spmm_step", "spmm_step16", "to_bf16"):
        monkeypatch.setattr(ops, fn, getattr(rec, fn))
    monkeypatch.setattr(ops, "_PLANES", planes)
    ops.cheb_stack_(sset, s, gather16)
    ops.adjoint_stack_(sset, s)
    return rec.calls


@pytest.mark.parametrize("ks", [1, 2, 3, 4, 6])
@pytest.mark.parametrize("planes,gather16", [(2, True), (1, True), (1, False)])
def test_chebyshev_stack_issues_the_same_launches(monkeypatch, ks, planes, gather16):
    """One chain (a Chebyshev stack): the launches of the stack and its adjoint, written out as they were before the
    stack was parametrised by chain."""
    from stmgcn_b200.graph import SupportSet
    g = _Graph()
    sset = SupportSet("cheb", 4, ks, [g] if ks > 1 else [], torch.device("cpu"))
    got = _record(monkeypatch, sset, ks, planes, gather16)
    want = []
    if ks > 1:
        if planes == 1 and gather16:
            want.append(("to_bf16", "s0"))
            for k in range(1, ks):
                want.append(("spmm16", g, False, 1.0 if k == 1 else 2.0, 0.0 if k == 1 else -1.0,
                             None if k == 1 else f"s{k - 2}", 0.0, None, f"s{k}", k < ks - 1))
        else:
            want.append(("spmm", g, False, 1.0, "s0", 0.0, None, 0.0, None, "s1"))
            for k in range(2, ks):
                want.append(("spmm", g, False, 2.0, f"s{k - 1}", -1.0, f"s{k - 2}", 0.0, None, f"s{k}"))
        k_ord = ks - 1
        for k in range(k_ord - 1, 0, -1):
            z = f"s{k + 2}" if k + 2 <= k_ord else None
            want.append(("spmm", g, True, 2.0, f"s{k + 1}", -1.0 if z else 0.0, z, 1.0, f"s{k}", f"s{k}"))
        z = "s2" if k_ord >= 2 else None
        want.append(("spmm", g, True, 1.0, "s1", -1.0 if z else 0.0, z, 1.0, "s0", "s0"))
    assert got == want


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("planes", [2, 1])
def test_diffusion_chains_run_the_chebyshev_code(monkeypatch, order, planes):
    """Two chains: each runs exactly the launches of a one-chain stack of order K over its own segments (T_0 = s0 shared,
    the adjoint of both adds into s0)."""
    from stmgcn_b200.graph import SupportSet
    gf, gb = _Graph(), _Graph()
    ks = 2 * order + 1
    got = _record(monkeypatch, SupportSet("cheb", 4, ks, [gf, gb], torch.device("cpu")), ks, planes, True)
    one = _record(monkeypatch, SupportSet("cheb", 4, order + 1, [gf], torch.device("cpu")), order + 1, planes, True)

    def relabel(calls, g, seg):
        names = {f"s{k}": f"s{seg[k]}" for k in range(len(seg))}
        return [tuple(names.get(v, v) if isinstance(v, str) else (g if v is gf else v) for v in c) for c in calls]

    n_fwd = order + (1 if planes == 1 else 0)
    seg_f = [0] + list(range(1, order + 1))
    seg_b = [0] + list(range(order + 1, 2 * order + 1))
    want = (relabel(one[:n_fwd], gf, seg_f) + relabel(one[:n_fwd], gb, seg_b) + relabel(one[n_fwd:], gf, seg_f)
            + relabel(one[n_fwd:], gb, seg_b))
    assert got == want


def test_chain_oracle_equals_golden():
    """The sparse oracle with two chains [P_f^T, P_b^T] (fp64, hand-written backward) and the dense restatement (2K+1
    supports, autograd) against the reference run of diffusion_ref.npz: forward, loss, every parameter gradient and
    d obs_seq."""
    meta, params, grads, supports, adjs, blob = D.load_golden()
    ks = 2 * meta["k"] + 1
    orc = D.ChainOracle({k: v.numpy() for k, v in params.items()}, [D.diffusion_chains_csr(a.double()) for a in adjs],
                         ks, dtype=np.float64)
    out, loss, g = orc.loss_and_grads(blob["x"], blob["y"])
    assert_close(out, blob["out"], "oracle forward")
    assert abs(loss - float(blob["loss"])) <= 1e-5 * abs(float(blob["loss"]))
    assert set(g) == set(grads)
    for key in grads:
        assert_close(g[key], grads[key], f"oracle grad {key}")
    # dense restatement, with the gradient at obs_seq
    leaves = {k: v.double().requires_grad_(True) for k, v in params.items()}
    x = torch.from_numpy(blob["x"]).double().requires_grad_(True)
    out_d = O.dense_st_mgcn(leaves, x, [D.diffusion_supports_dense(a.double(), meta["k"]) for a in adjs])
    loss_d = nn.MSELoss()(out_d, torch.from_numpy(blob["y"]).double())
    loss_d.backward()
    assert_close(out_d.detach().numpy(), blob["out"], "dense forward")
    assert_close(x.grad.numpy(), blob["grad_x"], "dense d obs_seq")
    for key in grads:
        assert_close(leaves[key].grad.numpy(), grads[key], f"dense grad {key}")


def test_chain_oracle_backward_equals_autograd():
    """The chain oracle's hand-written backward agrees with autograd on the dense stack to fp64 precision (K = 3: two
    chains of three terms)."""
    a = _directed(17, 7)
    params = {k: v.double() for k, v in O.init_params(1, 5, 1, 8, 2, 6, 7, seed=2).items()}
    gen = torch.Generator().manual_seed(1)
    x, y = torch.randn(2, 5, 17, 1, generator=gen).double(), torch.randn(2, 17, 1, generator=gen).double()
    orc = D.ChainOracle({k: v.numpy() for k, v in params.items()}, [D.diffusion_chains_csr(a)], 7)
    out, loss, g = orc.loss_and_grads(x.numpy(), y.numpy())
    o_d, l_d, g_d = O.dense_loss_and_grads(params, x, y, [D.diffusion_supports_dense(a, 3)])
    assert_close(out, o_d.numpy(), "chain oracle forward", 1e-12)
    for key in g_d:
        assert_close(g[key], g_d[key].numpy(), f"chain oracle grad {key}", 1e-10)


def test_one_chain_oracle_equals_the_chebyshev_oracle():
    """ChainOracle with one chain per graph (L~) is SparseOracle: the same forward, loss and gradients, bit for bit."""
    from stmgcn_b200 import synth
    n, m, k = 15, 2, 3
    sups = [O.chebyshev_supports_dense(synth.make_adjacency(n, g, 0.3), k) for g in range(m)]
    laps = [O.laplacian_csr_from_supports(s) for s in sups]
    params = {k_: v.numpy() for k_, v in O.init_params(m, 4, 1, 8, 2, 6, k + 1, seed=5).items()}
    gen = torch.Generator().manual_seed(6)
    x, y = torch.randn(2, 4, n, 1, generator=gen).numpy(), torch.randn(2, n, 1, generator=gen).numpy()
    o0, l0, g0 = O.SparseOracle(params, laps, k + 1).loss_and_grads(x, y)
    o1, l1, g1 = D.ChainOracle(params, [[lap] for lap in laps], k + 1).loss_and_grads(x, y)
    assert np.array_equal(o0, o1) and l0 == l1 and all(np.array_equal(g0[key], g1[key]) for key in g0)
