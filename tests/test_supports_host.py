"""The supports on the host: how ``graph.py`` turns what a caller holds into the CSR and CSR^T the SpMM kernels read.

* a ``GraphHandle`` owns its tensors: editing the caller's CSR after the build reaches neither direction, so the
  forward and the backward always multiply by one matrix;
* ``SparseSupports.version()`` / ``graph.support_version`` change with every kind of in-place edit (the key on which a
  handle rebuilds its support set and ``graphs.GraphedStep`` refuses to replay);
* hand-made CSR with unsorted columns, repeated entries and stored zeros gives the CSR^T of scipy, entry for entry;
* a malformed CSR raises a ``ValueError`` naming the fault;
* the Chebyshev classifier of dense stacks at its tolerance.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from kernel_cases import MALFORMED, handmade_csr, malformed, scipy_of, valid_csr


def test_handmade_csr_has_the_advertised_edges():
    n = 300
    rp, ci, v = handmade_csr(n, 0)
    deg = np.diff(rp.numpy())
    assert set(range(10)) <= set(deg.tolist()) and deg.max() >= n - 1
    a = scipy_of(rp, ci, v, n)
    assert not a.has_sorted_indices
    b = a.copy()
    b.sum_duplicates()
    assert b.nnz < a.nnz                                                    # repeated entries
    assert int((v == 0).sum()) > 0 and bool(torch.signbit(v[v == 0]).any())    # stored 0.0 and -0.0
    assert (np.diff(sp.csr_matrix(a.T).indptr) >= n // 2).any()            # a hub column: a hub row of A^T


def _process_sparse_handle(n=50):
    import GCN
    from stmgcn_b200 import synth
    return GCN.Adj_Preprocessor("chebyshev", 3).process_sparse(synth.make_adjacency(n, 0, 0.1))


@pytest.mark.parametrize("edit", ["mul_", "setitem", "copy_"])
def test_graph_handle_is_a_snapshot_of_the_callers_csr(edit):
    """``GraphHandle.from_csr`` on a handle's CSR, then an in-place edit of the handle's values: the CSR and the CSR^T
    the kernels read both still hold the matrix of build time, and share no memory with the caller's tensors.  (Before
    handles copied their values, the CSR was the caller's ``vals`` itself while the CSR^T was a copy, so after this edit
    the forward and the backward multiplied by two matrices 100 % of max|L~| apart.)"""
    from stmgcn_b200.graph import GraphHandle
    h = _process_sparse_handle()
    before = scipy_of(*h.mats[0], h.n).toarray()
    g = GraphHandle.from_csr(h.n, *h.mats[0])
    mine = {t.untyped_storage().data_ptr() for t in h.mats[0]}
    for transpose in (False, True):
        assert not mine & {t.untyped_storage().data_ptr() for t in g.export(transpose)}, transpose
    with torch.no_grad():
        if edit == "mul_":
            h.vals.mul_(0.5)
        elif edit == "setitem":
            h.vals[::3] = 0.25
        else:
            h.vals.copy_(torch.flip(h.vals, [0]))
    assert np.abs(scipy_of(*h.mats[0], h.n).toarray() - before).max() > 0.1
    fwd = scipy_of(*g.export(False), h.n).toarray()
    bwd = scipy_of(*g.export(True), h.n).toarray()
    assert np.array_equal(fwd, before)
    assert np.array_equal(bwd, before.T)


def test_every_in_place_edit_changes_the_support_version():
    """``support_version`` of a handle changes with each in-place edit of any of its tensors (values, column indices,
    either chain of a two-chain handle) and with a replaced tensor; a dense stack's with an edit of one of its slices."""
    import GCN
    from stmgcn_b200 import synth
    from stmgcn_b200.graph import support_version
    h = _process_sparse_handle()
    diff = GCN.Adj_Preprocessor("random_walk_diffusion", 2).process_sparse(synth.make_directed_adjacency(40, 0, 0.1))
    dense = GCN.Adj_Preprocessor("chebyshev", 3).process(synth.make_adjacency(40, 0, 0.1))
    edits = [(h, lambda: h.vals.mul_(0.5)), (h, lambda: h.vals.__setitem__(3, 1.0)),
             (h, lambda: h.vals.copy_(h.vals)), (h, lambda: h.colidx.copy_(h.colidx)),
             (h, lambda: h.mats.__setitem__(0, (h.rowptr, h.colidx, h.vals.clone()))),
             (diff, lambda: diff.mats[1][2].mul_(2.0)), (diff, lambda: diff.mats[0][2].add_(0.0)),
             (dense, lambda: dense.mul_(0.5)), (dense, lambda: dense[2].zero_())]
    for i, (obj, edit) in enumerate(edits):
        v0 = support_version(obj)
        assert support_version(obj) == v0
        with torch.no_grad():
            edit()
        assert support_version(obj) != v0, f"edit {i} left the version unchanged"


@pytest.mark.parametrize("n", [1, 33, 300])
def test_handmade_csr_exports_scipys_csr_and_transpose(n):
    """``GraphHandle.from_csr`` on hand-made CSR keeps every stored entry (repeats and zeros included): its CSR is the
    caller's matrix entry for entry, its CSR^T lists A^T's entries with sorted columns, repeats in their order, so both
    densify (summing repeats) to exactly scipy's A and A^T."""
    from stmgcn_b200.graph import GraphHandle
    rp, ci, v = handmade_csr(n, n, hub_row=0, hub_col=min(1, n - 1))
    a = scipy_of(rp, ci, v, n)
    g = GraphHandle.from_csr(n, rp, ci, v)
    assert g.nnz == a.nnz
    for transpose, want in ((False, a.toarray()), (True, a.toarray().T)):
        rp_g, ci_g, v_g = g.export(transpose)
        assert rp_g.dtype == ci_g.dtype == torch.int32 and v_g.dtype == torch.float32
        assert int(rp_g[-1]) == a.nnz
        got = scipy_of(rp_g, ci_g, v_g, n)
        assert np.array_equal(got.toarray(), want), transpose
    rp_t, ci_t, _ = g.export(True)
    for i in range(n):
        row = ci_t[rp_t[i]:rp_t[i + 1]].numpy()
        assert (np.diff(row) >= 0).all(), f"CSR^T row {i} is not sorted"


@pytest.mark.parametrize("case", MALFORMED)
def test_malformed_csr_raises_a_value_error_naming_the_fault(case):
    from stmgcn_b200.graph import GraphHandle
    n, rp, ci, v, msg = malformed(case)
    with pytest.raises(ValueError, match=msg):
        GraphHandle.from_csr(n, rp, ci, v)


def test_the_valid_csr_the_malformed_ones_come_from_is_accepted():
    from stmgcn_b200.graph import GraphHandle
    n = 40
    assert GraphHandle.from_csr(n, *valid_csr(n)).nnz == valid_csr(n)[1].numel()


TOL_CHEB = 5e-5          # graph._is_chebyshev_stack's default tolerance


@pytest.mark.parametrize("slice_k", [0, 2, 3])
@pytest.mark.parametrize("factor", [10.0, 0.1])
def test_chebyshev_classifier_at_its_tolerance(slice_k, factor):
    """A ``process`` stack (K = 3) with slice ``k`` scaled by ``1 + factor * 5e-5``: at 10x the classifier's tolerance
    the recurrence probe misses by 5e-4 and the stack goes generic; at 0.1x it stays Chebyshev (the GPU suite checks that
    the model's results on such a stack are still those of the stack as given).  Unperturbed it is Chebyshev."""
    import GCN
    from stmgcn_b200 import synth
    from stmgcn_b200.graph import _is_chebyshev_stack
    a = GCN.Adj_Preprocessor("chebyshev", 3).process(synth.make_adjacency(60, 1, 0.1))
    assert _is_chebyshev_stack(a)
    b = a.clone()
    b[slice_k] *= 1.0 + factor * TOL_CHEB
    assert _is_chebyshev_stack(b) == (factor < 1.0)
