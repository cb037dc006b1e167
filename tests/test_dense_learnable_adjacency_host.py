"""Host tests of a learnable adjacency multiplied dense: which path each mode picks (no GPU: the choice reads the
pattern's size only), and the new entry points refusing bad arguments before any launch."""
import ctypes

import pytest
import torch

import learnable_adjacency_cases as LA


def _adj(kind, a, order=2, lam=2.0):
    import GCN
    return GCN.Adj_Preprocessor(kind, order, lambda_max=lam).process_learnable(a)


@pytest.mark.parametrize("mode", ["auto", "on", "off"])
def test_the_mode_and_the_rule_choose_the_path(monkeypatch, mode):
    from stmgcn_b200 import graph, ops
    from stmgcn_b200.synth import make_similarity_adjacency
    monkeypatch.setattr(ops, "_DENSE_SUPPORTS", mode)
    sim = _adj("chebyshev", make_similarity_adjacency(600, 0))
    sparse = _adj("random_walk_diffusion", LA.graph(600, 1, directed=True, density=0.01).float())
    small = _adj("localpool", make_similarity_adjacency(100, 1), order=1)
    assert graph.dense_rule(sim.n, sim.colidx.numel()) and not graph.dense_rule(sparse.n, sparse.colidx.numel())
    assert sim.dense() == (mode != "off")
    assert sparse.dense() == (mode == "on")
    assert small.dense() == (mode == "on")          # below DENSE_MIN_N only "on" goes dense


def _ptrs(*vals):
    return (ctypes.c_void_p * len(vals))(*vals)


def test_bad_arguments_are_refused_before_any_launch():
    from stmgcn_b200 import _lib
    lib = _lib.lib
    n0 = lib.stmgcn_launch_count()
    a, b, out = 0x10000, 0x20000, 0x40000000
    coef = _lib.float_array([1.0, 2.0])
    cases = [
        (lambda: lib.stmgcn_dense_chain_grad(8, 8, 0, _ptrs(a), _ptrs(b), coef, 0, out, None), b"nterms=0"),
        (lambda: lib.stmgcn_dense_chain_grad(8, 8, 9, _ptrs(*[a] * 9), _ptrs(*[b] * 9), coef, 0, out, None), b"nterms=9"),
        (lambda: lib.stmgcn_dense_chain_grad(0, 8, 1, _ptrs(a), _ptrs(b), coef, 0, out, None), b"n=0"),
        (lambda: lib.stmgcn_dense_chain_grad(8, 0, 1, _ptrs(a), _ptrs(b), coef, 0, out, None), b"f_total=0"),
        (lambda: lib.stmgcn_dense_chain_grad(8, 8, 1, _ptrs(a), _ptrs(b), coef, 2, out, None), b"round_b16=2"),
        (lambda: lib.stmgcn_dense_chain_grad(8, 8, 1, _ptrs(a), _ptrs(b), coef, 0, None, None), b"null pointer"),
        (lambda: lib.stmgcn_dense_chain_grad(8, 8, 2, _ptrs(a, None), _ptrs(b, b), coef, 0, out, None), b"term 1"),
        (lambda: lib.stmgcn_dense_chain_grad(8, 8, 1, _ptrs(a), _ptrs(b), coef, 0, a + 64, None), b"overlap"),
        (lambda: lib.stmgcn_pattern_scatter(0, a, b, 4, 0x30000, out, None), b"pattern_scatter: n=0"),
        (lambda: lib.stmgcn_pattern_scatter(8, None, b, 4, 0x30000, out, None), b"null rowptr"),
        (lambda: lib.stmgcn_pattern_scatter(8, a, None, 4, 0x30000, out, None), b"null colidx"),
        (lambda: lib.stmgcn_pattern_scatter(8, a, b, 4, 0x30000, 0x30000 + 8, None), b"overlaps an input"),
        (lambda: lib.stmgcn_pattern_gather(8, a, b, -1, out, 0x30000, None), b"nnz=-1"),
        (lambda: lib.stmgcn_pattern_gather(8, a, b, 4, out, None, None), b"null colidx / input / output"),
        (lambda: lib.stmgcn_pattern_gather(8, a, b, 4, out, out + 16, None), b"overlaps an input"),
    ]
    for call, msg in cases:
        rc = call()
        assert rc < 0 and msg in lib.stmgcn_last_error(), (msg, rc, lib.stmgcn_last_error())
    assert lib.stmgcn_launch_count() == n0


def test_dense_graph_without_a_copy_holds_the_matrix_itself():
    from stmgcn_b200.graph import DenseGraph
    m = torch.rand(5, 5)
    assert DenseGraph(m, copy=False).mat.data_ptr() == m.data_ptr()
    assert DenseGraph(m).mat.data_ptr() != m.data_ptr()
