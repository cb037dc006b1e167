"""Host tests of dense support matrices multiplied dense: the dispatch rule at and around its constants, the
dense-supports switch, the conversion cache keyed on the mode, and the SDDMM's refusal of a dense handle.  No GPU
needed."""
import os
import subprocess
import sys

import pytest
import torch

from stmgcn_b200 import graph, ops


@pytest.fixture
def mode():
    old = ops.dense_supports()
    yield ops.set_dense_supports
    ops.set_dense_supports(old)


def test_rule_at_and_around_its_constants():
    n0, d = graph.DENSE_MIN_N, graph.DENSE_MIN_DENSITY
    at = int(-(-d * n0 * n0 // 1))                     # the least nnz at the density threshold
    assert graph.dense_rule(n0, at) and graph.dense_rule(n0, n0 * n0)
    assert not graph.dense_rule(n0, at - 1)
    assert not graph.dense_rule(n0 - 1, (n0 - 1) ** 2)  # below the size threshold even fully dense
    n = 4096
    assert graph.dense_rule(n, n * n) and graph.dense_rule(n, int(-(-d * n * n // 1)))
    assert not graph.dense_rule(n, int(0.01 * n * n))   # the benchmarks' 1 % graphs stay CSR
    assert not graph.dense_rule(n, 0)


def test_switch_values_and_rejections(mode):
    for m in ("auto", "on", "off"):
        mode(m)
        assert ops.dense_supports() == m
    for bad in ("", "ON", "dense", "1", None):
        with pytest.raises(ValueError):
            mode(bad)


@pytest.mark.parametrize("value,ok", [("on", True), ("off", True), ("auto", True), ("yes", False)])
def test_environment_switch_is_read_and_checked_at_import(value, ok):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, STMGCN_DENSE_SUPPORTS=value, PYTHONPATH=os.path.join(root, "st-mgcn_b200"))
    res = subprocess.run([sys.executable, "-c", "from stmgcn_b200 import ops; print(ops.dense_supports())"],
                         capture_output=True, text=True, env=env)
    if ok:
        assert res.returncode == 0 and res.stdout.strip() == value, res.stderr
    else:
        assert res.returncode != 0 and "STMGCN_DENSE_SUPPORTS" in res.stderr


def test_cache_key_includes_the_mode(mode):
    """A stack converted under one mode is converted again under another (the key differs), not served stale."""
    a = torch.zeros(2, 8, 8)
    keys = {}
    for m in ("off", "on", "auto"):
        mode(m)
        keys[m] = graph._cache_key(a)
    assert len(set(keys.values())) == 3
    mode("off")
    assert graph._cache_key(a) == keys["off"]


def test_conversion_follows_the_mode(mode, monkeypatch):
    """Under off every matrix becomes CSR with no count; under on a DenseGraph (an fp32 snapshot) with no count; under
    auto the rule decides on the non-zero count, and a CSR build takes that count (no second count)."""
    built = []
    monkeypatch.setattr(graph.GraphHandle, "from_dense",
                        classmethod(lambda cls, m, nnz=None: built.append(nnz) or "csr"))
    n = graph.DENSE_MIN_N
    full = torch.ones(n, n)
    sparse = torch.zeros(n, n)
    sparse[0, 0] = 1.0
    sparse[3, 1] = float("nan")                          # NaN is a non-zero entry
    mode("off")
    assert graph._graph_from_dense(full) == "csr"
    mode("on")
    g = graph._graph_from_dense(sparse)
    assert isinstance(g, graph.DenseGraph) and g.nnz == n * n and g.n == n
    sparse[0, 1] = 2.0                                  # the snapshot does not see an edit after the build
    assert float(g.mat[0, 1]) == 0.0 and g.mat.is_contiguous() and g.mat.dtype == torch.float32
    mode("auto")
    assert isinstance(graph._graph_from_dense(full), graph.DenseGraph)
    assert graph._graph_from_dense(sparse) == "csr"
    assert built == [None, 3]


def test_csr_from_a_known_count_equals_the_counting_build():
    gen = torch.Generator().manual_seed(0)
    m = torch.where(torch.rand(50, 50, generator=gen) < 0.1, torch.randn(50, 50, generator=gen), torch.zeros(50, 50))
    m[4, 7] = -0.0
    m[9, 2] = float("nan")
    a, b = graph.GraphHandle.from_dense(m), graph.GraphHandle.from_dense(m, int((m != 0).sum()))
    for t in (False, True):
        for x, y in zip(a.export(t), b.export(t)):
            assert torch.equal(x, y) if x.dtype != torch.float32 else torch.equal(x.nan_to_num(7.0), y.nan_to_num(7.0))


def test_csr_sddmm_refuses_a_dense_graph():
    g = graph.DenseGraph(torch.eye(4))
    dv = torch.zeros(4)
    with pytest.raises(AssertionError, match="DenseGraph"):
        ops.csr_sddmm_(g, [(torch.zeros(4, 2), torch.zeros(4, 2), 1.0)], dv)
