"""The reference semantics for NaN and +-Inf that tests/test_gpu_nonfinite.py holds the kernels to: torch's ReLU and
its backward, and what the dense fp64 oracle does with NaN supports and with a NaN in one window's observations."""
import math

import torch

import stmgcn_oracle as O


def test_torch_relu_propagates_nan_and_its_backward_passes_the_gradient_there():
    """relu(NaN) = NaN, relu(+-Inf) = +Inf / 0; the backward is ``out <= 0 ? 0 : grad``, so it passes the gradient at
    NaN.  clamp_min(0), which the finite-value tests use as a reference, differs there: its gradient at NaN is 0."""
    x = torch.tensor([math.nan, -1.0, 2.0, math.inf, -math.inf], dtype=torch.float64, requires_grad=True)
    y = torch.relu(x)
    assert torch.equal(torch.isnan(y), torch.tensor([True, False, False, False, False]))
    assert y[1:].tolist() == [0.0, 2.0, math.inf, 0.0]
    (g,) = torch.autograd.grad(y.sum(), x)
    assert g.tolist() == [1.0, 0.0, 1.0, 1.0, 0.0]
    (g_clamp,) = torch.autograd.grad(x.clamp_min(0).sum(), x)
    assert g_clamp.tolist() == [0.0, 0.0, 1.0, 1.0, 0.0]


def _isolated_setup():
    """test_gpu_exact_kernels' isolated-region model at H = G = 64 (the tensor-core shapes): graph 0 has a region
    without edges."""
    from stmgcn_b200 import synth
    shape = dict(n=60, m=2, k=2, t=6, b=3, c=1, hid=64, layers=2, gcn_hid=64)
    adjs = [synth.make_adjacency(shape["n"], g, 0.08) for g in range(shape["m"])]
    iso = 17
    adjs[0][iso, :] = 0.0
    adjs[0][:, iso] = 0.0
    adjs[0][iso - 1, iso + 1] = adjs[0][iso + 1, iso - 1] = 1.0
    return shape, adjs, iso


def test_dense_oracle_loss_is_nan_on_process_supports_with_an_isolated_region():
    """Adj_Preprocessor.process follows the reference's symmetric_normalize: D^-1/2 is infinite on an isolated region,
    so the supports have a NaN row and column there, and the dense oracle's output and loss are NaN."""
    import GCN
    shape, adjs, iso = _isolated_setup()
    sups = [GCN.Adj_Preprocessor("chebyshev", shape["k"]).process(a) for a in adjs]
    assert bool(torch.isnan(sups[0][1][iso]).all()) and bool(torch.isnan(sups[0][1][:, iso]).all())
    assert bool(torch.isfinite(sups[1]).all())
    params = O.init_params(shape["m"], shape["t"], shape["c"], shape["hid"], shape["layers"], shape["gcn_hid"],
                           shape["k"] + 1, seed=5)
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(shape["b"], shape["t"], shape["n"], shape["c"], generator=gen)
    y = torch.randn(shape["b"], shape["n"], shape["c"], generator=gen)
    out, loss, _ = O.dense_loss_and_grads({k: v.double() for k, v in params.items()}, x.double(), y.double(),
                                          [s.double() for s in sups])
    assert math.isnan(float(loss))
    assert not bool(torch.isfinite(out).any())


def test_dense_oracle_keeps_a_nan_observation_in_its_window():
    """A NaN in one window's obs makes that window's outputs and obs gradient NaN and leaves the other windows' finite:
    the windows meet only in the parameter gradients, which are all non-finite."""
    shape, adjs, _ = _isolated_setup()
    sups = [O.chebyshev_supports_dense(a.double(), shape["k"]) for a in adjs[1:]]
    params = {k: v.double() for k, v in O.init_params(1, shape["t"], shape["c"], shape["hid"], shape["layers"],
                                                      shape["gcn_hid"], shape["k"] + 1, seed=6).items()}
    gen = torch.Generator().manual_seed(6)
    x = torch.randn(shape["b"], shape["t"], shape["n"], shape["c"], generator=gen).double()
    x[1, 2, 5, 0] = math.nan
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    xg = x.clone().requires_grad_(True)
    out = O.dense_st_mgcn(leaves, xg, sups)
    loss = out.square().mean()
    grads = torch.autograd.grad(loss, [xg] + list(leaves.values()))
    assert not bool(torch.isfinite(out[1]).any()) and bool(torch.isfinite(out[[0, 2]]).all())
    assert not bool(torch.isfinite(grads[0][1]).any()) and bool(torch.isfinite(grads[0][[0, 2]]).all())
    assert all(not bool(torch.isfinite(g).any()) for g in grads[1:])
