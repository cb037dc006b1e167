"""CUDA-graph replay of a whole training step (stmgcn_b200.graphs.GraphedStep) against the eager step: same loss, same
gradients; weights updated between replays are seen by the replay (the weight-image pack kernels are part of the graph);
a batch of another size falls back to the eager path."""
import pytest
import torch
from torch import nn

import stmgcn_oracle as O
from helpers import DEV, assert_close, build_model

pytestmark = pytest.mark.gpu


def _eager(model, crit, x, y, sups):
    for p in model.parameters():
        p.grad = None
    loss = crit(model(obs_seq=x, sta_adj_list=sups), y)
    loss.backward()
    return loss.item(), {k: p.grad.detach().clone() for k, p in model.named_parameters()}


def test_graphed_step_matches_eager_and_tracks_weight_updates():
    from stmgcn_b200 import dp, graphs, synth
    meta = dict(n=96, m=3, k=3, t=12, b=6, c=1, hid=64, layers=3, gcn_hid=64)
    adjs = [synth.make_adjacency(meta["n"], g, 0.05) for g in range(meta["m"])]
    sups = [O.chebyshev_supports_dense(a, meta["k"]).to(DEV) for a in adjs]
    torch.manual_seed(5)
    model = build_model(meta, DEV)
    crit = nn.MSELoss(reduction="mean")
    gen = torch.Generator().manual_seed(6)
    xs = [torch.randn(meta["b"], meta["t"], meta["n"], 1, generator=gen).to(DEV) for _ in range(3)]
    ys = [torch.randn(meta["b"], meta["n"], 1, generator=gen).to(DEV) for _ in range(3)]
    ref = [_eager(model, crit, x, y, sups) for x, y in zip(xs[:2], ys[:2])]
    bucket = dp.GradBucket(model)
    gstep = graphs.GraphedStep(model, crit, xs[0], ys[0], sups, bucket=bucket)
    for i in range(2):                                   # replay on two different batches
        loss = gstep(xs[i], ys[i])
        assert abs(loss.item() - ref[i][0]) <= 1e-5 * abs(ref[i][0])
        for key, p in model.named_parameters():
            assert_close(p.grad.cpu().numpy(), ref[i][1][key].cpu().numpy(), f"graph replay {i} grad {key}", 2e-5)
    # an optimizer step between replays: the replay must use the NEW weights
    with torch.no_grad():
        for p in model.parameters():
            p.add_(0.01 * torch.randn(p.shape, generator=gen).to(DEV))
    loss = gstep(xs[2], ys[2])
    g_graph = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    l_graph = loss.item()
    l_eager, g_eager = _eager(model, crit, xs[2], ys[2], sups)
    assert abs(l_graph - l_eager) <= 1e-5 * abs(l_eager), (l_graph, l_eager)
    for key in g_eager:
        assert_close(g_graph[key].cpu().numpy(), g_eager[key].cpu().numpy(), f"after weight update, grad {key}", 2e-5)
    # short last batch (Data_Container.py:122): eager fallback inside GraphedStep
    bucket = dp.GradBucket(model)
    gstep = graphs.GraphedStep(model, crit, xs[0], ys[0], sups, bucket=bucket)
    xs_short, ys_short = xs[1][:2].contiguous(), ys[1][:2].contiguous()
    loss_s = gstep(xs_short, ys_short)
    g_s = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    l_ref, g_ref = _eager(model, crit, xs_short, ys_short, sups)
    assert abs(loss_s.item() - l_ref) <= 1e-5 * abs(l_ref)
    for key in g_ref:
        assert_close(g_s[key].cpu().numpy(), g_ref[key].cpu().numpy(), f"short batch grad {key}", 2e-5)
