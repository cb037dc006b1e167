"""Cost of learning the graphs at cfg3 (4096 regions, 3 graphs, K = 3, seq_len 12, batch 64, fp32-grade mode).

    python bench_learnable_adjacency.py [--steps 10] [--rounds 4] [--reps 50]

* step: the training step (forward + MSE + backward) five ways, alternating in rounds, each timed with CUDA events:
  fixed handles (``process_sparse`` once); ``process_sparse`` rebuilt from the edge weights every step; three
  ``LearnableAdjacency`` modules, eager; the same in a ``GraphedStep``; fixed handles in a ``GraphedStep``;
* kernels: the normalisation's forward launches (``stmgcn_adj_norm_fwd``) and backward launches (``stmgcn_adj_norm_bwd``)
  of one graph alone.

Before any time is printed, the loss and d weight of the modules on two windows are checked against a dense fp64
restatement (``oracle/stmgcn_oracle.py``, Laplacians built from the weights as leaves) that takes the step's own ReLU
masks, at 1e-4.  Prints one JSON line, with the card's name and power limit.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json

from benchlib import alternate, device_record, require_cuda, setup_paths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    require_cuda("bench_learnable_adjacency.py")
    setup_paths()

    import torch
    from torch import nn
    import GCN
    import STMGCN
    import stmgcn_oracle as O
    from stmgcn_b200 import _lib, ops, synth
    from stmgcn_b200.graphs import GraphedStep

    dev = torch.device("cuda:0")
    w = synth.WORKLOADS["cfg3"]
    ops.set_lstm_planes(2)
    pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
    adjs = [a.to(dev).to_sparse_coo().coalesce() for a in synth.make_adjacency_list(w)]
    idx = [a.indices() for a in adjs]
    weights = [nn.Parameter(a.values().clone()) for a in adjs]
    fixed = [pre.process_sparse(a) for a in adjs]
    mods = [pre.process_learnable(a).to(dev) for a in adjs]
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(**synth.model_kwargs(w)).to(dev)
    crit = nn.MSELoss()
    x, y = (t.to(dev) for t in synth.make_inputs(w, seed=0))

    def rebuilt():
        return [pre.process_sparse(torch.sparse_coo_tensor(i, v, a.shape)) for i, v, a in zip(idx, weights, adjs)]

    def step(sups):
        model.zero_grad(set_to_none=False)
        for v in weights + [m.weight for m in mods]:
            v.grad = None
        loss = crit(model(obs_seq=x, sta_adj_list=sups() if callable(sups) else sups), y)
        loss.backward()
        return loss

    # ---- correctness first: two windows against dense fp64 ------------------------------------------------------------
    x2, y2 = x[:2], y[:2]
    model.zero_grad()
    masks = []                          # the step's own ReLU masks (out > 0) of every GCN, in launch order
    real_proj_fwd = ops._proj_fwd

    def recording_proj_fwd(*a, **k):
        out_ = real_proj_fwd(*a, **k)
        masks.append(out_ > 0)
        return out_
    ops._proj_fwd = recording_proj_fwd
    try:
        loss2 = crit(model(obs_seq=x2, sta_adj_list=mods), y2)
    finally:
        ops._proj_fwd = real_proj_fwd
    loss2.backward()
    params = {k: p.detach().double() for k, p in model.state_dict().items()}
    leaves, stacks = [], []
    for m in mods:
        leaf = m.weight.detach().double().clone().requires_grad_(True)
        adj64 = torch.zeros(m.n, m.n, dtype=torch.float64, device=dev).index_put(m.edges(), leaf, accumulate=True)
        stacks.append(O.chain_stack_dense([O.rescaled_laplacian_dense(adj64, m.lambda_max)], m.order))
        leaves.append(leaf)
    out64 = O.dense_st_mgcn(params, x2.double(), stacks, masks=masks)
    loss64 = ((out64 - y2.double()) ** 2).mean()
    loss64.backward()
    err_loss = abs(loss2.item() - loss64.item()) / abs(loss64.item())
    err_grad = max(O.max_rel_err(m.weight.grad.cpu().numpy(), leaf.grad.cpu().numpy()) for m, leaf in zip(mods, leaves))
    del stacks, out64, loss64, leaves, masks, loss2      # no autograd graph of an eager step outlives it into a capture
    torch.cuda.empty_cache()
    if not (err_loss <= 1e-4 and err_grad <= 1e-4):
        raise SystemExit(f"bench_learnable_adjacency: parity failed: loss {err_loss:.3e}, d weight {err_grad:.3e}")

    # ---- the step, five ways, alternating -----------------------------------------------------------------------------
    graphed_fixed = GraphedStep(model, crit, x, y, fixed)
    graphed_mods = GraphedStep(model, crit, x, y, mods)
    variants = {"fixed": lambda: step(fixed), "process_sparse_per_step": lambda: step(rebuilt),
                "module_eager": lambda: step(mods), "module_graphed": lambda: graphed_mods(),
                "fixed_graphed": lambda: graphed_fixed()}
    ms, _ = alternate(variants, args.rounds, args.steps, 3)

    # ---- the normalisation's launches alone ---------------------------------------------------------------------------
    m = mods[0]
    n, nnz = m.n, m.colidx.numel()
    wt = m.weight.detach()
    work_f = torch.empty(2 * n, device=dev)
    work_b = torch.empty(3 * n + nnz, device=dev)
    vals, g, dw = torch.empty(nnz, device=dev), torch.randn(nnz, device=dev), torch.empty_like(wt)
    head = ops._norm_args(m.kind, m.pattern(), wt, m.scale)

    def fwd():
        _lib.check(ops.L.stmgcn_adj_norm_fwd(*head, work_f.data_ptr(), work_f.numel(), vals.data_ptr(), None,
                                             ops._stream()), "adj_norm_fwd")

    def bwd():
        _lib.check(ops.L.stmgcn_adj_norm_bwd(*head, g.data_ptr(), None, work_b.data_ptr(), work_b.numel(), dw.data_ptr(),
                                             ops._stream()), "adj_norm_bwd")
    norm_ms, _ = alternate({"fwd": fwd, "bwd": bwd}, args.rounds, args.reps, 5)

    name, power = device_record()
    med = lambda v: sorted(v)[len(v) // 2]      # noqa: E731
    print(json.dumps(dict(
        bench="learnable_adjacency", workload="cfg3", card=name, power_limit=power, learnable_graphs=len(mods),
        nnz_per_graph=[int(i.shape[1]) for i in idx], step_ms_median={k: med(v) for k, v in ms.items()},
        step_ms_rounds=ms, norm_fwd_us_median=med(norm_ms["fwd"]) * 1e3,
        norm_bwd_us_median=med(norm_ms["bwd"]) * 1e3,
        parity=dict(windows=2, loss_rel_err=err_loss, d_weight_rel_err=err_grad))))


if __name__ == "__main__":
    main()
