#!/usr/bin/env python
"""bench_diffusion.py -- the training step with random-walk diffusion supports against the same step with Chebyshev
supports, at cfg3 shapes.

    python bench_diffusion.py [--steps K] [--warmup W] [--rounds R] [--order 2] [--workload cfg3]

Both models see the same DIRECTED synthetic graphs (``synth.make_directed_adjacency``, seeded) and the same inputs:
``chebyshev`` with ``K`` (``K+1`` supports, one recurrence chain of ``L~``) and ``random_walk_diffusion`` with ``K``
(``2K+1`` supports, two chains: ``P_f^T`` and ``P_b^T``), both from ``Adj_Preprocessor.process_sparse``.  A step is
forward + MSE + backward through the public modules, timed with CUDA events; the two kinds alternate for ``R`` rounds of
``K`` steps each and the median round is reported per kind.  Before any time is printed, the loss of two picked windows
of each kind's step is checked against the fp64 sparse oracle (``oracle/diffusion_oracle.py``'s ``ChainOracle``;
windows are independent, so the oracle runs on those two only), at the 1e-4 bar.  Prints one JSON line with the card's name and power limit.
Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys

from benchlib import alternate, device_record, require_cuda, setup_paths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--order", type=int, default=2)
    ap.add_argument("--workload", default="cfg3")
    args = ap.parse_args()
    require_cuda("bench_diffusion.py")
    setup_paths()

    import numpy as np
    import scipy.sparse as sp
    import torch
    from torch import nn
    import GCN
    import STMGCN
    import diffusion_oracle as D
    from stmgcn_b200 import synth

    w = synth.WORKLOADS[args.workload]
    dev = torch.device("cuda:0")
    adjs = [synth.make_directed_adjacency(w.n_regions, m, w.density) for m in range(w.n_graphs)]
    x_cpu, y_cpu = synth.make_inputs(w, seed=0)
    x, y = x_cpu.to(dev), y_cpu.to(dev)
    crit = nn.MSELoss(reduction="mean")
    kinds = {}
    for kind in ("chebyshev", "random_walk_diffusion"):
        pre = GCN.Adj_Preprocessor(kind, args.order)
        sups = [pre.process_sparse(a) for a in adjs]
        kw = synth.model_kwargs(w)
        kw["sta_kernel_config"] = {"kernel_type": kind, "K": args.order}
        torch.manual_seed(0)
        model = STMGCN.ST_MGCN(**kw)
        params = {k: v.detach().clone().numpy() for k, v in model.state_dict().items()}
        kinds[kind] = dict(model=model.to(dev), sups=[s.to(dev) for s in sups], sups_cpu=sups, params=params,
                           ks=len(sups[0]))

    def step(k):
        m = kinds[k]["model"]
        for p in m.parameters():
            p.grad = None
        loss = crit(m(obs_seq=x, sta_adj_list=kinds[k]["sups"]), y)
        loss.backward()
        return loss

    # correctness first: the picked windows' loss of each kind against the fp64 sparse oracle
    picks = [0, w.batch - 1]
    checks = {}
    for kind, k in kinds.items():
        with torch.no_grad():
            out = k["model"](obs_seq=x, sta_adj_list=k["sups"])
        got = float(((out[picks] - y[picks]) ** 2).mean().double())
        chains = [[sp.csr_matrix(m.numpy()) for m in h.matrices_dense()] for h in k["sups_cpu"]]
        orc = D.ChainOracle(k["params"], chains, k["ks"], dtype=np.float64)
        o_ref = orc.forward(x_cpu[picks].numpy())
        want = float(np.mean((o_ref - y_cpu[picks].numpy().astype(np.float64)) ** 2))
        checks[kind] = abs(got - want) / abs(want)
        if not checks[kind] <= 1e-4:
            sys.exit(f"{kind}: loss of windows {picks} {got:.8f} vs fp64 oracle {want:.8f} "
                     f"(relative error {checks[kind]:.2e} > 1e-4): no time reported")
        del out

    times, _ = alternate({kind: lambda kind=kind: step(kind) for kind in kinds}, args.rounds, args.steps, args.warmup)
    assert all(bool(torch.isfinite(step(kind))) for kind in kinds)     # every timed step computes this same loss
    name, limit = device_record()
    ms = {kind: statistics.median(t) for kind, t in times.items()}
    result = {
        "workload": args.workload, "n_regions": w.n_regions, "graphs": w.n_graphs, "seq_len": w.seq_len,
        "batch": w.batch, "hidden": w.lstm_hidden, "K": args.order, "graphs_kind": "directed (synth.make_directed_adjacency)",
        "step": "fwd + MSE + bwd", "device": name, "power_limit": limit,
        "chebyshev": {"supports": kinds["chebyshev"]["ks"], "ms_per_step": round(ms["chebyshev"], 3),
                      "rounds_ms": [round(t, 3) for t in times["chebyshev"]],
                      "loss_rel_err_vs_fp64_oracle": checks["chebyshev"]},
        "random_walk_diffusion": {"supports": kinds["random_walk_diffusion"]["ks"],
                                  "ms_per_step": round(ms["random_walk_diffusion"], 3),
                                  "rounds_ms": [round(t, 3) for t in times["random_walk_diffusion"]],
                                  "loss_rel_err_vs_fp64_oracle": checks["random_walk_diffusion"]},
        "diffusion_over_chebyshev": round(ms["random_walk_diffusion"] / ms["chebyshev"], 3),
    }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
