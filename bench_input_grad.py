"""Extra cost of the input gradient: one cfg3 training step (forward, MSE, backward) with and without
``obs_seq.requires_grad``, timed alternately with CUDA events on one GPU.  Prints one JSON line with the card's name
and power limit.

    python bench_input_grad.py [--workload cfg3] [--steps 20] [--rounds 3]

The extra work is the temporal GCN's adjoint (K SpMM steps on B*T features and one projection U per graph), the LSTM's
d_xo, and the adjoint of the observation transpose.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json

from benchlib import alternate, device_record, require_cuda, setup_paths


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    require_cuda("bench_input_grad.py")
    setup_paths()

    import torch
    from torch import nn
    import GCN
    import STMGCN
    from stmgcn_b200 import synth

    w = synth.WORKLOADS[args.workload]
    dev = torch.device("cuda:0")
    pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
    sups = [pre.process_sparse(a).to(dev) for a in synth.make_adjacency_list(w)]
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(**synth.model_kwargs(w)).to(dev)
    x, y = (v.to(dev) for v in synth.make_inputs(w))
    crit = nn.MSELoss()

    def step(grad: bool) -> None:
        model.zero_grad(set_to_none=True)
        xs = x.detach().requires_grad_(grad)
        crit(model(obs_seq=xs, sta_adj_list=sups), y).backward()

    runs, launches = alternate({"base": lambda: step(False), "obs_grad": lambda: step(True)},
                               args.rounds, args.steps, args.warmup)
    name, power_limit = device_record()
    print(json.dumps({"workload": w.name, "device": name, "power_limit": power_limit, "steps": args.steps,
                      "ms_per_step": [round(v, 3) for v in runs["base"]],
                      "ms_per_step_obs_grad": [round(v, 3) for v in runs["obs_grad"]],
                      "extra_ms": round(min(runs["obs_grad"]) - min(runs["base"]), 3),
                      "gpu_launches": launches["base"], "gpu_launches_obs_grad": launches["obs_grad"]}))


if __name__ == "__main__":
    main()
