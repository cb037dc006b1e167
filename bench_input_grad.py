"""Extra cost of the input gradient: one cfg3 training step (forward, MSE, backward) with and without
``obs_seq.requires_grad``, timed alternately with CUDA events on one GPU.  Prints one JSON line.

    python bench_input_grad.py [--workload cfg3] [--steps 20] [--rounds 3]

The extra work is the temporal GCN's adjoint (K SpMM steps on B*T features and one projection U per graph), the LSTM's
d_xo, and the adjoint of the observation transpose.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.abspath(__file__))
for _p in (REPO, os.path.join(REPO, "st-mgcn_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    from torch import nn
    import GCN
    import STMGCN
    from stmgcn_b200 import _lib, synth

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

    def timed(grad: bool):
        for _ in range(args.warmup):
            step(grad)
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.steps):
            step(grad)
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) / args.steps, (_lib.launch_count() - n0) // args.steps

    runs = {False: [], True: []}
    launches = {}
    for _ in range(args.rounds):
        for grad in (False, True):
            ms, launches[grad] = timed(grad)
            runs[grad].append(ms)
    base, with_dx = min(runs[False]), min(runs[True])
    print(json.dumps({"workload": w.name, "device": torch.cuda.get_device_name(dev), "steps": args.steps,
                      "ms_per_step": [round(v, 3) for v in runs[False]],
                      "ms_per_step_obs_grad": [round(v, 3) for v in runs[True]],
                      "extra_ms": round(with_dx - base, 3), "gpu_launches": launches[False],
                      "gpu_launches_obs_grad": launches[True]}))


if __name__ == "__main__":
    main()
