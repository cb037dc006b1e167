"""Cost of packing the tensor-core weight images on every forward: one training step (forward, MSE, backward) with the
product code ("new": every forward packs the LSTM and projection images from the weights as they are) against a
memoised packer local to this script ("old": each image packed once per weight storage and reused, which is what a
cache keyed on the weights' version did in a loop without an optimizer step).  Both run in one process, alternated
round by round, each step timed with CUDA events.  Prints one JSON line.

    python bench_pack.py [--steps 10] [--rounds 5] [--warmup 3]

Workloads: cfg2 (1024 regions, batch 32, one bf16 plane) and cfg3 (4096 regions, batch 64, two planes).  Also times
the pack launches alone and checks that "old" and "new" give the same output, loss and gradients: no further apart
than two runs of "new" (the region pooling and the gradient reductions accumulate with atomics, a ReLU pre-activation
at the kink can then land on either side, and in the one-plane mode a hidden state can round to the neighbouring bf16
value), or SAME.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json
import statistics

from benchlib import device_record, require_cuda, setup_paths, timed

CASES = (("cfg2", 1), ("cfg3", 2))      # (workload, bf16 planes of the LSTM)
SAME = 2e-5                             # two-plane bar of two fresh copies of one model (tests/test_gpu_param_updates.py)


def memoised(ops):
    """("old") drop-in replacements of ops._lstm16_images / ops._proj_images that pack once per weight storage."""
    real_lstm, real_proj, memo = ops._lstm16_images, ops._proj_images, {}

    def lstm_images(weights, n_layers, c_in):
        key = ("lstm",) + tuple(w.data_ptr() for w in weights) + (n_layers, c_in)
        if key not in memo:
            memo[key] = real_lstm(weights, n_layers, c_in)
        return memo[key]

    def proj_images(w, ks, p, need_bwd):
        key = ("proj", w.data_ptr(), ks, p, need_bwd, ops.lstm_path())
        if key not in memo:
            memo[key] = real_proj(w, ks, p, need_bwd)
        return memo[key]

    return lstm_images, proj_images, memo


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10, help="timed steps per variant per round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    require_cuda("bench_pack.py")
    setup_paths()

    import torch
    from torch import nn
    import GCN
    import STMGCN
    import stmgcn_oracle as O
    from stmgcn_b200 import ops, synth

    dev = torch.device("cuda:0")
    gpu, limit = device_record()
    result = dict(gpu=gpu, power_limit=limit, steps_per_variant=args.steps * args.rounds)
    real = (ops._lstm16_images, ops._proj_images)
    old_planes = ops.lstm_planes()
    for name, planes in CASES:
        ops.set_lstm_planes(planes)
        w = synth.WORKLOADS[name]
        pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
        sups = [pre.process_sparse(a).to(dev) for a in synth.make_adjacency_list(w)]
        torch.manual_seed(0)
        model = STMGCN.ST_MGCN(**synth.model_kwargs(w)).to(dev)
        x, y = (v.to(dev) for v in synth.make_inputs(w))
        crit = nn.MSELoss()
        old_lstm, old_proj, memo = memoised(ops)

        def use(variant):
            ops._lstm16_images, ops._proj_images = (old_lstm, old_proj) if variant == "old" else real

        def step():
            model.zero_grad(set_to_none=True)
            out = model(obs_seq=x, sta_adj_list=sups)
            loss = crit(out, y)
            loss.backward()
            return out, loss

        try:
            # same results: one step of each, and a second step of "new" for the run-to-run spread
            res = {}
            for variant in ("new", "new again", "old"):
                use(variant.split()[0])
                out, loss = step()
                res[variant] = [out.detach().cpu().numpy(), loss.detach().cpu().numpy()] + \
                    [p.grad.cpu().numpy() for p in model.parameters()]
            spread = max(O.max_rel_err(a, b) for a, b in zip(res["new again"], res["new"]))
            diff = max(O.max_rel_err(a, b) for a, b in zip(res["old"], res["new"]))
            del res
            assert diff <= max(SAME, 4 * spread), f"{name}: old and new differ by {diff:.2e} (new vs new: {spread:.2e})"

            # one sample per step, not per round: the summary is a distribution over steps (median, p10, p90)
            times = {"new": [], "old": []}
            for _ in range(args.rounds):
                for variant in ("old", "new"):
                    use(variant)
                    for _ in range(args.warmup):
                        step()
                    times[variant] += [timed(step, 1)[0] for _ in range(args.steps)]
        finally:
            ops._lstm16_images, ops._proj_images = real
            memo.clear()

        # the pack launches of one step alone (every branch's LSTM images and its projection images), one stream
        ks = model.sta_K

        def packs():
            for cg, gcn in zip(model.rnn_list, model.gcn_list):
                ops._lstm16_images([wt.detach() for wt in cg._lstm_weights()], cg.lstm_num_layers, cg.input_dim)
                ops._proj_images(gcn.W.detach(), ks, gcn.input_dim, True)

        pack_ms, _ = timed(packs, 50, args.warmup)

        def summary(v):
            q = statistics.quantiles(v, n=10)
            return {"median_ms": round(statistics.median(v), 3), "p10_ms": round(q[0], 3), "p90_ms": round(q[-1], 3)}

        result[name] = {"planes": planes, "old": summary(times["old"]), "new": summary(times["new"]),
                        "new_minus_old_median_ms": round(statistics.median(times["new"]) - statistics.median(times["old"]), 3),
                        "pack_ms_per_step_serial": round(pack_ms, 4),
                        "max_rel_diff_old_vs_new": float(f"{diff:.2e}"),
                        "max_rel_diff_new_vs_new": float(f"{spread:.2e}")}
        del model, sups, x, y
        torch.cuda.empty_cache()
    ops.set_lstm_planes(old_planes)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
