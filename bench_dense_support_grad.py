"""Cost of dense support-stack gradients at cfg3 (4096 regions, 3 graphs, K = 3, seq_len 12, batch 64, fp32-grade mode).

    python bench_dense_support_grad.py [--steps 5] [--rounds 3] [--reps 10]

* kernels: ``stmgcn_dense_support_grad`` (dA_k = U_k x^T, 3xTF32 wgmma) for 4 slices against ``torch.matmul(U_k, x.T)``
  in fp32 with TF32 off, the fp32-grade alternative, at the spatial GCN's shape (F = B*64 = 4096) and the temporal one's
  (F = B*T = 768), alternated round by round; achieved TFLOP/s from the shapes (2 N^2 F per slice);
* step: the training step (forward + MSE + backward) on constant Chebyshev stacks against the same step on stacks
  ``process(adj)`` built from adjacencies that require grad (the step then also runs ``process`` and its backward, and
  converts the stacks at every forward).

Before any time is printed, the kernel's dA at both shapes is checked against an fp64 matmul of the same U and x, at
5e-5.  Prints one JSON line, with the card's name and power limit.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json

from benchlib import alternate, device_record, require_cuda, setup_paths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    require_cuda("bench_dense_support_grad.py")
    setup_paths()

    import torch
    from torch import nn
    import GCN
    import STMGCN
    from stmgcn_b200 import ops, synth

    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    w = synth.WORKLOADS["cfg3"]
    n, ks = w.n_regions, w.cheb_order + 1
    ops.set_lstm_planes(2)

    # ---- the kernel against the fp32 matmul, correctness first ----------------------------------------------------------
    kernels = {}
    for name, f_total in (("spatial", w.batch * w.gcn_hidden), ("temporal", w.batch * w.seq_len)):
        gen = torch.Generator(device=dev).manual_seed(1)
        u = torch.randn((ks, n, f_total), device=dev, generator=gen)
        x = torch.randn((n, f_total), device=dev, generator=gen)
        da = ops.dense_support_grad(u, x)
        err = 0.0
        for k in range(ks):
            ref = u[k].double() @ x.double().t()
            err = max(err, float((da[k].double() - ref).abs().max() / ref.abs().max()))
        del ref
        if err > 5e-5:
            raise SystemExit(f"bench_dense_support_grad: kernel parity failed at {name}: {err:.3e}")
        out = torch.empty_like(da)

        def torch_fp32():
            for k in range(ks):
                torch.matmul(u[k], x.t(), out=out[k])
        ms, _ = alternate({"kernel": lambda: ops.dense_support_grad(u, x), "torch_fp32": torch_fp32},
                          args.rounds, args.reps, 3)
        flop = 2.0 * n * n * f_total * ks
        t_k, t_t = min(ms["kernel"]), min(ms["torch_fp32"])
        kernels[name] = dict(f_total=f_total, slices=ks, kernel_ms=t_k, torch_fp32_ms=t_t, speedup=t_t / t_k,
                             kernel_tflops=flop / t_k * 1e-9, torch_fp32_tflops=flop / t_t * 1e-9, parity_rel_err=err)
        del u, x, da, out
        torch.cuda.empty_cache()

    # ---- the cfg3 step: constant stacks against stacks from adjacencies that require grad -----------------------------
    pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
    adjs = [a.to(dev) for a in synth.make_adjacency_list(w)]
    const = [pre.process(a) for a in adjs]
    learn = [a.clone().requires_grad_(True) for a in adjs]
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(**synth.model_kwargs(w)).to(dev)
    crit = nn.MSELoss()
    x, y = (t.to(dev) for t in synth.make_inputs(w, seed=0))

    def step(grad):
        model.zero_grad(set_to_none=False)
        for a in learn:
            a.grad = None
        sups = [pre.process(a) for a in learn] if grad else const
        loss = crit(model(obs_seq=x, sta_adj_list=sups), y)
        loss.backward()
        return loss

    step_ms, launches = alternate({"constant": lambda: step(False), "requires_grad": lambda: step(True)},
                                  args.rounds, args.steps, 2)
    card, power = device_record()
    print(json.dumps(dict(
        bench="dense_support_grad", workload="cfg3", card=card, power_limit=power, kernels=kernels,
        step_ms_constant=min(step_ms["constant"]), step_ms_requires_grad=min(step_ms["requires_grad"]),
        step_added_ms=min(step_ms["requires_grad"]) - min(step_ms["constant"]),
        step_ms_constant_rounds=step_ms["constant"], step_ms_requires_grad_rounds=step_ms["requires_grad"],
        launches_per_step=launches)))


if __name__ == "__main__":
    main()
