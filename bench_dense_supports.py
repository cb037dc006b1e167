"""Dense support matrices multiplied dense on the tensor cores (stmgcn_dense_mm_step, K1e) against the CSR gather (K1).

    python bench_dense_supports.py [--steps 3] [--rounds 3] [--reps 10] [--skip-steps]

* kernels: one step ``Y = 2 op(A) X - Z`` at N = 4096 and F = 768 / 4096 (cfg3's temporal / spatial widths), op(A) = A
  and A^T, for random matrices of density 0.5 .. 100 %: the dense step, the CSR step of the same matrix and
  ``torch.matmul`` in fp32 with TF32 off, alternated round by round; achieved TFLOP/s of the dense step (2 N^2 F).  These
  set ``graph.dense_rule``'s density (from which the dense step wins);
* smaller graphs: the dense and the CSR step at N = 128 .. 2048, at the rule's density and fully dense, which set its
  size bound;
* dense graphs: the cfg3 training step (4096 regions, 3 graphs, K = 3, T = 12, B = 64) on ``process()`` of three dense
  similarity adjacencies (``synth.make_similarity_adjacency``), under ``STMGCN_DENSE_SUPPORTS`` off and auto;
* learned dense stacks: the same step with the adjacencies requiring grad (``process(adj)`` at every step) and an Adam
  step between the timed steps, so the stacks are dense as in training, under off and auto.

Before any time is printed, every dense kernel step is checked against an fp64 product at 5e-5, and every step variant's
loss on two windows against the fp64 dense restatement at 1e-4.  Prints one JSON line, with the card's name and power
limit.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json

from benchlib import alternate, device_record, require_cuda, setup_paths

DENSITIES = (0.005, 0.01, 0.02, 0.04, 0.08, 0.25, 1.0)
SMALL_N = (128, 256, 512, 1024, 2048)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--skip-steps", action="store_true", help="time the kernels only")
    args = ap.parse_args()
    require_cuda("bench_dense_supports.py")
    setup_paths()

    import torch
    from torch import nn
    import GCN
    import STMGCN
    import stmgcn_oracle as O
    from stmgcn_b200 import graph, ops, synth

    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    w = synth.WORKLOADS["cfg3"]
    n = w.n_regions
    ops.set_lstm_planes(2)

    # ---- the kernel against the CSR step and torch.matmul, correctness first ---------------------------------------------
    kernels = []
    for f_total in (w.batch * w.seq_len, w.batch * w.gcn_hidden):
        gen = torch.Generator(device=dev).manual_seed(f_total)
        x = torch.randn((n, f_total), device=dev, generator=gen)
        z = torch.randn((n, f_total), device=dev, generator=gen)
        y = torch.empty_like(x)
        for dens in DENSITIES:
            a = torch.rand((n, n), device=dev, generator=gen)
            a = torch.where(a < dens, torch.randn((n, n), device=dev, generator=gen), torch.zeros_like(a))
            nnz = int((a != 0).sum())
            dg, cg = graph.DenseGraph(a), graph.GraphHandle.from_dense(a)
            for tr in (False, True):
                ops.spmm_step(dg, tr, 2.0, x, -1.0, z, 0.0, None, y)
                ref = 2.0 * ((a.t() if tr else a).double() @ x.double()) - z.double()
                err = float((y.double() - ref).abs().max() / ref.abs().max())
                if err > 5e-5:
                    raise SystemExit(f"bench_dense_supports: dense step parity failed (F={f_total}, density {dens}, "
                                     f"transpose {tr}): {err:.3e}")
                del ref
                at = (a.t() if tr else a).contiguous()
                ms, _ = alternate({
                    "dense": lambda: ops.spmm_step(dg, tr, 2.0, x, -1.0, z, 0.0, None, y),
                    "csr": lambda: ops.spmm_step(cg, tr, 2.0, x, -1.0, z, 0.0, None, y),
                    "torch_fp32": lambda: torch.matmul(at, x, out=y),
                }, args.rounds, args.reps, 2)
                t = {k: min(v) for k, v in ms.items()}
                kernels.append(dict(f_total=f_total, density=dens, nnz=nnz, transpose=tr, dense_ms=t["dense"],
                                    csr_ms=t["csr"], torch_fp32_ms=t["torch_fp32"],
                                    dense_tflops=2.0 * n * n * f_total / t["dense"] * 1e-9,
                                    torch_fp32_tflops=2.0 * n * n * f_total / t["torch_fp32"] * 1e-9,
                                    csr_over_dense=t["csr"] / t["dense"], parity_rel_err=err))
                del at
            del a, dg, cg
            torch.cuda.empty_cache()
        del x, z, y
    # ---- smaller graphs: where the rule's size bound lies ------------------------------------------------------------------
    small = []
    for n_s in SMALL_N:
        for f_total in (w.batch * w.seq_len, w.batch * w.gcn_hidden):
            gen = torch.Generator(device=dev).manual_seed(n_s + f_total)
            x = torch.randn((n_s, f_total), device=dev, generator=gen)
            z = torch.randn((n_s, f_total), device=dev, generator=gen)
            y = torch.empty_like(x)
            for dens in (graph.DENSE_MIN_DENSITY, 1.0):
                a = torch.rand((n_s, n_s), device=dev, generator=gen)
                a = torch.where(a < dens, torch.randn((n_s, n_s), device=dev, generator=gen), torch.zeros_like(a))
                dg, cg = graph.DenseGraph(a), graph.GraphHandle.from_dense(a)
                ops.spmm_step(dg, False, 2.0, x, -1.0, z, 0.0, None, y)
                ref = 2.0 * (a.double() @ x.double()) - z.double()
                err = float((y.double() - ref).abs().max() / ref.abs().max())
                if err > 5e-5:
                    raise SystemExit(f"bench_dense_supports: dense step parity failed (N={n_s}, F={f_total}): {err:.3e}")
                ms, _ = alternate({"dense": lambda: ops.spmm_step(dg, False, 2.0, x, -1.0, z, 0.0, None, y),
                                   "csr": lambda: ops.spmm_step(cg, False, 2.0, x, -1.0, z, 0.0, None, y)},
                                  args.rounds, args.reps, 2)
                small.append(dict(n=n_s, f_total=f_total, density=dens, dense_ms=min(ms["dense"]), csr_ms=min(ms["csr"]),
                                  csr_over_dense=min(ms["csr"]) / min(ms["dense"]), parity_rel_err=err))
    card, power = device_record()
    result = dict(bench="dense_supports", card=card, power_limit=power, n=n, kernels=kernels, small_n=small,
                  rule=dict(min_density=graph.DENSE_MIN_DENSITY, min_n=graph.DENSE_MIN_N))
    if args.skip_steps:
        print(json.dumps(result))
        return

    # ---- the cfg3 step on three dense graphs, and learning three dense stacks ---------------------------------------------
    pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
    adjs = [synth.make_similarity_adjacency(n, m).to(dev) for m in range(w.n_graphs)]
    const = [pre.process(a) for a in adjs]
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(**synth.model_kwargs(w)).to(dev)
    crit = nn.MSELoss()
    x, y = (t.to(dev) for t in synth.make_inputs(w, seed=0))

    def check(mode, sups, what):
        """The loss of windows 0 and 1 against the fp64 dense restatement."""
        ops.set_dense_supports(mode)
        with torch.no_grad():
            loss = float(crit(model(obs_seq=x[:2], sta_adj_list=sups), y[:2]))
            params = {k: v.detach().double() for k, v in model.named_parameters()}
            out64 = O.dense_st_mgcn(params, x[:2].double(), [s.detach().double() for s in sups])
            loss64 = float(torch.mean((out64 - y[:2].double()) ** 2))
        if abs(loss - loss64) > 1e-4 * abs(loss64):
            raise SystemExit(f"bench_dense_supports: {what} loss {loss:.8f} is off fp64 {loss64:.8f}")

    def step(mode, sups):
        ops.set_dense_supports(mode)
        model.zero_grad(set_to_none=False)
        loss = crit(model(obs_seq=x, sta_adj_list=sups), y)
        loss.backward()
        return loss

    for mode in ("off", "auto"):
        check(mode, const, f"dense graphs ({mode})")
    dense_ms, dense_launches = alternate({"off": lambda: step("off", const), "auto": lambda: step("auto", const)},
                                         args.rounds, args.steps, 2)
    del const
    torch.cuda.empty_cache()

    # learned stacks: each variant its own adjacencies, filled in by Adam steps before and between the timed steps
    learn = {mode: [a.clone().requires_grad_(True) for a in adjs] for mode in ("off", "auto")}
    opts = {mode: torch.optim.Adam(learn[mode], lr=1e-3) for mode in learn}

    def learned_step(mode):
        opts[mode].zero_grad(set_to_none=False)
        loss = step(mode, [pre.process(a) for a in learn[mode]])
        opts[mode].step()
        return loss

    for mode in learn:
        learned_step(mode)
        with torch.no_grad():
            stacks = [pre.process(a) for a in learn[mode]]
        fill = min(float((s[1] != 0).float().mean()) for s in stacks)
        check(mode, stacks, f"learned stacks ({mode}, L~ {100 * fill:.1f} % non-zero)")
        del stacks
    learned_ms, learned_launches = alternate({m: (lambda m=m: learned_step(m)) for m in learn}, args.rounds, args.steps, 1)
    ops.set_dense_supports("auto")
    result.update(
        dense_graphs=dict(step_ms_off=min(dense_ms["off"]), step_ms_auto=min(dense_ms["auto"]),
                          speedup=min(dense_ms["off"]) / min(dense_ms["auto"]), rounds=dense_ms,
                          launches_per_step=dense_launches),
        learned_stacks=dict(step_ms_off=min(learned_ms["off"]), step_ms_auto=min(learned_ms["auto"]),
                            speedup=min(learned_ms["off"]) / min(learned_ms["auto"]), rounds=learned_ms,
                            launches_per_step=learned_launches))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
