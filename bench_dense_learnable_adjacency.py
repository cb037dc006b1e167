"""Learning dense graphs: a LearnableAdjacency whose matrices are multiplied and differentiated dense (K1f) against the
other ways to learn the same graphs.

    python bench_dense_learnable_adjacency.py [--steps 3] [--rounds 3] [--reps 10] [--skip-steps]

* kernels, at N = 4096 on a dense similarity graph's own chain (K = 3): the chain gradient stmgcn_dense_chain_grad at
  cfg3's spatial (F = 64 * 64) and temporal (F = 64 * 12) widths, its error against fp64 and the error of the
  alternative it replaces (K1d's truncating split, accumulated in the tensor cores, one slice at a time, summed), and
  achieved TFLOP/s from shapes (2 N^2 F per term); the pattern scatter and gather of one N x N matrix;
* the cfg3 training step (4096 regions, 3 graphs, K = 3, T = 12, B = 64; forward and backward, no optimizer step) on
  three dense similarity adjacencies (``synth.make_similarity_adjacency``), alternated round by round:
  (a) fixed ``process()`` stacks; (b) ``process(adj)`` with ``adj.requires_grad`` (learning the dense stacks);
  (c) ``process_learnable(adj)`` under ``STMGCN_DENSE_SUPPORTS=off`` (the CSR gather and the SDDMM);
  (d) ``process_learnable(adj)`` under ``auto`` (dense); (e) (d) captured in a ``GraphedStep``.

Before any time is printed, each chain-gradient run is checked against fp64 at 5e-5 and each step variant's loss on two
windows against the fp64 dense restatement at 1e-4 (every learnable graph starts at its adjacency, so all variants
compute the same loss).  Prints one JSON line, with the card's name and power limit.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json

from benchlib import alternate, device_record, require_cuda, setup_paths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--skip-steps", action="store_true", help="time the kernels only")
    args = ap.parse_args()
    require_cuda("bench_dense_learnable_adjacency.py")
    setup_paths()

    import torch
    from torch import nn
    import GCN
    import STMGCN
    import stmgcn_oracle as O
    from stmgcn_b200 import ops, synth
    from stmgcn_b200.graphs import GraphedStep

    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    w = synth.WORKLOADS["cfg3"]
    n, k_ord = w.n_regions, w.cheb_order
    ops.set_lstm_planes(2)
    pre = GCN.Adj_Preprocessor("chebyshev", k_ord)

    # ---- kernels on a similarity graph's own chain --------------------------------------------------------------------
    ops.set_dense_supports("on")
    adj0 = pre.process_learnable(synth.make_similarity_adjacency(n, 0).to(dev)).to(dev)
    with torch.no_grad():
        sset = adj0()
        lt = sset.values[0].detach()
    kernels = []
    for f_total in (w.batch * w.gcn_hidden, w.batch * w.seq_len):
        gen = torch.Generator(device=dev).manual_seed(f_total)
        lt64 = lt.double()
        t = [torch.randn((n, f_total), device=dev, generator=gen, dtype=torch.float64)]
        t.append(lt64 @ t[0])
        for _ in range(2, k_ord + 1):
            t.append(2 * (lt64 @ t[-1]) - t[-2])
        g = [None] * (k_ord + 1)
        for k in range(k_ord, 0, -1):
            u = torch.randn((n, f_total), device=dev, generator=gen, dtype=torch.float64)
            g[k] = u + (2 * (lt64.T @ g[k + 1]) if k < k_ord else 0) - (g[k + 2] if k + 2 <= k_ord else 0)
        del lt64
        t = [x.float().contiguous() for x in t]
        g = [None] + [x.float().contiguous() for x in g[1:]]
        terms = [(g[k], t[k - 1], 1.0 if k == 1 else 2.0) for k in range(1, k_ord + 1)]
        ref = sum(c * (a.double() @ b.double().T) for a, b, c in terms)
        den = float(ref.abs().max())
        got = ops.dense_chain_grad(terms)
        err = float((got.double() - ref).abs().max()) / den
        if err > 5e-5:
            raise SystemExit(f"bench_dense_learnable_adjacency: chain gradient parity failed (F={f_total}): {err:.3e}")
        # the alternative: K1d (truncating split, tensor-core accumulation) slice by slice, summed in fp32
        k1d = sum(c * ops.dense_support_grad(a.unsqueeze(0), b)[0] for a, b, c in terms)
        err_k1d = float((k1d.double() - ref).abs().max()) / den
        del ref, k1d
        ms, _ = alternate({"chain": lambda: ops.dense_chain_grad(terms)}, args.rounds, args.reps, 2)
        t_ms = min(ms["chain"])
        kernels.append(dict(n=n, f_total=f_total, terms=k_ord, chain_grad_ms=t_ms,
                            chain_grad_tflops=2.0 * n * n * f_total * k_ord / t_ms * 1e-9, rel_err=err,
                            k1d_summed_rel_err=err_k1d))
        del t, g, terms, got
        torch.cuda.empty_cache()
    vals = ops.AdjNorm.apply(adj0.weight.detach(), adj0.kind, adj0.scale, *adj0.pattern())
    dense = ops.PatternToDense.apply(vals, adj0.rowptr, adj0.colidx)
    ms, _ = alternate({"scatter": lambda: ops.pattern_scatter(vals, adj0.rowptr, adj0.colidx),
                       "gather": lambda: ops.pattern_gather(dense, adj0.rowptr, adj0.colidx)}, args.rounds, args.reps, 2)
    card, power = device_record()
    result = dict(bench="dense_learnable_adjacency", card=card, power_limit=power, n=n, kernels=kernels,
                  scatter_ms=min(ms["scatter"]), gather_ms=min(ms["gather"]), pattern_entries=int(adj0.colidx.numel()))
    del sset, lt, vals, dense, adj0
    torch.cuda.empty_cache()
    if args.skip_steps:
        print(json.dumps(result))
        return

    # ---- the cfg3 training step ---------------------------------------------------------------------------------------
    adjs = [synth.make_similarity_adjacency(n, m).to(dev) for m in range(w.n_graphs)]
    const = [pre.process(a) for a in adjs]
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(**synth.model_kwargs(w)).to(dev)
    crit = nn.MSELoss()
    x, y = (t.to(dev) for t in synth.make_inputs(w, seed=0))
    with torch.no_grad():
        params = {k: v.detach().double() for k, v in model.named_parameters()}
        out64 = O.dense_st_mgcn(params, x[:2].double(), [pre.process(a.double()) for a in adjs])
        loss64 = float(torch.mean((out64 - y[:2].double()) ** 2))
        del out64

    learn_b = [a.clone().requires_grad_(True) for a in adjs]
    learn_c = [pre.process_learnable(a).to(dev) for a in adjs]
    learn_d = [pre.process_learnable(a).to(dev) for a in adjs]
    variants = {
        "a_fixed": ("auto", lambda: const),
        "b_process_requires_grad": ("auto", lambda: [pre.process(a) for a in learn_b]),
        "c_learnable_off": ("off", lambda: learn_c),
        "d_learnable_auto": ("auto", lambda: learn_d),
    }

    def check(name, mode, sups_fn):
        ops.set_dense_supports(mode)
        with torch.no_grad():
            loss = float(crit(model(obs_seq=x[:2], sta_adj_list=sups_fn()), y[:2]))
        if abs(loss - loss64) > 1e-4 * abs(loss64):
            raise SystemExit(f"bench_dense_learnable_adjacency: {name} loss {loss:.8f} is off fp64 {loss64:.8f}")

    def step(mode, sups_fn, leaves):
        ops.set_dense_supports(mode)
        model.zero_grad(set_to_none=False)
        for p in leaves:
            p.grad = None
        loss = crit(model(obs_seq=x, sta_adj_list=sups_fn()), y)
        loss.backward()
        return loss

    leaves = {"a_fixed": [], "b_process_requires_grad": learn_b, "c_learnable_off": [a.weight for a in learn_c],
              "d_learnable_auto": [a.weight for a in learn_d]}
    for name, (mode, fn) in variants.items():
        check(name, mode, fn)
    ops.set_dense_supports("auto")
    small = GraphedStep(model, crit, x[:2], y[:2], learn_d)
    loss = float(small(x[:2], y[:2]))
    if abs(loss - loss64) > 1e-4 * abs(loss64):
        raise SystemExit(f"bench_dense_learnable_adjacency: e_learnable_auto_graphed loss {loss:.8f} is off fp64 {loss64:.8f}")
    del small
    graphed = GraphedStep(model, crit, x, y, learn_d)
    fns = {name: (lambda name=name: step(variants[name][0], variants[name][1], leaves[name])) for name in variants}
    fns["e_learnable_auto_graphed"] = lambda: (ops.set_dense_supports("auto"), graphed(x, y))
    ms, launches = alternate(fns, args.rounds, args.steps, 1)
    ops.set_dense_supports("auto")
    result.update(step_ms={k: min(v) for k, v in ms.items()}, rounds=ms, launches_per_step=launches,
                  loss64_two_windows=loss64)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
