"""Cost of learnable edge weights at cfg3 (4096 regions, 3 graphs, K = 3, seq_len 12, batch 64, fp32-grade mode).

    python bench_support_grad.py [--steps 10] [--rounds 4] [--reps 50]

* step: the training step (forward + MSE + backward) with three learnable Chebyshev handles, rebuilt from their edge
  weights by ``Adj_Preprocessor.process_sparse`` every step, against the same step on fixed handles built once.  The two
  alternate in rounds, each timed with CUDA events;
* kernels: the SDDMM launches of one graph convolution's value gradient (``ops.csr_sddmm_``, K terms) against the K
  forward SpMM launches of the same convolution (``ops.spmm_step``), same gather volume, timed in the same run -- for the
  spatial GCN (F = B*64) and the temporal one (F = B*T).

Before any time is printed, the loss and the gradients of the handles' values on two windows are checked against a
dense fp64 restatement (``oracle/stmgcn_oracle.py``) that takes the step's own ReLU masks, at 1e-4.  Prints one JSON line, with the card's name and power limit.
Writes nothing.
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
    require_cuda("bench_support_grad.py")
    setup_paths()

    import torch
    from torch import nn
    import GCN
    import STMGCN
    import stmgcn_oracle as O
    from stmgcn_b200 import ops, synth

    dev = torch.device("cuda:0")
    w = synth.WORKLOADS["cfg3"]
    ops.set_lstm_planes(2)
    pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
    adjs = [a.to(dev).to_sparse_coo().coalesce() for a in synth.make_adjacency_list(w)]
    idx = [a.indices() for a in adjs]
    weights = [nn.Parameter(a.values().clone()) for a in adjs]
    fixed = [pre.process_sparse(a) for a in adjs]
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(**synth.model_kwargs(w)).to(dev)
    crit = nn.MSELoss()
    x, y = (t.to(dev) for t in synth.make_inputs(w, seed=0))

    def learnable():
        return [pre.process_sparse(torch.sparse_coo_tensor(i, v, a.shape)) for i, v, a in zip(idx, weights, adjs)]

    def step(sups):
        model.zero_grad(set_to_none=False)
        for v in weights:
            v.grad = None
        loss = crit(model(obs_seq=x, sta_adj_list=sups() if callable(sups) else sups), y)
        loss.backward()
        return loss

    # ---- correctness first: two windows against dense fp64 ------------------------------------------------------------
    # the gradient at the handles' values (the rescaled Laplacians' stored entries), against a dense fp64 restatement
    # whose Laplacians are built from the same values as leaves
    x2, y2 = x[:2], y[:2]
    model.zero_grad()
    hs = learnable()
    for h in hs:
        h.vals.retain_grad()
    masks = []                          # the step's own ReLU masks (out > 0) of every GCN, in launch order
    real_proj_fwd = ops._proj_fwd

    def recording_proj_fwd(*a, **k):
        out_ = real_proj_fwd(*a, **k)
        masks.append(out_ > 0)
        return out_
    ops._proj_fwd = recording_proj_fwd
    try:
        loss2 = crit(model(obs_seq=x2, sta_adj_list=hs), y2)
    finally:
        ops._proj_fwd = real_proj_fwd
    loss2.backward()
    n = w.n_regions
    params = {k: p.detach().double() for k, p in model.state_dict().items()}
    leaves, stacks = [], []
    for h in hs:
        leaf = h.vals.detach().double().clone().requires_grad_(True)
        rows = torch.repeat_interleave(torch.arange(n, device=dev), (h.rowptr[1:] - h.rowptr[:-1]).long())
        lap = torch.zeros(n, n, dtype=torch.float64, device=dev).index_put((rows, h.colidx.long()), leaf, accumulate=True)
        leaves.append(leaf)
        stacks.append(O.chain_stack_dense([lap], h.ks - 1))
    # the reference takes the step's ReLU masks: a pre-activation within rounding distance of the kink takes the same
    # branch in both (one flipped entry moves a d vals entry, a sum over one row's B*64 features, by about 1/64)
    out64 = O.dense_st_mgcn(params, x2.double(), stacks, masks=masks)
    loss64 = ((out64 - y2.double()) ** 2).mean()
    loss64.backward()
    err_loss = abs(loss2.item() - loss64.item()) / abs(loss64.item())
    err_grad = max(O.max_rel_err(h.vals.grad.cpu().numpy(), leaf.grad.cpu().numpy()) for h, leaf in zip(hs, leaves))
    del stacks, out64, loss64, leaves, hs, masks
    torch.cuda.empty_cache()
    if not (err_loss <= 1e-4 and err_grad <= 1e-4):
        raise SystemExit(f"bench_support_grad: parity failed: loss {err_loss:.3e}, d vals {err_grad:.3e}")

    # ---- the step, alternating learnable and fixed handles ------------------------------------------------------------
    step_ms, _ = alternate({"learnable": lambda: step(learnable), "fixed": lambda: step(fixed)},
                           args.rounds, args.steps, 3)
    ms_learn, ms_fixed = step_ms["learnable"], step_ms["fixed"]

    # ---- the SDDMM launches of one GCN against its K forward SpMM launches ------------------------------------------
    g = fixed[0].support_set().graphs[0]
    k = w.cheb_order
    kernels = {}
    for name, f_total in (("spatial", w.batch * w.gcn_hidden), ("temporal", w.batch * w.seq_len)):
        gen = torch.Generator(device=dev).manual_seed(1)
        s = torch.randn((k + 1, n, f_total), device=dev, generator=gen)
        u = torch.randn((k + 1, n, f_total), device=dev, generator=gen)
        dv = torch.zeros(g.nnz, device=dev)
        terms = [(u[j], s[j - 1], 1.0 if j == 1 else 2.0) for j in range(1, k + 1)]

        def sddmm():
            ops.csr_sddmm_(g, terms, dv)

        def spmm():
            ops.spmm_step(g, False, 1.0, s[0], 0.0, None, 0.0, None, s[1])
            for j in range(2, k + 1):
                ops.spmm_step(g, False, 2.0, s[j - 1], -1.0, s[j - 2], 0.0, None, s[j])

        kernel_ms, _ = alternate({"sddmm": sddmm, "spmm": spmm}, args.rounds, args.reps, 5)
        t_sd, t_sp = min(kernel_ms["sddmm"]) * 1e3, min(kernel_ms["spmm"]) * 1e3
        kernels[name] = dict(f_total=f_total, sddmm_us=t_sd, spmm_forward_us=t_sp, ratio=t_sd / t_sp)

    name, power = device_record()
    print(json.dumps(dict(
        bench="support_grad", workload="cfg3", card=name, power_limit=power, learnable_graphs=len(weights),
        nnz_per_graph=[int(i.shape[1]) for i in idx],
        step_ms_learnable=min(ms_learn), step_ms_fixed=min(ms_fixed), step_added_ms=min(ms_learn) - min(ms_fixed),
        step_ms_learnable_rounds=ms_learn, step_ms_fixed_rounds=ms_fixed, kernels=kernels,
        parity=dict(windows=2, loss_rel_err=err_loss, d_vals_rel_err=err_grad))))


if __name__ == "__main__":
    main()
