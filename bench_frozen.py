"""Cost of the weight gradients nobody asked for: one cfg3 training step (forward, MSE, backward) in three variants,
alternated over rounds and timed with CUDA events on one GPU.  Prints one JSON line.

    python bench_frozen.py [--workload cfg3] [--steps 20] [--rounds 3]

  all_trainable : every parameter requires grad (the plain training step);
  frozen_obs    : every parameter frozen, obs_seq.requires_grad (input attribution);
  lstm_frozen   : the shared LSTM of every CG_LSTM frozen, everything else trainable (fine-tuning).

Also timed: the LSTM backward alone (one CG_LSTM's stack at the workload's shape, on the current path) with and
without its weight gradients.  Before any time is printed, the gradients each variant asks for are checked against the
all-trainable run's, on the same shapes without the GCN activation: with it, cfg3's obs gradient is vanishing
(max |d obs| ~ 4e-9) and a ReLU mask that flips between two forwards (the forward's pooling sums with atomics) moves it
by up to 6e-2 between two all-trainable runs, frozen or not (H100, measured).  The card's name and power limit are read
in the same run.  Nothing is written to the tree.
"""
from __future__ import annotations

import argparse
import json

from benchlib import alternate, device_record, require_cuda, setup_paths

VARIANTS = ("all_trainable", "frozen_obs", "lstm_frozen")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg3")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    require_cuda("bench_frozen.py")
    setup_paths()

    import torch
    from torch import nn
    import GCN
    import STMGCN
    import stmgcn_oracle as O
    from stmgcn_b200 import ops, synth

    w = synth.WORKLOADS[args.workload]
    dev = torch.device("cuda:0")
    pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
    sups = [pre.process_sparse(a).to(dev) for a in synth.make_adjacency_list(w)]
    x, y = (v.to(dev) for v in synth.make_inputs(w))
    crit = nn.MSELoss()

    def make(**kw):
        torch.manual_seed(0)
        return STMGCN.ST_MGCN(**dict(synth.model_kwargs(w), **kw)).to(dev)

    def frozen_of(model, variant):
        return {"all_trainable": set(), "frozen_obs": {k for k, _ in model.named_parameters()},
                "lstm_frozen": {k for k, _ in model.named_parameters() if ".lstm." in k}}[variant]

    def step(model, variant: str, obs_grad: bool = None):
        frozen = frozen_of(model, variant)
        for k, p in model.named_parameters():
            p.requires_grad_(k not in frozen)
            p.grad = None
        xs = x.detach().requires_grad_(variant == "frozen_obs" if obs_grad is None else obs_grad)
        crit(model(obs_seq=xs, sta_adj_list=sups), y).backward()
        return xs

    # ---- the requested gradients against the all-trainable run's (which also takes d obs) ----
    model = make(gconv_activation=None)
    params = dict(model.named_parameters())
    base_x = step(model, "all_trainable", obs_grad=True)
    base = {k: p.grad.clone() for k, p in params.items()}
    base["obs"] = base_x.grad.clone()
    check = {}
    for variant in VARIANTS[1:]:
        xs = step(model, variant)
        frozen = frozen_of(model, variant)
        got = {k: p.grad for k, p in params.items() if k not in frozen}
        if variant == "frozen_obs":
            got["obs"] = xs.grad
        assert all(params[k].grad is None for k in frozen), f"{variant}: a frozen parameter has a gradient"
        errs = {k: O.max_rel_err(g.cpu(), base[k].cpu()) for k, g in got.items()}
        check[variant] = max(errs.values())
        assert check[variant] <= 1e-4, f"{variant}: {max(errs, key=errs.get)} is {check[variant]:.2e} off"
    del model, params, base, base_x
    model = make()                                  # the timed model: the workload's own activation

    # ---- the LSTM backward alone: one CG_LSTM's stack, the tape of one forward, backward with / without wgrad ----
    cg = model.rnn_list[0]
    lyr, hid = cg.lstm_num_layers, cg.lstm_hidden_dim
    xo, xt = ops.obs_to_node_major(x)
    n, b, t, c = xo.shape
    s_gate = torch.rand(b, t, device=dev)
    ws = [wt.detach() for wt in cg._lstm_weights()]
    d_top = torch.randn(n, b, hid, device=dev)
    on_tc = hid == 64 and ops.lstm_path() == "tc" and c <= 4 and t <= 64
    if on_tc:
        _, _, _, tape = ops._lstm16_forward(xo, s_gate, None, None, lyr, False, ws, ops.lstm_planes(), True)
        lstm_bwd = lambda wgrad: ops._lstm16_backward_ex(xo, s_gate, tape, lyr, ops.lstm_planes(), d_top,  # noqa: E731
                                                         wgrad=wgrad)
    else:
        # the exact path overwrites its gate tape: a fresh forward per backward (timed with it, both variants alike)
        def lstm_bwd(wgrad):
            _, _, _, tape = ops._exact_forward(xo, s_gate, None, None, lyr, hid, False, ws, True)
            return ops._exact_backward_ex(xo, s_gate, tape, lyr, hid, d_top, wgrad=wgrad)
    full, part = lstm_bwd(True), lstm_bwd(False)
    check["lstm_bwd_d_s"] = O.max_rel_err(part[0].cpu(), full[0].cpu())
    assert check["lstm_bwd_d_s"] <= 1e-4 and all(g is None for g in part[1])

    lstm = {"with_wgrad": lambda: lstm_bwd(True), "without_wgrad": lambda: lstm_bwd(False)}
    runs, launches = alternate({**{v: lambda v=v: step(model, v) for v in VARIANTS}, **lstm},
                               args.rounds, args.steps, args.warmup)
    name, power_limit = device_record()
    print(json.dumps({
        "workload": w.name, "device": name, "power_limit": power_limit,
        "lstm_path": ops.lstm_path(), "planes": ops.lstm_planes() if on_tc else None, "steps": args.steps,
        "ms_per_step": {v: [round(r, 3) for r in runs[v]] for v in VARIANTS},
        "gpu_launches": {v: launches[v] for v in VARIANTS},
        "lstm_bwd_ms": {k: [round(r, 3) for r in runs[k]] for k in lstm},
        "lstm_bwd_launches": {k: launches[k] for k in lstm},
        "lstm_bwd_includes_forward": not on_tc,
        "max_rel_err_vs_all_trainable": {k: float(f"{v:.3e}") for k, v in check.items()}}))


if __name__ == "__main__":
    main()
