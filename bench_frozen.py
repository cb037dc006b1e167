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
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.abspath(__file__))
for _p in (REPO, os.path.join(REPO, "st-mgcn_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

VARIANTS = ("all_trainable", "frozen_obs", "lstm_frozen")


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


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
    from stmgcn_b200 import _lib, ops, synth

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

    def rel(a, b):
        return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))

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
        errs = {k: rel(g, base[k]) for k, g in got.items()}
        check[variant] = max(errs.values())
        assert check[variant] <= 1e-4, f"{variant}: {max(errs, key=errs.get)} is {check[variant]:.2e} off"
    del model, params, base, base_x
    model = make()                                  # the timed model: the workload's own activation

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(args.steps):
            fn()
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) / args.steps, (_lib.launch_count() - n0) // args.steps

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
    check["lstm_bwd_d_s"] = rel(part[0], full[0])
    assert check["lstm_bwd_d_s"] <= 1e-4 and all(g is None for g in part[1])

    runs = {v: [] for v in VARIANTS}
    launches = {}
    lstm_runs = {True: [], False: []}
    lstm_launches = {}
    for _ in range(args.rounds):
        for v in VARIANTS:
            ms, launches[v] = timed(lambda: step(model, v))
            runs[v].append(ms)
        for wgrad in (True, False):
            ms, lstm_launches[wgrad] = timed(lambda: lstm_bwd(wgrad))
            lstm_runs[wgrad].append(ms)
    print(json.dumps({
        "workload": w.name, "device": torch.cuda.get_device_name(dev), "power_limit": _power_limit(),
        "lstm_path": ops.lstm_path(), "planes": ops.lstm_planes() if on_tc else None, "steps": args.steps,
        "ms_per_step": {v: [round(r, 3) for r in runs[v]] for v in VARIANTS},
        "gpu_launches": launches,
        "lstm_bwd_ms": {"with_wgrad": [round(r, 3) for r in lstm_runs[True]],
                        "without_wgrad": [round(r, 3) for r in lstm_runs[False]]},
        "lstm_bwd_launches": {"with_wgrad": lstm_launches[True], "without_wgrad": lstm_launches[False]},
        "lstm_bwd_includes_forward": not on_tc,
        "max_rel_err_vs_all_trainable": {k: float(f"{v:.3e}") for k, v in check.items()}}))


if __name__ == "__main__":
    main()
