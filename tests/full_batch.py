"""Full-batch gradient check at the benchmarked sizes: one training step of the CUDA model, every window carrying its true
target, against :class:`O.BF16ModeReference` with rounding off (fp64 torch autograd on the GPU, pinned to
``SparseOracle`` / ``ChainOracle`` in ``tests/test_oracle.py``).

Every window feeds the reductions the kernels split across tiles and CTAs (the LSTM's per-CTA weight-gradient slices,
the projection's ``dW`` / ``dbias`` / pool atomics, the fusion and gate ``fc`` sums, ``d_s``), so a lost or doubled
contribution, or rounding that builds up along a long sum, shows in the gradients.  The reference runs a chunk of windows
at a time (``window_chunk``): windows are independent (``STMGCN.py:47``), so its full-batch gradient is the sum of the
chunks' gradients, and only one chunk's fp64 tape is alive at once.

ReLU models: the reference takes the ReLU masks of the GPU's own forward (recorded through ``ops._proj_fwd``), so a
pre-activation within rounding distance of the kink follows the same branch in both.

Diagnostic (printed, not asserted): the same reference in fp32 (no TF32), i.e. what fp32 arithmetic of this model gets
at this size, next to the kernels' error of every gradient.

The bf16-arithmetic mode is checked by :func:`run_forced`: the reference rounds where the kernels round and is forced
with the step's own values at every rounding point, recorded for every row of the batch.
"""
import time

import numpy as np
import torch
from torch import nn

import stmgcn_oracle as O
from helpers import DEV, rel_err
from lstm_cases import step_local_error
from model_cases import FullBatchRecorder
from per_step import per_step_rel_err, worst_step


def _errors(got, ref, want_obs):
    """Output (worst window, each held to its own maximum), loss, every parameter gradient and, with ``want_obs``,
    d obs (worst window and worst time step)."""
    errs = {"out": float(np.max(per_step_rel_err(got["out"], ref["out"], 0))),
            "loss": abs(got["loss"] - ref["loss"]) / abs(ref["loss"])}
    for key, g in got["grads"].items():
        if key != "obs":
            errs["grad " + key] = rel_err(g, ref["grads"][key])
    if want_obs:
        errs["d obs"] = rel_err(got["d_obs"], ref["grads"]["obs"])
        errs["d obs (worst window)"] = float(np.max(per_step_rel_err(got["d_obs"], ref["grads"]["obs"], 0)))
        errs["d obs (worst step)"] = worst_step(got["d_obs"], ref["grads"]["obs"], 1)[0]
    return errs


def gpu_step(model, sups, x, y, want_obs=False, keep_masks=True):
    """One forward and backward of ``model`` on the whole batch with the true targets.  Returns the output, the loss,
    every parameter gradient (copies; the model's own are released), d obs with ``want_obs`` and, with ``keep_masks``,
    the ReLU mask of every GCN as a bool tensor (N, B, q) (order temporal 0, spatial 0, temporal 1, ...)."""
    from stmgcn_b200 import ops
    masks = []
    real_proj_fwd = ops._proj_fwd

    def recording_proj_fwd(*a, **k):
        out_ = real_proj_fwd(*a, **k)
        masks.append(out_ > 0)
        return out_
    xd = x.to(DEV).requires_grad_(want_obs)
    model.zero_grad(set_to_none=True)
    ops._proj_fwd = recording_proj_fwd
    try:
        out = model(obs_seq=xd, sta_adj_list=sups)
    finally:
        ops._proj_fwd = real_proj_fwd
    assert len(masks) == 2 * len(sups)
    loss = nn.MSELoss()(out, y.to(DEV))
    loss.backward()
    torch.cuda.synchronize()
    res = dict(out=out.detach(), loss=loss.item(), d_obs=xd.grad if want_obs else None,
               grads={k: p.grad.detach().clone() for k, p in model.named_parameters()},
               masks=masks if keep_masks else None)
    model.zero_grad(set_to_none=True)
    return res


def reference(params, chains, ks, x, y, relu, masks, window_chunk, want_obs, dtype=torch.float64):
    """:class:`O.BF16ModeReference` without rounding, in ``dtype`` on the GPU, ``window_chunk`` windows at a time."""
    ref = O.BF16ModeReference(params, chains, ks, relu=relu, rounding=False, relu_masks=masks, device=DEV, dtype=dtype)
    out, loss, grads = ref.loss_and_grads(x, y, want_obs=want_obs, window_chunk=window_chunk)
    del ref
    return dict(out=out, loss=float(loss), grads=grads)


def run(label, model, sups, params, chains, ks, x, y, *, relu, window_chunk, want_obs=False, repeat=False,
        fp32_diagnostic=True):
    """The GPU step on the full batch against the fp64 reference; prints and returns every error (see
    :func:`_errors`).

    ``repeat``: a second step at the same weights, checked against the reference at its own ReLU masks; the errors
    returned are the larger of the two steps'.  Printed beside them: per gradient, how far the second step moves from
    the first (max-norm relative; the order of the kernels' atomic sums), and how many ReLU mask entries differ."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    steps = [gpu_step(model, sups, x, y, want_obs, keep_masks=relu) for _ in range(2 if repeat else 1)]
    torch.cuda.empty_cache()
    t1 = time.perf_counter()
    lines = [f"{label}: B={x.shape[0]} relu={relu}, every window against the fp64 reference in chunks of {window_chunk}"]
    step_errs, f32 = [], None
    for i, got in enumerate(steps):
        ref = reference(params, chains, ks, x, y, relu, got["masks"], window_chunk, want_obs)
        step_errs.append(_errors(got, ref, want_obs))
        if i == 0 and fp32_diagnostic:
            assert not torch.backends.cuda.matmul.allow_tf32, "the fp32 diagnostic needs fp32 GEMMs, not TF32"
            ref32 = reference(params, chains, ks, x, y, relu, got["masks"], window_chunk, want_obs, torch.float32)
            f32 = _errors(dict(ref32, d_obs=ref32["grads"].get("obs")), ref, want_obs)
            del ref32
        del ref
        torch.cuda.empty_cache()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    spread = None
    if repeat:
        first, second = steps
        spread = {"grad " + k: rel_err(second["grads"][k], g) for k, g in first["grads"].items()}
        spread["out"] = rel_err(second["out"], first["out"])
        if relu:
            flips = [int((a != b).sum()) for a, b in zip(first["masks"], second["masks"])]
            lines.append(f"  ReLU mask entries that differ between the two steps, per GCN (temporal 0, spatial 0, "
                         f"temporal 1, ...): {flips}")
    head = f"  {'':<44} {'kernels':>9} {'fp32 ref':>9}"
    lines.append(head + (f" {'2nd step':>9} {'2-step spread':>13}" if repeat else ""))
    for k, v in sorted(step_errs[0].items(), key=lambda kv: -kv[1]):
        row = f"  {k:<44} {v:9.2e} " + (f"{f32[k]:9.2e}" if f32 else f"{'-':>9}")
        if repeat:
            row += f" {step_errs[1][k]:9.2e} " + (f"{spread[k]:13.2e}" if k in spread else f"{'-':>13}")
        lines.append(row)
    lines.append(f"  peak memory {peak:.1f} GiB; wall time: GPU step{'s' if repeat else ''} {t1 - t0:.1f} s, fp64 "
                 f"reference{'s' if repeat else ''}{' and fp32 diagnostic' if fp32_diagnostic else ''} {t2 - t1:.1f} s")
    print("\n".join(lines))
    for got in steps:
        assert bool(torch.isfinite(got["out"]).all())
    return {k: max(e[k] for e in step_errs) for k in step_errs[0]}


def _windows_rolled(tape, n, shift):
    """``tape`` with window b holding the recording of window (b + shift) mod B (rows ``n*B + b``)."""
    def roll(v, axis):
        shape = v.shape
        v = v.reshape(shape[:axis] + (n, shape[axis] // n) + shape[axis + 1:])
        return torch.roll(v, -shift, axis + 1).reshape(shape)
    return {k: torch.roll(v, -shift, 2) if k == "s" else roll(v, 1 if k == "h0" else 2) for k, v in tape.items()}


def run_forced(label, model, sups, params, chains, ks, x, y, *, relu, window_chunk, want_obs=False, window_offset=0):
    """The bf16-arithmetic mode on the full batch: one GPU step, every window with its true target, recorded for every
    row (:class:`FullBatchRecorder`), against :class:`O.BF16ModeReference` forced with that recording and the step's
    ReLU masks, ``window_chunk`` windows at a time.  The recording stays in the kernels' precision; each chunk's slice is
    widened to fp64 only when the reference reaches it.

    Returns (step-local errors: every LSTM layer-step and h_top of each graph, every spatial S_k, each the worst over
    the chunks; whole-model errors as :func:`_errors`; the worst whole-model error of the same step against the
    unrounded reference, which says the single-plane arithmetic ran).  Prints them with the peak memory and wall time.

    ``window_offset`` (negative controls only): the reference for window b is forced with window b + offset's
    recording."""
    n = x.shape[2]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    with FullBatchRecorder() as rec:
        got = gpu_step(model, sups, x, y, want_obs, keep_masks=relu)
    rec.check_intact()
    assert len(rec.lstm) == len(rec.stacks) == len(chains), "a graph branch ran without the bf16 mode's LSTM or stack"
    tapes = rec.take_tapes()
    if window_offset:
        tapes = [_windows_rolled(t, n, window_offset) for t in tapes]
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    ref = O.BF16ModeReference(params, chains, ks, relu=relu, relu_masks=got["masks"] if relu else None, device=DEV)
    step = {}

    def worst(key, v):
        step[key] = float(np.maximum(step.get(key, 0.0), v))          # NaN stays NaN

    def on_branch(m, br):
        tape = O._tape_windows(tapes[m], n, br["windows"], torch.float64)
        worst(f"g{m} LSTM layer-steps", step_local_error(tape, br["hs"], br["cs"], 1))
        worst(f"g{m} h_top", rel_err(tape["s"][0].reshape(n, -1), br["hs"][-1][-1].reshape(n, -1)))
        for k in range(1, ks):
            worst(f"g{m} S_{k}", rel_err(tape["s"][k].reshape(n, -1), br["stack"][k]))
    out, loss, grads = ref.loss_and_grads(x, y, tapes=tapes, want_obs=want_obs, on_branch=on_branch,
                                          window_chunk=window_chunk)
    errs = _errors(got, dict(out=out, loss=float(loss), grads=grads), want_obs)
    del ref, tapes, out, grads
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    unrounded = max(_errors(got, reference(params, chains, ks, x, y, relu, got["masks"], window_chunk, want_obs),
                            want_obs).values())
    torch.cuda.synchronize()
    t3 = time.perf_counter()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    lines = [f"{label}: B={x.shape[0]} relu={relu}, every window against the forced fp64 reference in chunks of "
             f"{window_chunk}" + (f", tapes {window_offset} window(s) off" if window_offset else ""),
             f"  step-local worst {max(step.values()):.2e}; whole model worst {max(errs.values()):.2e}; against the "
             f"unrounded reference {unrounded:.2e}"]
    for k, v in sorted({**step, **errs}.items(), key=lambda kv: -kv[1])[:8]:
        lines.append(f"  {k:<44} {v:9.2e}")
    lines.append(f"  peak memory {peak:.1f} GiB; wall time: GPU step and recording {t1 - t0:.1f} s, forced fp64 "
                 f"reference {t2 - t1:.1f} s, unrounded reference {t3 - t2:.1f} s")
    print("\n".join(lines))
    assert bool(torch.isfinite(got["out"]).all())
    return step, errs, unrounded


def assert_within(errs, tol, what=""):
    """Every error at ``tol``."""
    bad = {k: v for k, v in errs.items() if not v <= tol}
    assert not bad, f"{what}: above {tol:.0e}: {bad}"
