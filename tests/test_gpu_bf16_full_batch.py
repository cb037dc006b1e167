"""The bf16-arithmetic mode (``ops.set_lstm_planes(1)``: one bf16 hidden-state plane in the tensor-core LSTM, bf16
gather copies in the spatial Chebyshev recurrence) held to 1e-4 (``helpers.TOL``) on every window of the benchmarked
batches.

Each case is one training step of the whole batch with every window's true target, so every window feeds every
reduction the kernels split across tiles and CTAs (the LSTM's per-CTA weight-gradient slices, the projection's
``dW`` / ``dbias`` / pool atomics, ``d_s``, the fusion and gate ``fc`` sums).  The step is recorded for every row
(``model_cases.FullBatchRecorder``: the LSTM tapes and the spatial stacks the step keeps for its backward, by
reference and in the kernels' precision) and checked against ``stmgcn_oracle.BF16ModeReference`` forced with that
recording, a chunk of windows at a time (``full_batch.run_forced``).  ``tests/test_gpu_bf16_mode.py`` explains the
forcing and holds the small cases.

Each case also shows that the single-plane arithmetic ran: the recorded hidden-state tape has one plane, and the same
step is more than the bar away from the unrounded reference.
"""
import pytest
import torch

import full_batch
from helpers import TOL
from model_cases import CHUNK, bf16_mode, diffusion_case, forced_errors, gpu_run, workload_case  # noqa: F401

pytestmark = pytest.mark.gpu

PICKS = [0, 17, 31]                 # the cfg2 windows the picked-window check of the bf16 mode looks at

CASES = {
    "cfg2": lambda relu: (workload_case("cfg2", 32, relu), CHUNK["cfg2"]),
    "cfg2_diffusion": lambda relu: (diffusion_case(32, relu), CHUNK["cfg2"]),
    # bench.py's rank-0 inputs of cfg4: cfg3's shapes, batch 64, inputs of seed 100, supports from process_sparse
    "cfg4": lambda relu: (workload_case("cfg4", 64, relu), CHUNK["cfg4"]),
    # one window per chunk: beside the step's own tapes, kept for the forcing (11.5 GB), a chunk of two windows took
    # the peak to 25.3 GiB, one takes 18.4 GiB (H100)
    "cfg5": lambda relu: (workload_case("cfg5", 8, relu), 1),
}


def _run(case, relu, want_obs=False, **kw):
    (model, sups, chains, ks, params, x, y), chunk = CASES[case](relu)
    return full_batch.run_forced(f"bf16 mode {case}", model, sups, params, chains, ks, x, y, relu=relu,
                                 window_chunk=chunk, want_obs=want_obs, **kw)


def _bad(step, errs):
    return {k: v for k, v in {**step, **errs}.items() if not v <= TOL}


@pytest.mark.parametrize("relu", [True, False], ids=["relu", "smooth"])
@pytest.mark.parametrize("case", list(CASES))
def test_bf16_mode_on_every_window_matches_the_forced_reference(case, relu, bf16_mode):  # noqa: F811
    """Step-local: every (layer, step) of each shared LSTM (cell state; hidden state as the excess over half a bf16
    ulp), its fp32 h_top and every S_k of every spatial chain, on every chunk of windows.  Whole model: every window's
    output (each held to its own maximum), the loss and every parameter gradient; at cfg4 without the GCN activation
    also d obs, per window and per time step.  All at 1e-4, with ReLU at the kernels' own masks and without it.
    Sizes: cfg2 (1024 regions, batch 32) with Chebyshev and with random_walk_diffusion supports (two bf16 chains per
    graph); cfg4 (cfg3's shapes: 4096 regions, batch 64, 262 144 LSTM rows in 2 048 tiles); cfg5's shapes (16 384
    regions, K = 5, T = 24) at batch 8.

    Measured on an H100 80GB HBM3 at 700 W: step-local at most 1.1e-6 (cfg5; cfg2 and cfg4 6e-7 .. 7e-7), whole
    model at most 2.2e-5 (cfg4 smooth, d obs at its worst time step; cfg2 ReLU in one of three runs,
    rnn_list.0.gconv_temporal_feats.b); against the unrounded reference 4.8e-3 .. 1.8e-2."""
    step, errs, unrounded = _run(case, relu, want_obs=case == "cfg4" and not relu)
    bad = _bad(step, errs)
    assert not bad, f"{case}: above {TOL:.0e}: {bad}"
    assert unrounded > TOL, f"{case}: {unrounded:.2e} from the unrounded reference: the single-plane path did not run"


# ======================================================================================================================
# negative controls: each must fail the check above
# ======================================================================================================================
def test_a_backward_that_drops_unpicked_windows_fails_here_and_passes_the_picked_window_check(bf16_mode,  # noqa: F811
                                                                                            monkeypatch):
    """The LSTM backward zeroes the ``d_top`` rows (``n*B + b``) of every cfg2 window but 0, 17 and 31.  The output is
    untouched; the full-batch check fails in the LSTM's gradients and everything upstream of them, while the
    picked-window check of the same mode (targets of the other windows set to the run's own output, windows 0, 17 and
    31 against the forced reference) passes it: that check cannot see the windows it does not pick.  Measured on an
    H100: 1.3 (rnn_list.0.gconv_temporal_feats.b) against 9.4e-6 for the picked-window check."""
    real = bf16_mode.SharedLSTM.backward

    def lossy(ctx, d_top, dh_n, dc_n):
        keep = torch.zeros(d_top.shape[1], dtype=torch.bool, device=d_top.device)
        keep[PICKS] = True
        return real(ctx, d_top * keep[None, :, None], dh_n, dc_n)
    monkeypatch.setattr(bf16_mode.SharedLSTM, "backward", staticmethod(lossy))
    step, errs, _ = _run("cfg2", False)
    lost = _bad(step, errs)
    worst = max(lost.items(), key=lambda kv: kv[1]) if lost else None
    print(f"control drop-unpicked-windows: full-batch check worst {worst} ({worst[1] / TOL:.0f}x the bar)" if worst
          else "control drop-unpicked-windows: the full-batch check passed it")
    assert errs["out"] <= TOL
    assert any(".lstm." in k for k in lost), f"the full-batch check passed a backward that drops windows: {errs}"

    (model, sups, chains, ks, params, x, y), _ = CASES["cfg2"](False)
    run = gpu_run(model, sups, x, y, PICKS)
    del model
    torch.cuda.empty_cache()
    step_p, errs_p = forced_errors(run, params, chains, ks, x, y, PICKS, relu=False)
    worst_p = max({**step_p, **errs_p}.values())
    print(f"  the picked-window check (windows {PICKS}) on the same mutant: worst {worst_p:.2e} (bar {TOL:.0e})")
    assert worst_p <= TOL, "the picked-window check saw the dropped windows: the control no longer shows the gap"


def _fp32_spatial_gathers(ops, monkeypatch):
    """The spatial chain gathers from fp32 (no bf16 copies) while the LSTM keeps one plane."""
    monkeypatch.setattr(ops, "_gather16", lambda sset, x: False)


CONTROLS = {
    # the reference for window b forced with window b+1's recording: the harness's own row slicing (rows n*B + b, the
    # blocked cell states) must line the recording up with the windows the reference computes
    "tape_one_window_off": ("cfg2", None, dict(window_offset=1)),
    # the mistake the 2e-2 end-to-end check of this mode passes (test_gpu_bf16_mode), at cfg4's size
    "fp32_spatial_gathers_cfg4": ("cfg4", _fp32_spatial_gathers, {}),
}


@pytest.mark.parametrize("control", list(CONTROLS))
def test_negative_controls_fail_the_full_batch_check(control, bf16_mode, monkeypatch):  # noqa: F811
    """Each mistake, in the harness or in the kernels' arithmetic, lands above the bar (model without the GCN
    activation); the margin is printed.  Measured on an H100: one window off 1.2 (the LSTM layer-steps); fp32 spatial
    gathers at cfg4 2.0e-3 (S_3)."""
    case, mutate, kw = CONTROLS[control]
    if mutate is not None:
        mutate(bf16_mode, monkeypatch)
    step, errs, _ = _run(case, False, **kw)
    worst = max({**step, **errs}.items(), key=lambda kv: kv[1])
    print(f"control {control}: worst {worst[0]} {worst[1]:.2e} ({worst[1] / TOL:.0f}x the bar)")
    assert worst[1] > TOL, f"{control}: the full-batch check does not see it"
