"""The LSTM backward held to its bar at every time step (``per_step.per_step_rel_err``), not only in max-norm.

With the suite's input distribution the gradients decay going back in time: at T = 64 the first step's d_s is ~1e-9
(one layer) to ~1e-7 (two layers) of the largest, so a backward that dropped or corrupted its first 16 .. 30 steps would
still pass the max-norm checks of test_gpu_lstm16 / test_gpu_lstm16_chains / test_gpu_input_grads.  Here every step
of d_s (B, T) and d_xo (N, B, T, C), and dh0 / dc0 of every layer, is compared with the tape-forced fp64 reference
(test_gpu_input_grads._state_reference, seeds dh_n / dc_n, every extra wanted) relative to that step's own maximum, at
the suite's 5e-5:

* the tensor-core kernels (lstm16.cu) at every case of test_gpu_lstm16.CASES and test_gpu_lstm16_chains.CASES, both
  plane modes; the exact-fp32 kernels (lstm.cu) at every case of test_gpu_exact_kernels.LSTM_CASES and
  test_gpu_input_grads.EXACT_CASES;
* long-memory cases: +3 on the forget-gate rows of b_ih, so that every step carries weight in the summed gradients too
  (each case asserts that the reference's max|d_s[:, 0]| is at least 1e-2 of max|d_s|); there every output, the weight
  gradients included, is also held to 5e-5 in max-norm;
* negative controls in every case with T >= 2: the reference truncated to steps T/2 .. T-1 (started from the kernel's
  own state at T/2 - 1, no gradient into it) and the kernel's d_s with steps 0 and 1 swapped must both fail the
  per-step bar; in the long-memory cases the truncated reference must also fail the weight-gradient bar;
* module level: SharedLSTM at T = 64 / 65 and ST_MGCN's d obs at T = 24 against free-running fp64 references, where
  rounding builds up over the steps, at bars taken from measurement.
"""
import pytest
import torch
from torch import nn

import stmgcn_oracle as O
from per_step import per_step_rel_err, worst_step
from helpers import DEV, GRAD_TOL, sm_count
from lstm_cases import (EXACT, HID, PREMISE, TC_CASES, exact_run, grad_errors, lstm16_inputs, lstm16_run, lstm_inputs,
                        seeds, state_gradients, wave_regions, with_long_memory)
from model_cases import dense_grads, small_model

pytestmark = pytest.mark.gpu


def _per_step(got, ref):
    """{output: (worst per-step error, its step)}: d_s over T, d_xo over T, dh0 / dc0 over the layers."""
    return {k: worst_step(got[k], ref[k], axis) for k, axis in (("d_s", 1), ("d_xo", 2), ("dh0", 0), ("dc0", 0))}


def _truncated_reference(xo, s, ws, lyr, planes, ktape, d_top, dh_n, dc_n):
    """Truncated BPTT: the reference run over steps T/2 .. T-1 only, from the kernel's tape state at T/2 - 1 taken as a
    constant; d_s and d_xo of the steps before T/2 are zero."""
    t = xo.shape[2]
    k = t // 2
    h_k, c_k = ktape["h"][:, k - 1].clone(), ktape["c"][:, k - 1].clone()
    tape = dict(h=ktape["h"][:, k:], c=ktape["c"][:, k:], h0=h_k)
    r = state_gradients(xo[:, :, k:], s[:, k:], h_k, c_k, ws, lyr, planes, tape, d_top, dh_n, dc_n)
    r["d_s"] = torch.cat([r["d_s"].new_zeros(s.shape[0], k), r["d_s"]], dim=1)
    r["d_xo"] = torch.cat([r["d_xo"].new_zeros(xo.shape[:2] + (k,) + xo.shape[3:]), r["d_xo"]], dim=2)
    return r


def _check(what, xo, s, h0, c0, ws, lyr, planes, d_top, dh_n, dc_n, got, ktape, long_memory, bars=None):
    ref = state_gradients(xo, s, h0, c0, ws, lyr, planes, ktape, d_top, dh_n, dc_n)
    steps = _per_step(got, ref)
    line = f"{what}: per step " + ", ".join(f"{k} {e:.2e} (step {i})" for k, (e, i) in steps.items())
    bad = {k: e for k, (e, _) in steps.items() if not e <= (bars or {}).get(k, GRAD_TOL)}
    if long_memory:
        share = float(ref["d_s"][:, 0].abs().max()) / float(ref["d_s"].abs().max())
        errs = grad_errors(got, ref)
        line += f"; max-norm worst {max(errs.values()):.2e} ({max(errs, key=errs.get)}); d_s[:, 0] share {share:.2f}"
        assert share >= PREMISE, f"{what}: the long-memory premise fails: d_s[:, 0] is {share:.1e} of max|d_s|"
        bad.update({k: e for k, e in errs.items() if not e <= GRAD_TOL})
    t = xo.shape[2]
    if t >= 2:
        trunc = _truncated_reference(xo, s, ws, lyr, planes, ktape, d_top, dh_n, dc_n)
        tr_step = worst_step(trunc["d_s"], ref["d_s"], 1)[0]
        tr_old = O.max_rel_err(trunc["d_s"].cpu().numpy(), ref["d_s"].cpu().numpy())
        tr_w = max(v for k, v in grad_errors(trunc, ref).items() if k.startswith("param"))
        swapped = got["d_s"].clone()
        swapped[:, [0, 1]] = swapped[:, [1, 0]]
        sw_step = worst_step(swapped, ref["d_s"], 1)[0]
        line += (f"; controls: truncated at T/2 per step {tr_step:.1e}, max-norm d_s {tr_old:.1e} weights {tr_w:.1e}; "
                 f"steps 0 / 1 swapped per step {sw_step:.1e}")
        assert tr_step > GRAD_TOL, f"{what}: the truncated reference passes the per-step bar ({tr_step:.2e})"
        assert sw_step > GRAD_TOL, f"{what}: d_s with steps 0 and 1 swapped passes the per-step bar ({sw_step:.2e})"
        if long_memory:
            assert tr_w > GRAD_TOL, f"{what}: the truncated reference passes the weight-gradient bar ({tr_w:.2e})"
    print(line)
    assert not bad, f"{what}: above the bar: {bad}"


# The saturated case's dh0 of layer 1, held to 2e-3: measured 1.25e-3 (one plane) and 1.26e-3 (two planes) on an H100
# 80GB HBM3, while every other output of the case is within 7.1e-6 per step.  An absolute error, not a relative one:
# layer 1's dh0 is 3.4e-4 at most (layer 0's 0.45), and ~4e-7 off.  Layers > 0 of that case sit in saturation (biases
# i +10, f +20, g +-15 with W in +-0.25), and lstm16_bwd_kernel forms sigmoid' as s (1 - s) from the fp32 activation:
# 1 - s carries fp32's rounding of 1, ~6e-8 absolute, 1.3e-3 of sigmoid'(10) (an fp64 emulation of the formula gives
# 1.3e-2 on the worst gate of layer 1, 7e-7 with 1 - s = e^-v s from the exponential).  The exponential form held this
# case within 5e-5 and every other test, but spilled lstm16_bwd_kernel at its 168-register cap and made the cfg3 step
# 5 % slower (71.3 against 67.7-68.0 ms), so the kernel keeps s (1 - s) and the bar carries its error.
SATURATED_DH0_BAR = 2e-3


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", TC_CASES, ids=[c[0] for c in TC_CASES])
def test_tensor_core_backward_per_step(case, planes):
    name, n, b, t, lyr, c, state, long_memory = case
    if n is None:
        n = wave_regions(b)
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n, b, t, lyr, c, state, seed=3000 + 10 * TC_CASES.index(case) + planes,
                                       saturate=name == "saturated")
    if long_memory:
        ws = with_long_memory(ws, HID)
    dh_n, dc_n = seeds(lyr, n * b, HID, seed=3000 + TC_CASES.index(case))
    got, ktape, _ = lstm16_run(xo, s, h0, c0, ws, lyr, planes, d_top, dh_n, dc_n)
    _check(f"lstm16 {name} P={planes} rows={n * b}", xo, s, h0, c0, ws, lyr, planes, d_top, dh_n, dc_n, got, ktape,
           long_memory, bars={"dh0": SATURATED_DH0_BAR} if name == "saturated" else None)


@pytest.mark.parametrize("case", EXACT, ids=[c[0] for c in EXACT])
def test_exact_backward_per_step(case):
    name, hid, lyr, t, c, n, b, state, long_memory = case
    if n is None:
        n = (2 * 32 * sm_count()) // b + 1
    xo, s, h0, c0, ws, d_top = lstm_inputs(n, b, t, lyr, c, hid, state, seed=4000 + EXACT.index(case),
                                           saturate=name == "saturated")
    if long_memory:
        ws = with_long_memory(ws, hid)
    xo, s, d_top = xo.to(DEV), s.to(DEV), d_top.to(DEV)
    h0, c0 = (None, None) if h0 is None else (h0.to(DEV), c0.to(DEV))
    ws = [w.to(DEV) for w in ws]
    dh_n, dc_n = seeds(lyr, n * b, hid, seed=4000 + EXACT.index(case))
    got, ktape = exact_run(xo, s, h0, c0, ws, lyr, hid, d_top, dh_n, dc_n)
    _check(f"lstm {name} rows={n * b}", xo, s, h0, c0, ws, lyr, 2, d_top, dh_n, dc_n, got, ktape, long_memory)


# free-running fp64 references: the fp32 forward's rounding builds up over the steps, so these bars come from
# measurement (at most 4x the measured worst step, never above the 1e-4 parity bar).  Measured on an H100 80GB HBM3:
# SharedLSTM T = 64 (tensor cores, 3xBF16) d_s 5.8e-5, d_xo 7.9e-5 (4x would exceed 1e-4); T = 65 (exact FFMA) d_s
# 1.7e-6, d_xo 1.2e-6; ST_MGCN d obs 8.8e-6.
SHARED_LSTM_BAR = {64: 1e-4, 65: 6e-6}
ST_MGCN_BAR = 3e-5


@pytest.mark.parametrize("t_len", [64, 65])
def test_shared_lstm_input_gradients_per_step(t_len, monkeypatch):
    """ops.SharedLSTM at T = 64 (tensor cores, two planes) and T = 65 (exact-FFMA kernels) with xo and s requiring
    grad: d_s and d_xo per step against the free-running fp64 LSTM (O.lstm_explicit)."""
    from stmgcn_b200 import ops
    calls = []
    real = ops._lstm16_forward
    monkeypatch.setattr(ops, "_lstm16_forward", lambda *a: calls.append(1) or real(*a))
    monkeypatch.setattr(ops, "_PLANES", 2)
    monkeypatch.setattr(ops, "_LSTM_PATH", "tc")
    n, b, lyr, c = 3, 50, 3, 2
    xo, s, _, _, ws, d_top = lstm16_inputs(n, b, t_len, lyr, c, False, seed=5000 + t_len)
    xo_g, s_g = xo.clone().requires_grad_(True), s.clone().requires_grad_(True)
    h_top, _, _ = ops.SharedLSTM.apply(xo_g, s_g, None, None, lyr, HID, False, *ws)
    (h_top.reshape(n * b, HID) * d_top).sum().backward()
    torch.cuda.synchronize()
    assert len(calls) == (1 if t_len <= 64 else 0), "SharedLSTM took the wrong kernel family"
    xo64, s64 = xo.double().requires_grad_(True), s.double().requires_grad_(True)
    layers = [tuple(w.double() for w in ws[4 * l:4 * l + 4]) for l in range(lyr)]
    seq, _ = O.lstm_explicit(xo64.reshape(n * b, t_len, c) * s64.repeat(n, 1)[:, :, None], layers)
    d_xo, d_s = torch.autograd.grad((seq[:, -1] * d_top.double()).sum(), [xo64, s64])
    steps = {"d_s": worst_step(s_g.grad, d_s, 1), "d_xo": worst_step(xo_g.grad, d_xo, 2)}
    print(f"SharedLSTM T={t_len} ({'tensor cores' if calls else 'FFMA'}) free-running: "
          + ", ".join(f"{k} {e:.2e} (step {i})" for k, (e, i) in steps.items()) + f"; bar {SHARED_LSTM_BAR[t_len]:.0e}")
    bad = {k: e for k, (e, _) in steps.items() if not e <= SHARED_LSTM_BAR[t_len]}
    assert not bad, bad


def test_st_mgcn_obs_gradient_per_step():
    """ST_MGCN (two Chebyshev graphs, ReLU, H = 64 on the tensor cores) at T = 24 with obs_seq requiring grad: d obs
    per step against the dense fp64 oracle."""
    model, sups, n, t = small_model(2, 1, "chebyshev", "relu", seed=21, t=24)
    gen = torch.Generator().manual_seed(22)
    x = torch.randn(4, t, n, 1, generator=gen).to(DEV).requires_grad_(True)
    y = torch.randn(4, n, 1, generator=gen).to(DEV)
    out = model(obs_seq=x, sta_adj_list=[v.to(DEV) for v in sups])
    nn.MSELoss()(out, y).backward()
    d_obs, _ = dense_grads(model, sups, x, y, "relu")
    errs = per_step_rel_err(x.grad, d_obs, 1)
    share = (d_obs.abs().amax(dim=(0, 2, 3)) / d_obs.abs().max()).min()
    print(f"ST_MGCN T={t} d obs per step: worst {errs.max():.2e} (step {int(errs.argmax())}), "
          f"smallest step {float(share):.1e} of the largest; bar {ST_MGCN_BAR:.0e}")
    assert bool((errs <= ST_MGCN_BAR).all()), errs
