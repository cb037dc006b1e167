"""CPU tests of the per-step metric (tests/per_step.py) and of the premises of tests/test_gpu_lstm_per_step.py, in fp64
with the inputs of the GPU suite drawn on the CPU."""
import numpy as np
import pytest
import torch

import stmgcn_oracle as O
from per_step import per_step_rel_err, worst_step
from helpers import GRAD_TOL
from lstm_cases import EXACT, PREMISE, TC_CASES, lstm16_inputs, lstm_inputs, with_long_memory


# ======================================================================================================================
# the metric
# ======================================================================================================================
def test_each_step_is_judged_against_its_own_maximum():
    ref = np.array([[1e-9, 1.0], [2e-9, -3.0]])           # (B, T): step 0 is a billionth of step 1
    new = ref.copy()
    new[:, 0] += 1e-10
    new[1, 1] += 3e-6
    errs = per_step_rel_err(new, ref, axis=1)
    assert errs.shape == (2,)
    assert errs[0] == pytest.approx(1e-10 / 2e-9)
    assert errs[1] == pytest.approx(1e-6)
    assert O.max_rel_err(new, ref) < 1e-6                 # the whole-tensor metric does not see step 0
    assert worst_step(new, ref, 1) == (pytest.approx(0.05), 0)


def test_axis_and_shape_handling():
    gen = np.random.default_rng(0)
    ref = gen.standard_normal((3, 4, 5, 2))
    new = ref + 1e-3 * gen.standard_normal(ref.shape)
    for axis in range(4):
        errs = per_step_rel_err(new, ref, axis)
        assert errs.shape == (ref.shape[axis],)
        for i in range(ref.shape[axis]):
            sl = [slice(None)] * 4
            sl[axis] = i
            assert errs[i] == pytest.approx(O.max_rel_err(new[tuple(sl)], ref[tuple(sl)]))
    assert np.array_equal(per_step_rel_err(new, ref, -1), per_step_rel_err(new, ref, 3))
    assert np.array_equal(per_step_rel_err(torch.from_numpy(new), torch.from_numpy(ref), 2), per_step_rel_err(new, ref, 2))
    with pytest.raises(ValueError, match="shapes differ"):
        per_step_rel_err(new[:, :3], ref, 1)
    with pytest.raises(np.exceptions.AxisError):
        per_step_rel_err(new, ref, 4)


def test_a_zero_reference_slice_is_judged_against_the_global_maximum():
    ref = np.array([[0.0, 2.0], [0.0, -4.0]])
    assert per_step_rel_err(ref, ref, 1).tolist() == [0.0, 0.0]
    new = ref.copy()
    new[0, 0] = 1e-3
    assert per_step_rel_err(new, ref, 1)[0] == pytest.approx(1e-3 / 4.0)
    zero = np.zeros((2, 3))
    assert per_step_rel_err(zero, zero, 0).tolist() == [0.0, 0.0]
    assert per_step_rel_err(zero + 0.5, zero, 0).tolist() == [0.5, 0.5]


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("where", ["new", "ref"])
def test_nan_or_inf_fails_the_bar(bad, where):
    ref = np.ones((3, 4))
    new = ref.copy()
    (new if where == "new" else ref)[1, 2] = bad
    errs = per_step_rel_err(new, ref, 0)
    assert errs[0] == 0.0 and errs[2] == 0.0
    assert np.isnan(errs[1]) and not errs[1] <= GRAD_TOL
    err, step = worst_step(new, ref, 0)
    assert np.isnan(err) and step == 1 and not err <= GRAD_TOL
    # another step's NaN does not change how a zero slice is judged
    ref2 = np.array([[0.0, 1.0], [0.0, 4.0]])
    new2 = ref2.copy()
    new2[0, 0], new2[1, 1] = 2.0, np.nan
    assert per_step_rel_err(new2, ref2, 1)[0] == pytest.approx(0.5)


# ======================================================================================================================
# premises, in fp64 on the CPU
# ======================================================================================================================
def _reference(xo, s, ws, lyr, d_top, h0=None, c0=None, cut=0):
    """fp64 gradients (d_s (B, T), the weight gradients) of <h_top, d_top> through O.lstm_explicit; ``cut`` > 0:
    truncated BPTT, the backward only over steps cut .. T-1 from the (constant) state at cut - 1."""
    n, b, t, c = xo.shape
    s64 = s.double().requires_grad_(True)
    layers = [tuple(w.double().requires_grad_(True) for w in ws[4 * l:4 * l + 4]) for l in range(lyr)]
    x = xo.double().reshape(n * b, t, c) * s64.repeat(n, 1)[:, :, None]
    h0 = None if h0 is None else h0.double()
    c0 = None if c0 is None else c0.double()
    if cut:
        with torch.no_grad():
            _, (h0, c0) = O.lstm_explicit(x[:, :cut], layers, h0, c0)
    seq, _ = O.lstm_explicit(x[:, cut:], layers, h0, c0)
    g = torch.autograd.grad((seq[:, -1] * d_top.double()).sum(), [s64] + [w for layer in layers for w in layer])
    return g[0], list(g[1:])


def test_truncated_bptt_passes_the_max_norm_bar_and_fails_the_per_step_one():
    """The t64_l1_c4 case of test_gpu_lstm16 (N = 3, B = 43, T = 64, L = 1, C = 4) with its one-plane seed: a backward
    that skips the first 28 steps is within 5e-5 of the full one on d_s in max-norm, and fails the per-step metric.
    (With this seed, skipping T/2 = 32 steps puts d_s 9.2e-5 off in max-norm, 30 steps 6.1e-5, 28 steps 3.8e-5.)"""
    n, b, t, lyr, c = 3, 43, 64, 1, 4
    cut = 28
    xo, s, _, _, ws, d_top = lstm16_inputs(n, b, t, lyr, c, False, seed=21, device="cpu")
    d_s, _ = _reference(xo, s, ws, lyr, d_top)
    d_s_cut, _ = _reference(xo, s, ws, lyr, d_top, cut=cut)
    old = O.max_rel_err(d_s_cut.numpy(), d_s.numpy())
    new, step = worst_step(d_s_cut, d_s, 1)
    print(f"truncated at step {cut}: max-norm d_s {old:.1e}, per step {new:.1e} (step {step}); "
          f"d_s[:, 0] {float(d_s[:, 0].abs().max() / d_s.abs().max()):.1e} of the maximum")
    assert old <= GRAD_TOL, old
    assert new > GRAD_TOL, new


def _tc_long_inputs(case, planes, n_waves=4):
    name, n, b, t, lyr, c, state, _ = case
    seed = 3000 + 10 * TC_CASES.index(case) + planes
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n or n_waves, b, t, lyr, c, state, seed=seed, device="cpu")
    return xo, s, h0, c0, with_long_memory(ws, 64), d_top, lyr


def _exact_long_inputs(case):
    name, hid, lyr, t, c, n, b, state, _ = case
    xo, s, h0, c0, ws, d_top = lstm_inputs(n, b, t, lyr, c, hid, state, seed=4000 + EXACT.index(case))
    return xo, s, h0, c0, with_long_memory(ws, hid), d_top, lyr


LONG = ([("tc", c) for c in TC_CASES if c[-1]] + [("exact", c) for c in EXACT if c[-1]])


@pytest.mark.parametrize("family,case", LONG, ids=[f"{f}-{c[0]}" for f, c in LONG])
def test_long_memory_inputs_give_every_step_weight(family, case):
    """The long-memory cases of test_gpu_lstm_per_step (their seeds; the multi-wave one with 4 regions here): the
    fp64 max|d_s[:, 0]| is at least 1e-2 of max|d_s|, and a backward truncated at T/2 fails the weight-gradient bar."""
    xo, s, h0, c0, ws, d_top, lyr = _tc_long_inputs(case, 2) if family == "tc" else _exact_long_inputs(case)
    d_s, wg = _reference(xo, s, ws, lyr, d_top, h0, c0)
    share = float(d_s[:, 0].abs().max() / d_s.abs().max())
    _, wg_cut = _reference(xo, s, ws, lyr, d_top, h0, c0, cut=xo.shape[2] // 2)
    w_err = max(O.max_rel_err(a.numpy(), r.numpy()) for a, r in zip(wg_cut, wg))
    print(f"{case[0]}: d_s[:, 0] {share:.2f} of the maximum; truncated at T/2: weights {w_err:.1e}")
    assert share >= PREMISE, share
    assert w_err > GRAD_TOL, w_err


def test_without_the_forget_bias_the_early_steps_vanish():
    """The same draws as the first long-memory case without the +3: d_s[:, 0] falls far below 1e-2 of the maximum --
    what the forget bias is there to change."""
    case = next(c for c in TC_CASES if c[-1])
    name, n, b, t, lyr, c, state, _ = case
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n or 4, b, t, lyr, c, state, seed=3000 + 10 * TC_CASES.index(case) + 2,
                                       device="cpu")
    d_s, _ = _reference(xo, s, ws, lyr, d_top, h0, c0)
    share = float(d_s[:, 0].abs().max() / d_s.abs().max())
    print(f"{name} without the forget bias: d_s[:, 0] {share:.1e} of the maximum")
    assert share < PREMISE * 1e-2, share
