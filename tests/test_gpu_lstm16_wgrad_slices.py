"""Weight gradients of the tensor-core LSTM backward against the tape-forced fp64 reference where the per-CTA
weight-gradient slices see their unusual shapes: T = 1, 2 and odd T, a ragged row count whose last tile is partial, and
more tiles than one wave of CTAs, so that each slice element takes the adds of several (step, tile) items, the last of
them from a partial tile.  Layer 0 runs with one input channel (its compile-time variant) and with three (the runtime
variant, whose auxiliary x*s tile fills kd rows 64 .. 66 of the slice).  The bar is the kernel-level gradient bar of
tests/test_gpu_lstm16.py.
"""
import pytest
import torch

import stmgcn_oracle as O
from helpers import GRAD_TOL
from lstm_cases import lstm16_inputs, lstm16_kernel, reference, wave_regions

pytestmark = pytest.mark.gpu

# (T, layers, channels C, initial state)
SLICE_CASES = [(1, 2, 1, False), (2, 2, 3, True), (3, 3, 1, False), (5, 2, 3, False)]
NAMES = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", SLICE_CASES, ids=[f"t{t}_l{lyr}_c{c}{'_state' if s else ''}" for t, lyr, c, s in SLICE_CASES])
def test_lstm16_weight_gradients_at_short_and_odd_t_with_a_ragged_last_tile(case, planes):
    t, lyr, c, state = case
    b = 37                                  # b_inner does not divide 128
    n = wave_regions(b)                     # more than two tiles per CTA, the last one partial
    rows = n * b
    assert rows % 128 != 0
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n, b, t, lyr, c, state, seed=1000 + 10 * t + planes)
    _, _, ktape, d_s, grads = lstm16_kernel(xo, s, h0, c0, ws, lyr, planes, d_top)
    hs, _, layers, s64 = reference(xo, s, h0, c0, ws, lyr, planes, ktape)
    flat = [w for layer in layers for w in layer]
    ref = torch.autograd.grad((hs[-1][-1] * d_top.double()).sum(), [s64] + flat)
    errs = {"d_s": O.max_rel_err(d_s.cpu().numpy(), ref[0].cpu().numpy())}
    for i, (g, r) in enumerate(zip(grads, ref[1:])):
        l, j = divmod(i, 4)
        errs[f"{NAMES[j]}_l{l}"] = O.max_rel_err(g.cpu().numpy(), r.cpu().numpy())
    print(f"lstm16 weight gradients T={t} L={lyr} C={c} P={planes} rows={rows}: "
          + ", ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    bad = {k: v for k, v in errs.items() if not v <= GRAD_TOL}
    assert not bad, f"T={t} L={lyr} C={c} P={planes}: above the bar: {bad}"
