"""Long in-place chains of the tensor-core LSTM backward (lstm16.cu).

The backward walks each tile through all T steps before it takes the next (tile-major work items), so a tile's dh_rec
and dc are read back one item after they were written, and layer 0 adds its d_s contribution per item.  These cases
run the longest chain the kernels take (T = kBMaxSteps = 64) with several tiles per CTA and a ragged last tile, with
b_inner dividing the 128-row tile and not, against the tape-forced fp64 reference at the bars of test_gpu_lstm16.py.
"""
import pytest
import torch

import stmgcn_oracle as O
from helpers import FWD_TOL, GRAD_TOL
from lstm_cases import CHAIN_CASES, lstm16_inputs, lstm16_kernel, reference, step_local_error, wave_regions

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", CHAIN_CASES, ids=[c[0] for c in CHAIN_CASES])
def test_lstm16_t64_chains_over_several_tiles_per_cta(case, planes):
    name, b, c, state = case
    t, lyr = 64, 2
    n = wave_regions(b)
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n, b, t, lyr, c, state, seed=1000 + 10 * CHAIN_CASES.index(case) + planes)
    h_top, hc_n, ktape, d_s, grads = lstm16_kernel(xo, s, h0, c0, ws, lyr, planes, d_top)
    hs, cs, layers, s64 = reference(xo, s, h0, c0, ws, lyr, planes, ktape)
    errs = {"step-local forward": step_local_error(ktape, hs, cs, planes),
            "h_top": O.max_rel_err(h_top.cpu().numpy(), hs[-1][-1].detach().cpu().numpy())}
    if state:
        errs["c_n"] = O.max_rel_err(hc_n[1].cpu().numpy(), torch.stack([v[-1] for v in cs]).detach().cpu().numpy())
    flat = [w for layer in layers for w in layer]
    ref_grads = torch.autograd.grad((hs[-1][-1] * d_top.double()).sum(), [s64] + flat)
    gerrs = {"d_s": O.max_rel_err(d_s.cpu().numpy(), ref_grads[0].cpu().numpy())}
    for i, (g, r) in enumerate(zip(grads, ref_grads[1:])):
        l, j = divmod(i, 4)
        gerrs[f"{('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')[j]}_l{l}"] = O.max_rel_err(g.cpu().numpy(), r.cpu().numpy())
    print(f"lstm16 chain {name} P={planes} rows={n * b} T={t} L={lyr}: "
          + ", ".join(f"{k} {v:.2e}" for k, v in errs.items())
          + f"; worst gradient {max(gerrs.values()):.2e} ({max(gerrs, key=gerrs.get)})")
    bad = {k: v for k, v in errs.items() if not v <= FWD_TOL}
    bad.update({k: v for k, v in gerrs.items() if not v <= GRAD_TOL})
    assert not bad, f"{name} P={planes}: above the bar: {bad}"
