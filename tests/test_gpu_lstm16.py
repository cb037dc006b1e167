"""Kernel-level tests of the bf16-plane tensor-core LSTM (lstm16.cu) against the fp64 reference of its arithmetic,
``stmgcn_oracle.lstm_planes_reference``, for both plane modes.

The reference is forced with the kernel's own tape (hidden-state planes and cell states): every step consumes exactly
the values the kernel consumed, so the comparison is step-local (no rounding-boundary flips accumulate through time) and
its autograd backward has the kernel backward's semantics.  That holds the single-plane mode to an fp32-grade bar.
Bars: 2e-5 on forward values, 5e-5 on gradients (max-norm relative), for both plane modes and every case; a negative
control in every case shows that the bar tells the two plane modes apart.
"""
import pytest
import torch

import stmgcn_oracle as O
from helpers import FWD_TOL, GRAD_TOL
from lstm_cases import CASES, HID, lstm16_inputs, lstm16_kernel, reference, step_local_error, wave_regions

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_lstm16_kernels_match_the_fp64_plane_reference(case, planes):
    """Forward step by step (cell state, hidden-state planes, the fp32 h_top / h_n / c_n) and backward (d_s and the
    four gradients of every layer) of the tensor-core LSTM against the tape-forced fp64 reference.  Negative control:
    the reference in the other plane mode lands outside the forward bar.

    Measured on an H100 (max over the eight cases): one plane -- step-local forward 4.1e-7 (excess over half a bf16
    ulp for h), h_top / h_n / c_n 3.9e-7, gradients 6.5e-6, control 5.1e-4 .. 1.6e-3; two planes -- step-local forward
    8.5e-6 (the hi + lo representation of h keeps ~17 bits), h_top / h_n / c_n 3.1e-6, gradients 1.4e-5, control
    1.2e-3 .. 2.9e-3.  The saturated case: step-local forward 4.1e-7 / 4.9e-6, gradients 6.5e-6 / 1.1e-5 (one / two
    planes).  Before the layer-0 W_ih gradient took the lo plane of x*s, weight_ih_l0 was 8e-4 .. 2.2e-3 off
    with one plane."""
    name, n, b, t, lyr, c, state = case
    if n is None:
        n = wave_regions(b)
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n, b, t, lyr, c, state, seed=10 * CASES.index(case) + planes,
                                       saturate=name == "saturated")
    h_top, hc_n, ktape, d_s, grads = lstm16_kernel(xo, s, h0, c0, ws, lyr, planes, d_top)
    if name == "saturated":
        assert all(bool(torch.isfinite(v).all()) for v in (h_top, ktape["c"], d_s, *grads))
        assert float(ktape["c"].abs().max()) > 15.0, "the saturated case does not drive c far enough"
    hs, cs, layers, s64 = reference(xo, s, h0, c0, ws, lyr, planes, ktape)
    errs = {"step-local forward": step_local_error(ktape, hs, cs, planes),
            "h_top": O.max_rel_err(h_top.cpu().numpy(), hs[-1][-1].detach().cpu().numpy())}
    if state:
        errs["h_n"] = O.max_rel_err(hc_n[0].cpu().numpy(), torch.stack([h[-1] for h in hs]).detach().cpu().numpy())
        errs["c_n"] = O.max_rel_err(hc_n[1].cpu().numpy(), torch.stack([v[-1] for v in cs]).detach().cpu().numpy())
    flat = [w for layer in layers for w in layer]
    ref_grads = torch.autograd.grad((hs[-1][-1] * d_top.double()).sum(), [s64] + flat)
    gerrs = {"d_s": O.max_rel_err(d_s.cpu().numpy(), ref_grads[0].cpu().numpy())}
    for i, (g, r) in enumerate(zip(grads, ref_grads[1:])):
        l, j = divmod(i, 4)
        gerrs[f"{('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')[j]}_l{l}"] = O.max_rel_err(g.cpu().numpy(), r.cpu().numpy())
    # negative control: the other plane mode's arithmetic, same tape
    hs_o, cs_o, _, _ = reference(xo, s, h0, c0, ws, lyr, 3 - planes, ktape, grad=False)
    control = step_local_error(ktape, hs_o, cs_o, planes)
    print(f"lstm16 {name} P={planes} rows={n * b}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items())
          + f"; worst gradient {max(gerrs.values()):.2e} ({max(gerrs, key=gerrs.get)}); "
          + ", ".join(f"{k} {v:.1e}" for k, v in gerrs.items()) + f"; control (P={3 - planes} reference) {control:.2e}")
    bad = {k: v for k, v in errs.items() if not v <= FWD_TOL}
    bad.update({k: v for k, v in gerrs.items() if not v <= GRAD_TOL})
    assert not bad, f"{name} P={planes}: above the bar: {bad}"
    assert control > FWD_TOL, f"{name} P={planes}: the P={3 - planes} reference is within the bar ({control:.2e})"


@pytest.mark.parametrize("t_len", [64, 65])
def test_shared_lstm_routing_at_the_step_limit(t_len, monkeypatch):
    """ops.SharedLSTM at T = 64 (tensor-core kernels, the backward's whole step table) and T = 65 (exact-FFMA kernels)
    against the free-running fp64 reference with two planes (nn.LSTM arithmetic): forward and every gradient.
    Measured on an H100: T = 64 h_top 4.9e-6, gradients 7.0e-6; T = 65 h_top 5.2e-7, gradients 9.8e-7."""
    from stmgcn_b200 import ops
    calls = []
    real = ops._lstm16_forward
    monkeypatch.setattr(ops, "_lstm16_forward", lambda *a: calls.append(1) or real(*a))
    monkeypatch.setattr(ops, "_PLANES", 2)
    monkeypatch.setattr(ops, "_LSTM_PATH", "tc")
    n, b, lyr, c = 3, 50, 3, 1
    xo, s, _, _, ws, d_top = lstm16_inputs(n, b, t_len, lyr, c, False, seed=t_len)
    s_g = s.clone().requires_grad_(True)
    ws_g = [w.clone().requires_grad_(True) for w in ws]
    h_top, _, _ = ops.SharedLSTM.apply(xo, s_g, None, None, lyr, HID, False, *ws_g)
    (h_top.reshape(n * b, HID) * d_top).sum().backward()
    assert len(calls) == (1 if t_len <= 64 else 0), "SharedLSTM took the wrong kernel family"
    hs, _, layers, s64 = reference(xo, s, None, None, ws, lyr, 2, None)
    ref_grads = torch.autograd.grad((hs[-1][-1] * d_top.double()).sum(), [s64] + [w for layer in layers for w in layer])
    e_fwd = O.max_rel_err(h_top.detach().reshape(n * b, HID).cpu().numpy(), hs[-1][-1].detach().cpu().numpy())
    gerrs = [O.max_rel_err(g.grad.cpu().numpy(), r.cpu().numpy()) for g, r in zip([s_g] + ws_g, ref_grads)]
    print(f"SharedLSTM T={t_len} ({'tensor cores' if calls else 'FFMA'}): h_top {e_fwd:.2e}, worst gradient {max(gerrs):.2e}")
    assert e_fwd <= FWD_TOL, e_fwd
    assert max(gerrs) <= GRAD_TOL, gerrs


@pytest.mark.parametrize("lyr,t", [(3, 12), (2, 5), (1, 1)])
def test_lstm16_launch_sequence_packs_on_every_forward(lyr, t, monkeypatch):
    """Every forward of the tensor-core path packs each layer's weights and makes one launch per layer (the images are
    packed from the weights as they are at that forward, never reused from an earlier one); the backward is one fused
    launch and one weight-gradient reduction per layer."""
    from stmgcn_b200 import _lib, ops
    monkeypatch.setattr(ops, "_LSTM_PATH", "tc")
    xo, s, _, _, ws, d_top = lstm16_inputs(3, 40, t, lyr, 1, False, seed=3)
    ws_g = [w.requires_grad_(True) for w in ws]
    counts = []
    for _ in range(2):
        n0 = _lib.launch_count()
        h_top, _, _ = ops.SharedLSTM.apply(xo, s, None, None, lyr, HID, False, *ws_g)
        n1 = _lib.launch_count()
        (h_top.reshape(-1, HID) * d_top).sum().backward()
        counts.append((n1 - n0, _lib.launch_count() - n1))
    assert counts == [(2 * lyr, 2 * lyr), (2 * lyr, 2 * lyr)]


def test_lstm16_second_backward_repeats_the_first(monkeypatch):
    """The tensor-core backward leaves its tape intact: a second backward(retain_graph=True) over the same graph gives
    the first one's gradients (within the gradient bar: the kernels sum them with atomics)."""
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_LSTM_PATH", "tc")
    n, b, t, lyr, c = 5, 60, 7, 3, 2
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n, b, t, lyr, c, True, seed=4)
    leaves = [s.clone().requires_grad_(True)] + [w.clone().requires_grad_(True) for w in ws]
    h_top, _, _ = ops.SharedLSTM.apply(xo, leaves[0], h0, c0, lyr, HID, False, *leaves[1:])
    loss = (h_top.reshape(n * b, HID) * d_top).sum()
    grads = []
    for _ in range(2):
        for v in leaves:
            v.grad = None
        loss.backward(retain_graph=True)
        grads.append([v.grad.clone() for v in leaves])
    errs = [O.max_rel_err(a.cpu().numpy(), r.cpu().numpy()) for a, r in zip(grads[1], grads[0])]
    assert max(errs) <= GRAD_TOL, errs
