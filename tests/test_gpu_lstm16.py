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

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HID = 64
FWD_TOL, GRAD_TOL = 2e-5, 5e-5


def _sms():
    from stmgcn_b200 import _lib
    return int(_lib.lib.stmgcn_sm_count())


def _wave_regions(b):
    """Regions N such that N * b rows fill more than two 128-row tiles per SM and end in a partial tile."""
    n = (128 * (2 * _sms() + 1)) // b + 1
    while (n * b) % 128 == 0:
        n += 1
    return n


# (name, regions N (None: multi-wave, from the SM count), batch B, T, layers L, channels C, initial state)
CASES = [
    ("one_row", 1, 1, 3, 2, 1, False),                # one row, one partial tile, ds_fixed with B = 1
    ("t1_one_tile", 2, 64, 1, 3, 1, False),           # T = 1 (layer 0 has no MMA), exactly one tile
    ("t64_l1_c4", 3, 43, 64, 1, 4, False),            # T = kBMaxSteps, L = 1, C = 4, atomic d_s
    ("c3_l4_state", 5, 60, 7, 4, 3, True),            # C = 3, L = 4 (dx buffers reused), h0 / c0 forward and backward
    ("waves_b64", None, 64, 12, 3, 1, False),         # several tiles per CTA, ds_acc carried across items
    ("waves_b37_state", None, 37, 12, 3, 2, True),    # several tiles per CTA, atomic d_s, runtime-C variant
    ("b1100", 2, 1100, 4, 3, 1, False),               # windows spanning tiles
    ("saturated", 5, 40, 20, 3, 1, True),             # pre-activations to +-70 (capped exponentials), c to +-20
]


def _inputs(n, b, t, lyr, c, state, seed, saturate=False, device=DEV):
    """``saturate``: the terms the kernels add with fp32 FMAs drive the gates into saturation -- inputs x3 and layer 0's
    W_ih in +-3, biases i +10, f +20, g +-15 (one sign per unit), o uniform in +-50 -- so the pre-activations reach about
    +-70 and c about +-T, while the tensor-core operands W_hh and W_ih of layers > 0 keep their usual +-0.25.  (With
    those in +-2 as well, the two-plane kernel is 5.9e-5 off step-local and 1.1e-4 in the gradients, measured: three
    bf16 passes keep ~16 bits of each product, so the error of a pre-activation grows with sum |W| |h|, here 8-fold,
    while h stays within +-1.  The one-plane mode, whose reference rounds like the kernel, stayed within its bars.)
    The draws are made on the CPU; ``device`` is where the tensors land."""
    gen = torch.Generator().manual_seed(seed)
    xo = torch.randn(n, b, t, c, generator=gen) * (3.0 if saturate else 1.0)
    s = 0.2 + 0.8 * torch.rand(b, t, generator=gen)
    ws = []
    for l in range(lyr):
        in_l = c if l == 0 else HID
        amp_ih = 6.0 if saturate and l == 0 else 0.5
        ws += [(torch.rand(4 * HID, in_l, generator=gen) - 0.5) * amp_ih, (torch.rand(4 * HID, HID, generator=gen) - 0.5) * 0.5,
               (torch.rand(4 * HID, generator=gen) - 0.5) * 0.5, (torch.rand(4 * HID, generator=gen) - 0.5) * 0.5]
        if saturate:
            ws[-2] = torch.zeros(4 * HID)
            ws[-2][:HID], ws[-2][HID:2 * HID] = 10.0, 20.0
            ws[-2][2 * HID:3 * HID] = 15.0 * torch.sign(torch.randn(HID, generator=gen))
            ws[-2][3 * HID:] = (torch.rand(HID, generator=gen) - 0.5) * 100.0
            ws[-1] = torch.zeros(4 * HID)
    h0 = c0 = None
    if state:
        h0 = torch.randn(lyr, n * b, HID, generator=gen) * 0.3
        c0 = torch.randn(lyr, n * b, HID, generator=gen) * 0.5
    d_top = torch.randn(n * b, HID, generator=gen)
    dev = lambda v: None if v is None else v.to(device).contiguous()      # noqa: E731
    return dev(xo), dev(s), dev(h0), dev(c0), [dev(w) for w in ws], dev(d_top)


def _reference(xo, s, h0, c0, ws, lyr, planes, tape, grad=True):
    """fp64 reference (on the device) -> (hs, cs, fp64 LSTM parameters, fp64 s): autograd leaves when ``grad``."""
    n, b, t, c = xo.shape
    with torch.set_grad_enabled(grad):
        s64 = s.double().requires_grad_(grad)
        layers = [tuple(w.double().requires_grad_(grad) for w in ws[4 * l:4 * l + 4]) for l in range(lyr)]
        x = xo.double().reshape(n * b, t, c) * s64.repeat(n, 1)[:, :, None]           # row r = n * B + b -> s[b]
        h0d = None if h0 is None else h0.double()
        c0d = None if c0 is None else c0.double()
        _, _, (hs, cs) = O.lstm_planes_reference(x, layers, planes, h0d, c0d, tape)
        return hs, cs, layers, s64


def _kernel(xo, s, h0, c0, ws, lyr, planes, d_top):
    from stmgcn_b200 import ops
    n, b, t, c = xo.shape
    rows = n * b
    state = h0 is not None
    h_top, h_n, c_n, tape = ops._lstm16_forward(xo, s, h0, c0, lyr, state, ws, planes, True)
    d_s, grads = ops._lstm16_backward(xo, s, tape, lyr, planes, d_top)
    torch.cuda.synchronize()
    ktape = dict(h=tape["hp"].double().sum(dim=2),                                # (L, T, R, 64): planes summed
                 c=ops.from_blocked(tape["cs"], rows).double())
    if state:
        ktape["h0"] = tape["h0p"].double().sum(dim=1)
    return h_top.reshape(rows, HID), (h_n, c_n) if state else None, ktape, d_s, grads


def _half_ulp_bf16(v):
    _, e = torch.frexp(v)                     # |v| = m 2^e, m in [0.5, 1): bf16 keeps 8 significant bits
    return torch.ldexp(torch.ones_like(v), e - 9)


def _step_local_error(ktape, hs, cs, planes):
    """Max over every (layer, step) of the cell-state error and the hidden-state error.  Two planes: hi + lo against the
    reference h; one plane: the excess of |hi - h| over half a bf16 ulp of h (hi is h rounded to bf16)."""
    worst = 0.0
    for l in range(len(hs)):
        for t in range(len(hs[l])):
            h_ref, c_ref = hs[l][t].detach(), cs[l][t].detach()
            worst = max(worst, O.max_rel_err(ktape["c"][l, t].cpu().numpy(), c_ref.cpu().numpy()))
            hk = ktape["h"][l, t]
            if planes == 2:
                worst = max(worst, O.max_rel_err(hk.cpu().numpy(), h_ref.cpu().numpy()))
            else:
                excess = ((hk - h_ref).abs() - _half_ulp_bf16(h_ref)).clamp_min(0)
                worst = max(worst, float(excess.max()) / max(float(h_ref.abs().max()), 1e-30))
    return worst


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
        n = _wave_regions(b)
    xo, s, h0, c0, ws, d_top = _inputs(n, b, t, lyr, c, state, seed=10 * CASES.index(case) + planes,
                                       saturate=name == "saturated")
    h_top, hc_n, ktape, d_s, grads = _kernel(xo, s, h0, c0, ws, lyr, planes, d_top)
    if name == "saturated":
        assert all(bool(torch.isfinite(v).all()) for v in (h_top, ktape["c"], d_s, *grads))
        assert float(ktape["c"].abs().max()) > 15.0, "the saturated case does not drive c far enough"
    hs, cs, layers, s64 = _reference(xo, s, h0, c0, ws, lyr, planes, ktape)
    errs = {"step-local forward": _step_local_error(ktape, hs, cs, planes),
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
    hs_o, cs_o, _, _ = _reference(xo, s, h0, c0, ws, lyr, 3 - planes, ktape, grad=False)
    control = _step_local_error(ktape, hs_o, cs_o, planes)
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
    xo, s, _, _, ws, d_top = _inputs(n, b, t_len, lyr, c, False, seed=t_len)
    s_g = s.clone().requires_grad_(True)
    ws_g = [w.clone().requires_grad_(True) for w in ws]
    h_top, _, _ = ops.SharedLSTM.apply(xo, s_g, None, None, lyr, HID, False, *ws_g)
    (h_top.reshape(n * b, HID) * d_top).sum().backward()
    assert len(calls) == (1 if t_len <= 64 else 0), "SharedLSTM took the wrong kernel family"
    hs, _, layers, s64 = _reference(xo, s, None, None, ws, lyr, 2, None)
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
    xo, s, _, _, ws, d_top = _inputs(3, 40, t, lyr, 1, False, seed=3)
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
    xo, s, h0, c0, ws, d_top = _inputs(n, b, t, lyr, c, True, seed=4)
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
