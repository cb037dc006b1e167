"""The LSTM suites' shared cases, seeded inputs, tape-forced fp64 reference and kernel runners.

The reference is ``O.lstm_planes_reference`` forced with the kernel's own tape (hidden states, cell states, initial
hidden state): every layer-step starts from the values the kernel started from, so the comparison is step-local (no
rounding-boundary flips accumulate through time) and its autograd backward has the kernel backward's semantics.

The kernel runners look the entry points up in ``ops`` at call time, so a test that wraps one with ``monkeypatch`` sees
the calls.
"""
import torch

import stmgcn_oracle as O
from helpers import DEV, rel_err, sm_count

HID = 64                    # the tensor-core LSTM's hidden width


def wave_regions(b):
    """Regions N such that N * b rows fill more than two 128-row tiles per SM and end in a partial tile."""
    n = (128 * (2 * sm_count() + 1)) // b + 1
    while (n * b) % 128 == 0:
        n += 1
    return n


# ======================================================================================================================
# case tables
# ======================================================================================================================
# tensor-core LSTM: (name, regions N (None: multi-wave, from the SM count), batch B, T, layers L, channels C, initial state)
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

# T = 64 chains of the tensor-core backward over several tiles per CTA: (name, batch B (b_inner), channels C, initial state)
CHAIN_CASES = [
    ("b64", 64, 1, False),           # b_inner divides 128: every tile's rows cover the same windows
    ("b37_state", 37, 2, True),      # b_inner does not divide 128; h0 / c0; runtime-C layer-0 variant
]

# exact-fp32 LSTM: (name, H, L, T, C, regions N (None: multi-wave, from the SM count), batch B, initial state, forced
# "fma" path)
LSTM_CASES = [
    ("h4_one_row", 4, 2, 5, 1, 1, 1, False, False),          # one row; ul = 1, 28 idle lanes per warp
    ("h20_state", 20, 3, 9, 2, 37, 5, True, False),          # H % 32 != 0 forward and backward with h0 / c0
    ("h36_c3_state", 36, 2, 4, 3, 7, 36, True, False),       # ul = 2 with a partial second unit; bwd data TN = 128
    ("h100_c4_state", 100, 2, 6, 4, 13, 11, True, False),    # 4H = 400: partial second forward panel; bwd data TN = 128
                                                             # with two panels (2H = 200); partial second wgrad z-panel
    ("h128_waves", 128, 3, 7, 1, None, 37, False, False),    # kMaxUnitsPerLane; wgrad kd = 256 (two TMK panels);
                                                             # more than 32 * SMs rows: grid-stride pointwise rows
    ("h64_l8_state", 64, 8, 3, 1, 3, 50, True, True),        # kMaxLayers on the forced exact path
    ("h64_t70_b2100", 64, 2, 70, 1, 2, 2100, False, False),  # T > 64 routes H = 64 here; b_inner > 2048: global d_s
    ("h32_t1_state", 32, 1, 1, 1, 5, 9, True, False),        # T = 1: the backward's first step is also t = 0
    ("saturated", 64, 3, 20, 1, 11, 40, True, True),         # gate pre-activations to +-60, c to +-20
]

# exact-fp32 LSTM with the input and state gradients: (name, H, L, T, C, regions N, batch B, initial state)
EXACT_CASES = [("h16_c1", 16, 2, 5, 1, 7, 5, False),
               ("h48_c3_state", 48, 3, 6, 3, 9, 4, True),
               ("h128_l8_c4_state", 128, 8, 3, 4, 3, 11, True),
               ("h48_t1_c2", 48, 1, 1, 2, 5, 3, False)]

FORGET_BIAS = 3.0           # long-memory cases: added to b_ih's forget-gate rows [H, 2H)
PREMISE = 1e-2              # long-memory cases: max|d_s[:, 0]| / max|d_s| of the reference at least this

# per-step checks, tensor cores: (name, regions N (None: multi-wave, from the SM count), batch B, T, layers L,
# channels C, initial state, long memory)
TC_CASES = ([(name, n, b, t, lyr, c, state, False) for name, n, b, t, lyr, c, state in CASES]
            + [("chain_" + name, None, b, 64, 2, c, state, False) for name, b, c, state in CHAIN_CASES]
            + [("long_waves_b64", None, 64, 64, 2, 1, False, True),        # several tiles per CTA
               ("long_t64_l1_c4_state", 3, 43, 64, 1, 4, True, True),
               ("long_l3_c3_b37_state", 7, 37, 64, 3, 3, True, True)])     # 259 rows: a ragged third tile
# per-step checks, exact fp32: (name, H, L, T, C, regions N (None: multi-wave), batch B, initial state, long memory)
EXACT = ([(name, hid, lyr, t, c, n, b, state, False) for name, hid, lyr, t, c, n, b, state, _ in LSTM_CASES]
         + [(name, hid, lyr, t, c, n, b, state, False) for name, hid, lyr, t, c, n, b, state in EXACT_CASES]
         + [("long_h64_t70_b2100", 64, 2, 70, 1, 2, 2100, False, True),   # b_inner > 2048: d_s atomics in global memory
            ("long_h48_t40_state", 48, 3, 40, 2, 9, 20, True, True)])


# ======================================================================================================================
# inputs
# ======================================================================================================================
def lstm16_inputs(n, b, t, lyr, c, state, seed, saturate=False, device=DEV):
    """Seeded inputs of the tensor-core LSTM (H = 64): xo (N,B,T,C), s (B,T), h0 / c0 (L,R,H) or None, nn.LSTM
    parameters, d_top (R,H).

    ``saturate``: the terms the kernels add with fp32 FMAs drive the gates into saturation -- inputs x3 and layer 0's
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


def lstm_inputs(n, b, t, lyr, c, hid, state, seed, saturate=False):
    """Seeded CPU inputs of the exact-fp32 LSTM: xo (N,B,T,C), s (B,T), h0 / c0 (L,R,H) or None, nn.LSTM parameters,
    d_top (R,H).

    ``saturate``: inputs x4, weights in +-2 and biases i +10, f +20, g +-15 (one sign per unit), so the gate
    pre-activations reach about +-60 and c about +-T, while about a third of the pre-activations stay within +-8."""
    gen = torch.Generator().manual_seed(seed)
    xo = torch.randn(n, b, t, c, generator=gen) * (4.0 if saturate else 1.0)
    s = 0.2 + 0.8 * torch.rand(b, t, generator=gen)
    amp = 4.0 if saturate else 0.5
    ws = []
    for l in range(lyr):
        in_l = c if l == 0 else hid
        w_ih = (torch.rand(4 * hid, in_l, generator=gen) - 0.5) * amp
        w_hh = (torch.rand(4 * hid, hid, generator=gen) - 0.5) * amp
        b_ih = (torch.rand(4 * hid, generator=gen) - 0.5) * 0.5
        b_hh = (torch.rand(4 * hid, generator=gen) - 0.5) * 0.5
        if saturate:
            b_ih = torch.zeros(4 * hid)
            b_ih[:hid], b_ih[hid:2 * hid] = 10.0, 20.0
            b_ih[2 * hid:3 * hid] = 15.0 * torch.sign(torch.randn(hid, generator=gen))
            b_hh = torch.zeros(4 * hid)
        ws += [w_ih, w_hh, b_ih, b_hh]
    h0 = c0 = None
    if state:
        h0 = torch.randn(lyr, n * b, hid, generator=gen) * 0.3
        c0 = torch.randn(lyr, n * b, hid, generator=gen) * 0.5
    d_top = torch.randn(n * b, hid, generator=gen)
    return xo, s, h0, c0, ws, d_top


def seeds(lyr, rows, hid, seed):
    """Seeded dh_n / dc_n (L,R,H) on the device."""
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(lyr, rows, hid, generator=gen).to(DEV), torch.randn(lyr, rows, hid, generator=gen).to(DEV))


def with_long_memory(ws, hid):
    """``ws`` with FORGET_BIAS added to every layer's forget-gate rows of b_ih (in place), so every step carries weight
    in the summed gradients."""
    for l in range(len(ws) // 4):
        ws[4 * l + 2][hid:2 * hid] += FORGET_BIAS
    return ws


# ======================================================================================================================
# the tape-forced fp64 reference
# ======================================================================================================================
def reference(xo, s, h0, c0, ws, lyr, planes, tape, grad=True, state_leaves=False):
    """``O.lstm_planes_reference`` in fp64 on the device, forced with ``tape`` (None: free-running) -> (hs, cs, layers,
    leaves).  With two planes its arithmetic is ``O.lstm_explicit``'s.  ``layers`` are the fp64 LSTM parameters and
    ``leaves`` the fp64 s; both are autograd leaves when ``grad``.

    ``state_leaves``: xo, h0 and c0 are leaves too, a missing h0 / c0 becoming a zero leaf (the gradient at a zero
    initial state, which ``tape`` then starts from unless it has its own h0), and ``leaves`` is (xo, s, h0, c0).
    Without it a missing h0 / c0 is passed on as None."""
    n, b, t, c = xo.shape
    rows = n * b
    with torch.set_grad_enabled(grad):
        xo64 = xo.double().requires_grad_(grad and state_leaves)
        s64 = s.double().requires_grad_(grad)
        if state_leaves:
            hid = ws[1].shape[1]
            h0d = (h0.double() if h0 is not None else xo64.new_zeros(lyr, rows, hid)).requires_grad_(grad)
            c0d = (c0.double() if c0 is not None else xo64.new_zeros(lyr, rows, hid)).requires_grad_(grad)
            tape = dict(tape)
            if "h0" not in tape:
                tape["h0"] = h0d.detach()
        else:
            h0d = None if h0 is None else h0.double()
            c0d = None if c0 is None else c0.double()
        layers = [tuple(w.double().requires_grad_(grad) for w in ws[4 * l:4 * l + 4]) for l in range(lyr)]
        x = xo64.reshape(rows, t, c) * s64.repeat(n, 1)[:, :, None]           # row r = n * B + b -> s[b]
        _, _, (hs, cs) = O.lstm_planes_reference(x, layers, planes, h0d, c0d, tape)
        return hs, cs, layers, ((xo64, s64, h0d, c0d) if state_leaves else s64)


def state_gradients(xo, s, h0, c0, ws, lyr, planes, tape, d_top, dh_n, dc_n):
    """The tape-forced reference's gradients of <h_top, d_top> + <h_n, dh_n> + <c_n, dc_n> (dh_n / dc_n may be None)
    with respect to xo, s, h0, c0 (zeros when None) and the weights, as a dict."""
    hs, cs, layers, leaves = reference(xo, s, h0, c0, ws, lyr, planes, tape, state_leaves=True)
    loss = (hs[-1][-1] * d_top.double()).sum()
    if dh_n is not None:
        loss = loss + sum((hs[l][-1] * dh_n[l].double()).sum() for l in range(lyr))
    if dc_n is not None:
        loss = loss + sum((cs[l][-1] * dc_n[l].double()).sum() for l in range(lyr))
    flat = [w for layer in layers for w in layer]
    g = torch.autograd.grad(loss, list(leaves) + flat)
    return dict(d_xo=g[0], d_s=g[1], dh0=g[2], dc0=g[3], params=list(g[4:]))


def grad_errors(got, ref):
    """Max-norm errors of d_xo, d_s, dh0, dc0 and every weight gradient (``param i``)."""
    errs = {k: rel_err(got[k], ref[k]) for k in ("d_xo", "d_s", "dh0", "dc0")}
    errs.update({f"param {i}": rel_err(a, r) for i, (a, r) in enumerate(zip(got["params"], ref["params"]))})
    return errs


def _half_ulp_bf16(v):
    _, e = torch.frexp(v)                     # |v| = m 2^e, m in [0.5, 1): bf16 keeps 8 significant bits
    return torch.ldexp(torch.ones_like(v), e - 9)


def step_local_error(ktape, hs, cs, planes=2):
    """Max over every (layer, step) of the cell-state error and the hidden-state error.  Two planes: hi + lo against the
    reference h; one plane: the excess of |hi - h| over half a bf16 ulp of h (hi is h rounded to bf16)."""
    worst = 0.0
    for l in range(len(hs)):
        for t in range(len(hs[l])):
            h_ref, c_ref = hs[l][t].detach(), cs[l][t].detach()
            worst = max(worst, rel_err(ktape["c"][l, t], c_ref))
            hk = ktape["h"][l, t]
            if planes == 2:
                worst = max(worst, rel_err(hk, h_ref))
            else:
                excess = ((hk - h_ref).abs() - _half_ulp_bf16(h_ref)).clamp_min(0)
                worst = max(worst, float(excess.max()) / max(float(h_ref.abs().max()), 1e-30))
    return worst


# ======================================================================================================================
# kernel runners
# ======================================================================================================================
def kernel_tape(tape, rows, state):
    """The tensor-core forward's tape as the reference takes it, in fp64: h (planes summed), c (unblocked) and, with an
    initial ``state``, h0 (planes summed)."""
    from stmgcn_b200 import ops
    ktape = dict(h=tape["hp"].double().sum(dim=2), c=ops.from_blocked(tape["cs"], rows).double())
    if state:
        ktape["h0"] = tape["h0p"].double().sum(dim=1)
    return ktape


def lstm16_kernel(xo, s, h0, c0, ws, lyr, planes, d_top):
    """Tensor-core forward and backward through the plain entry points -> (h_top, (h_n, c_n) or None, tape, d_s,
    weight gradients)."""
    from stmgcn_b200 import ops
    n, b, t, c = xo.shape
    rows = n * b
    state = h0 is not None
    h_top, h_n, c_n, tape = ops._lstm16_forward(xo, s, h0, c0, lyr, state, ws, planes, True)
    d_s, grads = ops._lstm16_backward(xo, s, tape, lyr, planes, d_top)
    torch.cuda.synchronize()
    return h_top.reshape(rows, HID), (h_n, c_n) if state else None, kernel_tape(tape, rows, state), d_s, grads


def lstm16_run(xo, s, h0, c0, ws, lyr, planes, d_top, dh_n, dc_n):
    """Tensor-core forward and the _ex backward with every extra wanted -> (gradients dict, tape for the reference,
    the forward's tape)."""
    from stmgcn_b200 import ops
    rows = xo.shape[0] * xo.shape[1]
    _, _, _, tape = ops._lstm16_forward(xo, s, h0, c0, lyr, h0 is not None, ws, planes, True)
    d_s, grads, (d_xo, dh0, dc0) = ops._lstm16_backward_ex(xo, s, tape, lyr, planes, d_top, dh_n, dc_n, (True, True, True))
    torch.cuda.synchronize()
    return dict(d_xo=d_xo, d_s=d_s, dh0=dh0, dc0=dc0, params=grads), kernel_tape(tape, rows, h0 is not None), tape


def exact_run(xo, s, h0, c0, ws, lyr, hid, d_top, dh_n, dc_n):
    """Exact-fp32 forward and the _ex backward with every extra wanted -> (gradients dict, tape for the reference)."""
    from stmgcn_b200 import ops
    _, _, _, tape = ops._exact_forward(xo, s, h0, c0, lyr, hid, True, ws, True)
    ktape = dict(h=tape[2].double(), c=tape[3].double())
    if h0 is not None:
        ktape["h0"] = h0.double()
    d_s, grads, (d_xo, dh0, dc0) = ops._exact_backward_ex(xo, s, tape, lyr, hid, d_top, dh_n, dc_n, (True, True, True))
    torch.cuda.synchronize()
    return dict(d_xo=d_xo, d_s=d_s, dh0=dh0, dc0=dc0, params=grads), ktape
