"""Harness of the C ABI's caller-memory and stream contract (include/stmgcn_b200.h), and the calls that drive it.

A ``Buf`` is one caller buffer: a view into a larger allocation with GUARD bytes of sentinel before and after it.  A
``Call`` is one entry-point call on such buffers, with its fp64 reference and its launch count.  ``run_contract`` runs a
call clean, poisoned twice and with pre-filled accumulators; ``run_captured`` runs it eagerly on a side stream and from a
captured CUDA graph.  The ``*_calls`` generators yield the calls of one entry-point family in order, each receiving the
clean results of the one before; ``drive`` feeds them to a runner.  test_gpu_abi_contract.py states the contract and
holds the tests of the harness itself.

The calls go through ``lib()`` and ``ops`` at call time, never through names bound at import.
"""
import math

import torch

from helpers import DEV, FWD_TOL, GRAD_TOL, lib, rel_err
from kernel_cases import fuse_rows, proj_inputs, proj_ref_out
from lstm_cases import (HID, kernel_tape, lstm16_inputs, lstm_inputs, reference, grad_errors, seeds, state_gradients,
                        step_local_error, wave_regions)


GUARD = 64 * 1024                                   # bytes of sentinel on each side of a buffer


SENTINEL = {torch.float32: 0x7FA5A5A5, torch.bfloat16: 0x7FA5}


_INT = {4: torch.int32, 2: torch.int16, 1: torch.uint8}


POISON = ("nan", "big")


RESULTS = ("out", "out0", "inout", "acc")


def bits(x):
    return x.contiguous().view(_INT[x.element_size()])


def _poison(v, mode, seed):
    if mode == "nan":
        v.view(_INT[v.element_size()]).fill_(-1)                 # every byte 0xFF: NaN in fp32 and bf16
    else:
        gen = torch.Generator(device=v.device).manual_seed(seed)
        v.copy_(((torch.rand(v.shape, generator=gen, device=v.device) * 2 - 1) * 1e4).to(v.dtype))


class Buf:
    """One caller buffer ``t`` inside ``raw``, GUARD sentinel bytes on each side.  Roles: ``in`` (const input),
    ``inout`` (input the call overwrites), ``out`` (overwritten output), ``out0`` (output the caller zero-fills), ``acc``
    (+= output, caller zeroes), ``ws`` (workspace needing no initialisation), ``keep`` (a buffer the call is given but
    must not write).  ``part`` extracts the meaningful part of a result, ``keep`` lists the regions of an output the call
    must leave as they were, ``pad`` the padding regions of an input that are filled with poison too.  ``exact``: the
    output has no atomics (bit-identical across runs); ``finite``: every value of a result must be finite."""

    def __init__(self, role, init=None, shape=None, dtype=torch.float32, device=DEV, guard=None, exact=True, finite=True,
                 part=None, keep=None, pad=None):
        if init is not None:
            shape, dtype = init.shape, init.dtype
        self.role, self.exact, self.finite = role, exact, finite
        self.part = part or (lambda t: t)
        self.keep = keep or (lambda t: [])
        self.pad = pad or (lambda t: [])
        item = torch.empty(0, dtype=dtype).element_size()
        self.nbytes = math.prod(shape) * item
        self.raw = torch.empty(2 * GUARD + -(-self.nbytes // 512) * 512, dtype=torch.uint8, device=device)
        self.guard, self._gint = (SENTINEL[dtype] if guard is None else guard), _INT[item]
        self.raw.view(self._gint).fill_(self.guard)
        self.t = self.raw[GUARD:GUARD + self.nbytes].view(dtype).view(tuple(shape))
        self.init = None if init is None else init.to(self.t.device)
        if self.init is not None:
            self.t.copy_(self.init)
        self.acc_init = None

    @property
    def p(self):
        return self.t.data_ptr()

    def prepare(self, mode, seed):
        """Fill for a ``clean`` / ``nan`` / ``big`` / ``acc`` run; returns the snapshot the call must leave unchanged."""
        if self.role in ("in", "inout"):
            self.t.copy_(self.init)
            if mode in POISON:
                for i, v in enumerate(self.pad(self.t)):
                    _poison(v, mode, seed + i)
        elif self.role in ("out", "ws", "keep") and mode in POISON:
            _poison(self.t, mode, seed)
        elif self.role == "acc" and mode == "acc":
            self.t.copy_(self.acc_init)
        else:
            self.t.zero_()
        return [v.clone() for v in self._fixed()]

    def _fixed(self):
        return [self.t] if self.role in ("in", "keep") else self.keep(self.t)

    def unchanged(self, snap):
        return all(torch.equal(bits(a), bits(b)) for a, b in zip(self._fixed(), snap))

    def guards_intact(self):
        head = self.raw[:GUARD].view(self._gint)
        tail = self.raw[GUARD + self.nbytes:].view(self._gint)
        return bool((head == self.guard).all()) and bool((tail == self.guard).all())

    def result(self):
        return self.part(self.t).clone()


class Call:
    """One entry-point call: ``launch(stream)`` returns the library's rc; ``reference(results)`` asserts the clean run's
    results against fp64; ``launches``: kernels the call enqueues."""

    def __init__(self, name, bufs, launch, reference=None, launches=None):
        self.name, self.bufs, self.launch, self.reference, self.launches = name, bufs, launch, reference, launches
        self.cuda = next(iter(bufs.values())).t.is_cuda


def cuda_stream():
    return torch.cuda.current_stream().cuda_stream


def _same(call, name, got, want, what):
    buf = call.bufs[name]
    if buf.finite:
        assert bool(torch.isfinite(got).all()), f"{call.name} ({what}): {name} is not finite"
    if buf.exact and buf.role != "acc":
        assert torch.equal(bits(got), bits(want)), f"{call.name} ({what}): {name} differs from the clean run"
    else:
        err = rel_err(got, want)
        assert err <= GRAD_TOL, f"{call.name} ({what}): {name} is {err:.2e} off the clean run"


def run_once(call, mode):
    snaps = {k: b.prepare(mode, 101 * i) for i, (k, b) in enumerate(call.bufs.items())}
    n0 = lib().stmgcn_launch_count() if call.cuda else 0
    rc = call.launch(cuda_stream() if call.cuda else None)
    if call.cuda:
        torch.cuda.synchronize()
        assert rc == 0, f"{call.name} ({mode} run): rc={rc}: {lib().stmgcn_last_error()}"
        if call.launches is not None:
            got = lib().stmgcn_launch_count() - n0
            assert got == call.launches, f"{call.name} ({mode} run): {got} launches, expected {call.launches}"
    for k, b in call.bufs.items():
        assert b.guards_intact(), f"{call.name} ({mode} run): a guard band of {k} changed"
        assert b.unchanged(snaps[k]), f"{call.name} ({mode} run): {k} changed where the call must not write"
    return {k: b.result() for k, b in call.bufs.items() if b.role in RESULTS}


def run_contract(call):
    """Clean run against the reference, two poisoned runs, one run with pre-filled accumulators; returns the clean
    results (the inputs of the calls that follow)."""
    clean = run_once(call, "clean")
    if call.reference is not None:
        call.reference(clean)
    for mode in POISON:
        for k, v in run_once(call, mode).items():
            _same(call, k, v, clean[k], f"{mode}-poisoned run")
    accs = [k for k, b in call.bufs.items() if b.role == "acc"]
    if accs:
        gen = torch.Generator().manual_seed(7)
        for k in accs:
            c = clean[k]
            scale = float(c.abs().max()) or 1.0
            call.bufs[k].acc_init = ((torch.rand(c.shape, generator=gen) * 2 - 1) * scale).to(c.device)
        got = run_once(call, "acc")
        for k, v in got.items():
            if k in accs:
                err = rel_err(v.double() - call.bufs[k].acc_init.double(), clean[k])
                assert err <= GRAD_TOL, f"{call.name}: {k} started at V ends {err:.2e} away from V + the clean result (+=)"
            else:
                _same(call, k, v, clean[k], "run with pre-filled accumulators")
    return clean


def run_captured(call):
    """One eager call on a side stream, then the same call captured into a CUDA graph and replayed: the replay's results
    equal the eager ones (bit for bit without atomics, within the gradient bar for sums of atomics)."""
    def prep():
        for i, b in enumerate(call.bufs.values()):
            b.prepare("clean", i)

    def results():
        return {k: b.result() for k, b in call.bufs.items() if b.role in RESULTS}

    prep()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        rc = call.launch(side.cuda_stream)
    torch.cuda.synchronize()
    assert rc == 0, f"{call.name} (eager on a side stream): rc={rc}: {lib().stmgcn_last_error()}"
    eager = results()
    prep()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="global"):
        rc = call.launch(cuda_stream())
    assert rc == 0, f"{call.name} (captured): rc={rc}: {lib().stmgcn_last_error()}"
    prep()
    graph.replay()
    torch.cuda.synchronize()
    for k, v in results().items():
        _same(call, k, v, eager[k], "graph replay")
    for k, b in call.bufs.items():
        assert b.guards_intact(), f"{call.name} (graph replay): a guard band of {k} changed"
    return eager


def drive(calls, runner):
    """Run a generator of Calls; each receives the results of the one before (a forward's outputs feed its backward)."""
    try:
        call = next(calls)
        while True:
            call = calls.send(runner(call))
    except StopIteration:
        pass


def _tf32_image(bmat, tile_rows):
    """stmgcn_proj_pack_tc's image of a logical B[n][k]: per 32-wide k-block a hi and a lo [tile_rows][32] fp32 tile,
    element (n, k) at its 128-byte-swizzle offset, hi = the value with its low 13 mantissa bits cleared and lo = the
    rest, cleared likewise (tc_common.cuh); rows past n_rows zero."""
    n_rows, k_cols = bmat.shape
    v = bmat.float().contiguous()
    hi = (v.view(torch.int32) & -8192).view(torch.float32)
    lo = ((v - hi).view(torch.int32) & -8192).view(torch.float32)
    n = torch.arange(n_rows, device=v.device).view(-1, 1).expand(n_rows, k_cols)
    k = torch.arange(k_cols, device=v.device).view(1, -1).expand(n_rows, k_cols)
    tile = tile_rows * 32
    idx = (k // 32) * 2 * tile + n * 32 + (((k % 32) // 4) ^ (n % 8)) * 4 + k % 4
    img = torch.zeros(k_cols // 32 * 2 * tile, device=v.device)
    img[idx.reshape(-1)] = hi.reshape(-1)
    img[(idx + tile).reshape(-1)] = lo.reshape(-1)
    return img


def proj_calls(ks, p, q, n, b_sz, gap, tc, bcast, relu, bias, seed):
    """stmgcn_proj_pack_tc (``tc``: into a NaN-filled img_fwd and a zero-filled img_bwd), stmgcn_proj_fwd and
    stmgcn_proj_bwd on a stack whose segments lie rows*p + gap floats apart, the gaps NaN; U is written with the same
    stride and its gaps must stay untouched.  ``bcast``: the temporal GCN's gate pooling forward and broadcast backward."""
    rows = n * b_sz
    s, w, bv, d_out = proj_inputs(ks, p, q, rows, relu, bias, seed)
    sk = rows * p + gap
    stack = torch.full((ks * sk,), float("nan"))
    for k in range(ks):
        stack[k * sk:k * sk + rows * p] = s[k].reshape(-1)
    act = 1 if relu else 0
    s64, w64 = s.double().to(DEV), w.double().to(DEV)
    b64 = None if bv is None else bv.double().to(DEV)
    ref_out = proj_ref_out(s64, w64, b64, relu)
    what = f"ks={ks} p={p} q={q} rows={rows} gap={gap}"
    img_f = img_b = None
    if tc:
        n_bwd = 2 if ks > 4 else 1
        b = dict(w=Buf("in", w), img_fwd=Buf("out", shape=(ks * 64 * 64 * 2,)),
                 img_bwd=Buf("out0", shape=(n_bwd * 2 * 2 * 256 * 32,)))

        def ref_pack(res):
            wd = w.to(DEV)
            assert torch.equal(bits(res["img_fwd"]), bits(_tf32_image(wd.t(), 64))), f"forward image, {what}"
            want = torch.cat([_tf32_image(wd[g * 256:(g + 1) * 256], 256) for g in range(n_bwd)])
            assert torch.equal(bits(res["img_bwd"]), bits(want)), f"backward image, {what}"

        got = yield Call("proj_pack_tc", b, lambda st, b=b: lib().stmgcn_proj_pack_tc(
            b["w"].p, ks, b["img_fwd"].p, b["img_bwd"].p, st), ref_pack, 1 + n_bwd)
        img_f, img_b = got["img_fwd"], got["img_bwd"]

    b = dict(s=Buf("in", stack), w=Buf("in", w), out=Buf("out", shape=(rows, q)))
    if bias:
        b["bias"] = Buf("in", bv)
    if bcast:
        b["pool"] = Buf("acc", shape=(b_sz, q))
    if tc:
        b["wimg"] = Buf("in", img_f)
    opt = lambda b, k: b[k].p if k in b else None      # noqa: E731

    def ref_fwd(res):
        errs = {"out": rel_err(res["out"], ref_out)}
        if bcast:
            errs["pool"] = rel_err(res["pool"], (s64[0] + ref_out).view(n, b_sz, q).sum(0))
        assert max(errs.values()) <= FWD_TOL, f"proj_fwd {what}: {errs}"

    got = yield Call("proj_fwd", b, lambda st, b=b: lib().stmgcn_proj_fwd(
        b["s"].p, sk, ks, rows, p, b["w"].p, opt(b, "bias"), q, act, b["out"].p, opt(b, "pool"), b_sz, opt(b, "wimg"), st),
        ref_fwd, 2 if bcast else 1)
    out_k = got["out"]

    gen = torch.Generator().manual_seed(seed + 1)
    d_b = torch.randn(b_sz, q, generator=gen)
    scale = 0.37 if bcast else 1.0
    b = dict(s=Buf("in", stack), wt=Buf("in", w.t().contiguous()), out=Buf("in", out_k), dz=Buf("out", shape=(rows, q)),
             dw=Buf("acc", shape=(ks * p, q)),
             u=Buf("out", shape=(ks * sk,), part=lambda t: torch.stack([t[k * sk:k * sk + rows * p] for k in range(ks)]),
                   keep=lambda t: [t[k * sk + rows * p:(k + 1) * sk] for k in range(ks)]))
    b["d_bcast" if bcast else "d_out"] = Buf("in", d_b if bcast else d_out)
    if bias:
        b["db"] = Buf("acc", shape=(q,))
    if tc:
        b["wimg_t"] = Buf("in", img_b)
    # the tensor-core backward: p = q = 64, weight image, full d_out and 16-byte aligned segments; else dz, dW and U
    on_tc = tc and not bcast and gap % 4 == 0
    dz = (d_b.repeat(n, 1) * scale if bcast else d_out).double().to(DEV)
    if relu:
        dz = dz * (out_k > 0)

    def ref_bwd(res):
        errs = {"dz": rel_err(res["dz"], dz), "dW": rel_err(res["dw"], torch.einsum("krp,rq->kpq", s64, dz).reshape(ks * p, q)),
                "U": rel_err(res["u"], torch.einsum("rq,kpq->krp", dz, w64.reshape(ks, p, q)).reshape(ks, -1))}
        if bias:
            errs["db"] = rel_err(res["db"], dz.sum(0))
        assert max(errs.values()) <= GRAD_TOL, f"proj_bwd {what}: {errs}"

    yield Call("proj_bwd", b, lambda st, b=b: lib().stmgcn_proj_bwd(
        b["s"].p, sk, ks, rows, p, b["wt"].p, q, act, b["out"].p, opt(b, "d_out"), opt(b, "d_bcast"), scale, b_sz, b["dz"].p,
        b["dw"].p, opt(b, "db"), b["u"].p, sk, opt(b, "wimg_t"), st),
        ref_bwd, ((2 if ks > 4 else 1) + (ks + 1) // 2) if on_tc else 3)


def gate_calls(t, b_sz):
    n_regions = 50
    gen = torch.Generator().manual_seed(t + b_sz)
    pool = torch.randn(b_sz, t, generator=gen) * n_regions
    fcw = torch.randn(t, t, generator=gen) / t ** 0.5
    fcb = torch.rand(t, generator=gen) - 0.5
    d_s = torch.randn(b_sz, t, generator=gen)
    p64, w64, b64 = (v.double().to(DEV) for v in (pool, fcw, fcb))
    b = dict(pool=Buf("in", pool), fcw=Buf("in", fcw), fcb=Buf("in", fcb), z=Buf("out", shape=(b_sz, t)),
             a1=Buf("out", shape=(b_sz, t)), s=Buf("out", shape=(b_sz, t)))

    def ref_fwd(res):
        a1 = (p64 / n_regions) @ w64.t() + b64
        errs = {"z": rel_err(res["z"], p64 / n_regions), "a1": rel_err(res["a1"], a1),
                "s": rel_err(res["s"], torch.sigmoid(a1.clamp_min(0) @ w64.t() + b64))}
        assert max(errs.values()) <= FWD_TOL, f"gate_fwd T={t}: {errs}"

    got = yield Call("gate_fwd", b, lambda st: lib().stmgcn_gate_fwd(
        b["pool"].p, b_sz, t, n_regions, b["fcw"].p, b["fcb"].p, b["z"].p, b["a1"].p, b["s"].p, st), ref_fwd, 1)
    c = dict(d_s=Buf("in", d_s), z=Buf("in", got["z"]), a1=Buf("in", got["a1"]), s=Buf("in", got["s"]),
             fcw=Buf("in", fcw), d_fcw=Buf("acc", shape=(t, t)), d_fcb=Buf("acc", shape=(t,)), d_z=Buf("out", shape=(b_sz, t)))

    def ref_bwd(res):
        z64 = got["z"].double().requires_grad_(True)
        wg, bg = w64.clone().requires_grad_(True), b64.clone().requires_grad_(True)
        a1 = z64 @ wg.t() + bg
        s = torch.sigmoid((a1 * (got["a1"] > 0)) @ wg.t() + bg)              # the kernel's own ReLU mask
        g = torch.autograd.grad((s * d_s.double().to(DEV)).sum(), [z64, wg, bg])
        errs = {"d_z": rel_err(res["d_z"], g[0]), "d_fcw": rel_err(res["d_fcw"], g[1]), "d_fcb": rel_err(res["d_fcb"], g[2])}
        assert max(errs.values()) <= GRAD_TOL, f"gate_bwd T={t}: {errs}"

    yield Call("gate_bwd", c, lambda st: lib().stmgcn_gate_bwd(
        c["d_s"].p, c["z"].p, c["a1"].p, c["s"].p, b_sz, t, c["fcw"].p, c["d_fcw"].p, c["d_fcb"].p, c["d_z"].p, st), ref_bwd, 1)


def lstm_calls(n, b_sz, state):
    """H = 48, L = 3, T = 5, C = 2.  The backward's workspaces dh_rec, dc and dx_work are poisoned: the step t = T-1
    must not read them."""
    from stmgcn_b200 import ops
    hid, lyr, t, c = 48, 3, 5, 2
    rows = n * b_sz
    xo, s, h0, c0, ws, d_top = (None if v is None else v.to(DEV) if torch.is_tensor(v) else [w.to(DEV) for w in v]
                                for v in lstm_inputs(n, b_sz, t, lyr, c, hid, state, seed=rows))
    wx, wp, bp, wpt = ops._pack_lstm(ws, lyr, hid)
    b = dict(xo=Buf("in", xo), s=Buf("in", s), wx=Buf("in", wx), wp=Buf("in", wp), bp=Buf("in", bp),
             hs=Buf("out", shape=(lyr, t, rows, hid)), cs=Buf("out", shape=(lyr, t, rows, hid)),
             gates=Buf("out", shape=(lyr, t, rows, 4 * hid)))
    if state:
        b.update(h0=Buf("in", h0), c0=Buf("in", c0))
    opt = lambda b, k: b[k].p if k in b else None      # noqa: E731

    def tape(res):
        tp = dict(h=res["hs"].double(), c=res["cs"].double())
        if state:
            tp["h0"] = h0.double()
        return tp

    def ref_fwd(res):
        hs, cs, _, _ = reference(xo, s, h0, c0, ws, lyr, 2, tape(res), grad=False)
        err = step_local_error(tape(res), hs, cs)
        assert err <= FWD_TOL, f"lstm_fwd rows={rows}: step-local {err:.2e}"

    got = yield Call("lstm_fwd", b, lambda st: lib().stmgcn_lstm_fwd(
        t, lyr, rows, hid, c, b_sz, b["xo"].p, b["s"].p, b["wx"].p, b["wp"].p, b["bp"].p, opt(b, "h0"), opt(b, "c0"),
        b["hs"].p, b["cs"].p, b["gates"].p, st), ref_fwd, lyr * t)

    c_ = dict(xo=Buf("in", xo), s=Buf("in", s), wx=Buf("in", wx), wpt=Buf("in", wpt), cs=Buf("in", got["cs"]),
              hs=Buf("in", got["hs"]), gates=Buf("inout", got["gates"]), d_top=Buf("in", d_top),
              dh_rec=Buf("ws", shape=(lyr, rows, hid)), dc=Buf("ws", shape=(lyr, rows, hid)), dx_work=Buf("ws", shape=(rows, hid)),
              d_s=Buf("acc", shape=(b_sz, t)), dwx=Buf("acc", shape=wx.shape), dwp=Buf("acc", shape=wp.shape),
              dbp=Buf("acc", shape=bp.shape))
    if state:
        c_.update(h0=Buf("in", h0), c0=Buf("in", c0))

    def ref_bwd(res):
        hs, _, layers, s64 = reference(xo, s, h0, c0, ws, lyr, 2, tape(got))
        ref = torch.autograd.grad((hs[-1][-1] * d_top.double()).sum(), [s64] + [w for layer in layers for w in layer])
        grads = ops._unpack_lstm_grads(res["dwx"], res["dwp"], res["dbp"], lyr, hid, c)
        errs = {"d_s": rel_err(res["d_s"], ref[0])}
        errs.update({f"param {i}": rel_err(g, r) for i, (g, r) in enumerate(zip(grads, ref[1:]))})
        assert max(errs.values()) <= GRAD_TOL, f"lstm_bwd rows={rows}: {errs}"

    yield Call("lstm_bwd", c_, lambda st: lib().stmgcn_lstm_bwd(
        t, lyr, rows, hid, c, b_sz, c_["xo"].p, c_["s"].p, c_["wx"].p, c_["wpt"].p, opt(c_, "h0"), opt(c_, "c0"), c_["cs"].p,
        c_["hs"].p, c_["gates"].p, c_["d_top"].p, c_["dh_rec"].p, c_["dc"].p, c_["dx_work"].p, c_["d_s"].p, c_["dwx"].p,
        c_["dwp"].p, c_["dbp"].p, st), ref_bwd, 2 * lyr * t + lyr)


def blocked_pads(t, rows):
    """The padding rows rows .. R_pad-1 of a tile-blocked (..., R_pad, 64) tensor, as a view."""
    if rows % 128 == 0:
        return []
    *lead, rp, h = t.shape
    return [t.view(*lead, rp // 128, 16, 128, 4)[..., -1, :, rows % 128:, :]]


# (name, regions N (None: multi-wave), batch B, T, layers L, channels C, initial state)
LSTM16_CASES = [("one_row", 1, 1, 3, 2, 1, False),
                ("l1_no_dx_work", 3, 43, 4, 1, 1, False),
                ("c3_l4_state", 5, 60, 5, 4, 3, True),
                ("waves_b37_state", None, 37, 4, 2, 2, True)]


def lstm16_calls(case, planes):
    """stmgcn_lstm16_pack layer by layer into a NaN-filled image (the other layers' slots must stay untouched), then the
    forward (with h_n given, a separate h_top must stay untouched) and the backward with every workspace poisoned and
    the padding rows of c0 and d_top poisoned; hp and cs must come out of the backward bit-identical."""
    from stmgcn_b200 import ops
    name, n, b_sz, t, lyr, c, state = case
    if n is None:
        n = wave_regions(b_sz)
    rows = n * b_sz
    rp = -(-rows // 128) * 128
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n, b_sz, t, lyr, c, state, seed=20 * LSTM16_CASES.index(case) + planes)
    what = f"{name} P={planes} rows={rows}"
    slot = lambda l: (0, 32768) if l == 0 else (32768 * (2 * l - 1), 65536)      # noqa: E731  (bf16 elements)
    wimg_n = 32768 * (2 * lyr - 1)
    wimg, bias, wih_t = torch.empty(wimg_n, dtype=torch.bfloat16, device=DEV), torch.empty(lyr, 256, device=DEV), None
    for l in range(lyr):
        o, m = slot(l)
        b = dict(w_ih=Buf("in", ws[4 * l]), w_hh=Buf("in", ws[4 * l + 1]), b_ih=Buf("in", ws[4 * l + 2]),
                 b_hh=Buf("in", ws[4 * l + 3]),
                 wimg=Buf("out", shape=(wimg_n,), dtype=torch.bfloat16, part=lambda v, o=o, m=m: v[o:o + m],
                          keep=lambda v, o=o, m=m: [v[:o], v[o + m:]]),
                 bias=Buf("out", shape=(lyr, 256), part=lambda v, l=l: v[l], keep=lambda v, l=l: [v[:l], v[l + 1:]]),
                 wih_t=Buf("out" if l == 0 else "keep", shape=(c, 256)))
        got = yield Call(f"lstm16_pack layer {l}", b, lambda st, b=b, l=l: lib().stmgcn_lstm16_pack(
            b["w_ih"].p, b["w_hh"].p, b["b_ih"].p, b["b_hh"].p, l, c, b["wimg"].p, b["bias"].p, b["wih_t"].p, st), None, 1)
        wimg[o:o + m], bias[l] = got["wimg"], got["bias"]
        wih_t = got["wih_t"] if l == 0 else wih_t

    pads = lambda v: blocked_pads(v, rows)      # noqa: E731
    h0p = ops.to_planes(h0, planes) if state else None
    common = lambda: dict(xo=Buf("in", xo), s=Buf("in", s), wimg=Buf("in", wimg), bias=Buf("in", bias),     # noqa: E731
                          wih_t=Buf("in", wih_t),
                          **(dict(h0p=Buf("in", h0p), c0=Buf("in", ops.to_blocked(c0), pad=pads)) if state else {}))
    b = dict(common(), hp=Buf("out", shape=(lyr, t, planes, rows, 64), dtype=torch.bfloat16),
             cs=Buf("out", shape=(lyr, t, rp, 64), part=lambda v: ops.from_blocked(v, rows)),
             h_top=Buf("keep" if state else "out", shape=(rows, 64)))
    if state:
        b["h_n"] = Buf("out", shape=(lyr, rows, 64))
    opt = lambda b, k: b[k].p if k in b else None      # noqa: E731

    def tape(res):
        tp = dict(h=res["hp"].double().sum(dim=2), c=res["cs"].double())
        if state:
            tp["h0"] = h0p.double().sum(dim=1)
        return tp

    def ref_fwd(res):
        hs, cs, _, _ = reference(xo, s, h0, c0, ws, lyr, planes, tape(res), grad=False)
        errs = {"step-local": step_local_error(tape(res), hs, cs, planes),
                "h_top": rel_err(res["h_n"][-1] if state else res["h_top"], hs[-1][-1])}
        if state:
            errs["h_n"] = rel_err(res["h_n"], torch.stack([h[-1] for h in hs]))
        assert max(errs.values()) <= FWD_TOL, f"lstm16_fwd {what}: {errs}"

    got = yield Call("lstm16_fwd", b, lambda st: lib().stmgcn_lstm16_fwd(
        t, lyr, rows, c, b_sz, planes, b["xo"].p, b["s"].p, b["wimg"].p, b["bias"].p, b["wih_t"].p, opt(b, "h0p"),
        opt(b, "c0"), b["hp"].p, b["cs"].p, b["h_top"].p, opt(b, "h_n"), st), ref_fwd, lyr)

    shapes = [sh for l in range(lyr) for sh in ((256, c if l == 0 else 64), (256, 64), (256,), (256,))]
    grid = int(lib().stmgcn_lstm16_grid(rows))
    d = dict(common(), hp=Buf("in", got["hp"]), cs=Buf("in", ops.to_blocked(got["cs"])),
             d_top=Buf("in", ops.to_blocked(d_top), pad=pads), dh_rec=Buf("ws", shape=(rp, 64)), dc=Buf("ws", shape=(rp, 64)),
             dw_scratch=Buf("ws", shape=(grid, 128 * 256)), dbp=Buf("ws", shape=(lyr, 256)),
             zero_tile=Buf("in", torch.zeros(128 * 64, dtype=torch.bfloat16)), d_s=Buf("acc", shape=(b_sz, t)),
             grads=Buf("out", shape=(sum(math.prod(sh) for sh in shapes),), exact=False))
    if lyr > 1:
        d["dx_work"] = Buf("ws", shape=(min(2, lyr - 1), t, rp, 64))

    def ref_bwd(res):
        hs, _, layers, s64 = reference(xo, s, h0, c0, ws, lyr, planes, tape(got))
        ref = torch.autograd.grad((hs[-1][-1] * d_top.double()).sum(), [s64] + [w for layer in layers for w in layer])
        errs = {"d_s": rel_err(res["d_s"], ref[0])}
        for i, (g, r) in enumerate(zip(res["grads"].split([math.prod(sh) for sh in shapes]), ref[1:])):
            errs[f"param {i}"] = rel_err(g, r.reshape(-1))
        assert max(errs.values()) <= GRAD_TOL, f"lstm16_bwd {what}: {errs}"

    yield Call("lstm16_bwd", d, lambda st: lib().stmgcn_lstm16_bwd(
        t, lyr, rows, c, b_sz, planes, d["xo"].p, d["s"].p, d["wimg"].p, d["bias"].p, d["wih_t"].p, opt(d, "h0p"),
        opt(d, "c0"), d["hp"].p, d["cs"].p, d["d_top"].p, d["dh_rec"].p, d["dc"].p, opt(d, "dx_work"), d["dw_scratch"].p,
        d["dbp"].p, d["zero_tile"].p, d["d_s"].p, d["grads"].p, st), ref_bwd, 2 * lyr)


def fuse_calls(m, c):
    from stmgcn_b200 import _lib as lib_mod
    gdim = 20
    n, b_sz = fuse_rows("waves" if m == 3 else "small")
    rows = n * b_sz
    gen = torch.Generator().manual_seed(10 * m + c)
    gs = [0.3 + torch.randn(n, b_sz, gdim, generator=gen) for _ in range(m)]
    fcw = torch.randn(c, gdim, generator=gen) / gdim ** 0.5
    fcb = torch.randn(c, generator=gen) * 0.3
    d_y = 0.5 + torch.randn(b_sz, n, c, generator=gen)
    w64, b64 = fcw.double().to(DEV), fcb.double().to(DEV)
    b = {f"g{k}": Buf("in", g) for k, g in enumerate(gs)}
    b.update(fcw=Buf("in", fcw), fcb=Buf("in", fcb), feat=Buf("out", shape=(rows, gdim)), y=Buf("out", shape=(b_sz, n, c)))

    def ref_fwd(res):
        feat = sum(g.double() for g in gs).to(DEV).reshape(rows, gdim)
        errs = {"feat": rel_err(res["feat"], feat),
                "y": rel_err(res["y"], (feat @ w64.t() + b64).reshape(n, b_sz, c).permute(1, 0, 2))}
        assert max(errs.values()) <= FWD_TOL, f"fuse_out_fwd M={m} C={c}: {errs}"

    got = yield Call("fuse_out_fwd", b, lambda st: lib().stmgcn_fuse_out_fwd(
        lib_mod.ptr_array([b[f"g{k}"].p for k in range(m)]), m, n, b_sz, gdim, c, b["fcw"].p, b["fcb"].p, b["feat"].p,
        b["y"].p, st), ref_fwd, 1)
    e = dict(d_y=Buf("in", d_y), feat=Buf("in", got["feat"]), fcw=Buf("in", fcw), d_feat=Buf("out", shape=(rows, gdim)),
             d_fcw=Buf("acc", shape=(c, gdim)), d_fcb=Buf("acc", shape=(c,)))

    def ref_bwd(res):
        dy = d_y.double().to(DEV).permute(1, 0, 2).reshape(rows, c)
        errs = {"d_feat": rel_err(res["d_feat"], dy @ w64), "d_fcw": rel_err(res["d_fcw"], dy.t() @ got["feat"].double()),
                "d_fcb": rel_err(res["d_fcb"], dy.sum(0))}
        assert max(errs.values()) <= GRAD_TOL, f"fuse_out_bwd M={m} C={c}: {errs}"

    yield Call("fuse_out_bwd", e, lambda st: lib().stmgcn_fuse_out_bwd(
        e["d_y"].p, e["feat"].p, n, b_sz, gdim, c, e["fcw"].p, e["d_feat"].p, e["d_fcw"].p, e["d_fcb"].p, st), ref_bwd, 1)


def obs_grad_calls(c, which):
    b_sz, t, n = 5, 7, 33
    gen = torch.Generator().manual_seed(c)
    d_xo, d_xt = torch.randn(n, b_sz, t, c, generator=gen), torch.randn(n, b_sz, t, generator=gen)
    bufs = dict(d_obs=Buf("out", shape=(b_sz, t, n, c)))
    if "xo" in which:
        bufs["d_xo"] = Buf("in", d_xo)
    if "xt" in which:
        bufs["d_xt"] = Buf("in", d_xt)
    opt = lambda k: bufs[k].p if k in bufs else None      # noqa: E731

    def ref(res):
        want = torch.zeros(b_sz, t, n, c, dtype=torch.float64)
        if "xo" in which:
            want += d_xo.double().permute(1, 2, 0, 3)
        if "xt" in which:
            want += d_xt.double().permute(1, 2, 0)[..., None]
        assert torch.equal(res["d_obs"].double().cpu(), want.float().double())

    yield Call("obs_grad", bufs, lambda st: lib().stmgcn_obs_grad(opt("d_xo"), opt("d_xt"), bufs["d_obs"].p, b_sz, t, n,
                                                                    c, st), ref, 1)


def lstm16_ex_calls(n, b_sz, t, lyr, c, state, planes):
    """Forward through ops (not under test), then stmgcn_lstm16_bwd_ex with every extra: seeds with poisoned padding
    rows, dh0 / dc0 with unspecified padding rows, d_xo."""
    from stmgcn_b200 import ops
    rows = n * b_sz
    rp = -(-rows // 128) * 128
    xo, s, h0, c0, ws, d_top = lstm16_inputs(n, b_sz, t, lyr, c, state, seed=n + planes)
    dh_n, dc_n = seeds(lyr, rows, HID, seed=n)
    _, _, _, tape = ops._lstm16_forward(xo, s, h0, c0, lyr, state, ws, planes, True)
    ktape = kernel_tape(tape, rows, state)
    pads = lambda v: blocked_pads(v, rows)      # noqa: E731
    blocked = lambda v: ops.from_blocked(v, rows)      # noqa: E731
    shapes = [sh for l in range(lyr) for sh in ((256, c if l == 0 else 64), (256, 64), (256,), (256,))]
    grid = int(lib().stmgcn_lstm16_grid(rows))
    d = dict(xo=Buf("in", xo), s=Buf("in", s), wimg=Buf("in", tape["wimg"].view(torch.bfloat16)), bias=Buf("in", tape["bias"]),
             wih_t=Buf("in", tape["wih_t"]), hp=Buf("in", tape["hp"]), cs=Buf("in", tape["cs"]),
             d_top=Buf("in", ops.to_blocked(d_top), pad=pads), dh_rec=Buf("ws", shape=(rp, 64)),
             dc=Buf("ws", shape=(rp, 64)), dw_scratch=Buf("ws", shape=(grid, 128 * 256)), dbp=Buf("ws", shape=(lyr, 256)),
             zero_tile=Buf("in", torch.zeros(128 * 64, dtype=torch.bfloat16)), d_s=Buf("acc", shape=(b_sz, t)),
             grads=Buf("out", shape=(sum(math.prod(sh) for sh in shapes),), exact=False),
             dh_n=Buf("in", ops.to_blocked(dh_n), pad=pads), dc_n=Buf("in", ops.to_blocked(dc_n), pad=pads),
             dh0=Buf("out", shape=(lyr, rp, 64), part=blocked), dc0=Buf("out", shape=(lyr, rp, 64), part=blocked),
             d_xo=Buf("out", shape=xo.shape))
    if state:
        d.update(h0p=Buf("in", tape["h0p"]), c0=Buf("in", tape["c0b"], pad=pads))
    if lyr > 1:
        d["dx_work"] = Buf("ws", shape=(min(2, lyr - 1), t, rp, 64))
    opt = lambda k: d[k].p if k in d else None      # noqa: E731

    def ref(res):
        r = state_gradients(xo, s, h0, c0, ws, lyr, planes, ktape, d_top, dh_n, dc_n)
        got = dict(d_xo=res["d_xo"], d_s=res["d_s"], dh0=res["dh0"], dc0=res["dc0"],
                   params=[g.view(sh) for g, sh in zip(res["grads"].split([math.prod(sh) for sh in shapes]), shapes)])
        errs = grad_errors(got, r)
        assert max(errs.values()) <= GRAD_TOL, f"lstm16_bwd_ex rows={rows} P={planes}: {errs}"

    yield Call("lstm16_bwd_ex", d, lambda st: lib().stmgcn_lstm16_bwd_ex(
        t, lyr, rows, c, b_sz, planes, d["xo"].p, d["s"].p, d["wimg"].p, d["bias"].p, d["wih_t"].p, opt("h0p"), opt("c0"),
        d["hp"].p, d["cs"].p, d["d_top"].p, d["dh_rec"].p, d["dc"].p, opt("dx_work"), d["dw_scratch"].p, d["dbp"].p,
        d["zero_tile"].p, d["d_s"].p, d["grads"].p, d["dh_n"].p, d["dc_n"].p, d["dh0"].p, d["dc0"].p, d["d_xo"].p, st),
        ref, 2 * lyr)


def lstm_ex_calls(n, b_sz, state):
    from stmgcn_b200 import ops
    hid, lyr, t, c = 48, 3, 5, 2
    rows = n * b_sz
    xo, s, h0, c0, ws, d_top = (None if v is None else v.to(DEV) if torch.is_tensor(v) else [w.to(DEV) for w in v]
                                for v in lstm_inputs(n, b_sz, t, lyr, c, hid, state, seed=rows))
    dh_n, dc_n = seeds(lyr, rows, hid, seed=rows)
    _, _, _, tape = ops._exact_forward(xo, s, h0, c0, lyr, hid, True, ws, True)
    _, _, hs, cs, gates, wx, wpt = tape
    ktape = dict(h=hs.double(), c=cs.double())
    if state:
        ktape["h0"] = h0.double()
    bp = ops._pack_lstm(ws, lyr, hid)[2]
    d = dict(xo=Buf("in", xo), s=Buf("in", s), wx=Buf("in", wx), wpt=Buf("in", wpt), cs=Buf("in", cs), hs=Buf("in", hs),
             gates=Buf("inout", gates), d_top=Buf("in", d_top), dh_rec=Buf("ws", shape=(lyr, rows, hid)),
             dc=Buf("ws", shape=(lyr, rows, hid)), dx_work=Buf("ws", shape=(rows, hid)), d_s=Buf("acc", shape=(b_sz, t)),
             dwx=Buf("acc", shape=wx.shape), dwp=Buf("acc", shape=wpt.shape), dbp=Buf("acc", shape=bp.shape),
             dh_n=Buf("in", dh_n), dc_n=Buf("in", dc_n), dh0=Buf("out", shape=(lyr, rows, hid)),
             dc0=Buf("out", shape=(lyr, rows, hid)), d_xo=Buf("out", shape=xo.shape))
    if state:
        d.update(h0=Buf("in", h0), c0=Buf("in", c0))
    opt = lambda k: d[k].p if k in d else None      # noqa: E731

    def ref(res):
        r = state_gradients(xo, s, h0, c0, ws, lyr, 2, ktape, d_top, dh_n, dc_n)
        got = dict(d_xo=res["d_xo"], d_s=res["d_s"], dh0=res["dh0"], dc0=res["dc0"],
                   params=ops._unpack_lstm_grads(res["dwx"], res["dwp"], res["dbp"], lyr, hid, c))
        errs = grad_errors(got, r)
        assert max(errs.values()) <= GRAD_TOL, f"lstm_bwd_ex rows={rows}: {errs}"

    yield Call("lstm_bwd_ex", d, lambda st: lib().stmgcn_lstm_bwd_ex(
        t, lyr, rows, hid, c, b_sz, d["xo"].p, d["s"].p, d["wx"].p, d["wpt"].p, opt("h0"), opt("c0"), d["cs"].p, d["hs"].p,
        d["gates"].p, d["d_top"].p, d["dh_rec"].p, d["dc"].p, d["dx_work"].p, d["d_s"].p, d["dwx"].p, d["dwp"].p,
        d["dbp"].p, d["dh_n"].p, d["dc_n"].p, d["dh0"].p, d["dc0"].p, d["d_xo"].p, st), ref, 2 * lyr * t + lyr)
