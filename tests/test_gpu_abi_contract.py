"""The C ABI's caller-memory and stream contract (include/stmgcn_b200.h), entry point by entry point, called directly
through ``_lib.lib`` -- no ``ops`` wrapper zeroes an accumulator or sizes a buffer on the kernels' behalf.

Every buffer of a call -- inputs, outputs, workspaces -- is a view into a larger allocation with 64 KiB of sentinel
before and after it (more than one 128 x 64 fp32 tile; the view keeps the allocation's 512-byte alignment).  The fp32
sentinel is the NaN 0x7FA5A5A5 and the bf16 one 0x7FA5, so a read past a buffer reaches the results as NaN and a write
past it changes guard bytes; the int32 CSR arrays are guarded with values valid for them (0 after colidx, nnz after
rowptr), so an overrun cannot turn into a wild address.  Each call then runs

1. clean: outputs, accumulators and workspaces zeroed; the results against an fp64 reference, at 2e-5 (forward) and
   5e-5 (gradients), max-norm relative;
2. poisoned, twice: every workspace, every overwritten output and the padding rows of the tile-blocked inputs filled
   with all bytes 0xFF (NaN in fp32 and bf16), then with seeded finite values of both signs around 1e4 (which pass
   through comparisons such as a ReLU mask).  Outputs without atomics must equal the clean run bit for bit, sums of
   atomics must be within the gradient bar of it, and every output must be finite;
3. accumulators pre-filled with seeded values V of about the result's magnitude: out - V must match the clean run
   within the gradient bar (an overwrite instead of += fails, and so does double counting);

and after every run all guard bytes must be intact, every const input bit-identical to before, and the kernel launch
count must have grown by what the call launches.  Rejected calls must return < 0 with nothing enqueued and nothing
changed, and every entry point must replay from a CUDA graph captured on a side stream in global capture mode (a
device synchronisation, a launch on the legacy stream or an allocation fails the capture).

The CPU tests at the top show that each check of the harness catches what it is there for.
"""
import math

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from test_gpu_exact_kernels import (ACTS, FWD_TOL, GRAD_TOL, _err, _fuse_rows, _lstm_reference, _proj_ref_out, _proj_rows,
                                    _sms, isolated_matrix, lstm_inputs, proj_inputs)
from test_gpu_exact_kernels import _step_local_error as _exact_step_local_error
from test_gpu_lstm16 import _inputs as lstm16_inputs
from test_gpu_lstm16 import _reference as lstm16_reference
from test_gpu_lstm16 import _step_local_error as lstm16_step_local_error
from test_gpu_lstm16 import _wave_regions
from test_gpu_proj_tc import _shape as _tc_shape

DEV = "cuda:0"
GUARD = 64 * 1024                                   # bytes of sentinel on each side of a buffer
SENTINEL = {torch.float32: 0x7FA5A5A5, torch.bfloat16: 0x7FA5}
_INT = {4: torch.int32, 2: torch.int16, 1: torch.uint8}
POISON = ("nan", "big")
RESULTS = ("out", "out0", "inout", "acc")


def _bits(x):
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
        return all(torch.equal(_bits(a), _bits(b)) for a, b in zip(self._fixed(), snap))

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


def _lib():
    from stmgcn_b200 import _lib as lib
    return lib.lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _same(call, name, got, want, what):
    buf = call.bufs[name]
    if buf.finite:
        assert bool(torch.isfinite(got).all()), f"{call.name} ({what}): {name} is not finite"
    if buf.exact and buf.role != "acc":
        assert torch.equal(_bits(got), _bits(want)), f"{call.name} ({what}): {name} differs from the clean run"
    else:
        err = _err(got, want)
        assert err <= GRAD_TOL, f"{call.name} ({what}): {name} is {err:.2e} off the clean run"


def _run(call, mode):
    snaps = {k: b.prepare(mode, 101 * i) for i, (k, b) in enumerate(call.bufs.items())}
    n0 = _lib().stmgcn_launch_count() if call.cuda else 0
    rc = call.launch(_stream() if call.cuda else None)
    if call.cuda:
        torch.cuda.synchronize()
        assert rc == 0, f"{call.name} ({mode} run): rc={rc}: {_lib().stmgcn_last_error()}"
        if call.launches is not None:
            got = _lib().stmgcn_launch_count() - n0
            assert got == call.launches, f"{call.name} ({mode} run): {got} launches, expected {call.launches}"
    for k, b in call.bufs.items():
        assert b.guards_intact(), f"{call.name} ({mode} run): a guard band of {k} changed"
        assert b.unchanged(snaps[k]), f"{call.name} ({mode} run): {k} changed where the call must not write"
    return {k: b.result() for k, b in call.bufs.items() if b.role in RESULTS}


def run_contract(call):
    """Clean run against the reference, two poisoned runs, one run with pre-filled accumulators; returns the clean
    results (the inputs of the calls that follow)."""
    clean = _run(call, "clean")
    if call.reference is not None:
        call.reference(clean)
    for mode in POISON:
        for k, v in _run(call, mode).items():
            _same(call, k, v, clean[k], f"{mode}-poisoned run")
    accs = [k for k, b in call.bufs.items() if b.role == "acc"]
    if accs:
        gen = torch.Generator().manual_seed(7)
        for k in accs:
            c = clean[k]
            scale = float(c.abs().max()) or 1.0
            call.bufs[k].acc_init = ((torch.rand(c.shape, generator=gen) * 2 - 1) * scale).to(c.device)
        got = _run(call, "acc")
        for k, v in got.items():
            if k in accs:
                err = _err(v.double() - call.bufs[k].acc_init.double(), clean[k])
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
    assert rc == 0, f"{call.name} (eager on a side stream): rc={rc}: {_lib().stmgcn_last_error()}"
    eager = results()
    prep()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="global"):
        rc = call.launch(_stream())
    assert rc == 0, f"{call.name} (captured): rc={rc}: {_lib().stmgcn_last_error()}"
    prep()
    graph.replay()
    torch.cuda.synchronize()
    for k, v in results().items():
        _same(call, k, v, eager[k], "graph replay")
    for k, b in call.bufs.items():
        assert b.guards_intact(), f"{call.name} (graph replay): a guard band of {k} changed"
    return eager


def _drive(calls, runner):
    """Run a generator of Calls; each receives the results of the one before (a forward's outputs feed its backward)."""
    try:
        call = next(calls)
        while True:
            call = calls.send(runner(call))
    except StopIteration:
        pass


# ======================================================================================================================
# the harness catches what it is for (CPU, no library call)
# ======================================================================================================================
def _cpu_call(kernel, **bufs):
    return Call("cpu kernel", bufs, lambda st: kernel(bufs) or 0)


def _x():
    return torch.randn(33, 7, generator=torch.Generator().manual_seed(0))


def test_harness_guard_check_catches_a_one_element_overrun():
    def kernel(b, over):
        b["y"].raw[GUARD:GUARD + b["y"].nbytes + 4 * over].view(torch.float32).copy_(
            torch.arange(33 * 7 + over, dtype=torch.float32))

    run_contract(_cpu_call(lambda b: kernel(b, 0), x=Buf("in", _x(), device="cpu"), y=Buf("out", shape=(33, 7), device="cpu")))
    with pytest.raises(AssertionError, match="a guard band of y changed"):
        run_contract(_cpu_call(lambda b: kernel(b, 1), x=Buf("in", _x(), device="cpu"),
                               y=Buf("out", shape=(33, 7), device="cpu")))


def test_harness_poison_check_catches_a_read_of_an_unwritten_workspace():
    def kernel(b, leak):
        b["y"].t.copy_(2 * b["x"].t + (b["ws"].t * 0 if leak else 0))

    def ref(res):
        assert torch.equal(res["y"], 2 * _x())

    bufs = lambda: dict(x=Buf("in", _x(), device="cpu"), ws=Buf("ws", shape=(33, 7), device="cpu"),      # noqa: E731
                        y=Buf("out", shape=(33, 7), device="cpu"))
    b = bufs()
    run_contract(Call("cpu kernel", b, lambda st: kernel(b, False), ref))
    b = bufs()
    with pytest.raises(AssertionError, match=r"nan-poisoned run\): y is not finite"):
        run_contract(Call("cpu kernel", b, lambda st: kernel(b, True), ref))


def test_harness_accumulator_check_catches_an_overwrite():
    def kernel(b, overwrite):
        s = b["x"].t.sum(0)
        b["acc"].t.copy_(s) if overwrite else b["acc"].t.add_(s)

    bufs = lambda: dict(x=Buf("in", _x(), device="cpu"), acc=Buf("acc", shape=(7,), device="cpu"))   # noqa: E731
    b = bufs()
    run_contract(Call("cpu kernel", b, lambda st: kernel(b, False)))
    b = bufs()
    with pytest.raises(AssertionError, match=r"acc started at V ends .* \(\+=\)"):
        run_contract(Call("cpu kernel", b, lambda st: kernel(b, True)))


# ======================================================================================================================
# K1: Chebyshev steps and the bf16 copy
# ======================================================================================================================
SPMM_CASES = [(n, f, ("A", "AT", "alias")[(i + j) % 3]) for i, n in enumerate((1, 33, 1000)) for j, f in enumerate((7, 40, 264))]


def _csr_bufs(op):
    csr = sp.csr_matrix(op)
    return dict(rowptr=Buf("in", torch.from_numpy(csr.indptr.astype(np.int32)), guard=csr.nnz),
                colidx=Buf("in", torch.from_numpy(csr.indices.astype(np.int32)), guard=0),
                vals=Buf("in", torch.from_numpy(csr.data.astype(np.float32))))


def _spmm_calls(n, f, variant):
    """Y = 2 op(A) X - Z + 0.5 U through stmgcn_cheb_spmm_step and (f % 8 == 0) _step16, then stmgcn_to_bf16 of X.
    ``AT``: the CSR of A^T is passed; ``alias``: U is Y (the adjoint recurrence's in-place update)."""
    a = isolated_matrix(n, seed=7 * n + f)
    op = a.T if variant == "AT" else a
    if n > 1:
        assert (sp.csr_matrix(op).getnnz(axis=1) == 0).any(), "the CSR has no empty row"
    gen = torch.Generator().manual_seed(n + f)
    x, z, u = (torch.randn(n, f, generator=gen) for _ in range(3))
    op64 = torch.from_numpy(op.astype(np.float64)).to(DEV)
    z64, u64 = z.double().to(DEV), u.double().to(DEV)
    uk = "y" if variant == "alias" else "u"

    def operands():
        bufs = dict(_csr_bufs(op), z=Buf("in", z))
        if variant == "alias":
            bufs["y"] = Buf("inout", u)
        else:
            bufs.update(u=Buf("in", u), y=Buf("out", shape=(n, f)))
        return bufs

    b = dict(operands(), x=Buf("in", x))

    def ref32(res):
        err = _err(res["y"], 2.0 * (op64 @ x.double().to(DEV)) - z64 + 0.5 * u64)
        assert err <= FWD_TOL, f"cheb_spmm_step n={n} f={f} {variant}: {err:.2e}"

    yield Call("cheb_spmm_step", b, lambda st, b=b: _lib().stmgcn_cheb_spmm_step(
        n, b["rowptr"].p, b["colidx"].p, b["vals"].p, 2.0, b["x"].p, -1.0, b["z"].p, 0.5, b[uk].p, b["y"].p, f, st), ref32, 1)
    x16 = x.to(torch.bfloat16)
    if f % 8 == 0:
        b = dict(operands(), x16=Buf("in", x16), y16=Buf("out", shape=(n, f), dtype=torch.bfloat16))

        def ref16(res):
            err = _err(res["y"], 2.0 * (op64 @ x16.double().to(DEV)) - z64 + 0.5 * u64)
            assert err <= FWD_TOL, f"cheb_spmm_step16 n={n} f={f} {variant}: {err:.2e}"
            assert torch.equal(_bits(res["y16"]), _bits(res["y"].to(torch.bfloat16))), "y16 is not bf16(y)"

        yield Call("cheb_spmm_step16", b, lambda st, b=b: _lib().stmgcn_cheb_spmm_step16(
            n, b["rowptr"].p, b["colidx"].p, b["vals"].p, 2.0, b["x16"].p, -1.0, b["z"].p, 0.5, b[uk].p, b["y"].p,
            b["y16"].p, f, st), ref16, 1)
    if (n * f) % 8 == 0:
        yield from _to_bf16_calls(x.reshape(-1))


def _to_bf16_calls(x, finite=True):
    b = dict(x=Buf("in", x), y16=Buf("out", shape=x.shape, dtype=torch.bfloat16, finite=finite))

    def ref(res):
        want = x.to(torch.bfloat16).to(DEV)
        nan = torch.isnan(x).to(DEV)
        assert torch.equal(_bits(res["y16"])[~nan], _bits(want)[~nan]), "to_bf16 differs from torch's rounding"
        assert bool(torch.isnan(res["y16"][nan]).all()), "to_bf16 turned a NaN into a number"

    yield Call("to_bf16", b, lambda st: _lib().stmgcn_to_bf16(b["x"].p, b["y16"].p, x.numel(), st), ref, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("n,f,variant", SPMM_CASES)
def test_spmm_steps_keep_the_memory_contract(n, f, variant):
    """f = 7: the scalar kernel; 40: float4 with a partial column tile; 264: several column tiles."""
    _drive(_spmm_calls(n, f, variant), run_contract)


@pytest.mark.gpu
def test_to_bf16_rounds_like_torch_at_the_edges():
    """+-0, subnormals (a tie, one rounding up into the normals), FLT_MIN, FLT_MAX (to +-Inf), ties to even at 1 and
    next to the largest bf16, +-Inf, quiet and signalling NaNs, then normals over 80 binades: bit for bit torch's
    round-to-nearest-even on every non-NaN input; every NaN stays NaN."""
    edges = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x00008000, 0x00018000, 0x007FFFFF, 0x00800000, 0x7F7FFFFF,
             0xFF7FFFFF, 0x7F7F7FFF, 0x7F7F8000, 0x7F7E8000, 0x3F808000, 0x3F818000, 0x3F808001, 0xBF818000, 0x7F800000,
             0xFF800000, 0x7FC00000, 0xFFFFFFFF, 0x7F800001, 0x7FA5A5A5, 0x00000000]
    gen = torch.Generator().manual_seed(3)
    normal = torch.randn(4096, generator=gen) * torch.pow(2.0, torch.randint(-40, 40, (4096,), generator=gen).float())
    x = torch.cat([torch.tensor(np.array(edges, dtype=np.uint32).view(np.int32)).view(torch.float32), normal])
    _drive(_to_bf16_calls(x, finite=False), run_contract)


# ======================================================================================================================
# layout
# ======================================================================================================================
def _obs_calls(c):
    b_sz, t, n = 5, 7, 33
    obs = torch.randn(b_sz, t, n, c, generator=torch.Generator().manual_seed(c))
    b = dict(obs=Buf("in", obs), xt=Buf("out", shape=(n, b_sz, t)))
    if c > 1:
        b["xo"] = Buf("out", shape=(n, b_sz, t, c))

    def ref(res):
        want = obs.permute(2, 0, 1, 3).to(DEV)
        xt = want[..., 0].clone()
        for k in range(1, c):
            xt = xt + want[..., k]
        assert torch.equal(res["xt"], xt)
        if c > 1:
            assert torch.equal(res["xo"], want)

    yield Call("obs_to_node_major", b, lambda st: _lib().stmgcn_obs_to_node_major(
        b["obs"].p, b["xo"].p if c > 1 else None, b["xt"].p, b_sz, t, n, c, st), ref, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [1, 3])
def test_obs_to_node_major_keeps_the_memory_contract(c):
    """C = 1 with xo NULL (xt alone), C = 3."""
    _drive(_obs_calls(c), run_contract)


# ======================================================================================================================
# K2: projection
# ======================================================================================================================
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


def _proj_calls(ks, p, q, n, b_sz, gap, tc, bcast, relu, bias, seed):
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
    ref_out = _proj_ref_out(s64, w64, b64, relu)
    what = f"ks={ks} p={p} q={q} rows={rows} gap={gap}"
    img_f = img_b = None
    if tc:
        n_bwd = 2 if ks > 4 else 1
        b = dict(w=Buf("in", w), img_fwd=Buf("out", shape=(ks * 64 * 64 * 2,)),
                 img_bwd=Buf("out0", shape=(n_bwd * 2 * 2 * 256 * 32,)))

        def ref_pack(res):
            wd = w.to(DEV)
            assert torch.equal(_bits(res["img_fwd"]), _bits(_tf32_image(wd.t(), 64))), f"forward image, {what}"
            want = torch.cat([_tf32_image(wd[g * 256:(g + 1) * 256], 256) for g in range(n_bwd)])
            assert torch.equal(_bits(res["img_bwd"]), _bits(want)), f"backward image, {what}"

        got = yield Call("proj_pack_tc", b, lambda st, b=b: _lib().stmgcn_proj_pack_tc(
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
        errs = {"out": _err(res["out"], ref_out)}
        if bcast:
            errs["pool"] = _err(res["pool"], (s64[0] + ref_out).view(n, b_sz, q).sum(0))
        assert max(errs.values()) <= FWD_TOL, f"proj_fwd {what}: {errs}"

    got = yield Call("proj_fwd", b, lambda st, b=b: _lib().stmgcn_proj_fwd(
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
        errs = {"dz": _err(res["dz"], dz), "dW": _err(res["dw"], torch.einsum("krp,rq->kpq", s64, dz).reshape(ks * p, q)),
                "U": _err(res["u"], torch.einsum("rq,kpq->krp", dz, w64.reshape(ks, p, q)).reshape(ks, -1))}
        if bias:
            errs["db"] = _err(res["db"], dz.sum(0))
        assert max(errs.values()) <= GRAD_TOL, f"proj_bwd {what}: {errs}"

    yield Call("proj_bwd", b, lambda st, b=b: _lib().stmgcn_proj_bwd(
        b["s"].p, sk, ks, rows, p, b["wt"].p, q, act, b["out"].p, opt(b, "d_out"), opt(b, "d_bcast"), scale, b_sz, b["dz"].p,
        b["dw"].p, opt(b, "db"), b["u"].p, sk, opt(b, "wimg_t"), st),
        ref_bwd, ((2 if ks > 4 else 1) + (ks + 1) // 2) if on_tc else 3)


PROJ_TC = [(ks, rows_id, (0, 36, 7)[(i + j) % 3]) for i, ks in enumerate((1, 3, 5, 8)) for j, rows_id in enumerate((1, 129, "waves"))]
# (name, ks, p, q, regions N (None: multi-wave), batch B, gap, gate pooling / broadcast dOut)
PROJ_FMA = [("temporal", 4, 12, 12, 33, 5, 0, True),
            ("temporal_odd_gap", 3, 12, 12, 300, 7, 5, True),
            ("p64_q32", 3, 64, 32, 43, 3, 4, False),
            ("p64_q32_waves", 2, 64, 32, None, 1, 0, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("ks,rows_id,gap", PROJ_TC)
def test_projection_tensor_core_entry_points_keep_the_memory_contract(ks, rows_id, gap):
    """p = q = 64 with weight images.  ks = 5 and 8 split U over two launches and end the weight-gradient pairs on an
    odd support; a gap that is a multiple of 4 keeps the tensor-core kernels, an odd gap routes to the FFMA kernels."""
    n, b_sz = _tc_shape(rows_id)
    relu, bias = ACTS[PROJ_TC.index((ks, rows_id, gap)) % 4]
    _drive(_proj_calls(ks, 64, 64, n, b_sz, gap, True, False, relu, bias, seed=10 * ks + gap), run_contract)


@pytest.mark.gpu
@pytest.mark.parametrize("case", PROJ_FMA, ids=[c[0] for c in PROJ_FMA])
def test_projection_ffma_entry_points_keep_the_memory_contract(case):
    name, ks, p, q, n, b_sz, gap, bcast = case
    if n is None:
        n = _proj_rows("waves")
    relu, bias = ACTS[PROJ_FMA.index(case) % 4]
    _drive(_proj_calls(ks, p, q, n, b_sz, gap, False, bcast, relu, bias, seed=100 + PROJ_FMA.index(case)), run_contract)


# ======================================================================================================================
# K3a: context gate
# ======================================================================================================================
def _gate_calls(t, b_sz):
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
        errs = {"z": _err(res["z"], p64 / n_regions), "a1": _err(res["a1"], a1),
                "s": _err(res["s"], torch.sigmoid(a1.clamp_min(0) @ w64.t() + b64))}
        assert max(errs.values()) <= FWD_TOL, f"gate_fwd T={t}: {errs}"

    got = yield Call("gate_fwd", b, lambda st: _lib().stmgcn_gate_fwd(
        b["pool"].p, b_sz, t, n_regions, b["fcw"].p, b["fcb"].p, b["z"].p, b["a1"].p, b["s"].p, st), ref_fwd, 1)
    c = dict(d_s=Buf("in", d_s), z=Buf("in", got["z"]), a1=Buf("in", got["a1"]), s=Buf("in", got["s"]),
             fcw=Buf("in", fcw), d_fcw=Buf("acc", shape=(t, t)), d_fcb=Buf("acc", shape=(t,)), d_z=Buf("out", shape=(b_sz, t)))

    def ref_bwd(res):
        z64 = got["z"].double().requires_grad_(True)
        wg, bg = w64.clone().requires_grad_(True), b64.clone().requires_grad_(True)
        a1 = z64 @ wg.t() + bg
        s = torch.sigmoid((a1 * (got["a1"] > 0)) @ wg.t() + bg)              # the kernel's own ReLU mask
        g = torch.autograd.grad((s * d_s.double().to(DEV)).sum(), [z64, wg, bg])
        errs = {"d_z": _err(res["d_z"], g[0]), "d_fcw": _err(res["d_fcw"], g[1]), "d_fcb": _err(res["d_fcb"], g[2])}
        assert max(errs.values()) <= GRAD_TOL, f"gate_bwd T={t}: {errs}"

    yield Call("gate_bwd", c, lambda st: _lib().stmgcn_gate_bwd(
        c["d_s"].p, c["z"].p, c["a1"].p, c["s"].p, b_sz, t, c["fcw"].p, c["d_fcw"].p, c["d_fcb"].p, c["d_z"].p, st), ref_bwd, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("t", [12, 300])
def test_context_gate_keeps_the_memory_contract(t):
    _drive(_gate_calls(t, 5), run_contract)


# ======================================================================================================================
# K3b: exact-fp32 LSTM
# ======================================================================================================================
def _lstm_calls(n, b_sz, state):
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
        hs, cs, _, _ = _lstm_reference(xo, s, h0, c0, ws, lyr, 2, tape(res), grad=False)
        err = _exact_step_local_error(tape(res), hs, cs)
        assert err <= FWD_TOL, f"lstm_fwd rows={rows}: step-local {err:.2e}"

    got = yield Call("lstm_fwd", b, lambda st: _lib().stmgcn_lstm_fwd(
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
        hs, _, layers, s64 = _lstm_reference(xo, s, h0, c0, ws, lyr, 2, tape(got))
        ref = torch.autograd.grad((hs[-1][-1] * d_top.double()).sum(), [s64] + [w for layer in layers for w in layer])
        grads = ops._unpack_lstm_grads(res["dwx"], res["dwp"], res["dbp"], lyr, hid, c)
        errs = {"d_s": _err(res["d_s"], ref[0])}
        errs.update({f"param {i}": _err(g, r) for i, (g, r) in enumerate(zip(grads, ref[1:]))})
        assert max(errs.values()) <= GRAD_TOL, f"lstm_bwd rows={rows}: {errs}"

    yield Call("lstm_bwd", c_, lambda st: _lib().stmgcn_lstm_bwd(
        t, lyr, rows, hid, c, b_sz, c_["xo"].p, c_["s"].p, c_["wx"].p, c_["wpt"].p, opt(c_, "h0"), opt(c_, "c0"), c_["cs"].p,
        c_["hs"].p, c_["gates"].p, c_["d_top"].p, c_["dh_rec"].p, c_["dc"].p, c_["dx_work"].p, c_["d_s"].p, c_["dwx"].p,
        c_["dwp"].p, c_["dbp"].p, st), ref_bwd, 2 * lyr * t + lyr)


@pytest.mark.gpu
@pytest.mark.parametrize("state", [False, True])
def test_exact_lstm_keeps_the_memory_contract(state):
    """Ragged rows: 35 with h0 / c0; without, more rows than the backward's pointwise grid covers in one pass."""
    n, b_sz = (7, 5) if state else ((2 * 32 * _sms()) // 5 + 1, 5)
    _drive(_lstm_calls(n, b_sz, state), run_contract)


# ======================================================================================================================
# K3b: tensor-core LSTM
# ======================================================================================================================
def _blocked_pads(t, rows):
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


def _lstm16_calls(case, planes):
    """stmgcn_lstm16_pack layer by layer into a NaN-filled image (the other layers' slots must stay untouched), then the
    forward (with h_n given, a separate h_top must stay untouched) and the backward with every workspace poisoned and
    the padding rows of c0 and d_top poisoned; hp and cs must come out of the backward bit-identical."""
    from stmgcn_b200 import ops
    name, n, b_sz, t, lyr, c, state = case
    if n is None:
        n = _wave_regions(b_sz)
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
        got = yield Call(f"lstm16_pack layer {l}", b, lambda st, b=b, l=l: _lib().stmgcn_lstm16_pack(
            b["w_ih"].p, b["w_hh"].p, b["b_ih"].p, b["b_hh"].p, l, c, b["wimg"].p, b["bias"].p, b["wih_t"].p, st), None, 1)
        wimg[o:o + m], bias[l] = got["wimg"], got["bias"]
        wih_t = got["wih_t"] if l == 0 else wih_t

    pads = lambda v: _blocked_pads(v, rows)      # noqa: E731
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
        hs, cs, _, _ = lstm16_reference(xo, s, h0, c0, ws, lyr, planes, tape(res), grad=False)
        errs = {"step-local": lstm16_step_local_error(tape(res), hs, cs, planes),
                "h_top": _err(res["h_n"][-1] if state else res["h_top"], hs[-1][-1])}
        if state:
            errs["h_n"] = _err(res["h_n"], torch.stack([h[-1] for h in hs]))
        assert max(errs.values()) <= FWD_TOL, f"lstm16_fwd {what}: {errs}"

    got = yield Call("lstm16_fwd", b, lambda st: _lib().stmgcn_lstm16_fwd(
        t, lyr, rows, c, b_sz, planes, b["xo"].p, b["s"].p, b["wimg"].p, b["bias"].p, b["wih_t"].p, opt(b, "h0p"),
        opt(b, "c0"), b["hp"].p, b["cs"].p, b["h_top"].p, opt(b, "h_n"), st), ref_fwd, lyr)

    shapes = [sh for l in range(lyr) for sh in ((256, c if l == 0 else 64), (256, 64), (256,), (256,))]
    grid = int(_lib().stmgcn_lstm16_grid(rows))
    d = dict(common(), hp=Buf("in", got["hp"]), cs=Buf("in", ops.to_blocked(got["cs"])),
             d_top=Buf("in", ops.to_blocked(d_top), pad=pads), dh_rec=Buf("ws", shape=(rp, 64)), dc=Buf("ws", shape=(rp, 64)),
             dw_scratch=Buf("ws", shape=(grid, 128 * 256)), dbp=Buf("ws", shape=(lyr, 256)),
             zero_tile=Buf("in", torch.zeros(128 * 64, dtype=torch.bfloat16)), d_s=Buf("acc", shape=(b_sz, t)),
             grads=Buf("out", shape=(sum(math.prod(sh) for sh in shapes),), exact=False))
    if lyr > 1:
        d["dx_work"] = Buf("ws", shape=(min(2, lyr - 1), t, rp, 64))

    def ref_bwd(res):
        hs, _, layers, s64 = lstm16_reference(xo, s, h0, c0, ws, lyr, planes, tape(got))
        ref = torch.autograd.grad((hs[-1][-1] * d_top.double()).sum(), [s64] + [w for layer in layers for w in layer])
        errs = {"d_s": _err(res["d_s"], ref[0])}
        for i, (g, r) in enumerate(zip(res["grads"].split([math.prod(sh) for sh in shapes]), ref[1:])):
            errs[f"param {i}"] = _err(g, r.reshape(-1))
        assert max(errs.values()) <= GRAD_TOL, f"lstm16_bwd {what}: {errs}"

    yield Call("lstm16_bwd", d, lambda st: _lib().stmgcn_lstm16_bwd(
        t, lyr, rows, c, b_sz, planes, d["xo"].p, d["s"].p, d["wimg"].p, d["bias"].p, d["wih_t"].p, opt(d, "h0p"),
        opt(d, "c0"), d["hp"].p, d["cs"].p, d["d_top"].p, d["dh_rec"].p, d["dc"].p, opt(d, "dx_work"), d["dw_scratch"].p,
        d["dbp"].p, d["zero_tile"].p, d["d_s"].p, d["grads"].p, st), ref_bwd, 2 * lyr)


@pytest.mark.gpu
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", LSTM16_CASES, ids=[c[0] for c in LSTM16_CASES])
def test_tensor_core_lstm_keeps_the_memory_contract(case, planes):
    _drive(_lstm16_calls(case, planes), run_contract)


# ======================================================================================================================
# fusion over graphs + output FC
# ======================================================================================================================
def _fuse_calls(m, c):
    from stmgcn_b200 import _lib as lib_mod
    gdim = 20
    n, b_sz = _fuse_rows("waves" if m == 3 else "small")
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
        errs = {"feat": _err(res["feat"], feat),
                "y": _err(res["y"], (feat @ w64.t() + b64).reshape(n, b_sz, c).permute(1, 0, 2))}
        assert max(errs.values()) <= FWD_TOL, f"fuse_out_fwd M={m} C={c}: {errs}"

    got = yield Call("fuse_out_fwd", b, lambda st: _lib().stmgcn_fuse_out_fwd(
        lib_mod.ptr_array([b[f"g{k}"].p for k in range(m)]), m, n, b_sz, gdim, c, b["fcw"].p, b["fcb"].p, b["feat"].p,
        b["y"].p, st), ref_fwd, 1)
    e = dict(d_y=Buf("in", d_y), feat=Buf("in", got["feat"]), fcw=Buf("in", fcw), d_feat=Buf("out", shape=(rows, gdim)),
             d_fcw=Buf("acc", shape=(c, gdim)), d_fcb=Buf("acc", shape=(c,)))

    def ref_bwd(res):
        dy = d_y.double().to(DEV).permute(1, 0, 2).reshape(rows, c)
        errs = {"d_feat": _err(res["d_feat"], dy @ w64), "d_fcw": _err(res["d_fcw"], dy.t() @ got["feat"].double()),
                "d_fcb": _err(res["d_fcb"], dy.sum(0))}
        assert max(errs.values()) <= GRAD_TOL, f"fuse_out_bwd M={m} C={c}: {errs}"

    yield Call("fuse_out_bwd", e, lambda st: _lib().stmgcn_fuse_out_bwd(
        e["d_y"].p, e["feat"].p, n, b_sz, gdim, c, e["fcw"].p, e["d_feat"].p, e["d_fcw"].p, e["d_fcb"].p, st), ref_bwd, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [1, 40])
@pytest.mark.parametrize("m", [1, 3])
def test_fuse_out_keeps_the_memory_contract(m, c):
    """M = 3 runs more rows than the forward's grid covers in one pass; C = 40 the second bias-gradient lane loop."""
    _drive(_fuse_calls(m, c), run_contract)


# ======================================================================================================================
# rejected calls and the stream contract
# ======================================================================================================================
# (what, call(lib, ptr_array, stream, a, b, c, d, e, f)): one or two representative argument errors per entry point
REJECTS = [
    ("cheb_spmm_step: n = 0", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_cheb_spmm_step(
        0, a, b, c, 1.0, d, 0.0, None, 0.0, None, e, 64, st)),
    ("cheb_spmm_step: y aliases x", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_cheb_spmm_step(
        64, a, b, c, 1.0, d, 0.0, None, 0.0, None, d, 64, st)),
    ("cheb_spmm_step16: f % 8 != 0", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_cheb_spmm_step16(
        64, a, b, c, 1.0, d, 0.0, None, 0.0, None, e, f, 12, st)),
    ("to_bf16: count % 8 != 0", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_to_bf16(a, b, 12, st)),
    ("obs_to_node_major: xo NULL with C = 3", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_obs_to_node_major(
        a, None, b, 4, 5, 6, 3, st)),
    ("proj_fwd: pooling with q != p", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_proj_fwd(
        a, 768, 2, 64, 12, b, c, 16, 1, d, e, 4, None, st)),
    ("proj_fwd: pooling with rows % b_inner != 0", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_proj_fwd(
        a, 768, 2, 64, 12, b, c, 12, 1, d, e, 5, None, st)),
    ("proj_pack_tc: ks = 9", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_proj_pack_tc(a, 9, b, c, st)),
    ("proj_bwd: d_out and d_out_bcast", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_proj_bwd(
        a, 768, 1, 64, 12, b, 12, 1, c, d, e, 1.0, 4, f, a, None, None, 0, None, st)),
    ("proj_bwd: u without wt", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_proj_bwd(
        a, 768, 1, 64, 12, None, 12, 1, c, d, None, 1.0, 4, e, f, None, b, 768, None, st)),
    ("gate_fwd: T = 5000", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_gate_fwd(a, 2, 5000, 10, b, c, d, e, f, st)),
    ("gate_bwd: T = 3000", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_gate_bwd(a, b, c, d, 2, 3000, e, f, a, b, st)),
    ("lstm_fwd: H = 6", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm_fwd(
        3, 2, 8, 6, 1, 2, a, b, c, d, e, None, None, f, a, b, st)),
    ("lstm_bwd: C = 5", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm_bwd(
        3, 2, 8, 8, 5, 2, a, b, c, d, None, None, e, f, a, b, c, d, e, f, a, b, c, st)),
    ("lstm16_pack: C = 5", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm16_pack(a, b, c, d, 0, 5, e, f, a, st)),
    ("lstm16_fwd: planes = 3", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm16_fwd(
        3, 2, 100, 1, 4, 3, a, b, c, d, e, None, None, f, a, b, None, st)),
    ("lstm16_bwd: T = 65", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm16_bwd(
        65, 2, 100, 1, 4, 2, a, b, c, d, e, None, None, f, a, b, c, d, e, f, a, b, c, d, st)),
    ("lstm16_bwd: dx_work NULL with L = 2", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_lstm16_bwd(
        5, 2, 100, 1, 4, 2, a, b, c, d, e, None, None, f, a, b, c, d, None, f, a, b, c, d, st)),
    ("fuse_out_fwd: M = 9", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_fuse_out_fwd(
        pa([a] * 9), 9, 4, 2, 8, 2, b, c, d, e, st)),
    ("fuse_out_bwd: C*G beyond shared memory", lambda L, pa, st, a, b, c, d, e, f: L.stmgcn_fuse_out_bwd(
        a, b, 4, 2, 400, 40, c, d, e, f, st)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", REJECTS, ids=[r[0] for r in REJECTS])
def test_rejected_calls_enqueue_nothing_and_change_nothing(case):
    """Valid guarded buffers, one bad argument: the call returns < 0 with a message, launches nothing and leaves every
    buffer bit-identical (the pooling checks of stmgcn_proj_fwd used to run after its GEMM had written ``out``)."""
    from stmgcn_b200 import _lib as lib_mod
    what, call = case
    gen = torch.Generator().manual_seed(0)
    bufs = [Buf("in", torch.randn(1 << 16, generator=gen)) for _ in range(6)]
    torch.cuda.synchronize()
    n0 = _lib().stmgcn_launch_count()
    rc = call(_lib(), lib_mod.ptr_array, _stream(), *(x.p for x in bufs))
    torch.cuda.synchronize()
    assert rc < 0, f"{what}: rc={rc}"
    assert _lib().stmgcn_last_error(), f"{what}: no message"
    assert _lib().stmgcn_launch_count() == n0, f"{what}: a kernel was launched"
    for i, x in enumerate(bufs):
        assert x.guards_intact() and torch.equal(_bits(x.t), _bits(x.init)), f"{what}: buffer {i} changed"


CAPTURED = {
    "spmm_steps_and_bf16_copy": lambda: _spmm_calls(1000, 264, "alias"),
    "obs_to_node_major": lambda: _obs_calls(3),
    "projection_tensor_cores": lambda: _proj_calls(5, 64, 64, *_tc_shape(129), 0, True, False, True, True, seed=1),
    "projection_ffma_pool": lambda: _proj_calls(4, 12, 12, 33, 5, 0, False, True, True, True, seed=2),
    "context_gate": lambda: _gate_calls(12, 5),
    "exact_lstm": lambda: _lstm_calls(7, 5, True),
    "tensor_core_lstm": lambda: _lstm16_calls(LSTM16_CASES[2], 2),
    "fuse_out": lambda: _fuse_calls(3, 40),
}


@pytest.mark.gpu
@pytest.mark.parametrize("family", list(CAPTURED))
def test_entry_points_enqueue_on_the_given_stream_and_replay_from_a_cuda_graph(family):
    """Every entry point: an eager call on a side stream, then the same call captured with torch.cuda.graph (global
    capture mode) and replayed; the replay equals the eager call.  Covers lstm.cu, the FFMA projection and fuse_out_bwd,
    which the model-level graph test does not capture."""
    _drive(CAPTURED[family](), run_captured)
