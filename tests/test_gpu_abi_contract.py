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
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from abi_harness import (GUARD, LSTM16_CASES, Buf, Call, bits, cuda_stream, drive, fuse_calls, gate_calls, lstm16_calls,
                         lstm_calls, proj_calls, run_captured, run_contract)
from helpers import DEV, FWD_TOL, lib, rel_err, sm_count
from kernel_cases import ACTS, isolated_matrix, proj_rows, tc_shape


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
        err = rel_err(res["y"], 2.0 * (op64 @ x.double().to(DEV)) - z64 + 0.5 * u64)
        assert err <= FWD_TOL, f"cheb_spmm_step n={n} f={f} {variant}: {err:.2e}"

    yield Call("cheb_spmm_step", b, lambda st, b=b: lib().stmgcn_cheb_spmm_step(
        n, b["rowptr"].p, b["colidx"].p, b["vals"].p, 2.0, b["x"].p, -1.0, b["z"].p, 0.5, b[uk].p, b["y"].p, f, st), ref32, 1)
    x16 = x.to(torch.bfloat16)
    if f % 8 == 0:
        b = dict(operands(), x16=Buf("in", x16), y16=Buf("out", shape=(n, f), dtype=torch.bfloat16))

        def ref16(res):
            err = rel_err(res["y"], 2.0 * (op64 @ x16.double().to(DEV)) - z64 + 0.5 * u64)
            assert err <= FWD_TOL, f"cheb_spmm_step16 n={n} f={f} {variant}: {err:.2e}"
            assert torch.equal(bits(res["y16"]), bits(res["y"].to(torch.bfloat16))), "y16 is not bf16(y)"

        yield Call("cheb_spmm_step16", b, lambda st, b=b: lib().stmgcn_cheb_spmm_step16(
            n, b["rowptr"].p, b["colidx"].p, b["vals"].p, 2.0, b["x16"].p, -1.0, b["z"].p, 0.5, b[uk].p, b["y"].p,
            b["y16"].p, f, st), ref16, 1)
    if (n * f) % 8 == 0:
        yield from _to_bf16_calls(x.reshape(-1))


def _to_bf16_calls(x, finite=True):
    b = dict(x=Buf("in", x), y16=Buf("out", shape=x.shape, dtype=torch.bfloat16, finite=finite))

    def ref(res):
        want = x.to(torch.bfloat16).to(DEV)
        nan = torch.isnan(x).to(DEV)
        assert torch.equal(bits(res["y16"])[~nan], bits(want)[~nan]), "to_bf16 differs from torch's rounding"
        assert bool(torch.isnan(res["y16"][nan]).all()), "to_bf16 turned a NaN into a number"

    yield Call("to_bf16", b, lambda st: lib().stmgcn_to_bf16(b["x"].p, b["y16"].p, x.numel(), st), ref, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("n,f,variant", SPMM_CASES)
def test_spmm_steps_keep_the_memory_contract(n, f, variant):
    """f = 7: the scalar kernel; 40: float4 with a partial column tile; 264: several column tiles."""
    drive(_spmm_calls(n, f, variant), run_contract)


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
    drive(_to_bf16_calls(x, finite=False), run_contract)


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

    yield Call("obs_to_node_major", b, lambda st: lib().stmgcn_obs_to_node_major(
        b["obs"].p, b["xo"].p if c > 1 else None, b["xt"].p, b_sz, t, n, c, st), ref, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [1, 3])
def test_obs_to_node_major_keeps_the_memory_contract(c):
    """C = 1 with xo NULL (xt alone), C = 3."""
    drive(_obs_calls(c), run_contract)


# ======================================================================================================================
# K2: projection
# ======================================================================================================================
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
    n, b_sz = tc_shape(rows_id)
    relu, bias = ACTS[PROJ_TC.index((ks, rows_id, gap)) % 4]
    drive(proj_calls(ks, 64, 64, n, b_sz, gap, True, False, relu, bias, seed=10 * ks + gap), run_contract)


@pytest.mark.gpu
@pytest.mark.parametrize("case", PROJ_FMA, ids=[c[0] for c in PROJ_FMA])
def test_projection_ffma_entry_points_keep_the_memory_contract(case):
    name, ks, p, q, n, b_sz, gap, bcast = case
    if n is None:
        n = proj_rows("waves")
    relu, bias = ACTS[PROJ_FMA.index(case) % 4]
    drive(proj_calls(ks, p, q, n, b_sz, gap, False, bcast, relu, bias, seed=100 + PROJ_FMA.index(case)), run_contract)


# ======================================================================================================================
# K3a: context gate
# ======================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("t", [12, 300])
def test_context_gate_keeps_the_memory_contract(t):
    drive(gate_calls(t, 5), run_contract)


# ======================================================================================================================
# K3b: exact-fp32 LSTM
# ======================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("state", [False, True])
def test_exact_lstm_keeps_the_memory_contract(state):
    """Ragged rows: 35 with h0 / c0; without, more rows than the backward's pointwise grid covers in one pass."""
    n, b_sz = (7, 5) if state else ((2 * 32 * sm_count()) // 5 + 1, 5)
    drive(lstm_calls(n, b_sz, state), run_contract)


# ======================================================================================================================
# K3b: tensor-core LSTM
# ======================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("planes", [1, 2])
@pytest.mark.parametrize("case", LSTM16_CASES, ids=[c[0] for c in LSTM16_CASES])
def test_tensor_core_lstm_keeps_the_memory_contract(case, planes):
    drive(lstm16_calls(case, planes), run_contract)


# ======================================================================================================================
# fusion over graphs + output FC
# ======================================================================================================================
@pytest.mark.gpu
@pytest.mark.parametrize("c", [1, 40])
@pytest.mark.parametrize("m", [1, 3])
def test_fuse_out_keeps_the_memory_contract(m, c):
    """M = 3 runs more rows than the forward's grid covers in one pass; C = 40 the second bias-gradient lane loop."""
    drive(fuse_calls(m, c), run_contract)


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
    n0 = lib().stmgcn_launch_count()
    rc = call(lib(), lib_mod.ptr_array, cuda_stream(), *(x.p for x in bufs))
    torch.cuda.synchronize()
    assert rc < 0, f"{what}: rc={rc}"
    assert lib().stmgcn_last_error(), f"{what}: no message"
    assert lib().stmgcn_launch_count() == n0, f"{what}: a kernel was launched"
    for i, x in enumerate(bufs):
        assert x.guards_intact() and torch.equal(bits(x.t), bits(x.init)), f"{what}: buffer {i} changed"


CAPTURED = {
    "spmm_steps_and_bf16_copy": lambda: _spmm_calls(1000, 264, "alias"),
    "obs_to_node_major": lambda: _obs_calls(3),
    "projection_tensor_cores": lambda: proj_calls(5, 64, 64, *tc_shape(129), 0, True, False, True, True, seed=1),
    "projection_ffma_pool": lambda: proj_calls(4, 12, 12, 33, 5, 0, False, True, True, True, seed=2),
    "context_gate": lambda: gate_calls(12, 5),
    "exact_lstm": lambda: lstm_calls(7, 5, True),
    "tensor_core_lstm": lambda: lstm16_calls(LSTM16_CASES[2], 2),
    "fuse_out": lambda: fuse_calls(3, 40),
}


@pytest.mark.gpu
@pytest.mark.parametrize("family", list(CAPTURED))
def test_entry_points_enqueue_on_the_given_stream_and_replay_from_a_cuda_graph(family):
    """Every entry point: an eager call on a side stream, then the same call captured with torch.cuda.graph (global
    capture mode) and replayed; the replay equals the eager call.  Covers lstm.cu, the FFMA projection and fuse_out_bwd,
    which the model-level graph test does not capture."""
    drive(CAPTURED[family](), run_captured)
