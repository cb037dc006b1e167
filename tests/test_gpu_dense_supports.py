"""GPU tests of dense support matrices multiplied dense (stmgcn_dense_mm_step / _step16, K1e): the kernels against fp64
at every edge, their C-ABI contract, the modules on the dense path against the fp64 dense restatement, the dispatch
rule at work, a cfg3-sized step on dense graphs, non-finite tracing, graph replay, and negative controls."""
import itertools

import pytest
import torch

import full_batch
from dense_support_grad_cases import (STACK_KINDS, DenseStackReference, chains_of, make_stack, model_reference,
                                      symmetric_graph)
from helpers import DEV, TOL, lib, rel_err
from model_cases import CHUNK, FullBatchRecorder, bf16_mode  # noqa: F401 (bf16_mode: a fixture)
from support_grad_cases import record_relu_masks

pytestmark = pytest.mark.gpu

KTOL = 2e-5          # the kernel-level bar: one 3xTF32 product against fp64


@pytest.fixture
def dense_mode():
    """Set the dense-supports mode for one test (restored afterwards; the conversion cache is keyed on it)."""
    from stmgcn_b200 import ops
    old = ops.dense_supports()
    yield ops.set_dense_supports
    ops.set_dense_supports(old)


@pytest.fixture(params=["tc", "fma"])
def path(request):
    from stmgcn_b200 import ops
    old = ops.lstm_path()
    ops.set_lstm_path(request.param)
    yield request.param
    ops.set_lstm_path(old)


def _step(n, a, lda, tr, alpha, x, beta, z, gamma, u, y, f):
    return lib().stmgcn_dense_mm_step(n, a.data_ptr(), lda, int(tr), alpha, x.data_ptr(), beta,
                                      None if z is None else z.data_ptr(), gamma, None if u is None else u.data_ptr(),
                                      y.data_ptr(), f, torch.cuda.current_stream().cuda_stream)


def _step16(n, a, lda, tr, alpha, x16, beta, z, gamma, u, y, y16, f):
    return lib().stmgcn_dense_mm_step16(n, a.data_ptr(), lda, int(tr), alpha, x16.data_ptr(), beta,
                                        None if z is None else z.data_ptr(), gamma,
                                        None if u is None else u.data_ptr(), y.data_ptr(),
                                        None if y16 is None else y16.data_ptr(), f,
                                        torch.cuda.current_stream().cuda_stream)


def _buf(numel, gen, off=0):
    return torch.randn(off + numel, device=DEV, generator=gen)[off:]


def _ref(n, a, lda, tr, alpha, x, beta, z, gamma, u, f):
    am = a.double().as_strided((n, n), (lda, 1))
    am = am.t() if tr else am
    r = alpha * (am @ x.double().view(n, f))
    if z is not None:
        r = r + beta * z.double().view(n, f)
    if u is not None:
        r = r + gamma * u.double().view(n, f)
    return r


SWEEP = [(n, f, i) for i, (n, f) in enumerate(itertools.product((1, 5, 127, 128, 129, 300, 1024),
                                                                 (1, 3, 4, 8, 31, 33, 768, 4096)))]
SWEEP.append((4096, 4096, len(SWEEP)))             # cfg3's spatial step: 4096-term contractions


@pytest.mark.parametrize("n,f,i", SWEEP)
def test_kernel_against_fp64(n, f, i):
    """Transpose on and off, z and u null or not, lda > n on every third case; reruns bit-identical."""
    gen = torch.Generator(device=DEV).manual_seed(i)
    lda = n + (3 if i % 3 == 0 else 0)
    a = _buf(n * lda, gen)
    x, z, u = (_buf(n * f, gen) for _ in range(3))
    for tr in (False, True):
        zz = z if i % 2 == 0 else None
        uu = u if i % 4 < 2 else None
        y = torch.full((n * f,), float("nan"), device=DEV)
        assert _step(n, a, lda, tr, 1.5, x, -0.5, zz, 0.75, uu, y, f) == 0
        assert rel_err(y.view(n, f), _ref(n, a, lda, tr, 1.5, x, -0.5, zz, 0.75, uu, f)) <= KTOL, (tr, zz is None, uu is None)
        again = torch.empty_like(y)
        assert _step(n, a, lda, tr, 1.5, x, -0.5, zz, 0.75, uu, again, f) == 0
        assert torch.equal(y, again)


@pytest.mark.parametrize("off", [1, 2, 3])
@pytest.mark.parametrize("tr", [False, True])
def test_kernel_misaligned_pointers_and_y_aliasing_u(off, tr):
    """Every operand off 16-byte alignment (the scalar variant), and y == u (the adjoint Clenshaw's y = u[k])."""
    n, f = 133, 64
    gen = torch.Generator(device=DEV).manual_seed(off)
    a, x, z, u = _buf(n * n, gen, off), _buf(n * f, gen, off), _buf(n * f, gen, off), _buf(n * f, gen, off)
    ref = _ref(n, a, n, tr, 2.0, x, -1.0, z, 1.0, u, f)
    assert _step(n, a, n, tr, 2.0, x, -1.0, z, 1.0, u, u, f) == 0
    assert rel_err(u.view(n, f), ref) <= KTOL


@pytest.mark.parametrize("n,f", [(1, 8), (129, 8), (300, 40), (1024, 768), (4096, 4096)])
@pytest.mark.parametrize("tr", [False, True])
def test_bf16_twin_against_fp64_of_the_bf16_operand(n, f, tr):
    """The product of the bf16 copy x16, fp32 z / u / y, and y16 == to_bf16(y) bit for bit."""
    from stmgcn_b200 import ops
    gen = torch.Generator(device=DEV).manual_seed(n + f)
    a, x, z = _buf(n * n, gen), _buf(n * f, gen), _buf(n * f, gen)
    x16 = x.to(torch.bfloat16)
    y = torch.empty(n * f, device=DEV)
    y16 = torch.empty(n * f, device=DEV, dtype=torch.bfloat16)
    assert _step16(n, a, n, tr, 2.0, x16, -1.0, z, 0.0, None, y, y16, f) == 0
    assert rel_err(y.view(n, f), _ref(n, a, n, tr, 2.0, x16.float(), -1.0, z, 0.0, None, f)) <= KTOL
    assert torch.equal(y16.view(torch.int16), ops.to_bf16(y).view(torch.int16))


# ---- C-ABI contract --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("captured", [False, True])
@pytest.mark.parametrize("twin", [False, True])
def test_c_abi_contract_guard_bands_poisoned_output_const_inputs_launch_count(captured, twin):
    """y (and y16) overwritten in full from a NaN-poisoned start, nothing outside them written, the inputs left bit for
    bit, one launch per call; eagerly and replayed from a graph captured on a side stream."""
    n, f, guard = 300, 40, 4096
    gen = torch.Generator(device=DEV).manual_seed(11)
    a, x, z, u = _buf(n * n, gen), _buf(n * f, gen), _buf(n * f, gen), _buf(n * f, gen)
    x16 = x.to(torch.bfloat16)
    ins = [t.clone() for t in (a, x, z, u, x16)]
    buf = torch.full((n * f + 2 * guard,), 7.25, device=DEV)
    y = buf[guard:guard + n * f]
    y.fill_(float("nan"))
    buf16 = torch.full((n * f + 2 * guard,), 3.5, device=DEV, dtype=torch.bfloat16)
    y16 = buf16[guard:guard + n * f]
    y16.fill_(float("nan"))

    def call():
        if twin:
            return _step16(n, a, n, True, 2.0, x16, -1.0, z, 1.0, u, y, y16, f)
        return _step(n, a, n, True, 2.0, x, -1.0, z, 1.0, u, y, f)

    n0 = lib().stmgcn_launch_count()
    if captured:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(side), torch.cuda.graph(g, stream=side):
            assert call() == 0
        torch.cuda.current_stream().wait_stream(side)
        g.replay()
    else:
        assert call() == 0
    torch.cuda.synchronize()
    assert lib().stmgcn_launch_count() - n0 == 1
    assert torch.isfinite(y).all()
    assert rel_err(y.view(n, f), _ref(n, a, n, True, 2.0, x16.float() if twin else x, -1.0, z, 1.0, u, f)) <= KTOL
    assert (buf[:guard] == 7.25).all() and (buf[guard + n * f:] == 7.25).all()
    if twin:
        assert torch.isfinite(y16.float()).all()
        assert (buf16[:guard] == 3.5).all() and (buf16[guard + n * f:] == 3.5).all()
    for t, t0 in zip((a, x, z, u, x16), ins):
        assert torch.equal(t, t0)


def test_rejected_arguments_launch_nothing():
    n, f = 64, 16
    gen = torch.Generator(device=DEV).manual_seed(2)
    a, x, z = _buf(n * n, gen), _buf(n * f, gen), _buf(n * f, gen)
    x16 = x.to(torch.bfloat16)
    y = torch.empty(n * f, device=DEV)
    y16 = torch.empty(n * f, device=DEV, dtype=torch.bfloat16)
    n0 = lib().stmgcn_launch_count()
    bad = [
        lambda: _step(0, a, n, False, 1.0, x, 0.0, None, 0.0, None, y, f),            # n
        lambda: _step(n, a, n - 1, False, 1.0, x, 0.0, None, 0.0, None, y, f),        # lda < n
        lambda: _step(n, a, n, 2, 1.0, x, 0.0, None, 0.0, None, y, f),                # transpose
        lambda: _step(n, a, n, False, 1.0, x, 0.0, None, 0.0, None, y, 0),            # f_total
        lambda: _step(n, a, n, False, 1.0, x, 0.0, None, 0.0, None, x, f),            # y is x
        lambda: _step(n, a, n, False, 1.0, x, 1.0, z, 0.0, None, z, f),               # y is z
        lambda: _step(n, a, n, False, 1.0, x, 0.0, None, 0.0, None, a[:n * f], f),    # y inside a
        lambda: _step(n, a, n, False, 1.0, x, 0.0, None, 1.0, y[1:], y[:-1], f),      # u overlaps y, not y
        lambda: _step16(n, a, n, False, 1.0, x16, 0.0, None, 0.0, None, y, y16, 12),  # f_total % 8
        lambda: _step16(n, a, n, False, 1.0, x16, 0.0, None, 0.0, None, y, x16, f),   # y16 is x16
        lambda: _step16(n, a, n, False, 1.0, x16, 0.0, None, 0.0, None, y[1:], y16, f - 8),  # y misaligned
    ]
    for i, call in enumerate(bad):
        assert call() < 0, i
    torch.cuda.synchronize()
    assert lib().stmgcn_launch_count() == n0


def test_nan_reaches_every_row_and_inf_gives_nan():
    """A dense product forms 0 * NaN: a NaN in row j of X reaches every row of Y in its column, whatever A's zeros; an Inf
    operand gives NaN (inf_through_split_operands)."""
    n, f = 150, 64
    gen = torch.Generator(device=DEV).manual_seed(4)
    a = _buf(n * n, gen)
    a.view(n, n)[:, 99] = 0.0                      # no row has a non-zero in column 99 ...
    x = _buf(n * f, gen)
    x.view(n, f)[99, 5] = float("nan")             # ... and the NaN there still reaches every row of column 5
    x.view(n, f)[10, 7] = float("inf")
    y = torch.empty(n * f, device=DEV)
    assert _step(n, a, n, False, 1.0, x, 0.0, None, 0.0, None, y, f) == 0
    yv = y.view(n, f)
    assert torch.isnan(yv[:, 5]).all() and torch.isnan(yv[:, 7]).all()
    keep = torch.ones(f, dtype=torch.bool, device=DEV)
    keep[[5, 7]] = False
    assert torch.isfinite(yv[:, keep]).all()
    ref = _ref(n, a, n, False, 1.0, x.view(n, f)[:, keep].contiguous(), 0.0, None, 0.0, None, f - 2)
    assert rel_err(yv[:, keep], ref) <= KTOL


# ---- modules on the dense path ---------------------------------------------------------------------------------------
N, B, T, C, H, LAYERS, G = 37, 3, 6, 1, 64, 2, 64


def _inputs(seed, b=B, n=N):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(b, T, n, C, device=DEV, generator=gen), torch.randn(b, n, C, device=DEV, generator=gen)


def _model(ks, m, n=N, seed=0):
    import STMGCN
    torch.manual_seed(seed)
    kt, k = ("localpool", 1) if ks == 1 else ("chebyshev", ks - 1)
    return STMGCN.ST_MGCN(M=m, seq_len=T, n_nodes=n, input_dim=C, lstm_hidden_dim=H, lstm_num_layers=LAYERS,
                          gcn_hidden_dim=G, sta_kernel_config={"kernel_type": kt, "K": k}, gconv_use_bias=True).to(DEV)


def _graph_types(stacks):
    from stmgcn_b200 import graph
    return {type(g).__name__ for s in stacks for g in graph.supports_from_dense(s).graphs}


def _check_st_mgcn(stacks, learn, seed=0, obs_grad=False, what=""):
    """Loss, output, parameter gradients (and, ``learn``, stack gradients; ``obs_grad``, obs.grad) of ST_MGCN against
    the fp64 dense restatement at the kernels' ReLU masks."""
    model = _model(stacks[0].shape[0], len(stacks), seed=seed)
    x, y = _inputs(seed)
    x.requires_grad_(obs_grad)
    sups = [s.detach().clone().requires_grad_(True) for s in stacks] if learn else stacks
    with record_relu_masks() as rec:
        out = model(obs_seq=x, sta_adj_list=sups)
    loss = torch.mean((out - y) ** 2)
    loss.backward()
    params = {k: v.detach() for k, v in model.named_parameters()}
    out64, loss64, grads, sgrads = model_reference(params, x, y, stacks, list(range(len(stacks))), masks=rec.masks,
                                                   device=DEV)
    assert rel_err(out, out64) <= TOL, what
    assert abs(float(loss.detach()) - loss64) <= TOL * abs(loss64), what
    for k, p in model.named_parameters():
        assert rel_err(p.grad, grads[k]) <= TOL, (what, k)
    if learn:
        for s, g in zip(sups, sgrads):
            assert rel_err(s.grad, g) <= TOL, what
    if obs_grad:
        x64 = x.detach().double().requires_grad_(True)
        import stmgcn_oracle as O
        o = O.dense_st_mgcn({k: v.double() for k, v in params.items()}, x64, [s.double() for s in stacks],
                            masks=rec.masks)
        torch.mean((o - y.double()) ** 2).backward()
        assert rel_err(x.grad, x64.grad) <= TOL, what


@pytest.mark.parametrize("kind", STACK_KINDS)
@pytest.mark.parametrize("streams", ["1", "0"])
def test_st_mgcn_on_the_dense_path_against_fp64(monkeypatch, dense_mode, path, kind, streams):
    monkeypatch.setenv("STMGCN_GRAPH_STREAMS", streams)
    dense_mode("on")
    stacks = [make_stack(kind, N, s, device=DEV) for s in range(3)]
    if kind != "k0":
        assert _graph_types(stacks) == {"DenseGraph"}
    _check_st_mgcn(stacks, learn=False, obs_grad=True, what=f"{kind} constant")
    _check_st_mgcn(stacks, learn=True, what=f"{kind} learned")


@pytest.mark.parametrize("kind", ["cheb", "generic", "diffusion"])
def test_gcn_and_cg_lstm_on_the_dense_path_against_fp64(dense_mode, path, kind):
    import GCN
    import STMGCN
    import stmgcn_oracle as O
    dense_mode("on")
    stack = make_stack(kind, N, 3, device=DEV)
    ks = stack.shape[0]
    torch.manual_seed(0)
    gcn = GCN.GCN(K=ks, input_dim=64, hidden_dim=64).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(B, N, 64, device=DEV, generator=gen)
    probe = torch.randn(B, N, 64, device=DEV, generator=gen)
    leaf = stack.clone().requires_grad_(True)
    with record_relu_masks() as rec:
        out = gcn(leaf, x)
    (out * probe).sum().backward()
    s64 = stack.double().requires_grad_(True)
    w64 = gcn.W.detach().double().requires_grad_(True)
    ref = O.dense_gcn(s64, x.double(), w64, gcn.b.detach().double(), True, rec.masks[0])
    (ref * probe.double()).sum().backward()
    assert rel_err(out, ref) <= TOL and rel_err(gcn.W.grad, w64.grad) <= TOL and rel_err(leaf.grad, s64.grad) <= TOL

    torch.manual_seed(0)
    cg = STMGCN.CG_LSTM(seq_len=T, n_nodes=N, input_dim=C, lstm_hidden_dim=H, lstm_num_layers=LAYERS, K=ks,
                        gconv_use_bias=True).to(DEV)
    xo, _ = _inputs(2)
    probe = torch.randn(B, N, H, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    leaf = stack.clone().requires_grad_(True)
    with record_relu_masks() as rec:
        out, _ = cg(leaf, xo, None)
    (out * probe).sum().backward()
    params = {"rnn_list.0." + k: v.detach() for k, v in cg.named_parameters()}
    out64, _, grads, sgrads = model_reference(params, xo, None, [stack], [0], masks=rec.masks, device=DEV, cg_probe=probe)
    assert rel_err(out, out64) <= TOL
    for k, p in cg.named_parameters():
        assert rel_err(p.grad, grads["rnn_list.0." + k]) <= TOL, k
    assert rel_err(leaf.grad, sgrads[0]) <= TOL


def test_learned_stacks_after_adam_steps_through_process(dense_mode):
    """adj.grad through process() after Adam steps have filled the stacks in, on the dense path, against fp64."""
    import GCN
    import stmgcn_oracle as O
    dense_mode("on")
    model = _model(3, 2)
    x, y = _inputs(5)
    adjs = [symmetric_graph(N, 20 + g, device=DEV).requires_grad_(True) for g in range(2)]
    pre = GCN.Adj_Preprocessor("chebyshev", 2)
    opt = torch.optim.Adam(adjs, lr=1e-2)
    for _ in range(2):
        opt.zero_grad()
        torch.mean((model(obs_seq=x, sta_adj_list=[pre.process(a) for a in adjs]) - y) ** 2).backward()
        opt.step()
    assert min(float((pre.process(a.detach())[1] != 0).float().mean()) for a in adjs) > 0.9   # filled in
    for a in adjs:
        a.grad = None
    model.zero_grad()
    with record_relu_masks() as rec:
        out = model(obs_seq=x, sta_adj_list=[pre.process(a) for a in adjs])
    torch.mean((out - y) ** 2).backward()
    a64 = [a.detach().double().requires_grad_(True) for a in adjs]
    params = {k: v.detach().double() for k, v in model.named_parameters()}
    o = O.dense_st_mgcn(params, x.double(), [GCN.Adj_Preprocessor("chebyshev", 2).process(a) for a in a64],
                        masks=rec.masks)
    torch.mean((o - y.double()) ** 2).backward()
    for a, r in zip(adjs, a64):
        assert rel_err(a.grad, r.grad) <= TOL


# ---- dispatch ----------------------------------------------------------------------------------------------------------
def test_auto_dispatches_dense_stacks_dense_and_sparse_ones_to_csr_and_the_modes_agree(dense_mode):
    import GCN
    from stmgcn_b200 import graph, synth
    n = 4096
    pre = GCN.Adj_Preprocessor("chebyshev", 3)
    dense = pre.process(synth.make_similarity_adjacency(n, 0).to(DEV))
    sparse = pre.process(synth.make_adjacency(n, 0, 0.01).to(DEV))
    dense_mode("auto")
    assert _graph_types([dense]) == {"DenseGraph"} and _graph_types([sparse]) == {"GraphHandle"}
    dense_mode("on")
    assert _graph_types([sparse]) == {"DenseGraph"}
    dense_mode("off")
    assert _graph_types([dense]) == {"GraphHandle"}
    # the two paths agree within the bar on one GCN
    gcn = GCN.GCN(K=4, input_dim=64, hidden_dim=64).to(DEV)
    x = torch.randn(2, n, 64, device=DEV, generator=torch.Generator(device=DEV).manual_seed(0))
    outs = {}
    for mode in ("on", "off"):
        dense_mode(mode)
        with torch.no_grad():
            outs[mode] = gcn(dense, x)
    assert rel_err(outs["on"], outs["off"]) <= TOL


def test_cfg3_step_on_three_dense_graphs_against_fp64(dense_mode):
    """cfg3 at full size (4096 regions, 3 graphs, K = 3, T = 12, batch 64, every window with its true target) on
    process() of three dense similarity graphs under auto: loss and every parameter gradient within 1e-4 of the fp64
    reference, taken at the step's ReLU masks, a chunk of windows at a time."""
    import GCN
    import STMGCN
    from stmgcn_b200 import synth
    dense_mode("auto")
    w = synth.WORKLOADS["cfg3"]
    pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
    stacks = [pre.process(synth.make_similarity_adjacency(w.n_regions, m).to(DEV)) for m in range(w.n_graphs)]
    assert _graph_types(stacks) == {"DenseGraph"}
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(**synth.model_kwargs(w)).to(DEV)
    params = {k: v.detach().clone() for k, v in model.state_dict().items()}
    x, y = synth.make_inputs(w, seed=0)
    got = full_batch.gpu_step(model, stacks, x, y)
    ref = DenseStackReference(params, [chains_of(s) for s in stacks], w.n_supports, relu=True, rounding=False,
                              relu_masks=got["masks"], device=DEV)
    out, loss, grads = ref.loss_and_grads(x, y, window_chunk=CHUNK["cfg3"])
    assert rel_err(got["out"], out) <= TOL
    assert abs(got["loss"] - float(loss)) <= TOL * abs(float(loss))
    errs = {k: rel_err(g, grads[k]) for k, g in got["grads"].items()}
    print(f"cfg3 B={w.batch} on dense graphs: worst gradient {max(errs.values()):.2e} against fp64")
    assert max(errs.values()) <= TOL, errs


def test_nan_in_one_window_stays_in_that_window_and_the_non_finite_pattern_is_the_oracles(dense_mode):
    """A NaN in one window's obs: that window's output is NaN, the others finite, and which outputs are non-finite is
    exactly what the fp64 dense oracle (torch's ReLU) gives; the finite ones agree with it."""
    import stmgcn_oracle as O
    dense_mode("on")
    stacks = [make_stack("cheb", N, s, device=DEV) for s in range(3)]
    assert _graph_types(stacks) == {"DenseGraph"}
    model = _model(3, 3)
    x, _ = _inputs(1)
    x[1, 2, 7, 0] = float("nan")
    with torch.no_grad():
        out = model(obs_seq=x, sta_adj_list=stacks)
        params = {k: v.detach().double() for k, v in model.named_parameters()}
        ref = O.dense_st_mgcn(params, x.double(), [s.double() for s in stacks])
    assert torch.isnan(out[1]).all()
    assert torch.isfinite(out[[0, 2]]).all()
    assert torch.equal(torch.isfinite(out), torch.isfinite(ref))
    fin = torch.isfinite(ref)
    assert rel_err(out[fin], ref[fin]) <= TOL


@pytest.mark.parametrize("streams", ["1", "0"])
def test_bf16_mode_on_the_dense_path_against_the_forced_reference(monkeypatch, bf16_mode, dense_mode, streams):
    """bf16-arithmetic mode with dense Chebyshev stacks on the dense path (the bf16 twin, stmgcn_dense_mm_step16, runs
    the spatial recurrence): every spatial Chebyshev term one step from the kernels' own bf16-rounded previous term,
    and the loss and every parameter gradient, within 1e-4 of the forced fp64 reference that rounds where the kernels
    round."""
    monkeypatch.setenv("STMGCN_GRAPH_STREAMS", streams)
    _bf16_dense_errors(dense_mode, fault=False)


def _bf16_dense_errors(dense_mode, fault, monkeypatch=None):
    from stmgcn_b200 import graph, ops
    dense_mode("on")
    stacks = [make_stack("cheb", N, s, device=DEV) for s in range(2)]
    assert _graph_types(stacks) == {"DenseGraph"}
    twin = []
    real16 = ops.spmm_step16

    def witness(g, *a):
        twin.append(isinstance(g, graph.DenseGraph))
        real16(g, *a)
    if fault:
        real_chain = ops._cheb_chain_

        def fp32_operand_chain(g, t, gather16):
            # the twin reading the fp32 operand: the dense steps multiply t[k - 1], not its bf16 copy
            real_chain(g, t, gather16 and not isinstance(g, graph.DenseGraph))
        monkeypatch.setattr(ops, "_cheb_chain_", fp32_operand_chain)
    else:
        ops_mp = pytest.MonkeyPatch()
        ops_mp.setattr(ops, "spmm_step16", witness)
    model = _model(stacks[0].shape[0], 2)
    x, y = _inputs(11)
    params = {k: v.detach().clone() for k, v in model.state_dict().items()}
    try:
        with FullBatchRecorder() as rec:
            got = full_batch.gpu_step(model, stacks, x, y)
    finally:
        if not fault:
            ops_mp.undo()
    rec.check_intact()
    if not fault:
        assert twin and all(twin)
    tapes = rec.take_tapes()
    # each spatial Chebyshev term one step from the kernels' own previous terms: S_1 = L~ bf16(S_0),
    # S_k = 2 L~ bf16(S_{k-1}) - S_{k-2}
    errs = []
    for m, st in enumerate(stacks):
        lap, t = st[1].double(), [v.reshape(N, -1) for v in tapes[m]["s"]]
        for k in range(1, st.shape[0]):
            want = lap @ t[k - 1].to(torch.bfloat16).double()
            if k > 1:
                want = 2.0 * want - t[k - 2].double()
            errs.append(rel_err(t[k], want))
    ref = DenseStackReference(params, [chains_of(s) for s in stacks], stacks[0].shape[0], relu=True,
                              relu_masks=got["masks"], device=DEV)
    _, loss, grads = ref.loss_and_grads(x, y, tapes=tapes)
    errs += [abs(got["loss"] - float(loss)) / abs(float(loss))] + [rel_err(g, grads[k]) for k, g in got["grads"].items()]
    if not fault:
        assert max(errs) <= TOL, errs
    return max(errs)


def test_negative_control_bf16_twin_reading_the_fp32_operand_fails_the_bar(monkeypatch, bf16_mode, dense_mode, capsys):
    worst = _bf16_dense_errors(dense_mode, fault=True, monkeypatch=monkeypatch)
    with capsys.disabled():
        print(f"\n[negative control fp32_operand] worst error {worst:.2e} against the forced bf16 reference, bar {TOL:.0e}")
    assert worst > TOL


def _eager_step(model, crit, x, y, sups):
    """Loss and gradients of one eager step (its autograd graph is freed on return, before any capture)."""
    for p in model.parameters():
        p.grad = None
    loss = crit(model(obs_seq=x, sta_adj_list=sups), y)
    loss.backward()
    return loss.item(), {k: p.grad.detach().clone() for k, p in model.named_parameters()}


def test_graphed_step_replay_equals_eager_on_the_dense_path(dense_mode):
    from torch import nn
    from stmgcn_b200 import dp, graphs
    dense_mode("on")
    stacks = [make_stack("cheb", N, s, device=DEV) for s in range(3)]
    assert _graph_types(stacks) == {"DenseGraph"}
    model = _model(3, 3)
    crit = nn.MSELoss()
    x, y = _inputs(3)
    eager, g_eager = _eager_step(model, crit, x, y, stacks)
    step = graphs.GraphedStep(model, crit, x, y, stacks, bucket=dp.GradBucket(model))
    loss = step(x, y).item()
    assert abs(loss - eager) <= 1e-5 * abs(eager)
    for k, p in model.named_parameters():
        assert rel_err(p.grad, g_eager[k]) <= 2e-5, k


# ---- negative controls -------------------------------------------------------------------------------------------------
def _fault(monkeypatch, which):
    from stmgcn_b200 import graph, ops
    step = ops.spmm_step

    def bad(g, transpose, alpha, x, beta, z, gamma, u, y):
        if isinstance(g, graph.DenseGraph):
            if which == "no_transpose":
                transpose = False
            elif which == "no_beta_z":
                beta, z = 0.0, None
        step(g, transpose, alpha, x, beta, z, gamma, u, y)

    monkeypatch.setattr(ops, "spmm_step", bad)


@pytest.mark.parametrize("which", ["no_transpose", "no_beta_z"])
def test_negative_controls_fail_the_bar(monkeypatch, dense_mode, capsys, which):
    """A in place of A^T in the adjoint (the asymmetric slices of a dense diffusion stack) and the beta Z term of the
    Chebyshev recurrence dropped (a Chebyshev stack): each misses the bar."""
    dense_mode("on")
    kind = "diffusion" if which == "no_transpose" else "cheb"
    stacks = [make_stack(kind, N, s, device=DEV) for s in range(3)]
    _fault(monkeypatch, which)
    with pytest.raises(AssertionError):
        _check_st_mgcn(stacks, learn=True, what=which)
    model = _model(stacks[0].shape[0], 3)
    x, y = _inputs(0)
    x.requires_grad_(True)
    with record_relu_masks() as rec:
        out = model(obs_seq=x, sta_adj_list=stacks)
    torch.mean((out - y) ** 2).backward()
    params = {k: v.detach() for k, v in model.named_parameters()}
    _, _, grads, _ = model_reference(params, x, y, stacks, [0, 1, 2], masks=rec.masks, device=DEV)
    worst = max(rel_err(p.grad, grads[k]) for k, p in model.named_parameters())
    with capsys.disabled():
        print(f"\n[negative control {which}] worst parameter gradient {worst:.2e} against the bar {TOL:.0e}")
    assert worst > TOL
