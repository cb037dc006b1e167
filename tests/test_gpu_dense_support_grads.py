"""GPU tests of the dense support-stack gradient: stmgcn_dense_support_grad against fp64 at every edge, its C-ABI
contract and non-finite tracing, and GCN / CG_LSTM / ST_MGCN stacks (and the adjacency behind process()) against the
fp64 dense restatement with the stacks as leaves, taken at the kernels' own ReLU masks."""
import itertools

import pytest
import torch

from dense_support_grad_cases import STACK_KINDS, dense_process, make_stack, model_reference, symmetric_graph
import full_batch
from dense_support_grad_cases import DenseStackReference, chains_of
from helpers import DEV, GRAD_TOL, TOL, lib, rel_err
from model_cases import CHUNK, FullBatchRecorder, bf16_mode, cheb_workload  # noqa: F401 (bf16_mode: a fixture)
from support_grad_cases import record_relu_masks

pytestmark = pytest.mark.gpu


def _call(n, f, ks, u, stride, x, da):
    from stmgcn_b200 import _lib
    _lib.check(lib().stmgcn_dense_support_grad(n, f, ks, u.data_ptr(), stride, x.data_ptr(), da.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream), "dense_support_grad")


def _operands(n, f, ks, seed, off=0):
    """u (ks segments of n*f floats), x, both starting ``off`` floats into their buffers."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    ub = torch.randn(off + ks * n * f, device=DEV, generator=gen)
    xb = torch.randn(off + n * f, device=DEV, generator=gen)
    return ub[off:], xb[off:]


def _ref(u, x, n, f, ks):
    return torch.einsum("kif,jf->kij", u.double().view(ks, n, f), x.double().view(n, f))


SWEEP = [(n, f, 1 + i % 8) for i, (n, f) in enumerate(itertools.product((1, 5, 127, 128, 129, 300, 1024),
                                                                        (1, 3, 4, 31, 32, 33, 768, 4096)))]


@pytest.mark.parametrize("n,f,ks", SWEEP)
def test_kernel_against_fp64(n, f, ks):
    u, x = _operands(n, f, ks, seed=n * 31 + f)
    da = torch.empty(ks, n, n, device=DEV)
    _call(n, f, ks, u, n * f, x, da)
    assert rel_err(da, _ref(u, x, n, f, ks)) <= GRAD_TOL


@pytest.mark.parametrize("ks", range(1, 9))
@pytest.mark.parametrize("off", [1, 2, 3])
def test_kernel_misaligned_pointers_and_every_ks(ks, off):
    """Operands and da off 16-byte (and 8-byte) alignment: the scalar loads and stores, same results."""
    n, f = 133, 64
    u, x = _operands(n, f, ks, seed=ks + 10 * off, off=off)
    dab = torch.empty(off + ks * n * n, device=DEV)
    da = dab[off:]
    _call(n, f, ks, u, n * f, x, da)
    assert rel_err(da.view(ks, n, n), _ref(u, x, n, f, ks)) <= GRAD_TOL


def test_kernel_at_the_cfg3_spatial_shape_and_bit_identical_reruns():
    n = f = 4096
    ks = 4
    u, x = _operands(n, f, ks, seed=7)
    da = torch.empty(ks, n, n, device=DEV)
    _call(n, f, ks, u, n * f, x, da)
    again = torch.empty_like(da)
    _call(n, f, ks, u, n * f, x, again)
    assert torch.equal(da, again)
    for k in range(ks):                                 # slice by slice: the fp64 product of all four is 4 GB
        ref = u.double().view(ks, n, f)[k] @ x.double().view(n, f).t()
        assert rel_err(da[k], ref) <= GRAD_TOL


@pytest.mark.parametrize("captured", [False, True])
def test_c_abi_contract_guard_bands_poisoned_output_const_inputs_launch_count(captured):
    """da is overwritten in full (a NaN-poisoned da comes out finite), nothing outside it is written (guard bands), u
    and x are left bit for bit, one launch per call; eagerly and replayed from a graph captured on a side stream."""
    n, f, ks, guard = 300, 33, 3, 4096
    u, x = _operands(n, f, ks, seed=5)
    u0, x0 = u.clone(), x.clone()
    buf = torch.full((ks * n * n + 2 * guard,), 7.25, device=DEV)
    da = buf[guard:guard + ks * n * n]
    da.fill_(float("nan"))
    n0 = lib().stmgcn_launch_count()
    if captured:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(side), torch.cuda.graph(g, stream=side):
            _call(n, f, ks, u, n * f, x, da)
        torch.cuda.current_stream().wait_stream(side)
        g.replay()
    else:
        _call(n, f, ks, u, n * f, x, da)
    torch.cuda.synchronize()
    assert lib().stmgcn_launch_count() - n0 == 1
    assert torch.isfinite(da).all()
    assert rel_err(da.view(ks, n, n), _ref(u, x, n, f, ks)) <= GRAD_TOL
    assert (buf[:guard] == 7.25).all() and (buf[guard + ks * n * n:] == 7.25).all()
    assert torch.equal(u, u0) and torch.equal(x, x0)


@pytest.mark.parametrize("f", [64, 33])
def test_nan_and_inf_tracing(f):
    """A NaN in row i of U_k poisons row i of dA_k alone; a NaN in row j of x column j of every dA_k; an Inf gives NaN."""
    n, ks = 150, 3
    u, x = _operands(n, f, ks, seed=9)
    uv, xv = u.view(ks, n, f), x.view(n, f)
    uv[1, 17, f - 1] = float("nan")
    uv[2, 140, 0] = float("inf")
    xv[99, 5] = float("nan")
    da = torch.empty(ks, n, n, device=DEV)
    _call(n, f, ks, u, n * f, x, da)
    bad = torch.zeros(ks, n, n, dtype=torch.bool, device=DEV)
    bad[1, 17, :] = True
    bad[2, 140, :] = True
    bad[:, :, 99] = True
    assert torch.isnan(da[bad]).all()
    assert torch.isfinite(da[~bad]).all()
    clean = torch.where(bad, torch.zeros_like(da), da)
    ref = torch.where(bad, torch.zeros_like(da, dtype=torch.float64), _ref(u, x, n, f, ks).nan_to_num())
    assert rel_err(clean, ref) <= GRAD_TOL


# ---- modules --------------------------------------------------------------------------------------------------------
N, B, T, C, H, LAYERS, G = 37, 3, 6, 1, 64, 2, 64


@pytest.fixture(params=["tc", "fma"])
def path(request):
    from stmgcn_b200 import ops
    old = ops.lstm_path()
    ops.set_lstm_path(request.param)
    yield request.param
    ops.set_lstm_path(old)


def _inputs(seed, b=B):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(b, T, N, C, device=DEV, generator=gen), torch.randn(b, N, C, device=DEV, generator=gen)


def _model_for(ks, m, seed=0):
    import STMGCN
    torch.manual_seed(seed)
    kt, k = ("localpool", 1) if ks == 1 else ("chebyshev", ks - 1)
    model = STMGCN.ST_MGCN(M=m, seq_len=T, n_nodes=N, input_dim=C, lstm_hidden_dim=H, lstm_num_layers=LAYERS,
                           gcn_hidden_dim=G, sta_kernel_config={"kernel_type": kt, "K": k}, gconv_use_bias=True)
    return model.to(DEV)


def _check_st_mgcn(stacks, branch_stack, seed=0, what=""):
    model = _model_for(stacks[0].shape[0], len(branch_stack), seed)
    x, y = _inputs(seed)
    leaves = [s.detach().clone().requires_grad_(True) for s in stacks]
    with record_relu_masks() as rec:
        out = model(obs_seq=x, sta_adj_list=[leaves[i] for i in branch_stack])
    loss = torch.mean((out - y) ** 2)
    loss.backward()
    params = {k: v.detach() for k, v in model.named_parameters()}
    out64, loss64, grads, sgrads = model_reference(params, x, y, stacks, branch_stack, masks=rec.masks, device=DEV)
    assert rel_err(out, out64) <= TOL, what
    assert abs(float(loss.detach()) - loss64) <= TOL * abs(loss64), what
    for k, p in model.named_parameters():
        assert rel_err(p.grad, grads[k]) <= TOL, (what, k)
    for leaf, g in zip(leaves, sgrads):
        assert leaf.grad is not None and leaf.grad.dtype == leaf.dtype
        assert rel_err(leaf.grad, g) <= TOL, what
    return leaves, sgrads


@pytest.mark.parametrize("kind", STACK_KINDS)
@pytest.mark.parametrize("streams", ["1", "0"])
def test_st_mgcn_stack_gradients_against_fp64(monkeypatch, path, kind, streams):
    """Separate stacks per branch and one stack shared by three branches (autograd sums the branches' gradients)."""
    monkeypatch.setenv("STMGCN_GRAPH_STREAMS", streams)
    stacks = [make_stack(kind, N, s, device=DEV) for s in range(3)]
    _check_st_mgcn(stacks, [0, 1, 2], what=f"{kind} separate")
    _check_st_mgcn(stacks[:1], [0, 0, 0], what=f"{kind} shared")


@pytest.mark.parametrize("kind", STACK_KINDS)
def test_gcn_module_stack_gradient_against_fp64(path, kind):
    import GCN
    import stmgcn_oracle as O
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
    assert rel_err(out, ref) <= TOL
    assert rel_err(gcn.W.grad, w64.grad) <= TOL
    assert rel_err(leaf.grad, s64.grad) <= TOL


@pytest.mark.parametrize("kind", ["cheb", "generic", "k0"])
@pytest.mark.parametrize("exotic", [False, True])
def test_cg_lstm_stack_gradient_against_fp64(path, kind, exotic):
    """The temporal GCN's stack gradient; ``exotic``: a Tanh activation, applied by torch after the kernels' GCN."""
    import STMGCN
    from torch import nn
    stack = make_stack(kind, N, 4, device=DEV)
    torch.manual_seed(0)
    cg = STMGCN.CG_LSTM(seq_len=T, n_nodes=N, input_dim=C, lstm_hidden_dim=H, lstm_num_layers=LAYERS,
                        K=stack.shape[0], gconv_use_bias=True, gconv_activation=nn.Tanh if exotic else nn.ReLU).to(DEV)
    x, _ = _inputs(2)
    probe = torch.randn(B, N, H, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    leaf = stack.clone().requires_grad_(True)
    with record_relu_masks() as rec:
        out, _ = cg(leaf, x, None)
    (out * probe).sum().backward()
    params = {"rnn_list.0." + k: v.detach() for k, v in cg.named_parameters()}
    relu = nn.Tanh() if exotic else True
    out64, _, grads, sgrads = model_reference(params, x, None, [stack], [0], relu=relu,
                                              masks=None if exotic else rec.masks, device=DEV, cg_probe=probe)
    assert rel_err(out, out64) <= TOL
    for k, p in cg.named_parameters():
        assert rel_err(p.grad, grads["rnn_list.0." + k]) <= TOL, k
    assert rel_err(leaf.grad, sgrads[0]) <= TOL


@pytest.mark.parametrize("kt,k", [("chebyshev", 2), ("localpool", 1)])
def test_process_adj_gradient_reaches_the_adjacency(path, kt, k):
    """ST_MGCN on process(adj) with adj requiring grad: autograd carries every dA_k on into adj.grad."""
    from stmgcn_b200 import graph
    ks = k + 1 if kt == "chebyshev" else 1
    model = _model_for(ks, 2)
    x, y = _inputs(5)
    adjs = [symmetric_graph(N, 20 + g, device=DEV).requires_grad_(True) for g in range(2)]
    with record_relu_masks() as rec:
        out = model(obs_seq=x, sta_adj_list=[dense_process(kt, k, a) for a in adjs])
    torch.mean((out - y) ** 2).backward()
    assert len(graph._CACHE) == 0 or all(not v[0].requires_grad for v in graph._CACHE.values())
    params = {kk: v.detach() for kk, v in model.named_parameters()}
    import stmgcn_oracle as O
    leaves = {kk: v.double().requires_grad_(True) for kk, v in params.items()}
    a64 = [a.detach().double().requires_grad_(True) for a in adjs]
    out64 = O.dense_st_mgcn(leaves, x.double(), [dense_process(kt, k, a) for a in a64], masks=rec.masks)
    torch.mean((out64 - y.double()) ** 2).backward()
    for a, r in zip(adjs, a64):
        assert rel_err(a.grad, r.grad) <= TOL


def test_fused_adam_on_a_parameter_stack_trains_at_the_updated_values():
    """Three Adam(fused=True) steps on an nn.Parameter stack (no version bump): every forward multiplies by the values
    the optimizer left, and every gradient is the fp64 one at those values."""
    stack = torch.nn.Parameter(make_stack("cheb", N, 6, device=DEV))
    model = _model_for(3, 2)
    opt = torch.optim.Adam([stack] + list(model.parameters()), lr=1e-2, fused=True)
    x, y = _inputs(8)
    for step in range(3):
        opt.zero_grad()
        with record_relu_masks() as rec:
            out = model(obs_seq=x, sta_adj_list=[stack, stack])
        torch.mean((out - y) ** 2).backward()
        params = {k: v.detach() for k, v in model.named_parameters()}
        out64, _, _, sgrads = model_reference(params, x, y, [stack.detach()], [0, 0], masks=rec.masks, device=DEV)
        assert rel_err(out, out64) <= TOL, step
        assert rel_err(stack.grad, sgrads[0]) <= TOL, step
        opt.step()


@pytest.mark.parametrize("kind", ["cheb", "k0"])
@pytest.mark.parametrize("streams", ["1", "0"])
def test_bf16_mode_stack_gradients_against_the_forced_reference(monkeypatch, bf16_mode, kind, streams):
    """bf16-arithmetic mode, every window carrying gradient: each stack's gradient within 1e-4 of the forced fp64
    reference's own, sum over the GCNs that read it of U_k x^T formed from that reference's U_k and x (the step's tapes
    and ReLU masks); within that mode's 2e-2 of the unrounded dense reference.  A K = 0 stack [I] included."""
    monkeypatch.setenv("STMGCN_GRAPH_STREAMS", streams)
    stacks = [make_stack(kind, N, s, device=DEV) for s in range(2)]
    model = _model_for(stacks[0].shape[0], 2)
    x, y = _inputs(11)
    leaves = [s.clone().requires_grad_(True) for s in stacks]
    params = {k: v.detach().clone() for k, v in model.state_dict().items()}
    with FullBatchRecorder() as rec:
        got = full_batch.gpu_step(model, leaves, x, y)
    rec.check_intact()
    ref = DenseStackReference(params, [chains_of(s) for s in stacks], stacks[0].shape[0], relu=True,
                              relu_masks=got["masks"], device=DEV)
    _, loss, grads = ref.loss_and_grads(x, y, tapes=rec.take_tapes())
    assert abs(got["loss"] - float(loss)) <= TOL * abs(float(loss))
    for k, g in got["grads"].items():
        assert rel_err(g, grads[k]) <= TOL, k
    errs = [rel_err(leaf.grad, ref.stack_grad([m])) for m, leaf in enumerate(leaves)]
    print(f"bf16 mode, {kind} stacks: stack gradients against the forced reference {errs}")
    assert max(errs) <= TOL
    _, _, _, sgrads = model_reference(params, x, y, stacks, [0, 1], masks=got["masks"], device=DEV)
    for leaf, g in zip(leaves, sgrads):
        assert rel_err(leaf.grad, g) <= 2e-2


def test_cfg2_full_size_every_stack_gradient_against_fp64():
    """cfg2 at full size (1024 regions, 3 graphs, K = 3, batch 32, every window with its true target) on dense Chebyshev
    stacks that require grad: every stack gradient -- many row and column tiles and k-blocks per slice, the real
    F = B*64 and B*T, the temporal and the spatial GCN of its branch -- and every parameter gradient within 1e-4 of the
    fp64 reference, taken at the step's ReLU masks, a chunk of windows at a time."""
    import GCN
    from stmgcn_b200 import synth
    w = synth.WORKLOADS["cfg2"]
    model, _, laps, params, x, y = cheb_workload(w, w.batch)
    pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
    stacks = [pre.process(a.to(DEV)) for a in synth.make_adjacency_list(w)]
    leaves = [s.clone().requires_grad_(True) for s in stacks]
    got = full_batch.gpu_step(model, leaves, x, y)
    ref = DenseStackReference(params, [chains_of(s) for s in stacks], w.n_supports, relu=True, rounding=False,
                              relu_masks=got["masks"], device=DEV)
    _, loss, grads = ref.loss_and_grads(x, y, window_chunk=CHUNK["cfg2"])
    assert abs(got["loss"] - float(loss)) <= TOL * abs(float(loss))
    for k, g in got["grads"].items():
        assert rel_err(g, grads[k]) <= TOL, k
    errs = [rel_err(leaf.grad, ref.stack_grad([m])) for m, leaf in enumerate(leaves)]
    print(f"cfg2 B={w.batch}: stack gradients against fp64 {errs}")
    assert max(errs) <= TOL


def _parent_tail(ctx, s, u, x, need_dx, round16):
    """The graph convolutions' backward tail as it was before dense stacks had gradients (sparse values only)."""
    from stmgcn_b200 import ops
    need_v = ctx.needs_input_grad[5:]
    dx = None
    if need_dx:
        dx = ops.adjoint_stack_(ctx.sset, u)
    elif any(need_v):
        ops.adjoint_stack_(ctx.sset, u, False)
    dvals = ops.support_value_grads(ctx.sset, s, u, x, round16, need_v) if any(need_v) else [None] * len(need_v)
    return dx, dvals


@pytest.mark.parametrize("supports", ["constant dense", "learnable sparse"])
def test_without_a_dense_stack_that_requires_grad_the_backward_is_the_parents(monkeypatch, supports):
    """Constant dense stacks and learnable sparse handles: the dense-stack kernel never runs, and the launch count, the
    saved tensors and the gradients equal those of the same step with the backward tail the graph convolutions had
    before dense stacks had gradients."""
    import GCN
    from stmgcn_b200 import ops
    model = _model_for(3, 2)
    x, y = _inputs(12)
    adjs = [symmetric_graph(N, 30 + g, device=DEV) for g in range(2)]

    def run():
        if supports == "constant dense":
            sups = [make_stack("generic", N, g, device=DEV) for g in range(2)]
        else:
            sups = [GCN.Adj_Preprocessor("chebyshev", 2).process_sparse(a.clone().requires_grad_(True)) for a in adjs]
        model.zero_grad(set_to_none=True)
        saved = []
        with torch.autograd.graph.saved_tensors_hooks(lambda t: saved.append((tuple(t.shape), t.dtype)) or t,
                                                      lambda t: t):
            loss = torch.mean((model(obs_seq=x, sta_adj_list=sups) - y) ** 2)
        torch.cuda.synchronize()
        n0 = lib().stmgcn_launch_count()
        loss.backward()
        torch.cuda.synchronize()
        grads = {k: p.grad.clone() for k, p in model.named_parameters()}
        return lib().stmgcn_launch_count() - n0, saved, grads
    run()
    real = ops.dense_support_grad
    monkeypatch.setattr(ops, "dense_support_grad", lambda *a: (_ for _ in ()).throw(AssertionError("launched")))
    launches, saved, grads = run()
    monkeypatch.setattr(ops, "dense_support_grad", real)
    monkeypatch.setattr(ops, "_support_grads", _parent_tail)
    p_launches, p_saved, p_grads = run()
    assert launches == p_launches and saved == p_saved
    for k, g in grads.items():
        assert rel_err(g, p_grads[k]) <= GRAD_TOL, k


def _variant_tail(variant):
    """The dense-stack backward tail with one deliberate fault (negative controls)."""
    from stmgcn_b200 import ops

    def tail(ctx, s, u, x, need_dx, round16):
        sset = ctx.sset
        if variant == "after_clenshaw":             # U_k after the adjoint Clenshaw: the chain adjoints G_k
            dx = ops.adjoint_stack_(sset, u, need_dx)
            return dx, [ops.dense_support_grad(u, s[0] if x is None else x).to(sset.dense.dtype)]
        da = ops.dense_support_grad(u, s[0] if variant == "s0_as_x" else (s[0] if x is None else x))
        if variant == "transposed":
            da = da.transpose(1, 2).contiguous()
        elif variant == "dA_0_left_out":
            da[0] = 0
        dx = ops.adjoint_stack_(sset, u) if need_dx else None
        return dx, [da.to(sset.dense.dtype)]
    return tail


@pytest.mark.parametrize("variant,kind", [("transposed", "cheb"), ("after_clenshaw", "cheb"), ("s0_as_x", "generic"),
                                          ("dA_0_left_out", "cheb")])
def test_negative_controls_in_the_backward_fail_the_bar(monkeypatch, variant, kind):
    """Each fault injected into the real backward -- dA_k^T for dA_k, U after the Clenshaw (G_k), s[0] = A_0 x as x on a
    generic stack, dA_0 left out -- moves the stack gradient past the 1e-4 bar (the margin is printed); the same run
    without the fault passes it."""
    from stmgcn_b200 import ops
    stacks = [make_stack(kind, N, 0, device=DEV)]
    _check_st_mgcn(stacks, [0, 0], what=f"{variant} control, unfaulted")
    monkeypatch.setattr(ops, "_support_grads", _variant_tail(variant))
    model = _model_for(stacks[0].shape[0], 2)
    x, y = _inputs(0)
    leaf = stacks[0].clone().requires_grad_(True)
    with record_relu_masks() as rec:
        out = model(obs_seq=x, sta_adj_list=[leaf, leaf])
    torch.mean((out - y) ** 2).backward()
    params = {k: v.detach() for k, v in model.named_parameters()}
    _, _, _, sgrads = model_reference(params, x, y, stacks, [0, 0], masks=rec.masks, device=DEV)
    err = rel_err(leaf.grad, sgrads[0])
    print(f"negative control {variant}: stack gradient {err:.3e} from fp64 (bar {TOL:.0e})")
    assert err > 100 * TOL
