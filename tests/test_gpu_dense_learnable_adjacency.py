"""A learnable adjacency multiplied dense on the H100: stmgcn_dense_chain_grad against fp64 at every edge and on a dense
similarity graph's own chain, its negative controls, the pattern <-> dense entry points bit for bit, their C-ABI
contract, the dispatch between the dense and the CSR paths, and GCN / CG_LSTM / ST_MGCN with dense learnable graphs
against the fp64 dense restatement (taken at the kernels' own ReLU masks), at cfg2's full size, in the bf16 mode, under
capture and with non-finite values."""
import itertools

import pytest
import torch
from torch import nn

import learnable_adjacency_cases as LA
from abi_harness import Buf, Call, drive, run_captured, run_contract
from dense_support_grad_cases import model_reference
from helpers import DEV, GRAD_TOL, TOL, build_model, lib, rel_err
from support_grad_cases import record_relu_masks

pytestmark = pytest.mark.gpu

ORDERS = {"chebyshev": 3, "localpool": 1, "random_walk_diffusion": 2}


def _adj(kind, a, lam=2.0, order=None):
    import GCN
    return GCN.Adj_Preprocessor(kind, ORDERS[kind] if order is None else order, lambda_max=lam).process_learnable(a).to(DEV)


@pytest.fixture
def dense_on(monkeypatch):
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_DENSE_SUPPORTS", "on")


# ======================================================================================================================
# stmgcn_dense_chain_grad
# ======================================================================================================================
def _chain(n, f, terms, round_b16=False, out=None):
    from stmgcn_b200 import _lib
    out = torch.empty(n, n, device=DEV) if out is None else out
    a = _lib.ptr_array([t[0].data_ptr() for t in terms])
    b = _lib.ptr_array([t[1].data_ptr() for t in terms])
    coef = _lib.float_array([float(t[2]) for t in terms])
    _lib.check(lib().stmgcn_dense_chain_grad(n, f, len(terms), a, b, coef, int(round_b16), out.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream), "dense_chain_grad")
    return out


def _chain_ref(n, terms, round_b16=False):
    def rb(b):
        return b.to(torch.bfloat16).double() if round_b16 else b.double()
    return sum(c * (a.double().reshape(n, -1) @ rb(b).reshape(n, -1).T) for a, b, c in terms)


def _operands(n, f, nterms, seed, off=0):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    terms = []
    for t in range(nterms):
        a = torch.randn(off + n * f, device=DEV, generator=gen)[off:]
        b = torch.randn(off + n * f, device=DEV, generator=gen)[off:]
        terms.append((a, b, 1.0 if t == 0 else 2.0))
    return terms


SWEEP = [(n, f, 1 + i % 7) for i, (n, f) in enumerate(itertools.product((1, 5, 127, 128, 129, 300, 1024),
                                                                        (1, 3, 4, 31, 32, 33, 768, 4096)))]


@pytest.mark.parametrize("n,f,nterms", SWEEP)
def test_chain_grad_against_fp64(n, f, nterms):
    terms = _operands(n, f, nterms, seed=n * 37 + f)
    assert rel_err(_chain(n, f, terms), _chain_ref(n, terms)) <= GRAD_TOL


@pytest.mark.parametrize("off", [1, 2, 3])
def test_chain_grad_misaligned_pointers(off):
    """Operands and out off 16-byte (and 8-byte) alignment: the scalar loads and stores, same bar."""
    n, f = 133, 64
    terms = _operands(n, f, 3, seed=off, off=off)
    outb = torch.empty(off + n * n, device=DEV)
    out = _chain(n, f, terms, out=outb[off:].view(n, n))
    assert rel_err(out, _chain_ref(n, terms)) <= GRAD_TOL


def _similarity_chain(n, f, order, seed=0):
    """A dense similarity graph's L~ (normalised and scattered by the kernels) and its own chain: T_k of random features,
    and the Clenshaw totals G_k of random U_k, fp64, plus the U_k (for a negative control)."""
    import GCN
    from stmgcn_b200 import ops, synth
    adj = GCN.Adj_Preprocessor("chebyshev", order).process_learnable(synth.make_similarity_adjacency(n, seed).to(DEV)).to(DEV)
    with torch.no_grad():
        lt = ops.PatternToDense.apply(ops.AdjNorm.apply(adj.weight, adj.kind, adj.scale, *adj.pattern()), adj.rowptr,
                                      adj.colidx).double()
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    t = [torch.randn(n, f, device=DEV, generator=gen, dtype=torch.float64)]
    t.append(lt @ t[0])
    for _ in range(2, order + 1):
        t.append(2 * (lt @ t[-1]) - t[-2])
    u = [torch.randn(n, f, device=DEV, generator=gen, dtype=torch.float64) for _ in range(order + 1)]
    g = [None] * (order + 1)
    for k in range(order, 0, -1):
        g[k] = u[k] + (2 * (lt.T @ g[k + 1]) if k + 1 <= order else 0) - (g[k + 2] if k + 2 <= order else 0)
    f32 = lambda xs: [None if x is None else x.float().contiguous() for x in xs]     # noqa: E731
    return f32(t), f32(g), f32(u)


def _chain_terms(t, g, order, c1=1.0):
    return [(g[k], t[k - 1], c1 if k == 1 else 2.0) for k in range(1, order + 1)]


def test_chain_grad_on_a_similarity_graph_at_cfg3_shapes_and_bit_identical_reruns():
    """cfg3's spatial (F = 64 * 64) and temporal (F = 64 * 12) widths on a 4096-region similarity graph's own G_k and
    T_k, where the products cancel."""
    n, order = 4096, 3
    for f in (4096, 768):
        t, g, _ = _similarity_chain(n, f, order)
        terms = _chain_terms(t, g, order)
        got = _chain(n, f, terms)
        err = rel_err(got, _chain_ref(n, terms))
        print(f"similarity chain N={n} F={f}: {err:.2e}")
        assert err <= GRAD_TOL
        assert torch.equal(_chain(n, f, terms), got)


def test_chain_grad_round_b16_against_the_rounded_operand():
    n, f, order = 300, 768, 3
    t, g, _ = _similarity_chain(n, f, order, seed=2)
    terms = _chain_terms(t, g, order)
    got = _chain(n, f, terms, round_b16=True)
    assert rel_err(got, _chain_ref(n, terms, round_b16=True)) <= GRAD_TOL
    assert rel_err(got, _chain_ref(n, terms)) > GRAD_TOL          # the rounding is there


@pytest.mark.parametrize("variant", ["G transposed", "U for G", "c1 = 2"])
def test_chain_grad_negative_controls_fail_the_bar(variant):
    n, f, order = 300, 768, 3
    t, g, u = _similarity_chain(n, f, order, seed=3)
    want = _chain_ref(n, _chain_terms(t, g, order))
    if variant == "G transposed":          # T_{k-1} G_k^T = (G_k T_{k-1}^T)^T
        terms = [(b, a, c) for a, b, c in _chain_terms(t, g, order)]
    elif variant == "U for G":             # the projection backward's U_k, before the Clenshaw
        terms = _chain_terms(t, u, order)
    else:
        terms = _chain_terms(t, g, order, c1=2.0)
    assert rel_err(_chain(n, f, terms), want) > 10 * GRAD_TOL, variant


# ======================================================================================================================
# pattern <-> dense
# ======================================================================================================================
def _scatter(n, rowptr, colidx, vals):
    from stmgcn_b200 import ops
    return ops.PatternToDense.apply(vals, rowptr, colidx)


def _gather(n, rowptr, colidx, dense):
    from stmgcn_b200 import _lib
    dv = torch.empty(colidx.numel(), device=DEV)
    _lib.check(lib().stmgcn_pattern_gather(n, rowptr.data_ptr(), colidx.data_ptr(), colidx.numel(), dense.data_ptr(),
                                           dv.data_ptr(), torch.cuda.current_stream().cuda_stream), "pattern_gather")
    return dv


def _handmade_pattern(n, seed):
    """Unsorted columns, repeated entries (also more than 32 apart within a row), stored zeros and empty rows; values
    dyadic, so every sum of them is exact in fp32 and the fp64 scatter rounded once is the exact matrix."""
    gen = torch.Generator().manual_seed(seed)
    rows, cols = [], []
    for i in range(n):
        cnt = 0 if i % 7 == 3 else int(torch.randint(1, 80, (1,), generator=gen))
        c = torch.randint(0, max(n // 3, 1), (cnt,), generator=gen)          # narrow range: many repeats
        rows += [i] * cnt
        cols += c.tolist()
    rows, cols = torch.tensor(rows), torch.tensor(cols)
    vals = torch.randint(-64, 65, (rows.numel(),), generator=gen).float() / 16
    vals[::5] = 0.0
    vals[1::11] = -0.0
    rowptr = torch.zeros(n + 1, dtype=torch.int64)
    rowptr[1:] = torch.cumsum(torch.bincount(rows, minlength=n), 0)
    return rowptr.int().to(DEV), cols.int().to(DEV), vals.to(DEV), rows, cols


@pytest.mark.parametrize("n", [1, 45, 300])
def test_scatter_and_gather_bit_exact_with_repeats_and_stored_zeros(n):
    rowptr, colidx, vals, rows, cols = _handmade_pattern(n, n)
    dense = _scatter(n, rowptr, colidx, vals)
    want = torch.zeros(n, n, dtype=torch.float64).index_put((rows, cols), vals.double().cpu(), accumulate=True).float()
    assert torch.equal(dense.cpu(), want)
    g = torch.randn(n, n, generator=torch.Generator().manual_seed(n)).to(DEV)
    assert torch.equal(_gather(n, rowptr, colidx, g).cpu(), g.cpu()[rows, cols])
    assert torch.equal(_scatter(n, rowptr, colidx, vals), dense)


@pytest.mark.parametrize("kind,lam", [("chebyshev", 1.37), ("localpool", 2.0), ("random_walk_diffusion", 2.0)])
def test_module_matrices_are_the_fp64_scatter_of_its_values(dense_on, kind, lam):
    """The dense set's matrices are the module's normalised values scattered (added diagonal slots included; P_f^T
    from its CSR^T order), and its graphs are DenseGraphs."""
    from stmgcn_b200 import ops
    from stmgcn_b200.graph import DenseGraph
    adj = _adj(kind, LA.graph(61, 3, directed=kind == "random_walk_diffusion").float(), lam)
    assert adj.widx is not None or kind == "random_walk_diffusion"
    sset = adj()
    assert sset.graphs and all(isinstance(gr, DenseGraph) for gr in sset.graphs)
    vals = ops.AdjNorm.apply(adj.weight, adj.kind, adj.scale, *adj.pattern())
    prow, pcol, _, perm_t = LA.pattern_of(adj)
    if kind == "random_walk_diffusion":
        vf, vb = (v.detach().double().cpu() for v in vals)
        want = [LA.dense_of(adj.n, pcol[perm_t], prow[perm_t], vf), LA.dense_of(adj.n, prow, pcol, vb)]
    else:
        want = [LA.dense_of(adj.n, prow, pcol, vals.detach().double().cpu())]
    for got, w, gr in zip(sset.values, want, sset.graphs):
        assert torch.equal(got.detach().cpu(), w.float())
        assert gr.mat.data_ptr() == got.data_ptr()


# ======================================================================================================================
# C ABI contract
# ======================================================================================================================
def _dense_calls(f):
    from stmgcn_b200 import _lib
    n, nterms = 70, 3
    ig = 0x7FA5A5A5
    terms = _operands(n, f, nterms, seed=f)
    b = {f"a{t}": Buf("in", terms[t][0].clone()) for t in range(nterms)}
    b.update({f"b{t}": Buf("in", terms[t][1].clone()) for t in range(nterms)})
    b["out"] = Buf("out", shape=(n, n))
    coefs = [t[2] for t in terms]

    def launch(st):
        a = _lib.ptr_array([b[f"a{t}"].p for t in range(nterms)])
        bb = _lib.ptr_array([b[f"b{t}"].p for t in range(nterms)])
        return lib().stmgcn_dense_chain_grad(n, f, nterms, a, bb, _lib.float_array(coefs), 0, b["out"].p, st)

    def ref(res):
        assert rel_err(res["out"], _chain_ref(n, terms)) <= GRAD_TOL

    yield Call("dense_chain_grad", b, launch, ref, 1)
    rowptr, colidx, vals, rows, cols = _handmade_pattern(n, 5)
    nnz = colidx.numel()
    s = {"rowptr": Buf("in", rowptr, guard=ig), "colidx": Buf("in", colidx, guard=ig), "vals": Buf("in", vals),
         "dense": Buf("out", shape=(n, n))}

    def ref_s(res):
        want = torch.zeros(n, n, dtype=torch.float64).index_put((rows, cols), vals.double().cpu(), accumulate=True)
        assert torch.equal(res["dense"].cpu(), want.float())

    yield Call("pattern_scatter", s, lambda st: lib().stmgcn_pattern_scatter(
        n, s["rowptr"].p, s["colidx"].p, nnz, s["vals"].p, s["dense"].p, st), ref_s, 1)
    dense = torch.randn(n, n, generator=torch.Generator().manual_seed(8)).to(DEV)
    g = {"rowptr": Buf("in", rowptr, guard=ig), "colidx": Buf("in", colidx, guard=ig), "dense": Buf("in", dense),
         "dvals": Buf("out", shape=(nnz,))}

    def ref_g(res):
        assert torch.equal(res["dvals"].cpu(), dense.cpu()[rows, cols])

    yield Call("pattern_gather", g, lambda st: lib().stmgcn_pattern_gather(
        n, g["rowptr"].p, g["colidx"].p, nnz, g["dense"].p, g["dvals"].p, st), ref_g, 1)


@pytest.mark.parametrize("f", [36, 33])
def test_dense_learnable_abi_contract(f):
    drive(_dense_calls(f), run_contract)
    drive(_dense_calls(f), run_captured)


# ======================================================================================================================
# dispatch
# ======================================================================================================================
def _gcn_case(adj, seed=0, b=3):
    """A GCN on ``adj``, its input and a probe: ``step()`` runs forward and backward and returns d weight."""
    import GCN
    torch.manual_seed(seed)
    gcn = GCN.GCN(K=adj.ks, input_dim=64, hidden_dim=64).to(DEV)
    x = torch.randn(b, adj.n, 64, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed + 1))
    probe = torch.randn(b, adj.n, 64, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed + 2))

    def step():
        adj.weight.grad = None
        (gcn(adj, x) * probe).sum().backward()
        return adj.weight.grad
    return step


def _gcn_step(adj, seed=0, b=3):
    return _gcn_case(adj, seed, b)().clone()


def test_auto_sends_a_similarity_graph_dense_and_keeps_a_sparse_graph_on_the_parents_launches(monkeypatch):
    from stmgcn_b200 import ops, synth
    from stmgcn_b200.graph import DenseGraph, GraphHandle
    monkeypatch.setattr(ops, "_DENSE_SUPPORTS", "auto")
    sim = _adj("chebyshev", synth.make_similarity_adjacency(1024, 0), order=2)
    assert sim.dense() and all(isinstance(g, DenseGraph) for g in sim().graphs)
    # every degree positive (the hub reaches every region), so d weight is finite and comparable bit for bit
    sparse = _adj("chebyshev", LA.graph(1000, 1, isolated=False, density=0.01).float(), 1.5, order=2)
    assert not sparse.dense() and all(isinstance(g, GraphHandle) for g in sparse().graphs)

    def launches(mode):
        monkeypatch.setattr(ops, "_DENSE_SUPPORTS", mode)
        _gcn_step(sparse)
        torch.cuda.synchronize()
        n0 = lib().stmgcn_launch_count()
        dw = _gcn_step(sparse)
        torch.cuda.synchronize()
        return lib().stmgcn_launch_count() - n0, dw

    (n_auto, dw_auto), (n_off, dw_off) = launches("auto"), launches("off")
    assert n_auto == n_off
    assert bool(torch.isfinite(dw_off).all()) and torch.equal(dw_auto, dw_off)


@pytest.mark.parametrize("kind", LA.KINDS)
def test_on_and_off_agree_on_one_model(monkeypatch, kind):
    from stmgcn_b200 import ops
    from stmgcn_b200.graph import DenseGraph, GraphHandle
    _, model, adjs, x, y = _model_case(kind, n_adj=2)
    res = {}
    for mode, cls in (("on", DenseGraph), ("off", GraphHandle)):
        monkeypatch.setattr(ops, "_DENSE_SUPPORTS", mode)
        assert all(isinstance(g, cls) for g in adjs[0]().graphs)
        model.zero_grad(set_to_none=True)
        for a in adjs:
            a.weight.grad = None
        loss = nn.MSELoss()(model(obs_seq=x, sta_adj_list=[adjs[i] for i in (0, 0, 1)]), y)
        loss.backward()
        res[mode] = (loss.item(), {k: p.grad.clone() for k, p in model.named_parameters()},
                     [a.weight.grad.clone() for a in adjs])
    (l1, g1, d1), (l2, g2, d2) = res["on"], res["off"]
    assert abs(l1 - l2) <= TOL * abs(l2)
    for k in g1:
        assert rel_err(g1[k], g2[k]) <= TOL, k
    for a, b in zip(d1, d2):
        assert rel_err(a, b) <= TOL


@pytest.mark.parametrize("kind", LA.KINDS)
def test_dense_forward_and_backward_never_synchronise(dense_on, kind):
    adj = _adj(kind, LA.graph(300, 6, directed=True, isolated=False, density=0.05).float(), 1.5)
    step = _gcn_case(adj)                 # module, inputs and the structure's conversion (one host sync) first
    step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        dw = step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert dw.shape == adj.weight.shape and bool(torch.isfinite(dw).all())


# ======================================================================================================================
# the models
# ======================================================================================================================
META = dict(n=24, m=3, k=2, t=4, b=3, c=1, hid=64, layers=2, gcn_hid=64)


def _model_case(kind, seed=0, lam=1.6, n_adj=3):
    meta = dict(META, kernel_type=kind, k=1 if kind == "localpool" else META["k"])
    torch.manual_seed(seed)
    model = build_model(meta, DEV)
    a = [LA.graph(meta["n"], 20 + g, directed=kind == "random_walk_diffusion", density=0.3).float() for g in range(n_adj)]
    adjs = [_adj(kind, x, lam, meta["k"]) for x in a]
    gen = torch.Generator().manual_seed(seed + 11)
    x = torch.randn(meta["b"], meta["t"], meta["n"], meta["c"], generator=gen).to(DEV)
    y = torch.randn(meta["b"], meta["n"], meta["c"], generator=gen).to(DEV)
    return meta, model, adjs, x, y


def _dw64(adj, stack_grad):
    """d weight in fp64: a stack gradient carried back through the fp64 normalisation and the dense chain."""
    w64 = adj.weight.detach().double().cpu().requires_grad_(True)
    (dw,) = torch.autograd.grad(LA.module_stack64(adj, w64), w64, stack_grad.detach().double().cpu())
    return dw


def _check_st_mgcn(model, adjs, branch, x, y, what):
    model.zero_grad(set_to_none=True)
    for a in adjs:
        a.weight.grad = None
    with record_relu_masks() as rec:
        out = model(obs_seq=x, sta_adj_list=[adjs[i] for i in branch])
    loss = nn.MSELoss()(out, y)
    loss.backward()
    stacks = [LA.module_stack64(a, a.weight.detach().double().cpu()) for a in adjs]
    params = {k: v.detach() for k, v in model.named_parameters()}
    out64, loss64, grads, sgrads = model_reference(params, x, y, stacks, branch, masks=rec.masks, device=DEV)
    assert rel_err(out, out64) <= TOL, f"{what} output"
    assert abs(loss.item() - loss64) <= TOL * abs(loss64), f"{what} loss"
    for k, p in model.named_parameters():
        assert rel_err(p.grad, grads[k]) <= TOL, f"{what} {k}"
    for i, a in enumerate(adjs):
        if i in branch:
            assert rel_err(a.weight.grad, _dw64(a, sgrads[i])) <= TOL, f"{what} d weight {i}"


@pytest.mark.parametrize("path", ["tc", "fma"])
@pytest.mark.parametrize("streams", ["1", "0"])
@pytest.mark.parametrize("kind", LA.KINDS)
def test_st_mgcn_dense_learnable_graphs_against_fp64(monkeypatch, dense_on, path, streams, kind):
    """One adjacency shared by two branches, and three separate ones: output, loss, every parameter gradient and
    d weight within 1e-4 of the fp64 dense restatement."""
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_LSTM_PATH", path)
    monkeypatch.setenv("STMGCN_GRAPH_STREAMS", streams)
    _, model, adjs, x, y = _model_case(kind)
    _check_st_mgcn(model, adjs, [0, 0, 1], x, y, f"{kind} shared path={path} streams={streams}")
    _check_st_mgcn(model, adjs, [0, 1, 2], x, y, f"{kind} separate path={path} streams={streams}")


@pytest.mark.parametrize("kind", LA.KINDS)
def test_gcn_module_dense_learnable_graph_against_fp64(dense_on, kind):
    import GCN
    import stmgcn_oracle as O
    adj = _adj(kind, LA.graph(40, 7, directed=kind == "random_walk_diffusion").float(), 1.37)
    torch.manual_seed(0)
    gcn = GCN.GCN(K=adj.ks, input_dim=64, hidden_dim=64).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(3, adj.n, 64, device=DEV, generator=gen)
    probe = torch.randn(3, adj.n, 64, device=DEV, generator=gen)
    with record_relu_masks() as rec:
        out = gcn(adj, x)
    (out * probe).sum().backward()
    w64 = adj.weight.detach().double().cpu().requires_grad_(True)
    s64 = LA.module_stack64(adj, w64).to(DEV)
    W64 = gcn.W.detach().double().requires_grad_(True)
    ref = O.dense_gcn(s64, x.double(), W64, gcn.b.detach().double(), True, rec.masks[0])
    (ref * probe.double()).sum().backward()
    assert rel_err(out, ref) <= TOL
    assert rel_err(gcn.W.grad, W64.grad) <= TOL
    assert rel_err(adj.weight.grad, w64.grad) <= TOL


@pytest.mark.parametrize("kind", LA.KINDS)
def test_cg_lstm_dense_learnable_graph_with_initial_state_against_fp64(dense_on, kind):
    import STMGCN
    import stmgcn_oracle as O
    n, t, b, hid, layers = 30, 5, 3, 64, 2
    adj = _adj(kind, LA.graph(n, 8, directed=kind == "random_walk_diffusion").float(), 1.37)
    torch.manual_seed(0)
    cg = STMGCN.CG_LSTM(seq_len=t, n_nodes=n, input_dim=1, lstm_hidden_dim=hid, lstm_num_layers=layers, K=adj.ks,
                        gconv_use_bias=True, gconv_activation=nn.ReLU).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(2)
    x = torch.randn(b, t, n, 1, device=DEV, generator=gen)
    h0 = torch.randn(layers, b * n, hid, device=DEV, generator=gen)
    c0 = torch.randn(layers, b * n, hid, device=DEV, generator=gen)
    probe = torch.randn(b, n, hid, device=DEV, generator=gen)
    r = torch.randn(layers, b * n, hid, device=DEV, generator=gen)
    with record_relu_masks() as rec:
        out, (h_n, _) = cg(adj, x, (h0, c0))
    ((out * probe).sum() + (h_n * r).sum()).backward()
    params = {"p." + k: v.detach().double().requires_grad_(True) for k, v in cg.named_parameters()}
    w64 = adj.weight.detach().double().cpu().requires_grad_(True)
    s64 = LA.module_stack64(adj, w64).to(DEV)
    out64, (h64, _) = O.dense_cg_lstm(s64, x.double(), params, "p.", True, hidden=(h0.double(), c0.double()),
                                      mask=rec.masks[0])
    ((out64 * probe.double()).sum() + (h64 * r.double()).sum()).backward()
    assert rel_err(out, out64) <= TOL
    for k, p in cg.named_parameters():
        assert rel_err(p.grad, params["p." + k].grad) <= TOL, k
    assert rel_err(adj.weight.grad, w64.grad) <= TOL


def test_cfg2_full_size_three_dense_similarity_graphs_against_fp64(monkeypatch):
    """cfg2 (1024 regions, three dense similarity graphs, K = 3, batch 32, every window carrying gradient) under
    ``auto``: the output, the loss, every parameter gradient and every d weight within 1e-4 of fp64."""
    import STMGCN
    from stmgcn_b200 import ops, synth
    monkeypatch.setattr(ops, "_DENSE_SUPPORTS", "auto")
    w = synth.WORKLOADS["cfg2"]
    torch.manual_seed(0)
    model = STMGCN.ST_MGCN(**synth.model_kwargs(w)).to(DEV)
    adjs = [_adj("chebyshev", synth.make_similarity_adjacency(w.n_regions, g), order=w.cheb_order)
            for g in range(w.n_graphs)]
    assert all(a.dense() for a in adjs)
    x, y = (t.to(DEV) for t in synth.make_inputs(w, seed=12))
    _check_st_mgcn(model, adjs, list(range(w.n_graphs)), x, y, "cfg2 full size")


@pytest.mark.parametrize("kind", ["chebyshev", "random_walk_diffusion"])
def test_bf16_mode_dense_learnable_graphs_against_the_forced_reference(monkeypatch, dense_on, kind):
    """The bf16-arithmetic mode multiplies bf16 copies of the chain terms: the dense path's loss, gradients and d weight
    within 1e-4 of the fp64 reference that rounds where the kernels round (forced with the step's own values and
    masks)."""
    import support_grad_cases as S
    from full_batch import gpu_step
    from model_cases import FullBatchRecorder
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_PLANES", 1)
    _, model, adjs, x, y = _model_case(kind, seed=4, n_adj=2)
    branch = [0, 1, 0]
    for a in adjs:
        a.weight.grad = None
    with FullBatchRecorder() as rec:
        got = gpu_step(model, [adjs[i] for i in branch], x.clone(), y, want_obs=True)
    rec.check_intact()
    tapes = rec.take_tapes()
    params = {k: v.detach() for k, v in model.state_dict().items()}
    handles = [a.supports() for a in adjs]
    ref = S.ForcedValueReference(params, handles, branch, relu_masks=got["masks"], device=DEV)
    loss, grads, d_obs, d_vals = ref.value_grads(x, y, tapes)
    assert abs(got["loss"] - loss) <= TOL * abs(loss)
    for name, g in got["grads"].items():
        assert rel_err(g, grads[name]) <= TOL, f"bf16 mode dense {kind} {name}"
    for a, dv in zip(adjs, d_vals):
        w64 = a.weight.detach().double().cpu().requires_grad_(True)
        v64 = LA.module_values64(a, w64)
        v64 = v64 if isinstance(v64, tuple) else (v64,)
        (dw64,) = torch.autograd.grad(v64, w64, tuple(d.double().cpu() for d in dv))
        assert rel_err(a.weight.grad, dw64) <= TOL, f"bf16 mode dense {kind} d weight"


def test_graphed_step_replays_match_eager_and_see_fused_adam_updates(dense_on):
    from stmgcn_b200.graphs import GraphedStep
    _, model, adjs, x, y = _model_case("chebyshev", seed=5, n_adj=2)
    sups = [adjs[0], adjs[1], adjs[0]]
    assert all(a.dense() for a in adjs)
    crit = nn.MSELoss()
    opt = torch.optim.Adam(list(model.parameters()) + [p for a in adjs for p in a.parameters()], lr=1e-2, fused=True)
    step = GraphedStep(model, crit, x, y, sups)
    w_ptr = adjs[0].weight.data_ptr()
    losses = []
    for i in range(3):
        loss = step(x, y).item()
        replay = step.bucket.flat.clone()
        step.bucket.zero_()
        eager = crit(model(obs_seq=x, sta_adj_list=sups), y)
        eager.backward()
        assert abs(loss - eager.item()) <= GRAD_TOL * abs(eager.item()), f"step {i}"
        assert rel_err(replay, step.bucket.flat) <= GRAD_TOL, f"step {i}"
        assert adjs[0].weight.grad.abs().max() > 0
        losses.append(loss)
        opt.step()
    assert adjs[0].weight.data_ptr() == w_ptr
    assert len(set(losses)) == 3, "the replays did not see the optimizer's updates"


@pytest.mark.parametrize("kind", LA.KINDS)
def test_nan_weight_and_zero_degree_row_non_finite_where_fp64_is(dense_on, kind):
    """A NaN edge weight, and a row of zero degree: output and d weight are non-finite exactly where the fp64 dense
    restatement's are."""
    import GCN
    import stmgcn_oracle as O
    a = LA.graph(29, 5, directed=kind == "random_walk_diffusion").float()
    adj = _adj(kind, a, 1.5)
    torch.manual_seed(0)
    gcn = GCN.GCN(K=adj.ks, input_dim=64, hidden_dim=64, activation=None).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(2, adj.n, 64, device=DEV, generator=gen)
    probe = torch.randn(2, adj.n, 64, device=DEV, generator=gen)
    w0 = adj.weight.detach().clone()
    for e in (0, int(w0.numel()) // 2):
        w = w0.clone()
        w[e] = float("nan")
        with torch.no_grad():
            adj.weight.copy_(w)
        adj.weight.grad = None
        out = gcn(adj, x)
        (out * probe).sum().backward()
        w64 = w.double().cpu().requires_grad_(True)
        ref = O.dense_gcn(LA.module_stack64(adj, w64).to(DEV), x.double(), gcn.W.detach().double(), gcn.b.detach().double(),
                          False)
        (ref * probe.double()).sum().backward()
        for got, want, what in ((out, ref.detach(), "output"), (adj.weight.grad, w64.grad, "d weight")):
            bad = ~torch.isfinite(want.cpu())
            assert torch.equal(~torch.isfinite(got.cpu()), bad), f"{kind} NaN at {e}: {what}"
            assert bad.any()
            if not bad.all():
                assert rel_err(got.cpu()[~bad], want.cpu()[~bad]) <= TOL
