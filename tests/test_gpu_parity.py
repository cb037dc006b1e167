"""GPU parity tests: the CUDA path (through the C ABI / the drop-in modules) against the oracle and the
golden vectors generated from the reference.  Tolerance: 1e-4 max-norm relative (BASELINE.json)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch
from torch import nn

import stmgcn_oracle as O
from helpers import DEV, TOL, assert_close, build_model, load_golden

pytestmark = pytest.mark.gpu


def _rand_csr(n, density, seed, asym=True):
    rng = np.random.default_rng(seed)
    a = (rng.random((n, n)) < density) * rng.standard_normal((n, n))
    if not asym:
        a = (a + a.T) / 2
    a[np.arange(n), (np.arange(n) + 1) % n] = 0.5          # no empty rows
    return a.astype(np.float32)


def test_graph_handle_roundtrip():
    from stmgcn_b200.graph import GraphHandle
    a = _rand_csr(97, 0.1, 0)
    g = GraphHandle.from_dense(torch.from_numpy(a).to(DEV))
    ref = sp.csr_matrix(a)
    assert g.n == 97 and g.nnz == ref.nnz
    rp, ci, va = [t.cpu().numpy() for t in g.export(False)]
    assert np.array_equal(rp, ref.indptr) and np.array_equal(ci, ref.indices) and np.array_equal(va, ref.data)
    ref_t = sp.csr_matrix(a.T)
    rp, ci, va = [t.cpu().numpy() for t in g.export(True)]
    assert np.array_equal(rp, ref_t.indptr) and np.array_equal(ci, ref_t.indices) and np.array_equal(va, ref_t.data)
    # CSR entry == dense entry
    g2 = GraphHandle.from_csr(97, torch.from_numpy(ref.indptr).to(DEV), torch.from_numpy(ref.indices).to(DEV),
                              torch.from_numpy(ref.data).to(DEV))
    rp2, ci2, va2 = [t.cpu().numpy() for t in g2.export(True)]
    assert np.array_equal(rp2, ref_t.indptr) and np.array_equal(ci2, ref_t.indices) and np.array_equal(va2, ref_t.data)


@pytest.mark.parametrize("n,f", [(64, 32), (97, 7), (300, 768), (128, 132), (1, 4)])
@pytest.mark.parametrize("transpose", [False, True])
def test_spmm_step(n, f, transpose):
    from stmgcn_b200 import ops
    from stmgcn_b200.graph import GraphHandle
    a = _rand_csr(n, 0.08, n + f)
    g = GraphHandle.from_dense(torch.from_numpy(a).to(DEV))
    rng = np.random.default_rng(1)
    x, z, u = (rng.standard_normal((n, f)).astype(np.float32) for _ in range(3))
    xd, zd, ud = (torch.from_numpy(v).to(DEV) for v in (x, z, u))
    y = torch.empty_like(xd)
    op = a.T if transpose else a
    ops.spmm_step(g, transpose, 2.0, xd, -1.0, zd, 0.5, ud, y)
    ref = 2.0 * (op.astype(np.float64) @ x) - z + 0.5 * u
    assert_close(y.cpu().numpy(), ref, "spmm full", 1e-5)
    ops.spmm_step(g, transpose, 1.0, xd, 0.0, None, 0.0, None, y)
    assert_close(y.cpu().numpy(), op.astype(np.float64) @ x, "spmm plain", 1e-5)
    # in-place on the U operand (used by the adjoint Clenshaw)
    ops.spmm_step(g, transpose, 2.0, xd, -1.0, zd, 1.0, ud, ud)
    assert_close(ud.cpu().numpy(), 2.0 * (op.astype(np.float64) @ x) - z + u, "spmm in-place", 1e-5)


@pytest.mark.parametrize("n,f", [(64, 32), (97, 8), (300, 768), (128, 136)])
@pytest.mark.parametrize("transpose", [False, True])
def test_spmm_step_with_bf16_gather_copy(n, f, transpose):
    """stmgcn_cheb_spmm_step16 (bf16-arithmetic mode): the gathered operand is the bf16 copy, everything else fp32 -- equal
    to the fp32 kernel run on the rounded operand; the bf16 copy of the result is the rounded result; u may alias y."""
    from stmgcn_b200 import ops
    from stmgcn_b200.graph import GraphHandle
    g = GraphHandle.from_dense(torch.from_numpy(_rand_csr(n, 0.08, n + f)).to(DEV))
    gen = torch.Generator().manual_seed(n + f)
    x, z, u = (torch.randn(n, f, generator=gen).to(DEV) for _ in range(3))
    x16 = ops.to_bf16(x)
    assert torch.equal(x16, x.to(torch.bfloat16))
    y_ref = torch.empty_like(x)
    ops.spmm_step(g, transpose, 2.0, x16.float(), -1.0, z, 1.0, u, y_ref)
    y, y16 = u.clone(), torch.empty_like(x16)
    ops.spmm_step16(g, transpose, 2.0, x16, -1.0, z, 1.0, y, y, y16)              # u aliases y
    assert_close(y.cpu().numpy(), y_ref.cpu().numpy(), "spmm16 vs fp32 kernel on the rounded operand", 1e-6)
    assert torch.equal(y16, y.to(torch.bfloat16))


@pytest.mark.parametrize("name", ["cfg1_ref", "ragged_ref", "cfg3_small_ref", "localpool_tanh_ref", "cheb7_linear_ref"])
def test_model_matches_reference_golden(name):
    """Forward output, loss and EVERY parameter gradient vs vectors produced by the unmodified reference.  The model is
    built as the fixture's reference model was: ``localpool_tanh_ref`` without GCN bias, with ``nn.Tanh`` (applied by
    torch, outside the kernels) and localpool supports; ``cheb7_linear_ref`` without bias or activation, 8 supports."""
    meta, params, grads, supports, _, blob = load_golden(name)
    model = build_model(meta, DEV)
    model.load_state_dict(params)
    x = torch.from_numpy(blob["x"]).to(DEV)
    y = torch.from_numpy(blob["y"]).to(DEV)
    sups = [s.to(DEV) for s in supports]
    out = model(obs_seq=x, sta_adj_list=sups)
    loss = nn.MSELoss(reduction="mean")(out, y)
    loss.backward()
    assert_close(out.detach().cpu().numpy(), blob["out"], f"{name} forward")
    assert abs(loss.item() - float(blob["loss"])) <= 1e-5 * max(1.0, abs(float(blob["loss"])))
    for key, p in model.named_parameters():
        assert p.grad is not None, key
        assert_close(p.grad.cpu().numpy(), grads[key], f"{name} grad {key}")
    # inference mode (Model_Trainer.py:33 set_grad_enabled(False)) gives the same output
    with torch.no_grad():
        out2 = model(obs_seq=x, sta_adj_list=sups)
    assert_close(out2.cpu().numpy(), blob["out"], f"{name} no_grad forward")


def _mid_case(n, m, k, t, b, c, hid, layers, gcn_hid, seed, dens=0.05):
    from stmgcn_b200 import synth
    adjs = [synth.make_adjacency(n, g, dens) for g in range(m)]
    gen = torch.Generator().manual_seed(seed)
    adjs = [a * (0.5 + torch.rand(n, n, generator=gen)) for a in adjs]          # weighted, asymmetric
    sups = [O.chebyshev_supports_dense(a, k, lambda_max=1.7) for a in adjs]     # non-unit diagonal in L~
    params = O.init_params(m, t, c, hid, layers, gcn_hid, k + 1, seed=seed)
    x = torch.randn(b, t, n, c, generator=gen)
    y = torch.randn(b, n, c, generator=gen)
    return sups, params, x, y


@pytest.mark.parametrize("shape", [
    dict(n=256, m=3, k=3, t=12, b=8, c=1, hid=64, layers=3, gcn_hid=64),      # cfg2/3 shapes, small N/B
    dict(n=130, m=2, k=5, t=24, b=3, c=1, hid=64, layers=3, gcn_hid=64),      # cfg5 shapes, ragged N
    dict(n=65, m=1, k=0, t=1, b=1, c=3, hid=32, layers=1, gcn_hid=20),        # K=0, T=1, B=1
    dict(n=50, m=2, k=2, t=7, b=5, c=2, hid=128, layers=2, gcn_hid=68),       # H=128 (two column panels)
])
def test_model_matches_sparse_oracle(shape):
    """fwd + bwd vs the fp64 sparse oracle (itself pinned to the reference in tests/test_oracle.py)."""
    from helpers import build_model
    sups, params, x, y = _mid_case(seed=3, **shape)
    model = build_model(shape, DEV)
    model.load_state_dict(params)
    out = model(obs_seq=x.to(DEV), sta_adj_list=[s.to(DEV) for s in sups])
    loss = nn.MSELoss()(out, y.to(DEV))
    loss.backward()
    orc = O.SparseOracle({k_: v.numpy() for k_, v in params.items()},
                         [O.laplacian_csr_from_supports(s) for s in sups], shape["k"] + 1, dtype=np.float64)
    o_ref, l_ref, g_ref = orc.loss_and_grads(x.numpy(), y.numpy())
    assert_close(out.detach().cpu().numpy(), o_ref, "forward")
    assert abs(loss.item() - l_ref) <= 1e-5 * max(1.0, abs(l_ref))
    for key, p in model.named_parameters():
        assert_close(p.grad.cpu().numpy(), g_ref[key], f"grad {key}")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_second_device_of_the_process_computes_the_same():
    """The dynamic shared-memory limit is a per-device kernel attribute.  After the H = 128 model (exact-fp32 LSTM and
    projection: tall GEMMs with more than 48 KB of shared memory) ran on cuda:0, the same model runs on cuda:1 in the
    same process and gives the same forward and gradients."""
    shape = dict(n=50, m=2, k=2, t=7, b=5, c=2, hid=128, layers=2, gcn_hid=68)
    sups, params, x, y = _mid_case(seed=3, **shape)
    results = []
    for dev in ("cuda:0", "cuda:1"):
        with torch.cuda.device(dev):
            model = build_model(shape, dev)
            model.load_state_dict(params)
            out = model(obs_seq=x.to(dev), sta_adj_list=[s.to(dev) for s in sups])
            nn.MSELoss()(out, y.to(dev)).backward()
            torch.cuda.synchronize()
        results.append((out.detach().cpu().numpy(), {k_: p.grad.cpu().numpy() for k_, p in model.named_parameters()}))
    (out0, grads0), (out1, grads1) = results
    assert_close(out1, out0, "cuda:1 forward vs cuda:0")
    for key, g in grads0.items():
        assert_close(grads1[key], g, f"cuda:1 grad {key} vs cuda:0")


def test_gcn_generic_supports_and_no_activation():
    """localpool-style supports (A[0] != I) take the generic path; activation=None; x with odd strides."""
    import GCN
    n, b, p, q = 70, 4, 6, 10
    adj = torch.from_numpy((_rand_csr(n, 0.1, 5, asym=False) != 0).astype(np.float32))
    adj.fill_diagonal_(0)
    sup = GCN.Adj_Preprocessor("localpool", 1).process(adj)
    assert sup.shape == (1, n, n)
    torch.manual_seed(0)
    layer = GCN.GCN(K=1, input_dim=p, hidden_dim=q, bias=True, activation=None).to(DEV)
    x = torch.randn(b, p, n).permute(0, 2, 1)                      # non-contiguous (B,N,p) view
    xd = x.to(DEV).requires_grad_(True)
    out = layer(sup.to(DEV), xd)
    ref_x = x.clone().requires_grad_(True)
    w, bias = layer.W.detach().cpu(), layer.b.detach().cpu()
    w.requires_grad_(True)
    ref = O.dense_gcn(sup, ref_x, w, bias, relu=False)
    assert_close(out.detach().cpu().numpy(), ref.detach().numpy(), "generic forward")
    gsum = torch.randn(b, n, q)
    (out * gsum.to(DEV)).sum().backward()
    (ref * gsum).sum().backward()
    assert_close(xd.grad.cpu().numpy(), ref_x.grad.numpy(), "generic dX")
    assert_close(layer.W.grad.cpu().numpy(), w.grad.numpy(), "generic dW")


def test_cg_lstm_with_initial_hidden_state():
    import STMGCN
    from stmgcn_b200 import synth
    n, b, t, c, hid, lyr, k = 40, 3, 5, 1, 16, 2, 2
    sup = O.chebyshev_supports_dense(synth.make_adjacency(n, 0, 0.2), k)
    torch.manual_seed(4)
    mod = STMGCN.CG_LSTM(seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=lyr, K=k + 1,
                         gconv_use_bias=True).to(DEV)
    obs = torch.randn(b, t, n, c)
    h0, c0 = torch.randn(lyr, b * n, hid) * 0.3, torch.randn(lyr, b * n, hid) * 0.3
    out, (hn, cn) = mod(sup.to(DEV), obs.to(DEV), (h0.to(DEV), c0.to(DEV)))
    params = {"p." + k_: v.detach().cpu() for k_, v in mod.state_dict().items()}
    ref, (hn_r, cn_r) = O.dense_cg_lstm(sup, obs, params, "p.", hidden=(h0, c0))
    assert_close(out.detach().cpu().numpy(), ref.numpy(), "cg_lstm out")
    assert_close(hn.detach().cpu().numpy(), hn_r.numpy(), "h_n")
    assert_close(cn.detach().cpu().numpy(), cn_r.numpy(), "c_n")


def test_sparse_native_supports_equal_dense():
    """Adj_Preprocessor.process_sparse (no dense polynomials) gives the same forward as the dense stack."""
    import GCN
    from stmgcn_b200 import synth
    meta = dict(n=200, m=2, k=3, t=6, b=4, c=1, hid=32, layers=2, gcn_hid=16)
    adjs = [synth.make_adjacency(200, g, 0.05) for g in range(2)]
    pre = GCN.Adj_Preprocessor("chebyshev", 3)
    dense = [pre.process(a).to(DEV) for a in adjs]
    sparse = [pre.process_sparse(a).to(DEV) for a in adjs]
    torch.manual_seed(1)
    model = build_model(meta, DEV)
    x = torch.randn(4, 6, 200, 1, device=DEV)
    with torch.no_grad():
        a = model(obs_seq=x, sta_adj_list=dense)
        b_ = model(obs_seq=x, sta_adj_list=sparse)
    assert_close(b_.cpu().numpy(), a.cpu().numpy(), "sparse-native vs dense supports", 1e-5)


def test_errors_are_loud():
    import GCN
    from stmgcn_b200 import ops
    layer = GCN.GCN(K=2, input_dim=4, hidden_dim=4).to(DEV)
    with pytest.raises(RuntimeError):
        layer(torch.eye(8).repeat(2, 1, 1), torch.randn(1, 8, 4, device=DEV))      # supports on CPU
    with pytest.raises(AssertionError):
        layer(torch.eye(8, device=DEV).repeat(3, 1, 1), torch.randn(1, 8, 4, device=DEV))   # K mismatch (GCN.py:31)
    with pytest.raises(RuntimeError):
        ops.obs_to_node_major(torch.randn(2, 3, 4, 1))                               # CPU tensor


@pytest.mark.parametrize("rows_n,b,t,c", [(5, 60, 3, 1), (3, 50, 2, 2), (40, 64, 4, 1), (7, 36, 8, 1), (2, 1100, 4, 1)])
def test_lstm_tensor_core_path_matches_exact_fp32_path(rows_n, b, t, c):
    """tensor-core (wgmma) LSTM forward vs the exact-FFMA kernels on the same inputs (ragged 128-row tiles)."""
    from stmgcn_b200 import ops
    hid, lyr = 64, 3
    gen = torch.Generator().manual_seed(rows_n * 100 + t)
    xo = torch.randn(rows_n, b, t, c, generator=gen).to(DEV)
    s = torch.rand(b, t, generator=gen).to(DEV)
    ws = []
    for l in range(lyr):
        in_l = c if l == 0 else hid
        ws += [torch.randn(4 * hid, in_l, generator=gen) * 0.2, torch.randn(4 * hid, hid, generator=gen) * 0.2,
               torch.randn(4 * hid, generator=gen) * 0.1, torch.randn(4 * hid, generator=gen) * 0.1]
    ws = [w.to(DEV) for w in ws]
    h0 = (torch.randn(lyr, rows_n * b, hid, generator=gen) * 0.3).to(DEV)
    c0 = (torch.randn(lyr, rows_n * b, hid, generator=gen) * 0.3).to(DEV)
    outs = {}
    old = ops.lstm_path()
    try:
        for path in ("fma", "tc"):
            ops.set_lstm_path(path)
            with torch.no_grad():
                outs[path] = [v.clone() for v in ops.SharedLSTM.apply(xo, s, h0, c0, lyr, hid, True, *ws)]
    finally:
        ops.set_lstm_path(old)
    for name, a, b_ in zip(("h_top", "h_n", "c_n"), outs["tc"], outs["fma"]):
        assert_close(a.cpu().numpy(), b_.cpu().numpy(), f"tc vs fma {name}", 2e-5)


# (7, 36, 8): ragged last tile with the TMA-fed layer-0 inputs; (2, 1100, 4): batch larger than the shared-memory gate
# column (global-atomic adjoint path)
@pytest.mark.parametrize("rows_n,b,t,c", [(5, 60, 3, 1), (40, 64, 4, 1), (3, 50, 2, 2), (7, 36, 8, 1), (2, 1100, 4, 1)])
def test_lstm_tensor_core_backward_matches_exact_fp32_path(rows_n, b, t, c):
    """tensor-core (wgmma) fused BPTT kernel (pointwise in the loader + dA.Wp^T) vs the exact-FFMA kernels: d_s and all
    LSTM weight gradients (C=2 exercises the mixed case: layer 0 on FFMA, layers > 0 on tensor cores)."""
    from stmgcn_b200 import ops
    hid, lyr = 64, 3
    gen = torch.Generator().manual_seed(7 + rows_n)
    xo = torch.randn(rows_n, b, t, c, generator=gen).to(DEV)
    s0 = torch.rand(b, t, generator=gen).to(DEV)
    ws0 = []
    for l in range(lyr):
        in_l = c if l == 0 else hid
        ws0 += [torch.randn(4 * hid, in_l, generator=gen) * 0.2, torch.randn(4 * hid, hid, generator=gen) * 0.2,
                torch.randn(4 * hid, generator=gen) * 0.1, torch.randn(4 * hid, generator=gen) * 0.1]
    proj = torch.randn(rows_n, b, hid, generator=gen).to(DEV)
    res = {}
    old = ops.lstm_path()
    try:
        for path in ("fma", "tc"):
            ops.set_lstm_path(path)
            s = s0.clone().requires_grad_(True)
            ws = [w.to(DEV).requires_grad_(True) for w in ws0]
            h_top, _, _ = ops.SharedLSTM.apply(xo, s, None, None, lyr, hid, False, *ws)
            (h_top * proj).sum().backward()
            res[path] = [s.grad.clone()] + [w.grad.clone() for w in ws]
    finally:
        ops.set_lstm_path(old)
    names = ["d_s"] + [f"w{i}" for i in range(4 * lyr)]
    for name, a, b_ in zip(names, res["tc"], res["fma"]):
        assert_close(a.cpu().numpy(), b_.cpu().numpy(), f"tc vs fma {name}", 5e-5)


def test_training_loop_like_model_trainer(tmp_path):
    """Drive the drop-in model the way Model_Trainer.py does (Adam with L2 weight decay :13, train/eval modes,
    set_grad_enabled :33, keyword forward :35, checkpoint save/load :52,:70-71) and compare the parameter
    trajectory with the dense CPU oracle trained identically."""
    meta = dict(n=48, m=2, k=2, t=5, b=6, c=1, hid=64, layers=3, gcn_hid=64)
    sups, params, x, y = _mid_case(seed=11, **meta)
    model = build_model(meta, DEV)
    model.load_state_dict(params)
    opt = torch.optim.Adam(params=model.parameters(), lr=2e-3, weight_decay=1e-4)       # Main.py:13, Model_Trainer.py:13
    crit = nn.MSELoss(reduction="mean")
    ref = {k_: v.clone().requires_grad_(True) for k_, v in params.items()}
    ref_opt = torch.optim.Adam(params=list(ref.values()), lr=2e-3, weight_decay=1e-4)
    sd = [s.to(DEV) for s in sups]
    xd, yd = x.to(DEV), y.to(DEV)
    for step in range(3):
        model.train()
        with torch.set_grad_enabled(True):
            loss = crit(model(obs_seq=xd, sta_adj_list=sd), yd)
            opt.zero_grad()
            loss.backward()
            opt.step()
        ref_loss = crit(O.dense_st_mgcn(ref, x, sups), y)
        ref_opt.zero_grad()
        ref_loss.backward()
        ref_opt.step()
        assert abs(loss.item() - ref_loss.item()) <= 2e-5 * max(1.0, abs(ref_loss.item())), step
    for key, p in model.named_parameters():
        # Adam divides by sqrt(v): where a gradient component is ~1e-8 the update direction is ill-conditioned, and the
        # 3xBF16 products (gradients within ~1e-5 of exact, still 10x inside the 1e-4 parity bar) move such components
        # by a few 1e-4 of the largest parameter after three steps (measured 2.4e-4)
        assert_close(p.detach().cpu().numpy(), ref[key].detach().numpy(), f"param after 3 Adam steps: {key}", 1e-3)
    # validate / test phase: eval mode, no grad, checkpoint round trip
    model.eval()
    with torch.set_grad_enabled(False):
        out_eval = model(obs_seq=xd, sta_adj_list=sd)
    path = tmp_path / "ST_MGCN_best_model.pkl"
    torch.save({"epoch": 1, "state_dict": model.state_dict()}, path)
    model2 = build_model(meta, DEV)
    model2.load_state_dict(torch.load(path)["state_dict"])
    model2.eval()
    with torch.no_grad():
        out2 = model2(obs_seq=xd, sta_adj_list=sd)
    # (not bit-identical: the region pooling accumulates with atomics in a run-dependent order)
    assert_close(out2.cpu().numpy(), out_eval.cpu().numpy(), "checkpoint round trip", 1e-5)
    assert_close(out_eval.cpu().numpy(), O.dense_st_mgcn({k_: v.detach() for k_, v in ref.items()}, x, sups).numpy(),
                 "eval forward after training", 2e-4)


@pytest.mark.parametrize("ks", [1, 3, 4, 6])
def test_projection_tensor_core_path_matches_exact_fp32_path(ks):
    """tensor-core (wgmma) projection (fwd, dZ/U, dW) vs the exact-FFMA kernels; ks = 3 exercises the odd 64-row tail block of dW."""
    from stmgcn_b200 import ops
    from stmgcn_b200.graph import GraphHandle, SupportSet
    n, b, p, q = 37, 9, 64, 64                                  # 333 rows: ragged 128-row tiles
    lap = _rand_csr(n, 0.2, 3)
    g = GraphHandle.from_dense(torch.from_numpy(lap).to(DEV))
    sset = SupportSet("cheb", n, ks, [g] if ks > 1 else [], torch.device(DEV))
    gen = torch.Generator().manual_seed(ks)
    x0 = torch.randn(n, b, p, generator=gen)
    w0 = torch.randn(ks * p, q, generator=gen) * 0.1
    b0 = torch.randn(q, generator=gen) * 0.1
    proj = torch.randn(n, b, q, generator=gen).to(DEV)
    res = {}
    old = ops.lstm_path()
    try:
        for path in ("fma", "tc"):
            ops.set_lstm_path(path)
            x = x0.to(DEV).requires_grad_(True)
            w = w0.to(DEV).requires_grad_(True)
            bb = b0.to(DEV).requires_grad_(True)
            out = ops.ChebGCN.apply(x, w, bb, sset, 1)
            (out * proj).sum().backward()
            res[path] = [out.detach().clone(), x.grad.clone(), w.grad.clone(), bb.grad.clone()]
    finally:
        ops.set_lstm_path(old)
    for name, a, c in zip(("out", "dx", "dW", "db"), res["tc"], res["fma"]):
        assert_close(a.cpu().numpy(), c.cpu().numpy(), f"proj tc vs fma {name}", 2e-5)


def test_bf16_arithmetic_mode_within_the_reference_bf16_tolerance():
    """STMGCN_LSTM_PLANES=1 / ops.set_lstm_planes(1): hidden states are stored as ONE bf16 plane and the shared LSTM's
    tensor-core products with them run single-pass (fp32 cell state, accumulation and on-chip dA) -- the arithmetic of the
    bf16-quoted BASELINE configs.  The 1e-4 bar is an fp32 statement; SURVEY.md section 8(d) measured the reference's OWN
    bf16 execution at 1.9-2.2e-2 from its fp32 output, which is the tolerance here.
    Forward: against the reference's golden output (ReLU model).  Gradients: on the same model WITHOUT the GCN activation --
    with ReLU, bf16-level noise in h flips ~1e-3 of the masks of a 37 k-element GCN output and moves the gradients of a
    6-window batch by ~10 % (measured), which says nothing about the kernels; the smooth model isolates the arithmetic."""
    from stmgcn_b200 import ops
    meta, params, grads, supports, _, blob = load_golden("cfg3_small_ref")
    x = torch.from_numpy(blob["x"]).to(DEV)
    y = torch.from_numpy(blob["y"]).to(DEV)
    sups = [s.to(DEV) for s in supports]
    old = ops.lstm_planes()
    try:
        ops.set_lstm_planes(1)
        model = build_model(meta, DEV)
        model.load_state_dict(params)
        with torch.no_grad():
            out = model(obs_seq=x, sta_adj_list=sups)
        smooth = build_model(meta, DEV, relu=False)
        smooth.load_state_dict(params)
        out_s = smooth(obs_seq=x, sta_adj_list=sups)
        nn.MSELoss(reduction="mean")(out_s, y).backward()
    finally:
        ops.set_lstm_planes(old)
    e_out = assert_close(out.cpu().numpy(), blob["out"], "bf16 mode forward (ReLU model, reference golden)", 2e-2)
    orc = O.SparseOracle({k_: v.numpy() for k_, v in params.items()},
                         [O.laplacian_csr_from_supports(s) for s in supports], meta["k"] + 1, relu=False, dtype=np.float64)
    o_ref, _, g_ref = orc.loss_and_grads(blob["x"], blob["y"])
    e_out_s = assert_close(out_s.detach().cpu().numpy(), o_ref, "bf16 mode forward (smooth model)", 2e-2)
    errs = {key: O.max_rel_err(p.grad.cpu().numpy(), g_ref[key]) for key, p in smooth.named_parameters()}
    print(f"bf16 arithmetic mode: forward error {e_out:.2e} (ReLU) / {e_out_s:.2e} (smooth); worst gradient error "
          f"{max(errs.values()):.2e} ({max(errs, key=errs.get)}); tolerance 2e-2; all: "
          + ", ".join(f"{k} {v:.1e}" for k, v in sorted(errs.items(), key=lambda kv: -kv[1])[:12]))
    bad = {k: v for k, v in errs.items() if not v <= 2e-2}
    assert not bad, f"bf16 mode gradients above 2e-2: {bad}"
    assert e_out > 1e-6, "the bf16 mode produced fp32-grade results: the single-pass path did not run"
