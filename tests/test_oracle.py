"""CPU tests of the oracle (test infrastructure): pinned against the golden vectors generated from the
unmodified reference modules (tests/golden/*.npz, oracle/make_golden.py) and against closed-form known answers."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import stmgcn_oracle as O
from helpers import TOL, assert_close, load_golden


@pytest.mark.parametrize("name", ["cfg1_ref", "ragged_ref", "cfg3_small_ref"])
def test_dense_oracle_matches_reference_golden(name):
    meta, params, grads, supports, adjs, blob = load_golden(name)
    x, y = torch.from_numpy(blob["x"]), torch.from_numpy(blob["y"])
    out, loss, g = O.dense_loss_and_grads(params, x, y, supports)
    assert_close(out.numpy(), blob["out"], "forward", 1e-5)
    assert abs(float(loss) - float(blob["loss"])) < 1e-6
    for key in grads:
        assert_close(g[key].numpy(), grads[key], f"grad {key}", 2e-5)
    # support construction (GCN.py:57-97) restated
    for a, s in zip(adjs, supports):
        assert_close(O.chebyshev_supports_dense(a, meta["k"]).numpy(), s.numpy(), "supports", 1e-6)


@pytest.mark.parametrize("name", ["cfg1_ref", "ragged_ref", "cfg3_small_ref"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_sparse_oracle_matches_reference_golden(name, dtype):
    """Recurrence-on-features + hand-written backward == the reference's dense forward + autograd."""
    meta, params, grads, supports, _, blob = load_golden(name)
    orc = O.SparseOracle({k: v.numpy() for k, v in params.items()},
                         [O.laplacian_csr_from_supports(s) for s in supports], meta["k"] + 1, dtype=dtype)
    out, loss, g = orc.loss_and_grads(blob["x"], blob["y"])
    assert_close(out, blob["out"], "forward", 1e-5)
    assert abs(loss - float(blob["loss"])) < 1e-5
    for key in grads:
        assert_close(g[key], grads[key], f"grad {key}", 2e-5)


NEW_GOLDENS = ["localpool_tanh_ref", "cheb7_linear_ref"]


@pytest.mark.parametrize("name", NEW_GOLDENS)
def test_dense_oracle_matches_configured_reference_golden(name):
    """The dense restatement with the fixture's configuration (no GCN bias; ``nn.Tanh`` or no activation; localpool or
    Chebyshev K = 7) in fp64 reproduces the unmodified reference's fp32 forward, loss and every gradient."""
    from helpers import oracle_activation
    meta, params, grads, supports, adjs, blob = load_golden(name)
    assert not meta["bias"] and not any(k.endswith(".b") for k in params)
    x, y = torch.from_numpy(blob["x"]).double(), torch.from_numpy(blob["y"]).double()
    out, loss, g = O.dense_loss_and_grads({k: v.double() for k, v in params.items()}, x, y,
                                          [s.double() for s in supports], relu=oracle_activation(meta["activation"]))
    assert_close(out.numpy(), blob["out"], "forward", 1e-5)
    assert abs(float(loss) - float(blob["loss"])) < 1e-6
    assert set(g) == set(grads)
    for key in grads:
        assert_close(g[key].numpy(), grads[key], f"grad {key}", 2e-5)
    for a, s in zip(adjs, supports):            # support construction (GCN.py:57-97) restated
        if meta["kernel_type"] == "localpool":
            d = a.sum(1).pow(-0.5)
            want = (torch.eye(a.shape[0]) + d[:, None] * a * d[None, :])[None]
        else:
            want = O.chebyshev_supports_dense(a, meta["k"])
        assert_close(want.numpy(), s.numpy(), "supports", 1e-6)


def _small_model(relu_case, seed=0):
    from stmgcn_b200 import synth
    n, m, k, t, b, c, hid, lyr, g = 14, 2, 2, 4, 3, 2, 8, 2, 6
    adjs = [synth.make_adjacency(n, i, 0.3) for i in range(m)]
    sups = [O.chebyshev_supports_dense(a.double(), k, lambda_max=1.8) for a in adjs]
    params = {kk: v.double() for kk, v in O.init_params(m, t, c, hid, lyr, g, k + 1, seed=seed).items()}
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(b, t, n, c, generator=gen).double()
    y = torch.randn(b, n, c, generator=gen).double()
    return sups, params, x, y, k + 1


@pytest.mark.parametrize("relu", [True, False])
def test_dense_restatement_with_relu_or_none_is_the_sparse_oracle(relu):
    """The activation argument at ReLU (True, or an ``nn.ReLU()`` module) and at none (False, or None) gives the model of
    :class:`O.SparseOracle` at 1e-12 in fp64: forward, loss, every gradient and d obs."""
    sups, params, x, y, ks = _small_model(relu)
    orc = O.SparseOracle({k: v.numpy() for k, v in params.items()}, [O.laplacian_csr_from_supports(s) for s in sups],
                         ks, relu=relu, dtype=np.float64)
    o_ref, l_ref, g_ref = orc.loss_and_grads(x.numpy(), y.numpy())
    for act in ([True, torch.nn.ReLU()] if relu else [False, None]):
        out, loss, g = O.dense_loss_and_grads(params, x, y, sups, relu=act, want_obs=True)
        assert_close(out.numpy(), o_ref, "forward", 1e-12)
        assert abs(float(loss) - l_ref) <= 1e-12 * l_ref
        for key in g_ref:
            assert_close(g[key].numpy(), g_ref[key], f"grad {key}", 1e-12)
        # d obs against autograd through the restatement itself (the sparse oracle has no d obs)
        xd = x.clone().requires_grad_(True)
        (d_obs,) = torch.autograd.grad(torch.mean((O.dense_st_mgcn(params, xd, sups, relu) - y) ** 2), [xd])
        assert_close(g["obs"].numpy(), d_obs.numpy(), "d obs", 1e-12)


def test_dense_restatement_forced_with_its_own_relu_masks_changes_nothing():
    """Masks equal to the restatement's own ``z > 0``, handed back in the kernels' order and layout (temporal 0,
    spatial 0, temporal 1, ...; node-major (N, B, q)), change no value and no gradient; other masks do."""
    sups, params, x, y, _ = _small_model(True, seed=1)
    masks, real = [], O.dense_gcn

    def recording(supports, x_, w, b, relu=True, mask=None):
        z = real(supports, x_, w, b, False)
        masks.append((z > 0).permute(1, 0, 2))
        return real(supports, x_, w, b, relu, mask)
    O.dense_gcn = recording
    try:
        out0, loss0, g0 = O.dense_loss_and_grads(params, x, y, sups, want_obs=True)
    finally:
        O.dense_gcn = real
    assert len(masks) == 4 and [tuple(mk.shape) for mk in masks[:2]] == [(14, 3, 4), (14, 3, 6)]
    out1, loss1, g1 = O.dense_loss_and_grads(params, x, y, sups, masks=masks, want_obs=True)
    assert torch.equal(out1, out0) and float(loss1) == float(loss0)
    for key in g0:
        assert torch.allclose(g1[key], g0[key], rtol=0, atol=1e-15), key
    flipped = [mk.clone() for mk in masks]
    flipped[1][0] = ~flipped[1][0]              # one region of graph 0's spatial GCN takes the other branch
    out2, _, _ = O.dense_loss_and_grads(params, x, y, sups, masks=flipped)
    assert O.max_rel_err(out2.numpy(), out0.numpy()) > 1e-3
    with pytest.raises(ValueError, match="ReLU masks for 2 graphs"):
        O.dense_st_mgcn(params, x, sups, masks=masks[:3])
    with pytest.raises(ValueError, match="needs the ReLU activation"):
        O.dense_st_mgcn(params, x, sups, relu=False, masks=masks)


def test_lstm_explicit_equals_library_lstm():
    gen = torch.Generator().manual_seed(0)
    layers = []
    for l in range(3):
        in_l = 2 if l == 0 else 8
        layers.append(tuple(torch.randn(*s, generator=gen) * 0.3 for s in ((32, in_l), (32, 8), (32,), (32,))))
    x = torch.randn(5, 7, 2, generator=gen)
    h0, c0 = torch.randn(3, 5, 8, generator=gen), torch.randn(3, 5, 8, generator=gen)
    a, (ha, ca) = O.lstm_explicit(x, layers, h0, c0)
    b, (hb, cb) = O.lstm_library(x, layers, h0, c0)
    assert_close(a.numpy(), b.detach().numpy(), "seq", 1e-5)
    assert_close(ha.numpy(), hb.detach().numpy(), "h_n", 1e-5)
    assert_close(ca.numpy(), cb.detach().numpy(), "c_n", 1e-5)


def test_known_answer_chebyshev_eigenvector():
    """T_k(L) v = cos(k arccos(lambda)) v for an eigenvector v of a symmetric L with |lambda| <= 1."""
    n, k_ord = 12, 5
    # ring graph: A_norm has eigenvalues cos(2 pi j / n); L~ = -A_norm (lambda_max = 2)
    adj = torch.zeros(n, n)
    idx = torch.arange(n)
    adj[idx, (idx + 1) % n] = 1
    adj[(idx + 1) % n, idx] = 1
    sup = O.chebyshev_supports_dense(adj.double(), k_ord)
    j = 2
    v = torch.cos(2 * np.pi * j * idx.double() / n)
    lam = -np.cos(2 * np.pi * j / n)
    for k in range(k_ord + 1):
        want = np.cos(k * np.arccos(lam)) * v
        assert torch.allclose(sup[k] @ v, want, atol=1e-12)
    # the sparse oracle's feature recurrence gives the same
    orc = O.SparseOracle({"rnn_list.0.lstm.weight_ih_l0": np.zeros((4, 1))}, [sp.csr_matrix(sup[1].numpy())], k_ord + 1)
    st = orc._cheb_stack(orc.lap[0], v.numpy().reshape(n, 1, 1))
    for k in range(k_ord + 1):
        assert np.allclose(st[k].ravel(), np.cos(k * np.arccos(lam)) * v.numpy(), atol=1e-12)


def test_known_answer_ring_graph_spectrum():
    """Ring graph: the normalised adjacency has eigenvalues cos(2 pi j / n), so the rescaled Laplacian supports[1]
    (lambda_max = 2, GCN.py:86-93) has spectrum -cos(2 pi j / n) and supports[k] has spectrum T_k of it."""
    n, k_ord = 16, 3
    adj = torch.zeros(n, n, dtype=torch.float64)
    idx = torch.arange(n)
    adj[idx, (idx + 1) % n] = 1
    adj[(idx + 1) % n, idx] = 1
    sup = O.chebyshev_supports_dense(adj, k_ord)
    lam = np.sort(-np.cos(2 * np.pi * np.arange(n) / n))
    got = np.sort(np.linalg.eigvalsh(sup[1].numpy()))
    assert np.allclose(got, lam, atol=1e-12)
    for k in range(k_ord + 1):
        want = np.sort(np.cos(k * np.arccos(np.clip(lam, -1, 1))))
        assert np.allclose(np.sort(np.linalg.eigvalsh(sup[k].numpy())), want, atol=1e-10)


def test_chain_stack_of_one_chain_is_the_chebyshev_stack():
    """``chain_stack_dense`` of the single chain L~ is ``chebyshev_supports_dense`` of the adjacency, T_0 .. T_K."""
    from stmgcn_b200 import synth
    adj = synth.make_adjacency(40, 0, 0.2).double()
    for order in (1, 2, 5):
        want = O.chebyshev_supports_dense(adj, order)
        got = O.chain_stack_dense([O.rescaled_laplacian_dense(adj)], order)
        assert got.shape == want.shape, (order, got.shape, want.shape)
        assert_close(got.numpy(), want.numpy(), f"chain stack, K = {order}", 1e-12)


def test_known_answer_order_zero_gcn_is_a_linear_layer():
    x = torch.randn(3, 9, 4)
    w, b = torch.randn(4, 5), torch.randn(5)
    out = O.dense_gcn(torch.eye(9)[None], x, w, b, relu=False)
    assert torch.allclose(out, x @ w + b, atol=1e-6)


def test_known_answer_lstm_zero_weights():
    """Zero weights: h = sigmoid(b_o) tanh(sigmoid(b_i) tanh(b_g)) after one step."""
    hid = 3
    bias = torch.tensor([0.3] * hid + [9.9] * hid + [-0.7] * hid + [1.1] * hid)
    layers = [(torch.zeros(4 * hid, 2), torch.zeros(4 * hid, hid), bias, torch.zeros(4 * hid))]
    seq, _ = O.lstm_explicit(torch.randn(4, 1, 2), layers)
    want = torch.sigmoid(torch.tensor(1.1)) * torch.tanh(torch.sigmoid(torch.tensor(0.3)) * torch.tanh(torch.tensor(-0.7)))
    assert torch.allclose(seq, want.expand_as(seq), atol=1e-7)


def test_sparse_oracle_handles_asymmetric_laplacian_and_hypothesis_shapes():
    """Dense (autograd) vs sparse (hand backward) on random asymmetric weighted graphs, odd shapes."""
    from stmgcn_b200 import synth
    for seed, (n, m, k, t, b, c, hid, lyr, g) in enumerate([(20, 2, 4, 3, 2, 2, 8, 2, 6), (33, 1, 1, 1, 1, 1, 4, 1, 4),
                                                            (17, 3, 5, 6, 3, 1, 8, 3, 8)]):
        gen = torch.Generator().manual_seed(seed)
        adjs = [synth.make_adjacency(n, i, 0.3) * (0.2 + torch.rand(n, n, generator=gen)) for i in range(m)]
        sups = [O.chebyshev_supports_dense(a, k, lambda_max=1.6) for a in adjs]
        params = O.init_params(m, t, c, hid, lyr, g, k + 1, seed=seed)
        x, y = torch.randn(b, t, n, c, generator=gen), torch.randn(b, n, c, generator=gen)
        o1, l1, g1 = O.dense_loss_and_grads(params, x, y, sups)
        orc = O.SparseOracle({k_: v.numpy() for k_, v in params.items()},
                             [O.laplacian_csr_from_supports(s) for s in sups], k + 1, dtype=np.float64)
        o2, l2, g2 = orc.loss_and_grads(x.numpy(), y.numpy())
        assert_close(o2, o1.numpy(), "forward", 2e-5)
        for key in g1:
            assert_close(g2[key], g1[key].numpy(), f"grad {key}", 5e-5)


def test_dense_matches_reference_modules():
    """The restatement against the unmodified reference modules' own forward and autograd (tests/golden/small_ref.npz,
    oracle/make_golden.py: two graphs, two LSTM layers, H=16, G=8)."""
    _, params, grads, supports, _, blob = load_golden("small_ref")
    x, y = torch.from_numpy(blob["x"]), torch.from_numpy(blob["y"])
    o2, _, g2 = O.dense_loss_and_grads(params, x, y, supports)
    assert_close(o2.numpy(), blob["out"], "forward", 1e-5)
    assert set(g2) >= set(grads) and len(grads) > 0
    for key in grads:
        assert_close(g2[key].numpy(), grads[key], f"grad {key}", 2e-5)


def _rand_lstm(seed, c_in, hid, n_layers, rows, t_len, scale=0.3):
    gen = torch.Generator().manual_seed(seed)
    layers = []
    for l in range(n_layers):
        in_l = c_in if l == 0 else hid
        layers.append(tuple((torch.randn(*s, generator=gen, dtype=torch.float64) * scale).requires_grad_(True)
                            for s in ((4 * hid, in_l), (4 * hid, hid), (4 * hid,), (4 * hid,))))
    x = torch.randn(rows, t_len, c_in, generator=gen, dtype=torch.float64).requires_grad_(True)
    return gen, layers, x


def test_round_bf16_is_bf16_rounding_with_a_straight_through_gradient():
    v = (torch.randn(1000, dtype=torch.float64) * 3).requires_grad_(True)
    r = O.round_bf16(v)
    assert torch.equal(r.detach(), v.detach().float().to(torch.bfloat16).double())
    err = (r - v).detach().abs()
    assert 0 < float(err.max()) and bool((err <= v.detach().abs() * 2.0 ** -8).all())      # half an ulp: 8 significant bits
    r.backward(torch.arange(1000, dtype=torch.float64))
    assert torch.equal(v.grad, torch.arange(1000, dtype=torch.float64))


def test_lstm_planes_reference_two_planes_equals_the_lstm_oracles():
    """Two planes, no tape: the reference of the tensor-core LSTM is plain nn.LSTM arithmetic -- outputs equal
    lstm_explicit (with an initial state), autograd gradients equal SparseOracle's hand-written BPTT, to fp64 rounding."""
    hid, lyr, rows, t_len, c_in = 8, 3, 5, 6, 2
    gen, layers, x = _rand_lstm(0, c_in, hid, lyr, rows, t_len)
    h0, c0 = (torch.randn(lyr, rows, hid, generator=gen, dtype=torch.float64) * 0.3 for _ in range(2))
    seq, (hn, cn), (hs, cs) = O.lstm_planes_reference(x, layers, 2, h0, c0)
    seq_e, (hn_e, cn_e) = O.lstm_explicit(x, layers, h0, c0)
    for a, b, what in ((seq, seq_e, "seq"), (hn, hn_e, "h_n"), (cn, cn_e, "c_n"),
                       (torch.stack(hs[-1], 1), seq_e, "hs"), (torch.stack([c[-1] for c in cs]), cn_e, "cs")):
        assert_close(a.detach().numpy(), b.detach().numpy(), what, 1e-14)
    # gradients (no initial state: the sparse oracle's LSTM starts from zeros)
    seq, _, _ = O.lstm_planes_reference(x, layers, 2)
    d_top = torch.randn(rows, hid, generator=gen, dtype=torch.float64)
    flat = [w for layer in layers for w in layer]
    got = torch.autograd.grad((seq[:, -1] * d_top).sum(), [x] + flat)
    pre = "rnn_list.0.lstm."
    params = {}
    for l, layer in enumerate(layers):
        for name, w in zip(("weight_ih", "weight_hh", "bias_ih", "bias_hh"), layer):
            params[f"{pre}{name}_l{l}"] = w.detach().numpy()
    orc = O.SparseOracle(params, [], 1)
    h_top, saved = orc._lstm_fwd(x.detach().numpy(), pre)
    assert_close(seq[:, -1].detach().numpy(), h_top, "h_top vs SparseOracle", 1e-14)
    grads = {}
    dx = orc._lstm_bwd(d_top.numpy(), saved, pre, grads)
    assert_close(got[0].numpy(), dx, "dx vs SparseOracle", 1e-12)
    for i, g in enumerate(got[1:]):
        l, j = divmod(i, 4)
        name = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")[j]
        assert_close(g.numpy(), grads[f"{pre}{name}_l{l}"], f"{name}_l{l} vs SparseOracle", 1e-12)


@pytest.mark.parametrize("planes", [1, 2])
def test_lstm_planes_reference_tape_forcing_with_its_own_states_changes_nothing(planes):
    """Forcing the reference with a tape of its own states leaves outputs and autograd gradients unchanged: tape forcing
    only replaces VALUES, the gradient still flows through the computed states."""
    hid, lyr, rows, t_len, c_in = 8, 2, 4, 5, 3
    gen, layers, x = _rand_lstm(1, c_in, hid, lyr, rows, t_len)
    h0, c0 = (torch.randn(lyr, rows, hid, generator=gen, dtype=torch.float64) * 0.3 for _ in range(2))
    d_top = torch.randn(rows, hid, generator=gen, dtype=torch.float64)
    flat = [x] + [w for layer in layers for w in layer]
    seq, _, (hs, cs) = O.lstm_planes_reference(x, layers, planes, h0, c0)
    ref = torch.autograd.grad((seq[:, -1] * d_top).sum(), flat)
    tape = dict(h=torch.stack([torch.stack(v) for v in hs]).detach(), c=torch.stack([torch.stack(v) for v in cs]).detach(),
                h0=h0)
    seq_f, _, (hs_f, cs_f) = O.lstm_planes_reference(x, layers, planes, h0, c0, tape=tape)
    got = torch.autograd.grad((seq_f[:, -1] * d_top).sum(), flat)
    assert torch.allclose(seq_f, seq, rtol=0, atol=1e-15)
    for a, b in zip(got, ref):
        assert torch.allclose(a, b, rtol=1e-13, atol=1e-15)
    # one plane: the operands of the tensor-core products are bf16 -- a bf16-level change, far above fp64 rounding
    if planes == 1:
        seq2, _, _ = O.lstm_planes_reference(x, layers, 2, h0, c0)
        assert 1e-4 < O.max_rel_err(seq.detach().numpy(), seq2.detach().numpy()) < 2e-2


def test_lstm_planes_reference_rounds_only_the_tensor_core_operands():
    """One plane: h operands, W_hh and W_ih of layers > 0 are rounded to bf16; layer 0's W_ih (the fp32 FMA input term)
    and the biases are not.  A change far below one bf16 ulp moves the output only through the unrounded operands."""
    hid, lyr, rows, t_len, c_in = 8, 2, 3, 2, 1
    _, layers, x = _rand_lstm(2, c_in, hid, lyr, rows, t_len)
    def cells(ls):                     # the cell states of every layer-step (a change in h can vanish in its rounding)
        _, _, (_, cs) = O.lstm_planes_reference(x, ls, 1)
        return torch.stack([torch.stack(c) for c in cs])

    base = cells(layers)
    for l, j, moves in ((0, 0, True), (0, 1, False), (0, 2, True), (1, 0, False), (1, 1, False), (1, 3, True)):
        pert = [list(layer) for layer in layers]
        pert[l][j] = pert[l][j] + 1e-9 * torch.sign(pert[l][j].detach())
        assert bool((cells(pert) != base).any()) == moves, (l, j)


def test_sparse_oracle_relu_masks():
    """SparseOracle(relu_masks=...): the oracle's own masks (z > 0) change nothing; a flipped mask entry is followed in
    the forward (out = z * mask) and in the backward.  Without an activation the masks are ignored."""
    from stmgcn_b200 import synth
    n, m, k, t, b, c, hid, lyr, g = 15, 2, 2, 4, 2, 1, 8, 2, 6
    gen = torch.Generator().manual_seed(3)
    sups = [O.chebyshev_supports_dense(synth.make_adjacency(n, i, 0.3), k) for i in range(m)]
    params = {k_: v.numpy() for k_, v in O.init_params(m, t, c, hid, lyr, g, k + 1, seed=3).items()}
    x, y = torch.randn(b, t, n, c, generator=gen).numpy(), torch.randn(b, n, c, generator=gen).numpy()
    laps = [O.laplacian_csr_from_supports(s) for s in sups]

    class Recording(O.SparseOracle):
        def _gcn_fwd(self, lap, x_, w, b_):
            z, s = self._gcn_pre(lap, x_, w, b_)
            self.z.append(z)
            return super()._gcn_fwd(lap, x_, w, b_)

    rec = Recording(params, laps, k + 1)
    rec.z = []
    o0, l0, g0 = rec.loss_and_grads(x, y)
    masks = [z > 0 for z in rec.z]
    o1, l1, g1 = O.SparseOracle(params, laps, k + 1, relu_masks=masks).loss_and_grads(x, y)
    assert np.array_equal(o0, o1) and l0 == l1 and all(np.array_equal(g0[key], g1[key]) for key in g0)
    # flip the mask entry with the smallest |z| of graph 1's spatial GCN: the output moves by exactly that entry's change
    # (max(z, 0) -> z * mask) through the output layer, and the gradients follow the flipped branch
    z = rec.z[3]
    idx = np.unravel_index(np.argmin(np.abs(z)), z.shape)
    flipped = [mk.copy() for mk in masks]
    flipped[3][idx] = ~flipped[3][idx]
    o2, _, g2 = O.SparseOracle(params, laps, k + 1, relu_masks=flipped).loss_and_grads(x, y)
    want = o0.copy()
    delta = z[idx] * (1.0 if flipped[3][idx] else -1.0)            # out[idx] goes from max(z, 0) to z * mask
    fc_w = params["fc.weight"].astype(np.float64)
    want[idx[1], idx[0], :] += delta * fc_w[:, idx[2]]
    assert np.allclose(o2, want, rtol=0, atol=1e-12)
    assert any(not np.array_equal(g0[key], g2[key]) for key in g0)
    o3, _, g3 = O.SparseOracle(params, laps, k + 1, relu=False, relu_masks=flipped).loss_and_grads(x, y)
    o4, _, g4 = O.SparseOracle(params, laps, k + 1, relu=False).loss_and_grads(x, y)
    assert np.array_equal(o3, o4) and all(np.array_equal(g3[key], g4[key]) for key in g3)


def _bf16_case(seed, kind="chebyshev", n=17, m=2, k=3, t=5, b=3, c=2, hid=8, lyr=2, g=6):
    """A small random model for BF16ModeReference: (params (torch), chains per graph (scipy), n_supports, x, y)."""
    import diffusion_oracle as D
    from stmgcn_b200 import synth
    gen = torch.Generator().manual_seed(seed)
    if kind == "chebyshev":
        adjs = [synth.make_adjacency(n, i, 0.3) * (0.2 + torch.rand(n, n, generator=gen)) for i in range(m)]
        chains = [[O.laplacian_csr_from_supports(O.chebyshev_supports_dense(a.double(), k, lambda_max=1.6))] for a in adjs]
        ks = k + 1
    else:
        adjs = [synth.make_directed_adjacency(n, i, 0.3) for i in range(m)]
        chains = [D.diffusion_chains_csr(a.double()) for a in adjs]
        ks = 2 * k + 1
    params = O.init_params(m, t, c, hid, lyr, g, ks, seed=seed)
    x, y = torch.randn(b, t, n, c, generator=gen), torch.randn(b, n, c, generator=gen)
    return params, chains, ks, x, y


def test_csr_matmul_backward_is_the_transpose_product():
    a = sp.random(9, 9, 0.3, format="csr", random_state=0)
    lap, lap_t = O.torch_csr_pair(a)
    x = torch.randn(9, 4, dtype=torch.float64, requires_grad=True)
    g = torch.randn(9, 4, dtype=torch.float64)
    y = O.CsrMatmul.apply(x, lap, lap_t)
    (dx,) = torch.autograd.grad(y, x, g)
    dense = torch.from_numpy(a.toarray())
    assert torch.allclose(y, dense @ x, rtol=0, atol=1e-14)
    assert torch.allclose(dx, dense.t() @ g, rtol=0, atol=1e-14)


@pytest.mark.parametrize("relu", [True, False])
def test_bf16_mode_reference_without_rounding_is_the_sparse_oracle(relu):
    """Rounding off, no tapes: the fp64 torch model is the recurrence-on-features model of SparseOracle -- output, loss,
    every parameter gradient (one branch at a time through loss_and_grads) and the all-branches forward, to fp64
    rounding."""
    for seed, shape in enumerate([dict(), dict(n=23, m=3, k=2, t=4, b=2, c=1, lyr=3), dict(k=1, lyr=1, t=1)]):
        params, chains, ks, x, y = _bf16_case(seed, **shape)
        ref = O.BF16ModeReference(params, [ch for ch in chains], ks, relu=relu, rounding=False)
        out, loss, grads = ref.loss_and_grads(x, y, want_obs=True)
        orc = O.SparseOracle({k_: v.numpy() for k_, v in params.items()}, [ch[0] for ch in chains], ks, relu=relu)
        o2, l2, g2 = orc.loss_and_grads(x.numpy(), y.numpy())
        assert_close(out.numpy(), o2, "forward", 1e-12)
        assert abs(float(loss) - l2) <= 1e-12 * abs(l2)
        assert set(grads) == set(g2) | {"obs"}
        for key in g2:
            assert_close(grads[key].numpy(), g2[key], f"grad {key}", 1e-12)
        with torch.no_grad():
            assert_close(ref.forward(ref.leaves(), x.double()).numpy(), o2, "all-branch forward", 1e-12)
        # d obs against autograd through the dense restatement
        xd = x.double().requires_grad_(True)
        sups = []
        for ch in chains:
            lap = torch.from_numpy(ch[0].toarray())
            polys = [torch.eye(lap.shape[0], dtype=lap.dtype), lap]
            while len(polys) < ks:
                polys.append(2.0 * lap @ polys[-1] - polys[-2])
            sups.append(torch.stack(polys[:ks]))
        p64 = {k_: v.double() for k_, v in params.items()}
        (d_obs,) = torch.autograd.grad(torch.mean((O.dense_st_mgcn(p64, xd, sups, relu) - y.double()) ** 2), [xd])
        assert_close(grads["obs"].numpy(), d_obs.numpy(), "d obs", 1e-10)


def test_bf16_mode_reference_without_rounding_is_the_chain_oracle():
    """random_walk_diffusion (two chains per graph), rounding off: diffusion_oracle.ChainOracle, to fp64 rounding."""
    import diffusion_oracle as D
    params, chains, ks, x, y = _bf16_case(4, kind="random_walk_diffusion", k=2)
    out, loss, grads = O.BF16ModeReference(params, chains, ks, rounding=False).loss_and_grads(x, y)
    orc = D.ChainOracle({k_: v.numpy() for k_, v in params.items()}, chains, ks)
    o2, l2, g2 = orc.loss_and_grads(x.numpy(), y.numpy())
    assert_close(out.numpy(), o2, "forward", 1e-12)
    for key in g2:
        assert_close(grads[key].numpy(), g2[key], f"grad {key}", 1e-12)


def _random_masks(params, chains, ks, x, seed):
    """One random boolean ReLU mask (N, B, q) per GCN (temporal 0, spatial 0, temporal 1, ...): the model then follows
    branches no free-running forward would, so a mask sliced on the wrong axis or to the wrong windows shows."""
    gen = torch.Generator().manual_seed(seed)
    b, t, n, _ = x.shape
    g = params["gcn_list.0.W"].shape[1]
    return [torch.rand(n, b, q, generator=gen) < 0.6 for _ in chains for q in (t, g)]


@pytest.mark.parametrize("case", ["relu_masks", "smooth", "diffusion_relu_masks", "diffusion_smooth"])
def test_bf16_mode_reference_in_window_chunks_is_the_sparse_oracle(case):
    """``loss_and_grads(window_chunk=...)``: every branch's forward and backward a chunk of windows at a time, the
    gradients summed over chunks.  Chunks of 1 window, chunks that leave a ragged last chunk, and one chunk of the whole
    batch equal the unchunked model and SparseOracle / ChainOracle (Chebyshev / diffusion chains) to fp64 rounding:
    output, loss, every parameter gradient and d obs, with given ReLU masks (sliced to each chunk's windows) or without
    an activation."""
    import diffusion_oracle as D
    kind = "random_walk_diffusion" if case.startswith("diffusion") else "chebyshev"
    relu = case.endswith("relu_masks")
    params, chains, ks, x, y = _bf16_case(11, kind=kind, k=2, b=5, m=2, lyr=2)
    masks = _random_masks(params, chains, ks, x, 12) if relu else None
    ref = O.BF16ModeReference(params, chains, ks, relu=relu, rounding=False, relu_masks=masks)
    out, loss, grads = ref.loss_and_grads(x, y, want_obs=True)
    np_params = {k_: v.numpy() for k_, v in params.items()}
    np_masks = None if masks is None else [mk.numpy() for mk in masks]
    orc = (D.ChainOracle(np_params, chains, ks, relu=relu, relu_masks=np_masks) if kind != "chebyshev" else
           O.SparseOracle(np_params, [ch[0] for ch in chains], ks, relu=relu, relu_masks=np_masks))
    o2, l2, g2 = orc.loss_and_grads(x.numpy(), y.numpy())
    assert_close(out.numpy(), o2, "unchunked forward", 1e-12)
    for key in g2:
        assert_close(grads[key].numpy(), g2[key], f"unchunked grad {key}", 1e-12)
    for chunk in (1, 2, 3, x.shape[0]):                    # 2 and 3 leave a last chunk of 1 and 2 windows
        out_c, loss_c, grads_c = ref.loss_and_grads(x, y, want_obs=True, window_chunk=chunk)
        assert_close(out_c.numpy(), o2, f"chunk {chunk} forward", 1e-12)
        assert abs(float(loss_c) - l2) <= 1e-12 * abs(l2)
        assert set(grads_c) == set(g2) | {"obs"}
        for key in g2:
            assert_close(grads_c[key].numpy(), g2[key], f"chunk {chunk} grad {key}", 1e-12)
        assert_close(grads_c["obs"].numpy(), grads["obs"].numpy(), f"chunk {chunk} d obs", 1e-12)


def test_bf16_mode_reference_in_window_chunks_slices_the_tapes():
    """Rounding on and forced with tapes (rows n*B + b, and the spatial stacks (Ks, N, B, H)): each chunk takes its own
    windows' rows of the tapes, so the chunked model equals the unchunked one to fp64 rounding.  Forcing is per window
    (a tape with two windows swapped moves the output), so that agreement needs every chunk to take its own windows'."""
    params, chains, ks, x, y = _bf16_case(13, hid=16, b=5)
    ref = O.BF16ModeReference(params, chains, ks, relu=True)
    tapes = _own_tapes(ref, x)
    out, loss, grads = ref.loss_and_grads(x, y, tapes=tapes, want_obs=True)
    for chunk in (1, 2, 5):
        out_c, loss_c, grads_c = ref.loss_and_grads(x, y, tapes=tapes, want_obs=True, window_chunk=chunk)
        assert_close(out_c.numpy(), out.numpy(), f"chunk {chunk} forced forward", 1e-12)
        assert abs(float(loss_c) - float(loss)) <= 1e-12 * abs(float(loss))
        for key in grads:
            assert_close(grads_c[key].numpy(), grads[key].numpy(), f"chunk {chunk} forced grad {key}", 1e-12)
    n, b = x.shape[2], x.shape[0]
    perm = torch.tensor([1, 0, 2, 3, 4])
    swapped = [dict(h=t["h"].reshape(*t["h"].shape[:2], n, b, -1)[:, :, :, perm].reshape(t["h"].shape),
                    c=t["c"].reshape(*t["c"].shape[:2], n, b, -1)[:, :, :, perm].reshape(t["c"].shape),
                    s=t["s"][:, :, perm]) for t in tapes]
    out_s, _, _ = ref.loss_and_grads(x, y, tapes=swapped, window_chunk=2)
    assert O.max_rel_err(out_s.numpy(), out.numpy()) > 1e-6


def test_bf16_mode_reference_window_chunk_rejects_bad_sizes():
    params, chains, ks, x, y = _bf16_case(14, b=2)
    ref = O.BF16ModeReference(params, chains, ks, rounding=False)
    for bad in (0, -1):
        with pytest.raises(ValueError):
            ref.loss_and_grads(x, y, window_chunk=bad)


def test_bf16_mode_reference_takes_tapes_in_kernel_precision():
    """Tapes in the kernels' precision (h bf16, c and s fp32), whole-batch, are widened one chunk's slice at a time:
    output, loss, every gradient and d obs are bit-identical to those of the same tapes given in fp64, unchunked, in
    chunks of 1, in ragged chunks and in one whole-batch chunk."""
    params, chains, ks, x, y = _bf16_case(15, hid=16, b=5)
    ref = O.BF16ModeReference(params, chains, ks, relu=True)
    native = [dict(h=t["h"].to(torch.bfloat16), c=t["c"].float(), s=t["s"].float()) for t in _own_tapes(ref, x)]
    wide = [{k: v.double() for k, v in t.items()} for t in native]
    for chunk in (None, 1, 2, 5):
        out_n, loss_n, grads_n = ref.loss_and_grads(x, y, tapes=native, want_obs=True, window_chunk=chunk)
        out_w, loss_w, grads_w = ref.loss_and_grads(x, y, tapes=wide, want_obs=True, window_chunk=chunk)
        assert torch.equal(out_n, out_w) and torch.equal(loss_n, loss_w), f"chunk {chunk}"
        assert set(grads_n) == set(grads_w)
        for key in grads_w:
            assert torch.equal(grads_n[key], grads_w[key]), f"chunk {chunk} grad {key}"


def test_bf16_mode_reference_on_branch_per_chunk_is_the_whole_branch():
    """``on_branch`` with ``window_chunk``: called once per chunk and branch, ``branch["windows"]`` that chunk's.  Each value it
    sees (every LSTM layer-step's h and c, every spatial S_k, the branch output), put back together over the chunks,
    equals the unchunked branch's value to fp64 rounding -- with chunks of 1, ragged chunks and one whole-batch chunk.
    The model is forced with another model's tapes, so every chunk's values depend on it taking its own windows' rows."""
    params, chains, ks, x, y = _bf16_case(16, hid=16, b=5, m=2)
    params_other, chains_other, _, _, _ = _bf16_case(17, hid=16, b=5, m=2)
    tapes = _own_tapes(O.BF16ModeReference(params_other, chains_other, ks, relu=True), x)
    ref = O.BF16ModeReference(params, chains, ks, relu=True)
    n, bsz = x.shape[2], x.shape[0]

    def values(chunk):
        seen = {m: [] for m in range(ref.m)}

        def keep(m, br):
            win = br["windows"]
            nb = win.stop - win.start
            lstm = [torch.stack([torch.stack(v) for v in br[k]]) for k in ("hs", "cs")]       # (L, T, N*nb, H)
            seen[m].append((win, [v.reshape(*v.shape[:2], n, nb, -1) for v in lstm]
                            + [torch.stack(br["stack"]).reshape(ks, n, nb, -1), br["out"]]))
        ref.loss_and_grads(x, y, tapes=tapes, on_branch=keep, window_chunk=chunk)
        out = {}
        for m, parts in seen.items():
            wins = [w for w, _ in parts]
            assert [(w.start, w.stop) for w in wins] == [(i, min(i + (chunk or bsz), bsz))
                                                        for i in range(0, bsz, chunk or bsz)], f"chunk {chunk}: {wins}"
            # window axes: h and c (L, T, N, b, H) -> 3; S_k (Ks, N, b, H) -> 2; out (N, b, G) -> 1
            out[m] = [torch.cat([v[i] for _, v in parts], dim=axis) for i, axis in enumerate((3, 3, 2, 1))]
        return out
    whole = values(None)
    for chunk in (1, 2, bsz):
        got = values(chunk)
        for m in whole:
            for name, a, b in zip(("h", "c", "S", "out"), got[m], whole[m]):
                assert_close(a.detach().numpy(), b.detach().numpy(), f"chunk {chunk} branch {m} {name}", 1e-12)


def _own_tapes(ref, x):
    """The tapes of ``ref``'s own free-running forward, in the layout BF16ModeReference takes."""
    tapes = {}

    def keep(m, br):
        n, b = x.shape[2], x.shape[0]
        tapes[m] = dict(h=torch.stack([torch.stack(v) for v in br["hs"]]), c=torch.stack([torch.stack(v) for v in br["cs"]]),
                        s=torch.stack(br["stack"]).reshape(ref.ks, n, b, -1))
    ref.loss_and_grads(x, torch.zeros(x.shape[0], x.shape[2], x.shape[3]), on_branch=keep)
    return [tapes[m] for m in range(ref.m)]


@pytest.mark.parametrize("kind", ["chebyshev", "random_walk_diffusion"])
def test_bf16_mode_reference_forced_with_its_own_values_changes_nothing(kind):
    """Rounding on: forced with the tapes of its own free-running forward, the model reproduces its free-running output
    and gradients to fp64 rounding -- forcing replaces values only, and here the values agree.  And rounding on vs off
    differ at the bf16 level, above the 1e-4 bar in the output and tenfold in the gradients: the model really rounds."""
    params, chains, ks, x, y = _bf16_case(7, kind=kind, hid=16, b=4)
    ref = O.BF16ModeReference(params, chains, ks, relu=True)
    out, loss, grads = ref.loss_and_grads(x, y, want_obs=True)
    out_f, loss_f, grads_f = ref.loss_and_grads(x, y, tapes=_own_tapes(ref, x), want_obs=True)
    assert_close(out_f.numpy(), out.numpy(), "forced forward", 1e-12)
    assert abs(float(loss_f) - float(loss)) <= 1e-12 * abs(float(loss))
    for key in grads:
        assert_close(grads_f[key].numpy(), grads[key].numpy(), f"forced grad {key}", 1e-12)
    out_o, _, grads_o = O.BF16ModeReference(params, chains, ks, relu=True, rounding=False).loss_and_grads(x, y)
    assert 3 * TOL < O.max_rel_err(out.numpy(), out_o.numpy()) < 2e-2
    assert max(O.max_rel_err(grads[k_].numpy(), grads_o[k_].numpy()) for k_ in grads_o) > 1e-3


def test_bf16_mode_reference_rounds_the_spatial_gathers_only():
    """With the tapes of a free-running forward, each spatial term S_k is one step from the tape: 2 X bf16(S_{k-1}) -
    S_{k-2}.  Moving one tape term by far less than a bf16 ulp moves the next term through S_{k-2} (full precision) but
    not through the rounded gather; the temporal GCN does not round at all."""
    params, chains, ks, x, y = _bf16_case(8, k=3, hid=16, b=2, m=1)
    ref = O.BF16ModeReference(params, chains, ks)
    tapes = _own_tapes(ref, x)
    p = ref.leaves()
    xo = x.double().permute(2, 0, 1, 3)
    lap = torch.from_numpy(chains[0][0].toarray())
    with torch.no_grad():
        s = tapes[0]["s"].reshape(ks, 17, -1)
        bf = lambda v: v.float().to(torch.bfloat16).double()          # noqa: E731
        stack = ref.branch(p, 0, xo, tapes[0])["stack"]
        assert torch.allclose(stack[1], lap @ bf(s[0]), rtol=0, atol=1e-13)
        for k in range(2, ks):
            assert torch.allclose(stack[k], 2.0 * lap @ bf(s[k - 1]) - s[k - 2], rtol=0, atol=1e-13)
        # a change of 1e-12 relative: invisible through bf16(S_1) in S_2, visible through S_1 in S_3
        pert = dict(tapes[0])
        pert["s"] = tapes[0]["s"].clone()
        pert["s"][1] *= 1.0 + 1e-12
        stack2 = ref.branch(p, 0, xo, pert)["stack"]
        assert torch.equal(stack2[2], stack[2]) and not torch.equal(stack2[3], stack[3])
        # the temporal GCN's stack: full precision (the same as without rounding)
        _, comp = ref._stack(0, xo.sum(-1), False)
        _, comp_o = O.BF16ModeReference(params, chains, ks, rounding=False)._stack(0, xo.sum(-1), False)
        assert all(torch.equal(a, b) for a, b in zip(comp, comp_o))
