"""GPU parity at the sizes that are BENCHMARKED (BASELINE.json configs[1..4]), not only at toy sizes.

One training step on the full batch, every window with its true target, against the fp64 reference
(``tests/full_batch.py``: ``BF16ModeReference`` without rounding, on the GPU, a chunk of windows at a time).  Every
window then feeds every weight-gradient reduction -- the LSTM's per-CTA slices and their sum, the projection's ``dW`` /
``dbias`` / pool atomics, the fusion and gate ``fc`` sums, ``d_s`` -- at 262 144 LSTM rows, 2 048 tiles and > 2^31
element tapes at cfg3.  Every window's output, the loss and every parameter gradient are held to the bar.

Tolerance: 1e-4 max-norm relative (BASELINE.json north_star), fp32 arithmetic; 2e-2 for the bf16-arithmetic mode
against the unrounded reference.
"""
import pytest
import torch
from torch import nn

import full_batch
import stmgcn_oracle as O
from helpers import DEV, TOL, assert_close
from model_cases import CHUNK, cheb_workload

pytestmark = pytest.mark.gpu


def _run_full_batch(name, batch, relu=True, **kw):
    """``full_batch.run`` on workload ``name`` (Chebyshev supports); returns the errors."""
    from stmgcn_b200 import ops, synth
    w = synth.WORKLOADS[name]
    model, sups, laps, params, x, y = cheb_workload(w, batch, relu=relu)
    label = f"{name} path={ops.lstm_path()} planes={ops.lstm_planes()}"
    return full_batch.run(label, model, sups, params, [[lap] for lap in laps], w.n_supports, x, y, relu=relu,
                          window_chunk=CHUNK[name], **kw)


def _check_full_batch(name, batch, tol=TOL, relu=True, **kw):
    """:func:`_run_full_batch` and every error at ``tol``."""
    errs = _run_full_batch(name, batch, relu, **kw)
    full_batch.assert_within(errs, tol, what=f"{name} B={batch} relu={relu}")
    return errs


@pytest.mark.parametrize("relu", [True, False])
def test_cfg3_full_size_vs_fp64_reference_on_every_window(relu):
    """BASELINE configs[2]: 4096 regions, 3 graphs, K=3, T=12, batch 64, fp32 -- the size bench.py reports.  The step is
    taken twice at the same weights, and the spread of every gradient between the two is printed beside its error."""
    _check_full_batch("cfg3", 64, relu=relu, repeat=True)


@pytest.mark.parametrize("relu", [True, False])
def test_cfg2_full_size_vs_fp64_oracle(relu):
    """BASELINE configs[1] shapes (1024 regions, 3 graphs, K=3, T=12, batch 32) in fp32, every window."""
    _check_full_batch("cfg2", 32, relu=relu)


@pytest.mark.parametrize("relu", [True, False])
def test_cfg2_full_size_exact_fp32_path_vs_fp64_reference(relu):
    """The exact-fp32 CUDA-core path (``ops.set_lstm_path("fma")``: FFMA LSTM and projection kernels) at cfg2 full size,
    every window, at the same bar as the tensor-core path."""
    from stmgcn_b200 import ops
    old = ops.lstm_path()
    try:
        ops.set_lstm_path("fma")
        _check_full_batch("cfg2", 32, relu=relu)
    finally:
        ops.set_lstm_path(old)


@pytest.mark.parametrize("relu", [True, False])
def test_cfg5_shapes_vs_fp64_reference_on_every_window(relu):
    """BASELINE configs[4] shapes: 16384 regions, 3 graphs at 1 % density, K=5 (six supports), T=24; batch 8 of 32."""
    _check_full_batch("cfg5", 8, relu=relu)


@pytest.mark.parametrize("cfg,batch", [("cfg2", 32), ("cfg5", 8)])
def test_bf16_mode_at_the_quoted_sizes_vs_fp64_oracle(cfg, batch):
    """BASELINE configs[1] and [4] are quoted in the bf16 arithmetic mode (ops.set_lstm_planes(1): one bf16 hidden-state
    plane in the tensor-core LSTM, bf16 gather copies in the spatial Chebyshev recurrence, spmm_step16): the whole model at
    those sizes against the fp64 reference at the bf16 tolerance 2e-2 (SURVEY.md section 8(d)).  The model without the GCN
    activation, as in test_gpu_parity.py: bf16-level noise flips ReLU masks, which says nothing about the kernels.
    tests/test_gpu_lstm16.py is the tight check of the LSTM arithmetic in this mode; this is the end-to-end bound."""
    from stmgcn_b200 import ops
    old = ops.lstm_planes()
    try:
        ops.set_lstm_planes(1)
        errs = _check_full_batch(cfg, batch, tol=2e-2, relu=False, fp32_diagnostic=False)
    finally:
        ops.set_lstm_planes(old)
    assert errs["out"] > 1e-6, "the bf16 mode produced fp32-grade results: the single-plane path did not run"


def test_full_batch_check_fails_a_backward_that_drops_windows(monkeypatch):
    """Negative control: the LSTM backward loses the gradient of windows 1 .. B-2 (their rows ``n*B + b`` of ``d_top``
    are zeroed).  The output is untouched, so only a check in which those windows carry gradient can see it."""
    from stmgcn_b200 import ops
    real = ops.SharedLSTM.backward

    def lossy(ctx, d_top, dh_n, dc_n):
        d_top = d_top.clone()
        d_top[:, 1:-1] = 0
        return real(ctx, d_top, dh_n, dc_n)
    monkeypatch.setattr(ops.SharedLSTM, "backward", staticmethod(lossy))
    errs = _run_full_batch("cfg2", 32, fp32_diagnostic=False)
    assert errs["out"] <= TOL
    lost = {k: v for k, v in errs.items() if not v <= TOL}
    assert any(".lstm." in k for k in lost), f"the full-batch check passed a backward that drops windows: {errs}"


def test_lstm_tensor_core_vs_exact_fp32_at_cfg3_size():
    """tensor-core (wgmma) LSTM forward + BPTT + weight gradients against the exact-FFMA kernels ON DEVICE at cfg3's 262 144 rows."""
    from stmgcn_b200 import ops
    n, b, t, hid, lyr = 4096, 64, 12, 64, 3
    gen = torch.Generator().manual_seed(5)
    xo = torch.randn(n, b, t, 1, generator=gen).to(DEV)
    s0 = torch.rand(b, t, generator=gen).to(DEV)
    ws0 = []
    for l in range(lyr):
        in_l = 1 if l == 0 else hid
        ws0 += [(torch.rand(4 * hid, in_l, generator=gen) - 0.5) * 0.25, (torch.rand(4 * hid, hid, generator=gen) - 0.5) * 0.25,
                (torch.rand(4 * hid, generator=gen) - 0.5) * 0.25, (torch.rand(4 * hid, generator=gen) - 0.5) * 0.25]
    proj = (torch.randn(n, b, hid, generator=gen) * 1e-3).to(DEV)
    res = {}
    old = ops.lstm_path()
    try:
        for path in ("fma", "tc"):
            ops.set_lstm_path(path)
            s = s0.clone().requires_grad_(True)
            ws = [w_.to(DEV).requires_grad_(True) for w_ in ws0]
            h_top, _, _ = ops.SharedLSTM.apply(xo, s, None, None, lyr, hid, False, *ws)
            (h_top * proj).sum().backward()
            res[path] = [h_top.detach().clone(), s.grad.clone()] + [w_.grad.clone() for w_ in ws]
            del h_top, s, ws
            torch.cuda.empty_cache()
    finally:
        ops.set_lstm_path(old)
    names = ["h_top", "d_s"] + [f"w{i}" for i in range(4 * lyr)]
    # weight gradients are sums over 3.1 M (row, step) pairs: the two kernels add them in different orders in fp32, which
    # alone is worth ~1e-4 relative (measured 9.4e-5 between the 3xTF32 kernels and the FFMA kernels); the fp64-oracle tests
    # above are the pin, this one guards against indexing bugs at > 2^31-element sizes
    for name, a, c in zip(names, res["tc"], res["fma"]):
        assert_close(a.cpu().numpy(), c.cpu().numpy(), f"cfg3-size tc vs fma {name}", 5e-5 if name in ("h_top",) else 3e-4)


def test_cg_lstm_and_model_with_localpool_supports():
    """kernel_type='localpool' (A[0] = I + A_norm != I): the context gate's residual is x itself, not A_0 x
    (STMGCN.py:40-41).  CG_LSTM and ST_MGCN forward + every gradient against the dense oracle."""
    import GCN
    import STMGCN
    from stmgcn_b200 import synth
    n, b, t, c, hid, lyr, gh, m = 60, 5, 6, 1, 64, 2, 24, 2
    pre = GCN.Adj_Preprocessor("localpool", 1)
    sups = [pre.process(synth.make_adjacency(n, g, 0.15)) for g in range(m)]
    torch.manual_seed(3)
    model = STMGCN.ST_MGCN(M=m, seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=lyr,
                           gcn_hidden_dim=gh, sta_kernel_config={"kernel_type": "localpool", "K": 1},
                           gconv_use_bias=True, gconv_activation=nn.ReLU)
    params = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model = model.to(DEV)
    gen = torch.Generator().manual_seed(9)
    x, y = torch.randn(b, t, n, c, generator=gen), torch.randn(b, n, c, generator=gen)
    out = model(obs_seq=x.to(DEV), sta_adj_list=[s.to(DEV) for s in sups])
    loss = nn.MSELoss()(out, y.to(DEV))
    loss.backward()
    ref_p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    ref_out = O.dense_st_mgcn(ref_p, x, sups)
    ref_loss = nn.MSELoss()(ref_out, y)
    ref_loss.backward()
    assert_close(out.detach().cpu().numpy(), ref_out.detach().numpy(), "localpool model forward")
    for key, p in model.named_parameters():
        assert_close(p.grad.cpu().numpy(), ref_p[key].grad.numpy(), f"localpool grad {key}")
    # CG_LSTM alone (the advisor's case): gate computed from x + gconv(x)
    cg = model.rnn_list[0]
    h0 = cg.init_hidden(b)
    o1, _ = cg(sups[0].to(DEV), x.to(DEV), h0)
    o_ref, _ = O.dense_cg_lstm(sups[0], x, {"p." + k[len("rnn_list.0."):]: v for k, v in params.items()
                                             if k.startswith("rnn_list.0.")}, "p.")
    assert_close(o1.detach().cpu().numpy(), o_ref.numpy(), "localpool CG_LSTM forward")
