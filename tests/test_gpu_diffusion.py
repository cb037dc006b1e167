"""``kernel_type='random_walk_diffusion'`` on the GPU: the two-chain sparse supports of
``Adj_Preprocessor.process_sparse`` through ``ST_MGCN`` / ``CG_LSTM`` against the reference's golden vectors, the dense
``2K+1`` stack on the generic path, the fp64 reference on every window of a full cfg3 batch, both LSTM paths, the bf16
mode, CUDA-graph replay and training; negative controls that each break one part of the chain plumbing; and the launch
count of an unchanged Chebyshev step."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch
from torch import nn

import diffusion_oracle as D
import full_batch
import stmgcn_oracle as O
from helpers import DEV, TOL, assert_close
from model_cases import directed_workload

pytestmark = pytest.mark.gpu


def _model(meta, relu=True):
    import STMGCN
    return STMGCN.ST_MGCN(M=meta["m"], seq_len=meta["t"], n_nodes=meta["n"], input_dim=meta["c"],
                          lstm_hidden_dim=meta["hid"], lstm_num_layers=meta["layers"], gcn_hidden_dim=meta["gcn_hid"],
                          sta_kernel_config={"kernel_type": "random_walk_diffusion", "K": meta["k"]},
                          gconv_use_bias=True, gconv_activation=nn.ReLU if relu else None)


def _handles(adjs, k):
    import GCN
    pre = GCN.Adj_Preprocessor("random_walk_diffusion", k)
    return [pre.process_sparse(a).to(DEV) for a in adjs]


def _golden_errors(sups):
    """ST_MGCN on ``sups`` with the golden state_dict and inputs: max-norm relative errors against the reference run."""
    meta, params, grads, _, _, blob = D.load_golden()
    model = _model(meta).to(DEV)
    model.load_state_dict(params)
    x = torch.from_numpy(blob["x"]).to(DEV).requires_grad_(True)
    out = model(obs_seq=x, sta_adj_list=sups)
    loss = nn.MSELoss()(out, torch.from_numpy(blob["y"]).to(DEV))
    loss.backward()
    errs = {"out": O.max_rel_err(out.detach().cpu().numpy(), blob["out"]),
            "loss": abs(loss.item() - float(blob["loss"])) / abs(float(blob["loss"])),
            "d obs_seq": O.max_rel_err(x.grad.cpu().numpy(), blob["grad_x"])}
    for key, p in model.named_parameters():
        errs["grad " + key] = O.max_rel_err(p.grad.cpu().numpy(), grads[key])
    return errs


def _assert_errs(errs, tol=TOL, what=""):
    worst = sorted(errs.items(), key=lambda kv: -kv[1])
    print(what, ", ".join(f"{k} {v:.2e}" for k, v in worst[:5]))
    bad = {k: v for k, v in errs.items() if not v <= tol}
    assert not bad, f"{what} above {tol:.0e}: {bad}"


@pytest.mark.parametrize("path", ["tc", "fma"])
def test_st_mgcn_with_diffusion_handles_matches_the_reference(path):
    """Forward, loss, every parameter gradient and d obs_seq against the unmodified reference on the bidirectional
    stack (5 supports: the tensor-core projection's two support groups with path 'tc')."""
    from stmgcn_b200 import ops
    meta, *_, adjs, _ = D.load_golden()
    old = ops.lstm_path()
    try:
        ops.set_lstm_path(path)
        _assert_errs(_golden_errors(_handles(adjs, meta["k"])), what=f"diffusion golden ({path})")
    finally:
        ops.set_lstm_path(old)


def test_cg_lstm_with_a_diffusion_handle_matches_the_reference():
    """CG_LSTM (rnn_list.0 on graph 0, zero initial state): output, (h_n, c_n), its parameter gradients and d obs_seq of
    the golden probe sum(out * cg_w)."""
    meta, params, _, _, adjs, blob = D.load_golden()
    model = _model(meta).to(DEV)
    model.load_state_dict(params)
    cg = model.rnn_list[0]
    b = meta["b"]
    x = torch.from_numpy(blob["x"]).to(DEV).requires_grad_(True)
    out, (h_n, c_n) = cg(_handles(adjs[:1], meta["k"])[0], x, cg.init_hidden(b))
    (out * D.golden_probe(meta).to(DEV)).sum().backward()
    errs = {"out": O.max_rel_err(out.detach().cpu().numpy(), blob["cg_out"]),
            "h_n": O.max_rel_err(h_n.detach().cpu().numpy(), blob["cg_h_n"]),
            "c_n": O.max_rel_err(c_n.detach().cpu().numpy(), blob["cg_c_n"]),
            "d obs_seq": O.max_rel_err(x.grad.cpu().numpy(), blob["cg_grad_x"])}
    for key, p in cg.named_parameters():
        errs["grad " + key] = O.max_rel_err(p.grad.cpu().numpy(), blob["cg_grad." + key])
    _assert_errs(errs, what="diffusion CG_LSTM golden")


def test_handle_equals_the_dense_stack_on_the_generic_path():
    """The same model on the handle (two chains) and on the dense 2K+1 stack (every support applied on its own): 1e-5."""
    from stmgcn_b200.graph import supports_from_dense
    meta, params, _, supports, adjs, blob = D.load_golden()
    dense = [s.to(DEV) for s in supports]
    assert supports_from_dense(dense[0]).mode == "generic"
    res = []
    for sups in (_handles(adjs, meta["k"]), dense):
        model = _model(meta).to(DEV)
        model.load_state_dict(params)
        x = torch.from_numpy(blob["x"]).to(DEV).requires_grad_(True)
        out = model(obs_seq=x, sta_adj_list=sups)
        nn.MSELoss()(out, torch.from_numpy(blob["y"]).to(DEV)).backward()
        res.append([out.detach(), x.grad] + [p.grad for p in model.parameters()])
    for i, (a, b) in enumerate(zip(*res)):
        assert_close(a.cpu().numpy(), b.cpu().numpy(), f"handle vs dense stack, tensor {i}", 1e-5)


def _check_full_batch(name, batch, window_chunk, order=2, tol=TOL, relu=True, **kw):
    """test_gpu_fullsize.py's method on directed graphs with diffusion supports: one step on the full batch, every window
    with its true target, against the fp64 reference (two chains per graph) with the GPU forward's ReLU masks."""
    import GCN
    import STMGCN
    from stmgcn_b200 import ops, synth
    w, adjs = directed_workload(name, batch)
    pre = GCN.Adj_Preprocessor("random_walk_diffusion", order)
    sups_cpu = [pre.process_sparse(a) for a in adjs]
    chains = [[sp.csr_matrix(m.numpy()) for m in h.matrices_dense()] for h in sups_cpu]
    torch.manual_seed(0)
    kw_model = synth.model_kwargs(w)
    kw_model["sta_kernel_config"] = {"kernel_type": "random_walk_diffusion", "K": order}
    if not relu:
        kw_model["gconv_activation"] = None
    model = STMGCN.ST_MGCN(**kw_model)
    params = {k: v.detach().clone().numpy() for k, v in model.state_dict().items()}
    x, y = synth.make_inputs(w, seed=100, batch=batch)
    label = f"{name} diffusion K={order} planes={ops.lstm_planes()}"
    errs = full_batch.run(label, model.to(DEV), [s.to(DEV) for s in sups_cpu], params, chains, 2 * order + 1, x, y,
                          relu=relu, window_chunk=window_chunk, **kw)
    full_batch.assert_within(errs, tol, what=label)
    return errs


def test_cfg3_full_size_diffusion_vs_fp64_reference_on_every_window():
    """cfg3 shapes (4096 regions, 3 directed graphs, T=12, batch 64: 262 144 LSTM rows), K=2 (5 supports)."""
    _check_full_batch("cfg3", 64, 16)


def test_bf16_mode_with_diffusion_supports_vs_fp64_oracle():
    """The bf16 arithmetic mode (one bf16 LSTM plane, bf16 gather copies in both chains) at cfg2 shapes: the 2e-2 bar."""
    from stmgcn_b200 import ops
    old = ops.lstm_planes()
    try:
        ops.set_lstm_planes(1)
        errs = _check_full_batch("cfg2", 32, 32, tol=2e-2, relu=False, fp32_diagnostic=False)
    finally:
        ops.set_lstm_planes(old)
    assert errs["out"] > 1e-6, "the bf16 mode produced fp32-grade results: the single-plane path did not run"


def test_exact_and_tensor_core_paths_agree():
    """STMGCN_LSTM_PATH=fma (exact-fp32 LSTM and projection) against the tensor-core path on a directed cfg2-size case
    without the GCN activation (no ReLU mask can flip between the two)."""
    import GCN
    import STMGCN
    from stmgcn_b200 import ops, synth
    w, adjs = directed_workload("cfg2", 16)
    sups = [GCN.Adj_Preprocessor("random_walk_diffusion", 2).process_sparse(a).to(DEV) for a in adjs]
    kw = synth.model_kwargs(w)
    kw["sta_kernel_config"] = {"kernel_type": "random_walk_diffusion", "K": 2}
    kw["gconv_activation"] = None
    x, y = (t.to(DEV) for t in synth.make_inputs(w, seed=3, batch=16))
    res = {}
    old = ops.lstm_path()
    try:
        for path in ("fma", "tc"):
            ops.set_lstm_path(path)
            torch.manual_seed(0)
            model = STMGCN.ST_MGCN(**kw).to(DEV)
            out = model(obs_seq=x, sta_adj_list=sups)
            nn.MSELoss()(out, y).backward()
            res[path] = [out.detach()] + [p.grad for p in model.parameters()]
    finally:
        ops.set_lstm_path(old)
    for i, (a, b) in enumerate(zip(res["tc"], res["fma"])):
        assert_close(a.cpu().numpy(), b.cpu().numpy(), f"tc vs fma tensor {i}", 1e-4)


def test_graphed_step_replay_equals_the_eager_step():
    from stmgcn_b200 import dp, graphs
    meta, params, _, _, adjs, blob = D.load_golden()
    sups = _handles(adjs, meta["k"])
    model = _model(meta).to(DEV)
    model.load_state_dict(params)
    crit = nn.MSELoss()
    gen = torch.Generator().manual_seed(8)
    xs = [torch.randn(meta["b"], meta["t"], meta["n"], 1, generator=gen).to(DEV) for _ in range(2)]
    ys = [torch.randn(meta["b"], meta["n"], 1, generator=gen).to(DEV) for _ in range(2)]
    ref = []
    for x, y in zip(xs, ys):
        model.zero_grad(set_to_none=True)
        loss = crit(model(obs_seq=x, sta_adj_list=sups), y)
        loss.backward()
        ref.append((loss.item(), {k: p.grad.detach().clone() for k, p in model.named_parameters()}))
    del loss            # no autograd graph of an eager step may stay alive into the capture
    gstep = graphs.GraphedStep(model, crit, xs[0], ys[0], sups, bucket=dp.GradBucket(model))
    for i in range(2):
        loss = gstep(xs[i], ys[i])
        assert abs(loss.item() - ref[i][0]) <= 1e-5 * abs(ref[i][0])
        for key, p in model.named_parameters():
            assert_close(p.grad.cpu().numpy(), ref[i][1][key].cpu().numpy(), f"replay {i} grad {key}", 2e-5)


def test_adam_steps_lower_the_loss():
    meta, params, _, _, adjs, blob = D.load_golden()
    sups = _handles(adjs, meta["k"])
    model = _model(meta).to(DEV)
    model.load_state_dict(params)
    x, y = torch.from_numpy(blob["x"]).to(DEV), torch.from_numpy(blob["y"]).to(DEV)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    losses = []
    for _ in range(8):
        opt.zero_grad()
        loss = nn.MSELoss()(model(obs_seq=x, sta_adj_list=sups), y)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert all(np.isfinite(losses)), losses
    assert all(b < a for a, b in zip(losses, losses[1:])) and losses[-1] < 0.99 * losses[0], losses


def _variant(h, mats):
    from stmgcn_b200.graph import SparseSupports
    return SparseSupports("cheb", h.n, h.ks, mats)


def _transposed(m, n):
    dense = torch.sparse_csr_tensor(m[0].long(), m[1].long(), m[2], size=(n, n)).to_dense().t()
    from stmgcn_b200.graph import csr_from_coo
    r, c = (dense != 0).nonzero(as_tuple=True)
    return csr_from_coo(n, r, c, dense[r, c])


@pytest.mark.parametrize("control", ["swapped_chains", "no_backward_adjoint", "p_f_for_p_f_t"])
def test_negative_controls_fail(control, monkeypatch):
    """Each control breaks one part of the two-chain plumbing; the golden comparison must then fail."""
    from stmgcn_b200 import ops
    meta, *_, adjs, _ = D.load_golden()
    sups = _handles(adjs, meta["k"])
    if control == "swapped_chains":
        sups = [_variant(h, h.mats[::-1]) for h in sups]
    elif control == "p_f_for_p_f_t":
        sups = [_variant(h, [_transposed(h.mats[0], h.n), h.mats[1]]) for h in sups]
    else:
        def forward_chain_only(sset, u):
            if sset.mode == "cheb" and len(sset.graphs) == 2:
                ops._adjoint_chain_(sset.graphs[0], [u[i] for i in sset.chain_segments(0)])
                return u[0]
            return real(sset, u)
        real = ops.adjoint_stack_
        monkeypatch.setattr(ops, "adjoint_stack_", forward_chain_only)
    errs = _golden_errors(sups)
    print(control, {k: f"{v:.1e}" for k, v in sorted(errs.items(), key=lambda kv: -kv[1])[:4]})
    assert max(errs.values()) > 1e-2, f"negative control {control} passed the golden comparison"
    if control == "no_backward_adjoint":
        assert errs["out"] <= TOL            # only the backward is broken


# launches of libstmgcn_b200 kernels by one Chebyshev step (3 graphs, K=3, forward + MSE + backward), counted on an H100.
# The tensor-core columns include the weight packs every forward makes, 5 per graph branch (one per LSTM layer, the
# spatial projection's forward and backward images); the exact path packs nothing and keeps the count of the build
# before the support stacks were parametrised by chain
CHEB_LAUNCHES = {"planes2": 102, "planes1": 105, "fma": 393}


@pytest.mark.parametrize("mode", sorted(CHEB_LAUNCHES))
def test_chebyshev_step_launch_count_includes_the_weight_packs(mode):
    import GCN
    from stmgcn_b200 import _lib, ops, synth
    from helpers import build_model
    meta = dict(n=96, m=3, k=3, t=12, b=8, c=1, hid=64, layers=3, gcn_hid=64)
    pre = GCN.Adj_Preprocessor("chebyshev", meta["k"])
    sups = [pre.process_sparse(synth.make_adjacency(meta["n"], g, 0.05)).to(DEV) for g in range(meta["m"])]
    torch.manual_seed(0)
    model = build_model(meta, DEV)
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(meta["b"], meta["t"], meta["n"], 1, generator=gen).to(DEV)
    y = torch.randn(meta["b"], meta["n"], 1, generator=gen).to(DEV)
    old = (ops.lstm_path(), ops.lstm_planes())
    try:
        ops.set_lstm_path("fma" if mode == "fma" else "tc")
        ops.set_lstm_planes(1 if mode == "planes1" else 2)
        counts = []
        for _ in range(2):
            torch.cuda.synchronize()
            n0 = _lib.launch_count()
            nn.MSELoss()(model(obs_seq=x, sta_adj_list=sups), y).backward()
            torch.cuda.synchronize()
            counts.append(_lib.launch_count() - n0)
    finally:
        ops.set_lstm_path(old[0])
        ops.set_lstm_planes(old[1])
    print(mode, counts)
    assert counts[1] == CHEB_LAUNCHES[mode], counts
