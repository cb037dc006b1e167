"""The bf16-arithmetic mode (``ops.set_lstm_planes(1)``, the arithmetic of the bf16-quoted BASELINE configs) held to the
fp32 bar against ``stmgcn_oracle.BF16ModeReference``, an fp64 model that rounds where the kernels round.

A free-running fp64 model cannot hold this mode tightly: thousands of bf16 rounding boundaries per step fall on
different sides in fp32 and fp64, each moving an element by a bf16 ulp.  So the reference is forced with the kernels' own
values at every rounding point, recorded during the GPU forward by wrapping ``ops`` inside the test: the shared LSTM's
tape (one bf16 hidden-state plane, the cell states, the initial state's plane), the spatial Chebyshev stacks
(``ops.build_stack`` with bf16 gathers; ``S_0`` is the fp32 h_top) and the GCN outputs (their ReLU masks).  Every
layer-step and every ``S_k`` is then one step from the kernels' inputs, the gradients are the kernels' backward, and what
remains is fp32-vs-fp64 arithmetic: the 1e-4 bar (``helpers.TOL``) applies to every check.

Here only the rows of the picked windows are recorded (rows ``n*B + b``; windows are independent in this mode too),
and the full-batch gradient is ``|picked| / B`` times the reference's on the picked windows: the other windows' targets
are the run's own output, so their residual is zero and those windows carry no gradient.  At cfg2 and cfg5 such a check
cannot see a backward that loses the other windows (``test_gpu_bf16_full_batch`` shows one passing it).
``tests/test_gpu_bf16_full_batch.py`` holds the mode to the same bar on every window of the benchmarked batches (cfg2,
cfg2 with random_walk_diffusion supports, cfg4, cfg5's shapes), recording every row in the kernels' precision and
forcing the reference one chunk of windows at a time.

The 2e-2 tests (``test_gpu_parity``, ``test_gpu_fullsize``, ``test_gpu_diffusion``) bound the mode against unrounded fp64;
these checks say that the mode computes what it claims to, and the negative controls show that they catch the plausible
mistakes the 2e-2 bar can miss.
"""
import pytest
import torch

import stmgcn_oracle as O
from helpers import DEV, TOL, build_model, load_golden, rel_err
from model_cases import Recorder, bf16_mode, diffusion_case, forced_errors, gpu_run, workload_case  # noqa: F401

pytestmark = pytest.mark.gpu


# ======================================================================================================================
# recording the kernels' values
# ======================================================================================================================
def _summary(errs, n=6):
    return ", ".join(f"{k} {v:.2e}" for k, v in sorted(errs.items(), key=lambda kv: -kv[1])[:n])


# ======================================================================================================================
# cases
# ======================================================================================================================
def _golden_case(relu):
    meta, params, _, supports, _, blob = load_golden("cfg3_small_ref")
    model = build_model(meta, DEV, relu)
    model.load_state_dict(params)
    chains = [[O.laplacian_csr_from_supports(s)] for s in supports]
    x, y = torch.from_numpy(blob["x"]), torch.from_numpy(blob["y"])
    return model, [s.to(DEV) for s in supports], chains, meta["k"] + 1, params, x, y, list(range(x.shape[0]))


def _workload_case(name, batch, picks, relu):
    return workload_case(name, batch, relu) + (picks,)


def _diffusion_case(batch, picks, relu):
    return diffusion_case(batch, relu) + (picks,)


CASES = {
    "cfg3_small_golden": lambda relu: _golden_case(relu),
    "cfg2": lambda relu: _workload_case("cfg2", 32, [0, 17, 31], relu),
    "cfg5": lambda relu: _workload_case("cfg5", 8, [5], relu),
    "cfg2_diffusion": lambda relu: _diffusion_case(32, [0, 17, 31], relu),
}


@pytest.mark.parametrize("relu", [True, False], ids=["relu", "smooth"])
@pytest.mark.parametrize("case", list(CASES))
def test_bf16_mode_matches_the_forced_fp64_reference(case, relu, bf16_mode):  # noqa: F811
    """Step-local: every (layer, step) of each shared LSTM (cell state; hidden state as the excess over half a bf16 ulp,
    test_gpu_lstm16's measure), its fp32 h_top, and every S_k of every spatial chain.  Whole model: output, loss and
    every parameter gradient.  ReLU model (the reference takes the GPU's masks) and the model without the GCN activation;
    all at 1e-4.  Sizes: the cfg3_small golden case (all six windows), cfg2 full size (batch 32, windows 0, 17, 31),
    cfg5 shapes (16 384 regions, K = 5, T = 24, batch 8, window 5), cfg2 with random_walk_diffusion supports.

    Measured on an H100 80GB HBM3 at 700 W: step-local at most 1.0e-6 (cfg5's S_k; the LSTM layer-steps and h_top
    4e-7 .. 6e-7), whole model at most 2.2e-5 (cfg2_diffusion ReLU, fc.bias; cfg5 smooth 2.0e-5, cfg3_small smooth
    1.8e-5, in the LSTM's and the context gate's parameter gradients)."""
    model, sups, chains, ks, params, x, y, picks = CASES[case](relu)
    run = gpu_run(model, sups, x, y, picks)
    del model
    torch.cuda.empty_cache()
    assert len(run["rec"].stacks) == len(chains), "a spatial GCN ran without the bf16 gathers' stack call"
    step, errs = forced_errors(run, params, chains, ks, x, y, picks, relu)
    print(f"\nbf16 mode {case} {'relu' if relu else 'smooth'} windows {picks}: step-local worst "
          f"{max(step.values()):.2e} ({_summary(step, 4)}); whole model worst {max(errs.values()):.2e} ({_summary(errs)})")
    bad = {k: v for k, v in {**step, **errs}.items() if not v <= TOL}
    assert not bad, f"{case}: above {TOL:.0e}: {bad}"


def test_cg_lstm_with_an_initial_state_matches_the_forced_reference(bf16_mode):  # noqa: F811
    """CG_LSTM with (h0, c0): h0 enters the kernels as its bf16 plane (ops.to_planes(h0, 1)), c0 in fp32.  Output,
    h_n, c_n and the gradients of obs, h0, c0 and every parameter for <out, w> + <h_n, r1> + <c_n, r2>, against the
    reference forced with the recorded tape (h0's plane among it), at 1e-4.  Measured on an H100: 4.2e-6 (d h0)."""
    import STMGCN
    from stmgcn_b200 import synth
    n, b, t, c, hid, lyr, k = 37, 6, 7, 2, 64, 3, 3
    torch.manual_seed(11)
    model = STMGCN.CG_LSTM(seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=lyr, K=k + 1,
                           gconv_use_bias=True).to(DEV)
    params = {"rnn_list.0." + key: v.detach().clone() for key, v in model.state_dict().items()}
    sup = O.chebyshev_supports_dense(synth.make_adjacency(n, 0, 0.2).double(), k).float()
    gen = torch.Generator().manual_seed(12)
    x = torch.randn(b, t, n, c, generator=gen)
    h0, c0 = 0.5 * torch.randn(lyr, b * n, hid, generator=gen), torch.randn(lyr, b * n, hid, generator=gen)
    w_out, r1, r2 = (torch.randn(*s, generator=gen) for s in ((b, n, hid), (lyr, b * n, hid), (lyr, b * n, hid)))
    leaves = [v.to(DEV).requires_grad_(True) for v in (x, h0, c0)]
    with Recorder(range(b)) as rec:
        out, (h_n, c_n) = model(sup.to(DEV), leaves[0], (leaves[1], leaves[2]))
    ((out * w_out.to(DEV)).sum() + (h_n * r1.to(DEV)).sum() + (c_n * r2.to(DEV)).sum()).backward()
    torch.cuda.synchronize()
    (tape,) = rec.tapes()
    assert "h0" in tape
    ref = O.BF16ModeReference(params, [[O.laplacian_csr_from_supports(sup)]], k + 1, relu_masks=rec.masks, device=DEV)
    p = ref.leaves()
    r_leaves = [v.double().to(DEV).requires_grad_(True) for v in (x, h0, c0)]
    r_out, (r_hn, r_cn) = ref.cg_lstm(p, r_leaves[0], (r_leaves[1], r_leaves[2]), tape)
    loss = (r_out * w_out.double().to(DEV)).sum() + (r_hn * r1.double().to(DEV)).sum() + (r_cn * r2.double().to(DEV)).sum()
    names = [key for key, _ in model.named_parameters()]
    g = torch.autograd.grad(loss, r_leaves + [p["rnn_list.0." + key] for key in names])
    errs = {"out": rel_err(out, r_out), "h_n": rel_err(h_n, r_hn), "c_n": rel_err(c_n, r_cn)}
    errs.update({f"d {v}": rel_err(leaf.grad, gr) for v, leaf, gr in zip(("obs", "h0", "c0"), leaves, g[:3])})
    errs.update({"grad " + key: rel_err(prm.grad, gr) for (key, prm), gr in zip(model.named_parameters(), g[3:])})
    print(f"\nbf16 mode CG_LSTM with (h0, c0): worst {max(errs.values()):.2e} ({_summary(errs)})")
    bad = {key: v for key, v in errs.items() if not v <= TOL}
    assert not bad, f"above {TOL:.0e}: {bad}"


# ======================================================================================================================
# negative controls: plausible mistakes in the bf16 path, each of which must fail the forced bar
# ======================================================================================================================
def _fp32_spatial_gathers(ops, monkeypatch):
    """The spatial chain gathers from fp32 (no bf16 copies) while the LSTM keeps one plane."""
    monkeypatch.setattr(ops, "_gather16", lambda sset, x: False)


def _bf16_adjoint(ops, monkeypatch):
    """The adjoint Clenshaw gathers b_{k+1} from its bf16 copy."""
    real = ops._adjoint_chain_

    def adjoint16(g, u):
        if (u[0].numel() // g.n) % 8:
            return real(g, u)
        k_ord = len(u) - 1
        for k in range(k_ord - 1, 0, -1):
            z = u[k + 2] if k + 2 <= k_ord else None
            ops.spmm_step16(g, True, 2.0, ops.to_bf16(u[k + 1]), -1.0 if z is not None else 0.0, z, 1.0, u[k], u[k], None)
        z = u[2] if k_ord >= 2 else None
        ops.spmm_step16(g, True, 1.0, ops.to_bf16(u[1]), -1.0 if z is not None else 0.0, z, 1.0, u[0], u[0], None)
    monkeypatch.setattr(ops, "_adjoint_chain_", adjoint16)


def _bf16_temporal_gathers(ops, monkeypatch):
    """The temporal GCN's Chebyshev recurrence takes bf16 gathers too."""
    real = ops.build_stack
    monkeypatch.setattr(ops, "build_stack", lambda sset, x, gather16=False: real(sset, x, True))


def _bf16_t_k_minus_2(ops, monkeypatch):
    """The spatial recurrence reads T_{k-2} through its bf16 copy."""
    real = ops._cheb_chain_

    def chain(g, t, gather16):
        if not gather16:
            return real(g, t, gather16)
        src = ops.to_bf16(t[0])
        for k in range(1, len(t)):
            out16 = torch.empty_like(src) if k < len(t) - 1 else None
            z = None if k == 1 else ops.to_bf16(t[k - 2]).float()
            ops.spmm_step16(g, False, 1.0 if k == 1 else 2.0, src, 0.0 if k == 1 else -1.0, z, 0.0, None, t[k], out16)
            src = out16
    monkeypatch.setattr(ops, "_cheb_chain_", chain)


CONTROLS = {
    "fp32_spatial_gathers": _fp32_spatial_gathers,
    "bf16_adjoint_gathers": _bf16_adjoint,
    "bf16_temporal_gathers": _bf16_temporal_gathers,
    "bf16_t_k_minus_2": _bf16_t_k_minus_2,
    "two_plane_reference": None,                 # the kernels as they are, the reference without rounding
}


@pytest.mark.parametrize("control", list(CONTROLS))
def test_negative_controls_fail_the_forced_bar(control, bf16_mode, monkeypatch):  # noqa: F811
    """Each plausible mistake in the bf16 path, applied by wrapping ops, lands above the 1e-4 bar of the forced
    reference on the cfg3_small golden case (model without the GCN activation).  For information only, the error the
    2e-2 end-to-end check (the free-running fp64 SparseOracle) reports under the same mistake is printed too.

    Measured on an H100 (forced worst / 2e-2 check worst): fp32 spatial gathers 3.1e-3 (S_3) / 7.4e-3; bf16 adjoint
    gathers 3.0e-2 / 2.6e-2 (LSTM weight gradients); bf16 temporal gathers 3.8e-2 / 3.6e-2 (context-gate gradients);
    T_{k-2} through its bf16 copy 2.8e-3 (S_3) / 1.4e-2; the two-plane reference 7.5e-3 / 1.3e-2 (the unmutated run).
    The first and the fourth pass the 2e-2 check; unmutated, the forced checks stay within 2e-5."""
    if CONTROLS[control] is not None:
        CONTROLS[control](bf16_mode, monkeypatch)
    model, sups, chains, ks, params, x, y, picks = _golden_case(relu=False)
    run = gpu_run(model, sups, x, y, picks)
    step, errs = forced_errors(run, params, chains, ks, x, y, picks, relu=False,
                               rounding=control != "two_plane_reference")
    forced = {**step, **errs}
    orc = O.SparseOracle({k: v.numpy() for k, v in params.items()}, [c[0] for c in chains], ks, relu=False)
    o_ref, _, g_ref = orc.loss_and_grads(x.numpy(), y.numpy())
    free = {"out": O.max_rel_err(run["out"].cpu().numpy(), o_ref)}
    free.update({"grad " + k: O.max_rel_err(g.cpu().numpy(), g_ref[k]) for k, g in run["grads"].items()})
    print(f"\ncontrol {control}: forced worst {max(forced.values()):.2e} ({_summary(forced, 4)}); "
          f"2e-2 end-to-end check worst {max(free.values()):.2e} ({_summary(free, 2)})")
    assert max(forced.values()) > TOL, f"{control}: the forced bar does not see it ({_summary(forced)})"
