"""The model against the fp64 oracle at the weights it holds NOW, after every kind of parameter update.

The tensor-core path feeds its kernels operand images of the weights (the shared LSTM's bf16-plane images, the spatial
GCN's projection images).  Whatever writes the parameters between two forwards -- an optimizer of any flavour, a write
through ``.data``, ``load_state_dict``, an optimizer step replayed from a CUDA graph -- the next forward and its
gradients must be those of the new values.  Some of these writes do not bump a tensor's in-place version counter
(``Adam(fused=True)``, ``AdamW(fused=True)``, ``SGD(fused=True)``, ``p.data.add_``, ``p.data.copy_``, a captured
``Adam(capturable=True).step()`` replayed), so nothing keyed on that counter can tell that the weights moved.

Every case: one training forward + backward and one ``no_grad`` forward (so both the training and the inference
variants of every image exist), the update, then a ``no_grad`` forward and a training forward + backward that are
checked three ways:

* oracle: output, loss and every parameter gradient against ``O.SparseOracle`` in fp64, built from the parameters read
  back from the model and following the ReLU masks of the run (as test_gpu_diffusion.py's sub-batch checks do: at
  n = 96, B = 8 one pre-activation at the kink moves a branch's gradients by ~1e-3) -- 1e-4 with two planes and on the
  exact path; 2e-2 in the one-plane (bf16 arithmetic) mode, on the model without the GCN activation, as in
  ``test_bf16_arithmetic_mode_within_the_reference_bf16_tolerance``;
* fresh copy: the same quantities against a ``copy.deepcopy`` of the updated model (new storages).  This decides the
  one-plane cases, where a small step could hide under 2e-2.  Two runs are not bit-identical: the temporal GCN's region
  pooling and the weight-gradient reductions accumulate with atomics.  Measured on an H100 SXM (80 GB HBM3, 700 W power
  limit) over every case of this file in two runs: at most 1.7e-6 on the outputs and 4.8e-6 on the gradients with two
  planes and on the exact path, hence FRESH 2e-5; with one plane up to 8.5e-5 on the outputs and 9.4e-5 on the
  gradients (there a last-bit difference in the gate can round a hidden state to the neighbouring bf16 value), hence
  1e-3.  A stale weight image was 1.1e-2 or more away with two planes and 9e-2 or more with one;
* negative control: the oracle built from the parameters BEFORE the update lands outside the oracle bar on the output
  after it, so the update is large enough to be seen.

Plain gradient steps (``sgd_fused``, ``data_add_``) use lr = 2e-2 instead of Main.py's 2e-3: at 2e-3 one step moves the
output of the model without the GCN activation by 1.7e-2 of its largest value (fp64 oracle), inside the one-plane bar;
at 2e-2 by 0.17.
"""
import copy
import io

import numpy as np
import pytest
import scipy.sparse as sp
import torch
from torch import nn

import diffusion_oracle as D
import stmgcn_oracle as O
from helpers import DEV, TOL

pytestmark = pytest.mark.gpu

META = dict(n=96, m=3, k=3, t=12, b=8, c=1, hid=64, layers=3, gcn_hid=64)     # LSTM and projection on the tensor cores
LR, WD = 2e-3, 1e-4             # Main.py
LR_SGD = 2e-2                   # plain gradient steps: see the module docstring
BAR = {"tc2": TOL, "fma": TOL, "tc1": 2e-2}
FRESH = {"tc2": 2e-5, "fma": 2e-5, "tc1": 1e-3}

MECHANISMS = ["adam_foreach", "adam_fused", "adamw_fused", "sgd_fused", "data_add_", "data_copy_", "no_grad_copy_",
              "load_state_dict", "load_state_dict_assign", "captured_step"]
PATHS = ["tc2", "tc1", "fma"]


@pytest.fixture
def path(request):
    """Selects the kernel path of ``request.param``: tensor cores with two bf16 planes / one plane, or exact fp32."""
    from stmgcn_b200 import ops
    old = (ops.lstm_path(), ops.lstm_planes())
    ops.set_lstm_path("fma" if request.param == "fma" else "tc")
    ops.set_lstm_planes(1 if request.param == "tc1" else 2)
    yield request.param
    ops.set_lstm_path(old[0])
    ops.set_lstm_planes(old[1])


def _supports(kind):
    """(device supports, oracle matrices): Chebyshev (one L~ per graph) or diffusion (two chains per graph)."""
    import GCN
    from stmgcn_b200 import synth
    n, k = META["n"], META["k"]
    if kind == "cheb":
        adjs = [synth.make_adjacency(n, g, 0.05) for g in range(META["m"])]
        sups = [GCN.Adj_Preprocessor("chebyshev", k).process_sparse(a) for a in adjs]
        return [s.to(DEV) for s in sups], [sp.csr_matrix(s.laplacian_dense().numpy()) for s in sups]
    adjs = [synth.make_directed_adjacency(n, g, 0.05) for g in range(META["m"])]
    sups = [GCN.Adj_Preprocessor("random_walk_diffusion", k).process_sparse(a) for a in adjs]
    return [s.to(DEV) for s in sups], [[sp.csr_matrix(m.numpy()) for m in s.matrices_dense()] for s in sups]


def _model(kind, relu, seed):
    import STMGCN
    torch.manual_seed(seed)
    k = META["k"]
    return STMGCN.ST_MGCN(M=META["m"], seq_len=META["t"], n_nodes=META["n"], input_dim=META["c"],
                          lstm_hidden_dim=META["hid"], lstm_num_layers=META["layers"], gcn_hidden_dim=META["gcn_hid"],
                          sta_kernel_config={"kernel_type": "chebyshev" if kind == "cheb" else "random_walk_diffusion",
                                             "K": k},
                          gconv_use_bias=True, gconv_activation=nn.ReLU if relu else None).to(DEV)


def _oracle(model, mats, kind, relu, masks=None):
    params = {key: v.detach().cpu().numpy() for key, v in model.state_dict().items()}
    if kind == "cheb":
        return O.SparseOracle(params, mats, META["k"] + 1, relu=relu, dtype=np.float64, relu_masks=masks)
    return D.ChainOracle(params, mats, 2 * META["k"] + 1, relu=relu, dtype=np.float64, relu_masks=masks)


def _inputs(seed=1, b=META["b"]):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(b, META["t"], META["n"], META["c"], generator=gen)
    y = torch.randn(b, META["n"], META["c"], generator=gen)
    return x, y


def _fill(model, x, y, sups):
    """One training forward + backward (gradients accumulated into zeroed buffers, in place) and one no_grad forward."""
    for p in model.parameters():
        if p.grad is not None:
            p.grad.zero_()
    nn.MSELoss()(model(obs_seq=x, sta_adj_list=sups), y).backward()
    with torch.no_grad():
        model(obs_seq=x, sta_adj_list=sups)


def _run(model, x, y, sups):
    """A no_grad forward, then a training forward + backward: (output of each, loss and every parameter gradient; the
    ReLU masks of the training forward's GCNs in the oracle's order)."""
    from stmgcn_b200 import ops
    with torch.no_grad():
        out_ng = model(obs_seq=x, sta_adj_list=sups)
    for p in model.parameters():
        p.grad = None
    gcn_outs = []
    real_proj_fwd = ops._proj_fwd

    def recording_proj_fwd(*a, **k):
        gcn_outs.append(real_proj_fwd(*a, **k))
        return gcn_outs[-1]

    ops._proj_fwd = recording_proj_fwd
    try:
        out = model(obs_seq=x, sta_adj_list=sups)
    finally:
        ops._proj_fwd = real_proj_fwd
    loss = nn.MSELoss()(out, y)
    loss.backward()
    res = {"no_grad out": out_ng.cpu().numpy(), "out": out.detach().cpu().numpy(), "loss": loss.item()}
    res.update({"grad " + key: p.grad.cpu().numpy() for key, p in model.named_parameters()})
    return res, [(g > 0).cpu().numpy() for g in gcn_outs]


def _errs(res, ref):
    return {key: (abs(res[key] - ref[key]) / abs(ref[key]) if key == "loss" else O.max_rel_err(res[key], ref[key]))
            for key in ref}


def _oracle_ref(orc, x, y):
    out, loss, grads = orc.loss_and_grads(x.numpy(), y.numpy())
    ref = {"no_grad out": out, "out": out, "loss": loss}
    ref.update({"grad " + key: g for key, g in grads.items()})
    return ref


def _assert_within(errs, tol, what):
    worst = sorted(errs.items(), key=lambda kv: -kv[1])
    print(what, ", ".join(f"{k} {v:.2e}" for k, v in worst[:4]))
    bad = {k: f"{v:.2e}" for k, v in errs.items() if not v <= tol}
    assert not bad, f"{what}: above {tol:.0e}: {bad}"


def _mechanism(name, model, other, x, y, sups):
    """Sets up the update ``name`` on ``model`` and returns the callable that applies it (after the first step, with the
    gradients that step left).  ``other``: a differently seeded model, the source of the copies."""
    params = list(model.parameters())
    if name == "adam_foreach":
        return torch.optim.Adam(params, lr=LR, weight_decay=WD, foreach=True).step
    if name == "adam_fused":
        return torch.optim.Adam(params, lr=LR, weight_decay=WD, fused=True).step
    if name == "adamw_fused":
        return torch.optim.AdamW(params, lr=LR, weight_decay=WD, fused=True).step
    if name == "sgd_fused":
        return torch.optim.SGD(params, lr=LR_SGD, weight_decay=WD, fused=True).step
    if name == "data_add_":            # a hand-written SGD step
        def step():
            for p in params:
                p.data.add_(p.grad, alpha=-LR_SGD)
        return step
    if name == "data_copy_":           # loading weights the old way
        def step():
            for p, q in zip(params, other.parameters()):
                p.data.copy_(q)
        return step
    if name == "no_grad_copy_":
        def step():
            with torch.no_grad():
                for p, q in zip(params, other.parameters()):
                    p.copy_(q)
        return step
    if name == "load_state_dict":
        return lambda: model.load_state_dict(other.state_dict())
    if name == "load_state_dict_assign":
        return lambda: model.load_state_dict(other.state_dict(), assign=True)
    if name == "captured_step":
        # the optimizer step alone captured in a CUDA graph (warm-up on a side stream first, as torch.cuda.graphs asks);
        # the gradients it reads are the .grad tensors _fill accumulates into in place
        opt = torch.optim.Adam(params, lr=LR, weight_decay=WD, capturable=True)
        nn.MSELoss()(model(obs_seq=x, sta_adj_list=sups), y).backward()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            opt.step()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            opt.step()
        return graph.replay
    raise ValueError(name)


CASES = [("cheb", mech, p) for mech in MECHANISMS for p in PATHS] + [("diffusion", "adam_fused", "tc2")]


@pytest.mark.parametrize("kind,mechanism,path", CASES, indirect=["path"])
def test_model_after_update_matches_the_oracle_at_its_new_weights(kind, mechanism, path):
    relu = path != "tc1"
    sups, mats = _supports(kind)
    model = _model(kind, relu, seed=0)
    other = _model(kind, relu, seed=5)
    x, y = _inputs()
    xd, yd = x.to(DEV), y.to(DEV)
    update = _mechanism(mechanism, model, other, xd, yd, sups)
    _fill(model, xd, yd, sups)
    before = _oracle(model, mats, kind, relu)
    update()
    fresh = copy.deepcopy(model)
    res, masks = _run(model, xd, yd, sups)
    tag = f"{kind} {mechanism} {path}"
    _assert_within(_errs(res, _run(fresh, xd, yd, sups)[0]), FRESH[path], f"{tag} vs fresh copy")
    _assert_within(_errs(res, _oracle_ref(_oracle(model, mats, kind, relu, masks), x, y)), BAR[path], f"{tag} vs oracle")
    e_before = O.max_rel_err(res["out"], before.forward(x.numpy()))
    print(f"{tag}: output vs the oracle at the weights before the update {e_before:.2e}")
    assert e_before > BAR[path], f"{tag}: the update moved the output by only {e_before:.2e}"


@pytest.mark.parametrize("path", PATHS, indirect=True)
def test_two_fresh_copies_agree_within_the_fresh_copy_bar(path):
    """Two deep copies of one model, each packing its own images, agree within FRESH."""
    relu = path != "tc1"
    sups, _ = _supports("cheb")
    model = _model("cheb", relu, seed=0)
    x, y = (t.to(DEV) for t in _inputs())
    a, b = (_run(copy.deepcopy(model), x, y, sups)[0] for _ in range(2))
    errs = _errs(a, b)
    print(f"fresh-copy spread ({path}): outputs {max(errs['out'], errs['no_grad out']):.2e}, gradients "
          f"{max(v for k, v in errs.items() if k.startswith('grad')):.2e}")
    _assert_within(errs, FRESH[path], f"{path} fresh copies")


@pytest.mark.parametrize("ks", [1, 4, 5, 8])
def test_gcn_module_after_data_copy_matches_the_dense_oracle(ks):
    """GCN with p = q = 64 (the tensor-core projection; ks = 5 and 8 pack two backward images): forward, dX, dW and db
    after ``W.data.copy_`` / ``b.data.copy_`` against ``O.dense_gcn`` in fp64 at the new weights."""
    import GCN
    from stmgcn_b200 import synth
    n, b = 96, 8
    sup = O.chebyshev_supports_dense(synth.make_adjacency(n, 0, 0.05), ks - 1)
    supd = sup.to(DEV)
    torch.manual_seed(ks)
    layer = GCN.GCN(K=ks, input_dim=64, hidden_dim=64).to(DEV)
    other = GCN.GCN(K=ks, input_dim=64, hidden_dim=64)
    nn.init.normal_(other.b, std=0.1)
    gen = torch.Generator().manual_seed(10 + ks)
    x = torch.randn(b, n, 64, generator=gen)
    probe = torch.randn(b, n, 64, generator=gen)

    def run():
        with torch.no_grad():
            out_ng = layer(supd, x.to(DEV))
        xd = x.to(DEV).requires_grad_(True)
        layer.zero_grad(set_to_none=True)
        out = layer(supd, xd)
        (out * probe.to(DEV)).sum().backward()
        return dict(no_grad_out=out_ng, out=out.detach(), dx=xd.grad, dW=layer.W.grad, db=layer.b.grad)

    def reference(w, bias):
        x64 = x.double().requires_grad_(True)
        w64 = w.detach().cpu().double().requires_grad_(True)
        b64 = bias.detach().cpu().double().requires_grad_(True)
        out = O.dense_gcn(sup.double(), x64, w64, b64)
        (out * probe.double()).sum().backward()
        return dict(no_grad_out=out.detach(), out=out.detach(), dx=x64.grad, dW=w64.grad, db=b64.grad)

    run()
    before = reference(layer.W, layer.b)["out"]
    layer.W.data.copy_(other.W)
    layer.b.data.copy_(other.b)
    res, ref = run(), reference(layer.W, layer.b)
    errs = {key: O.max_rel_err(res[key].cpu().numpy(), ref[key].numpy()) for key in ref}
    _assert_within(errs, TOL, f"GCN ks={ks} after data.copy_")
    assert O.max_rel_err(res["out"].cpu().numpy(), before.numpy()) > TOL


def test_cg_lstm_module_after_data_copy_matches_the_dense_oracle():
    """CG_LSTM with C = 2, an initial state (h0, c0) and its final state: output, (h_n, c_n) and every parameter
    gradient after ``p.data.copy_`` of every parameter, against ``O.dense_cg_lstm`` in fp64 at the new weights."""
    import STMGCN
    from stmgcn_b200 import synth
    n, b, t, c, hid, lyr, k = 96, 8, 12, 2, 64, 3, 3
    sup = O.chebyshev_supports_dense(synth.make_adjacency(n, 0, 0.05), k)
    supd = sup.to(DEV)

    def make(seed):
        torch.manual_seed(seed)
        return STMGCN.CG_LSTM(seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=lyr, K=k + 1,
                              gconv_use_bias=True)

    mod, other = make(0).to(DEV), make(7)
    gen = torch.Generator().manual_seed(3)
    obs = torch.randn(b, t, n, c, generator=gen)
    h0, c0 = torch.randn(lyr, b * n, hid, generator=gen) * 0.3, torch.randn(lyr, b * n, hid, generator=gen) * 0.3
    probes = [torch.randn(b, n, hid, generator=gen), torch.randn(lyr, b * n, hid, generator=gen),
              torch.randn(lyr, b * n, hid, generator=gen)]

    def run():
        mod.zero_grad(set_to_none=True)
        out, (h_n, c_n) = mod(supd, obs.to(DEV), (h0.to(DEV), c0.to(DEV)))
        sum((v * pr.to(DEV)).sum() for v, pr in zip((out, h_n, c_n), probes)).backward()
        res = dict(out=out, h_n=h_n, c_n=c_n)
        res.update({"grad " + key: p.grad for key, p in mod.named_parameters()})
        return {key: v.detach().cpu().numpy() for key, v in res.items()}

    def reference():
        params = {"p." + key: v.detach().cpu().double().requires_grad_(True) for key, v in mod.state_dict().items()}
        out, (h_n, c_n) = O.dense_cg_lstm(sup.double(), obs.double(), params, "p.", hidden=(h0.double(), c0.double()))
        sum((v * pr.double()).sum() for v, pr in zip((out, h_n, c_n), probes)).backward()
        res = dict(out=out, h_n=h_n, c_n=c_n)
        res.update({"grad " + key[2:]: p.grad for key, p in params.items()})
        return {key: v.detach().numpy() for key, v in res.items()}

    run()
    before = reference()["out"]
    for p, q in zip(mod.parameters(), other.parameters()):
        p.data.copy_(q)
    res, ref = run(), reference()
    _assert_within({key: O.max_rel_err(res[key], ref[key]) for key in ref}, TOL, "CG_LSTM after data.copy_")
    assert O.max_rel_err(res["out"], before) > TOL


def test_trainer_flow_with_fused_adam_validates_what_a_checkpoint_reloads():
    """Model_Trainer.py's flow with ``Adam(fused=True)``: a few training steps, validation under
    ``torch.set_grad_enabled(False)`` (its :33), the state_dict saved and loaded into a fresh model: the reloaded model
    predicts what was validated (FRESH), and the validation is the oracle's at the trained weights."""
    sups, mats = _supports("cheb")
    model = _model("cheb", True, seed=0)
    x, y = _inputs()
    xv, _ = _inputs(seed=2)
    xd, yd, xvd = x.to(DEV), y.to(DEV), xv.to(DEV)
    opt = torch.optim.Adam(model.parameters(), lr=LR, weight_decay=WD, fused=True)
    crit = nn.MSELoss(reduction="mean")
    for _ in range(3):
        model.train()
        with torch.set_grad_enabled(True):
            loss = crit(model(obs_seq=xd, sta_adj_list=sups), yd)
            opt.zero_grad()
            loss.backward()
            opt.step()
    model.eval()
    with torch.set_grad_enabled(False):
        val = model(obs_seq=xvd, sta_adj_list=sups).cpu().numpy()
    buf = io.BytesIO()
    torch.save({"epoch": 3, "state_dict": model.state_dict()}, buf)
    buf.seek(0)
    reloaded = _model("cheb", True, seed=9)
    reloaded.load_state_dict(torch.load(buf)["state_dict"])
    reloaded.eval()
    with torch.no_grad():
        val2 = reloaded(obs_seq=xvd, sta_adj_list=sups).cpu().numpy()
    e_reload = O.max_rel_err(val, val2)
    e_oracle = O.max_rel_err(val, _oracle(model, mats, "cheb", True).forward(xv.numpy()))
    print(f"validation after 3 fused Adam steps: vs the reloaded checkpoint {e_reload:.2e}, vs the oracle {e_oracle:.2e}")
    assert e_reload <= FRESH["tc2"], f"the reloaded checkpoint predicts {e_reload:.2e} away from the validated model"
    assert e_oracle <= TOL, f"validation {e_oracle:.2e} from the oracle at the trained weights"


def test_graphed_step_and_its_eager_short_batch_after_a_fused_step():
    """GraphedStep: replay, a fused Adam step, replay again, then a short batch (eager: shapes are baked into the graph).
    Prediction, loss and every gradient of each against the oracle at the weights of that moment."""
    from stmgcn_b200 import graphs
    sups, mats = _supports("cheb")
    model = _model("cheb", True, seed=0)
    x, y = _inputs()
    xd, yd = x.to(DEV), y.to(DEV)
    gstep = graphs.GraphedStep(model, nn.MSELoss(), xd, yd, sups)
    opt = torch.optim.Adam(model.parameters(), lr=LR, weight_decay=WD, fused=True)

    def check(loss, xs, ys, what):
        res = {"out": gstep.out.cpu().numpy(), "loss": loss.item()}
        res.update({"grad " + key: p.grad.cpu().numpy() for key, p in model.named_parameters()})
        ref = _oracle_ref(_oracle(model, mats, "cheb", True), xs, ys)
        del ref["no_grad out"]
        _assert_within(_errs(res, ref), TOL, what)

    check(gstep(xd, yd), x, y, "first replay")
    opt.step()
    check(gstep(xd, yd), x, y, "replay after a fused Adam step")
    short = META["b"] - 3
    check(gstep(xd[:short], yd[:short]), x[:short], y[:short], "short batch (eager) after a fused Adam step")


def test_dense_support_stack_edited_in_place_is_picked_up():
    """``graph.supports_from_dense`` caches the conversion of a dense stack on its identity and in-place version.  An
    edit by a normal op (``sup.mul_`` under no_grad) bumps the version: the next forward converts the stack again, here
    from "cheb" (A[0] = I) to "generic" (A[0] = I / 2), and computes the edited stack's GCN (``O.dense_gcn`` in fp64)."""
    import GCN
    from stmgcn_b200 import synth
    from stmgcn_b200.graph import supports_from_dense
    n, b, k = 96, 8, 3
    sup = GCN.Adj_Preprocessor("chebyshev", k).process(synth.make_adjacency(n, 0, 0.05)).to(DEV)
    torch.manual_seed(0)
    layer = GCN.GCN(K=k + 1, input_dim=64, hidden_dim=64).to(DEV)
    gen = torch.Generator().manual_seed(4)
    x = torch.randn(b, n, 64, generator=gen)
    probe = torch.randn(b, n, 64, generator=gen)

    def run():
        layer.zero_grad(set_to_none=True)
        out = layer(sup, x.to(DEV))
        (out * probe.to(DEV)).sum().backward()
        return out.detach().cpu().numpy(), layer.W.grad.cpu().numpy()

    def reference():
        w = layer.W.detach().cpu().double().requires_grad_(True)
        out = O.dense_gcn(sup.cpu().double(), x.double(), w, layer.b.detach().cpu().double())
        (out * probe.double()).sum().backward()
        return out.detach().numpy(), w.grad.numpy()

    out0, _ = run()
    assert supports_from_dense(sup).mode == "cheb"
    with torch.no_grad():
        sup.mul_(0.5)
    assert supports_from_dense(sup).mode == "generic"
    (out, dw), (out_ref, dw_ref) = run(), reference()
    e_out, e_dw = O.max_rel_err(out, out_ref), O.max_rel_err(dw, dw_ref)
    print(f"after sup.mul_(0.5): forward {e_out:.2e}, dW {e_dw:.2e} from the oracle")
    assert e_out <= TOL and e_dw <= TOL, (e_out, e_dw)
    assert O.max_rel_err(out0, out_ref) > TOL
