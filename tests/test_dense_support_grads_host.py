"""Host tests of the dense support-stack gradient: the fp64 restatement against the reference's own gradients, the
kernel's formula against autograd (and its negative controls), the C entry point's argument checks, and the host policy
for stacks that require grad (never cached, refused by GraphedStep).  No GPU needed."""
import pytest
import torch

import stmgcn_oracle as O
from dense_support_grad_cases import (GOLDEN_CASES, STACK_KINDS, dense_process, gcn_autograd, gcn_formula, gcn_u,
                                      load_case, make_stack, model_reference)
from helpers import TOL, lib, rel_err
from support_grad_cases import chain_adjoints


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_the_dense_restatement_with_leaf_stacks_reproduces_the_reference_gradients(name):
    """The oracle's fp64 model with the stacks as leaves gives the reference's loss, parameter gradients and stack
    gradients; through ``process()`` (differentiated by autograd here, as in the reference) the adjacency's."""
    meta, params, sub = load_case(name)
    m, kt, k = meta["m"], meta["kernel_type"], meta["k"]
    obs = torch.from_numpy(sub["x"])
    cg = "probe" in sub
    adj_mode = "adj_grad.0" in sub
    if adj_mode:
        adjs = [torch.from_numpy(sub[f"adj.{g}"]).double().requires_grad_(True) for g in range(m)]
        stacks = [dense_process(kt, k, a) for a in adjs]
        assert max(rel_err(s, torch.from_numpy(sub[f"supports.{g}"])) for g, s in enumerate(stacks)) <= 1e-6
    else:
        stacks = [torch.from_numpy(sub[f"supports.{g}"]) for g in range(m)]
    y = None if cg else torch.from_numpy(sub["y"])
    probe = torch.from_numpy(sub["probe"]) if cg else None
    if adj_mode:
        # the stacks are not leaves here: autograd continues from them into the adjacencies
        leaves = {kk: v.double().requires_grad_(True) for kk, v in params.items()}
        if cg:
            out, _ = O.dense_cg_lstm(stacks[0], obs.double(), leaves, "rnn_list.0.")
            loss = (out * probe.double()).sum()
        else:
            out = O.dense_st_mgcn(leaves, obs.double(), stacks)
            loss = torch.mean((out - y.double()) ** 2)
        loss.backward()
        assert abs(float(loss) - float(sub["loss"])) <= TOL * abs(float(sub["loss"]))
        for g in range(m):
            key = f"adj_grad.{g}"
            if key in sub:
                assert rel_err(adjs[g].grad, torch.from_numpy(sub[key])) <= TOL, key
        return
    out, loss, grads, sgrads = model_reference(params, obs, y, stacks, list(range(m)))
    assert rel_err(out, torch.from_numpy(sub["out"])) <= TOL
    assert abs(loss - float(sub["loss"])) <= TOL * abs(float(sub["loss"]))
    for key, g in grads.items():
        assert rel_err(g, torch.from_numpy(sub["grad." + key])) <= TOL, key
    for g in range(m):
        assert rel_err(sgrads[g], torch.from_numpy(sub[f"stack_grad.{g}"])) <= TOL


def _gcn_case(kind, seed=0, n=17, b=3, p=6, q=5):
    gen = torch.Generator().manual_seed(seed)
    stack = make_stack(kind, n, seed, dtype=torch.float64)
    ks = stack.shape[0]
    x = torch.randn(b, n, p, generator=gen, dtype=torch.float64)
    w = torch.randn(ks * p, q, generator=gen, dtype=torch.float64)
    bias = torch.randn(q, generator=gen, dtype=torch.float64)
    probe = torch.randn(b, n, q, generator=gen, dtype=torch.float64)
    return stack, x, w, bias, probe


@pytest.mark.parametrize("kind", STACK_KINDS)
def test_the_formula_u_times_x_transposed_is_autograds_gradient_of_every_slice(kind):
    """dA_k = U_k x^T, U the projection's direct adjoint before any Clenshaw, for cheb, generic, dense 2K+1 diffusion
    and K = 0 stacks (A_0 = I gets a gradient too)."""
    stack, x, w, bias, probe = _gcn_case(kind)
    ref = gcn_autograd(stack, x, w, bias, probe)
    assert rel_err(gcn_formula(stack, x, w, bias, probe), ref) <= 1e-12
    assert float(ref[0].abs().max()) > 0


def test_the_formulas_negative_controls_fail_the_bar():
    """dA_k^T, the chain adjoints G_k (U after the Clenshaw), s[0] = A_0 x as x for a generic stack, and dA_0 left out
    each miss the bar by orders of magnitude."""
    stack, x, w, bias, probe = _gcn_case("cheb", seed=3)
    ref = gcn_autograd(stack, x, w, bias, probe)
    good = gcn_formula(stack, x, w, bias, probe)
    margins = {"transposed": rel_err(good.transpose(1, 2), ref)}
    u = gcn_u(stack, x, w, bias, probe)
    lap = stack[1]
    rows, cols = lap.nonzero(as_tuple=True)
    g = chain_adjoints(rows, cols, lap[rows, cols], list(u))
    xn = x.permute(1, 0, 2).reshape(x.shape[1], -1)
    after = torch.stack([u[0]] + list(g))
    margins["after_clenshaw"] = rel_err(torch.einsum("kif,jf->kij", after, xn), ref)
    no0 = good.clone()
    no0[0] = 0
    margins["dA_0_left_out"] = rel_err(no0, ref)
    gst, gx, gw, gb, gp = _gcn_case("generic", seed=4)
    gref = gcn_autograd(gst, gx, gw, gb, gp)
    s0 = torch.matmul(gst[0], gx).permute(1, 0, 2).reshape(gx.shape[1], -1)
    margins["s0_as_x"] = rel_err(torch.einsum("kif,jf->kij", gcn_u(gst, gx, gw, gb, gp), s0), gref)
    print({k: f"{v:.3e}" for k, v in margins.items()})
    for name, err in margins.items():
        assert err > 100 * TOL, (name, err)


def test_the_c_entry_rejects_bad_calls_before_any_launch():
    """Null pointers, ks outside 1..8, n or f_total below 1, a negative stride and a da overlapping u or x return a
    negative code with a message and launch nothing (no GPU needed: the checks come first)."""
    L = lib()
    n0 = L.stmgcn_launch_count()
    base = 1 << 20

    def call(n=4, f=8, ks=2, u=base, stride=32, x=base + 4096, da=base + 8192):
        return L.stmgcn_dense_support_grad(n, f, ks, u, stride, x, da, None)
    bad = [dict(u=None), dict(x=None), dict(da=None), dict(ks=0), dict(ks=9), dict(n=0), dict(f=0), dict(stride=-1),
           dict(da=base + 64), dict(da=base + 4096 + 64), dict(n=1 << 24)]
    for kw in bad:
        rc = call(**kw)
        assert rc < 0, kw
        assert L.stmgcn_last_error(), kw
    assert L.stmgcn_launch_count() == n0


def test_graphed_step_refuses_a_dense_stack_that_requires_grad():
    from stmgcn_b200.graphs import GraphedStep
    stack = torch.eye(4)[None].requires_grad_(True)
    with pytest.raises(ValueError, match=r"dense support stacks \[1\] require grad"):
        GraphedStep(torch.nn.Linear(1, 1), None, torch.zeros(1), torch.zeros(1), [torch.eye(4)[None], stack])


def test_the_cache_holds_no_stack_that_requires_grad_and_no_autograd_graph(monkeypatch):
    """A stack that requires grad is converted at every call and never enters the cache; a cached stack is held
    detached, so the cache keeps no autograd graph alive.  (The conversion itself is stubbed: it needs the device.)"""
    from stmgcn_b200 import graph
    calls = []
    monkeypatch.setattr(graph, "_convert_dense", lambda a, dense=None: calls.append(dense) or object())
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    graph.clear_cache()
    adj = symmetric = torch.rand(6, 6, dtype=torch.float64)
    adj = (symmetric + symmetric.t()).requires_grad_(True)
    stack = dense_process("chebyshev", 2, adj)
    assert stack.requires_grad and stack.grad_fn is not None
    graph.supports_from_dense(stack)
    graph.supports_from_dense(stack)
    assert len(calls) == 2 and all(d is stack for d in calls)
    assert len(graph._CACHE) == 0
    const = stack.detach().clone()
    graph.supports_from_dense(const)
    graph.supports_from_dense(const)
    assert len(calls) == 3 and calls[2] is None
    (held, _), = graph._CACHE.values()
    assert not held.requires_grad and held.grad_fn is None
    graph.clear_cache()
