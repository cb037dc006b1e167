"""CPU tests of the input- and state-gradient surface: the fp64 dense oracle against the reference's gradients at
obs_seq, h0 and c0 (tests/golden/inputgrad_ref.npz, oracle/make_golden_inputs.py), and the argument checks and
bindings of the entry points that compute them."""
import ctypes

import numpy as np
import torch

import stmgcn_oracle as O
from helpers import GOLDEN, assert_close

BAR = 2e-5


def _blob():
    return np.load(f"{GOLDEN}/inputgrad_ref.npz")


def _params(blob, prefix):
    return {k[len(prefix) + 6:]: torch.from_numpy(blob[k]).double().requires_grad_(True)
            for k in blob.files if k.startswith(prefix + "param.")}


def test_dense_oracle_matches_the_reference_input_gradient_of_st_mgcn():
    blob = _blob()
    m = int(blob["st.meta"][1])
    params = _params(blob, "st.")
    sups = [torch.from_numpy(blob[f"st.supports.{g}"]).double() for g in range(m)]
    x = torch.from_numpy(blob["st.x"]).double().requires_grad_(True)
    out = O.dense_st_mgcn(params, x, sups)
    loss = torch.mean((out - torch.from_numpy(blob["st.y"]).double()) ** 2)
    grads = torch.autograd.grad(loss, [x] + list(params.values()))
    assert_close(out.detach().numpy(), blob["st.out"], "forward", 1e-5)
    assert_close(grads[0].numpy(), blob["st.grad_obs"], "d obs", BAR)
    for key, g in zip(params, grads[1:]):
        assert_close(g.numpy(), blob["st.grad." + key], f"grad {key}", BAR)


def test_dense_oracle_matches_the_reference_state_gradients_of_cg_lstm():
    blob = _blob()
    params = _params(blob, "cg.")
    t64 = lambda k: torch.from_numpy(blob["cg." + k]).double()      # noqa: E731
    x, h0, c0 = (t64(k).requires_grad_(True) for k in ("x", "h0", "c0"))
    out, (h_n, c_n) = O.dense_cg_lstm(t64("supports"), x, params, "", hidden=(h0, c0))
    loss = torch.mean((out - t64("y")) ** 2) + (h_n * t64("r1")).sum() + (c_n * t64("r2")).sum()
    grads = torch.autograd.grad(loss, [x, h0, c0] + list(params.values()))
    assert_close(h_n.detach().numpy(), blob["cg.h_n"], "h_n", 1e-5)
    assert_close(c_n.detach().numpy(), blob["cg.c_n"], "c_n", 1e-5)
    for name, g in zip(("obs", "h0", "c0"), grads):
        assert_close(g.numpy(), blob["cg.grad_" + name], f"d {name}", BAR)
    for key, g in zip(params, grads[3:]):
        assert_close(g.numpy(), blob["cg.grad." + key], f"grad {key}", BAR)


def test_new_entry_points_are_bound_with_the_old_arguments_plus_the_extras():
    from stmgcn_b200 import _lib
    sig = {name: args for name, _, args in _lib.SIGNATURES}
    assert _lib.ABI_VERSION == 8
    assert sig["stmgcn_lstm_bwd_ex"][:-6] == sig["stmgcn_lstm_bwd"][:-1]
    assert sig["stmgcn_lstm16_bwd_ex"][:-6] == sig["stmgcn_lstm16_bwd"][:-1]
    assert len(sig["stmgcn_lstm_bwd_ex"]) == len(sig["stmgcn_lstm_bwd"]) + 5
    assert len(sig["stmgcn_lstm16_bwd_ex"]) == len(sig["stmgcn_lstm16_bwd"]) + 5
    assert sig["stmgcn_obs_grad"] == sig["stmgcn_obs_to_node_major"]


def test_new_entry_points_reject_bad_arguments_before_touching_cuda():
    """Nulls and unsupported shapes return a negative code with a message (no GPU needed)."""
    from stmgcn_b200 import _lib
    lib = _lib.lib
    p = ctypes.c_void_p(16)            # never dereferenced: every call below fails its argument checks first
    calls = {
        "obs_grad: d_obs NULL": lambda: lib.stmgcn_obs_grad(p, p, None, 2, 3, 4, 1, None),
        "obs_grad: C = 0": lambda: lib.stmgcn_obs_grad(p, p, p, 2, 3, 4, 0, None),
        "lstm_bwd_ex: C = 5": lambda: lib.stmgcn_lstm_bwd_ex(3, 2, 8, 8, 5, 2, *([p] * 17), p, p, p, p, p, None),
        "lstm_bwd_ex: gates NULL": lambda: lib.stmgcn_lstm_bwd_ex(3, 2, 8, 8, 1, 2, *([p] * 8), None, *([p] * 8),
                                                                 p, p, p, p, p, None),
        "lstm16_bwd_ex: T = 65": lambda: lib.stmgcn_lstm16_bwd_ex(65, 2, 100, 1, 4, 2, *([p] * 18), p, p, p, p, p, None),
        "lstm16_bwd_ex: planes = 3": lambda: lib.stmgcn_lstm16_bwd_ex(5, 2, 100, 1, 4, 3, *([p] * 18), p, p, p, p, p, None),
        "lstm16_bwd_ex: d_top NULL": lambda: lib.stmgcn_lstm16_bwd_ex(5, 2, 100, 1, 4, 2, *([p] * 9), None, *([p] * 8),
                                                                     p, p, p, p, p, None),
    }
    for what, call in calls.items():
        rc = call()
        assert rc < 0, f"{what}: rc={rc}"
        assert lib.stmgcn_last_error(), f"{what}: no message"
