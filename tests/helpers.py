"""Shared helpers for the test-suite (test infrastructure; may import the oracle)."""
import os

import numpy as np
import torch
from torch import nn

import stmgcn_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DEV = "cuda:0"
TOL = 1e-4          # BASELINE.json north_star: "within 1e-4 relative fp32" (max-norm form, SURVEY 8(d))
FWD_TOL, GRAD_TOL = 2e-5, 5e-5      # the kernel-level bars: forward values, gradients (max-norm relative)


def rel_err(a, b):
    """``max|a - b| / max|b|`` in fp64, with 1 as the denominator when ``max|b| = 0``, as ``O.max_rel_err``.  ``a`` and
    ``b`` are tensors (on any device) or numpy arrays; tensors are compared on ``a``'s device."""
    a, b = (torch.as_tensor(v).detach().double() for v in (a, b))
    b = b.to(a.device)
    den = float(b.abs().max())
    return float((a - b).abs().max()) / (den if den > 0 else 1.0)


def lib():
    """The library's ctypes handle (``_lib.lib``)."""
    from stmgcn_b200 import _lib
    return _lib.lib


def sm_count():
    return int(lib().stmgcn_sm_count())


def load_golden(name):
    """A fixture of ``oracle/make_golden.py``.  ``meta`` holds the sizes and the model configuration: ``kernel_type``,
    ``bias`` (``gconv_use_bias``) and ``activation`` (the activation's class name, or ``"None"``); fixtures written before
    those were recorded are Chebyshev models with bias and ReLU."""
    blob = np.load(os.path.join(GOLDEN, name + ".npz"))
    n, m, k, t, b, c, hid, layers, gcn_hid = [int(v) for v in blob["meta"]]
    meta = dict(n=n, m=m, k=k, t=t, b=b, c=c, hid=hid, layers=layers, gcn_hid=gcn_hid,
                kernel_type=str(blob["kernel_type"]) if "kernel_type" in blob.files else "chebyshev",
                bias=bool(blob["gconv_use_bias"]) if "gconv_use_bias" in blob.files else True,
                activation=str(blob["gconv_activation"]) if "gconv_activation" in blob.files else "ReLU")
    params = {key[len("param."):]: torch.from_numpy(blob[key]) for key in blob.files if key.startswith("param.")}
    grads = {key[len("grad."):]: blob[key] for key in blob.files if key.startswith("grad.")}
    supports = [torch.from_numpy(blob[f"supports.{g}"]) for g in range(m)]
    adjs = [torch.from_numpy(blob[f"adj.{g}"]) for g in range(m)]
    return meta, params, grads, supports, adjs, blob


def activation_class(name):
    """``nn.ReLU`` for ``"ReLU"`` etc.; None for ``"None"``."""
    return None if name == "None" else getattr(nn, name)


def oracle_activation(name):
    """The dense restatement's ``relu`` argument for an activation class name: True (ReLU), False (none) or a module."""
    fixed = {"ReLU": True, "None": False}
    return fixed[name] if name in fixed else activation_class(name)()


def build_model(meta, device, relu=None):
    """The repo's ``ST_MGCN`` for ``meta``: its ``kernel_type``, ``bias`` and ``activation`` when given, else a
    Chebyshev model with bias and ReLU.  ``relu`` True / False, when given, overrides the activation (ReLU / none)."""
    import STMGCN
    if relu is not None:
        act = nn.ReLU if relu else None
    else:
        act = activation_class(meta.get("activation", "ReLU"))
    model = STMGCN.ST_MGCN(M=meta["m"], seq_len=meta["t"], n_nodes=meta["n"], input_dim=meta["c"],
                           lstm_hidden_dim=meta["hid"], lstm_num_layers=meta["layers"],
                           gcn_hidden_dim=meta["gcn_hid"],
                           sta_kernel_config={"kernel_type": meta.get("kernel_type", "chebyshev"), "K": meta["k"]},
                           gconv_use_bias=meta.get("bias", True), gconv_activation=act)
    return model.to(device)


def assert_close(new, ref, what, tol=TOL):
    err = O.max_rel_err(new, ref)
    assert err <= tol, f"{what}: max-norm relative error {err:.3e} > {tol:.1e}"
    return err
