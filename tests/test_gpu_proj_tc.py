"""The tensor-core projection of the Chebyshev GCN (proj_tc.cu: forward, dZ / bias gradient / U, dW and the weight-image
pack) against an fp64 reference, on random stacks: every support count the kernels take (ks = 1..8; ks > 4
splits U over two launches), row counts around the 32-row weight-gradient chunk and the 128-row tile, a multi-wave
ragged size, ReLU and bias on and off.  Bars: 2e-5 forward, 5e-5 gradients (max-norm relative)."""
import pytest
import torch

import stmgcn_oracle as O
from helpers import DEV, FWD_TOL, GRAD_TOL
from kernel_cases import tc_shape

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("rows_id", [1, 31, 33, 129, "waves"])
@pytest.mark.parametrize("ks", list(range(1, 9)))
def test_projection_tensor_core_kernels_match_fp64(ks, rows_id, relu, bias):
    """out = act(sum_k S_k W_k + b); dZ = d_out * mask with the kernel's own mask (out > 0); db = sum dZ; dW_k = S_k^T dZ;
    U_k = dZ W_k^T.  Measured on an H100 (max over all 160 cases): out 6.3e-6, gradients 3.2e-6."""
    from stmgcn_b200 import ops
    n, b = tc_shape(rows_id)
    p = q = 64
    gen = torch.Generator().manual_seed(100 * ks + (rows_id if isinstance(rows_id, int) else 999) + 2 * relu + bias)
    s = torch.randn(ks, n, b, p, generator=gen).to(DEV)
    w = (torch.randn(ks * p, q, generator=gen) * 0.1).to(DEV)
    bv = (torch.randn(q, generator=gen) * 0.3).to(DEV) if bias else None
    d_out = torch.randn(n, b, q, generator=gen).to(DEV)
    act = 1 if relu else 0
    img_f, img_b = ops._proj_images(w, ks, p, True)
    assert img_f is not None and img_b is not None, "the tensor-core projection path did not run"
    out = ops._proj_fwd(s, w, bv, act, None, b, img_f)
    dw, db, u = ops._proj_bwd(s, w, act, out, d_out, None, 1.0, b, bias, True, img_b)
    torch.cuda.synchronize()

    rows = n * b
    s64 = s.double().reshape(ks, rows, p)
    w64 = w.double().reshape(ks, p, q)
    z = torch.einsum("krp,kpq->rq", s64, w64)
    if bias:
        z = z + bv.double()
    ref_out = z.clamp_min(0) if relu else z
    dz = d_out.double().reshape(rows, q)
    if relu:
        dz = dz * (out.reshape(rows, q) > 0)
    errs = {"out": O.max_rel_err(out.reshape(rows, q).cpu().numpy(), ref_out.cpu().numpy())}
    gerrs = {}
    if bias:
        gerrs["db"] = O.max_rel_err(db.cpu().numpy(), dz.sum(0).cpu().numpy())
    dw_ref = torch.einsum("krp,rq->kpq", s64, dz)
    u_ref = torch.einsum("rq,kpq->krp", dz, w64)
    for k in range(ks):
        gerrs[f"dW_{k}"] = O.max_rel_err(dw[k * p:(k + 1) * p].cpu().numpy(), dw_ref[k].cpu().numpy())
        gerrs[f"U_{k}"] = O.max_rel_err(u[k].reshape(rows, p).cpu().numpy(), u_ref[k].cpu().numpy())
    print(f"proj ks={ks} rows={rows} relu={relu} bias={bias}: out {errs['out']:.2e}, worst gradient "
          f"{max(gerrs.values()):.2e} ({max(gerrs, key=gerrs.get)})")
    bad = {k: v for k, v in errs.items() if not v <= FWD_TOL}
    bad.update({k: v for k, v in gerrs.items() if not v <= GRAD_TOL})
    assert not bad, f"ks={ks} rows={rows}: above the bar: {bad}"
