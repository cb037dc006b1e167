"""fp64 references of the dense support-stack gradient (``GCN.py:35`` differentiated in ``A[k]``) and the stacks its
suites run on.  Shared by the host and the GPU suites.

Two independent restatements:
* ``model_reference``: the dense restatement of the model (``stmgcn_oracle.dense_st_mgcn``) with the stacks as autograd
  leaves, so autograd gives every slice's gradient;
* ``gcn_formula``: the formula the kernel implements, ``dA_k = U_k x^T`` with ``U_k = dZ W_k^T`` the direct adjoint of
  ``S_k = A_k x`` in node-major form (``N, B*p``).
"""
import os

import numpy as np
import torch

import stmgcn_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN_CASES = ("cheb_leaf", "localpool_leaf", "cheb_adj", "cglstm_adj")


def load_case(name):
    """One case of ``dense_support_grad_ref.npz`` (oracle/make_dense_support_grad_golden.py): (meta dict, params, blob
    entries of the case without their prefix)."""
    blob = np.load(os.path.join(GOLDEN, "dense_support_grad_ref.npz"))
    p = name + "."
    sub = {k[len(p):]: blob[k] for k in blob.files if k.startswith(p)}
    n, m, k, t, b, c, hid, layers, gcn_hid = [int(v) for v in sub["meta"]]
    meta = dict(n=n, m=m, k=k, t=t, b=b, c=c, hid=hid, layers=layers, gcn_hid=gcn_hid,
                kernel_type=str(sub["kernel_type"]))
    params = {key[len("param."):]: torch.from_numpy(v) for key, v in sub.items() if key.startswith("param.")}
    return meta, params, sub


def dense_process(kernel_type, k, adj):
    """``Adj_Preprocessor.process`` of the repo (differentiable in ``adj``, any dtype and device)."""
    import GCN
    return GCN.Adj_Preprocessor(kernel_type, k).process(adj)


# ---- stacks ------------------------------------------------------------------------------------------------------
def symmetric_graph(n, seed, device="cpu", dtype=torch.float32):
    """Symmetric weighted connected adjacency (a ring plus random chords, no self-loops)."""
    gen = torch.Generator().manual_seed(seed)
    a = (torch.rand(n, n, generator=gen) < 0.2).double() * (0.5 + torch.rand(n, n, generator=gen, dtype=torch.float64))
    idx = torch.arange(n)
    a[idx, (idx + 1) % n] += 1.0
    a = 0.5 * (a + a.t())
    a.fill_diagonal_(0.0)
    return a.to(device, dtype)


def make_stack(kind, n, seed, device="cpu", dtype=torch.float32):
    """A dense (Ks, N, N) stack: ``"cheb"`` (Chebyshev K = 2 of the rescaled Laplacian: the kernels keep L~ only),
    ``"localpool"``, ``"generic"`` (three sparse random slices, a hand-made stack), ``"diffusion"`` (the 2K+1 = 5
    bidirectional random-walk stack, K = 2, densely) or ``"k0"`` (``[I]``)."""
    a = symmetric_graph(n, seed, "cpu", torch.float64)
    if kind == "cheb":
        st = dense_process("chebyshev", 2, a)
    elif kind == "localpool":
        st = dense_process("localpool", 1, a)
    elif kind == "k0":
        st = torch.eye(n, dtype=torch.float64)[None]
    elif kind == "generic":
        gen = torch.Generator().manual_seed(seed + 1)
        st = (torch.rand(3, n, n, generator=gen) < 0.25).double() * torch.randn(3, n, n, generator=gen, dtype=torch.float64)
    elif kind == "diffusion":
        gen = torch.Generator().manual_seed(seed + 2)
        d = a * (0.5 + torch.rand(n, n, generator=gen, dtype=torch.float64))      # directed weights
        pf = d / d.sum(1, keepdim=True)
        pb = d.t() / d.t().sum(1, keepdim=True)
        st = O.chain_stack_dense([pf.t(), pb.t()], 2)
    else:
        raise ValueError(kind)
    return st.to(device, dtype).contiguous()


STACK_KINDS = ("cheb", "localpool", "generic", "diffusion", "k0")


# ---- references --------------------------------------------------------------------------------------------------
def model_reference(params, obs, y, stacks, branch_stack, relu=True, masks=None, device="cpu", cg_probe=None):
    """fp64 (out, loss, parameter gradients, stack gradients) of the dense restatement with every stack a leaf; branch
    m reads ``stacks[branch_stack[m]]``.  ``y``: the MSE target (``ST_MGCN``), or None with ``cg_probe``: the first
    ``CG_LSTM`` alone (zero initial state) and the scalar ``sum(out * cg_probe)``.  ``masks``: the kernels' ReLU masks
    (:func:`support_grad_cases.record_relu_masks`)."""
    leaves = {k: v.detach().to(device, torch.float64).clone().requires_grad_(True) for k, v in params.items()}
    sl = [s.detach().to(device, torch.float64).clone().requires_grad_(True) for s in stacks]
    obs = obs.detach().to(device, torch.float64)
    if cg_probe is None:
        out = O.dense_st_mgcn(leaves, obs, [sl[i] for i in branch_stack], relu, masks=masks)
        loss = torch.mean((out - y.detach().to(device, torch.float64)) ** 2)
    else:
        out, _ = O.dense_cg_lstm(sl[branch_stack[0]], obs, leaves, "rnn_list.0.", relu,
                                 mask=None if masks is None else masks[0])
        loss = (out * cg_probe.detach().to(device, torch.float64)).sum()
    keys = [k for k in leaves if (cg_probe is None or k.startswith("rnn_list.0."))]
    res = torch.autograd.grad(loss, [leaves[k] for k in keys] + sl, allow_unused=True)
    return out.detach(), float(loss.detach()), dict(zip(keys, res[:len(keys)])), list(res[len(keys):])


def gcn_forward(stack, x, w, b, relu=True):
    """The reference GCN on a (B, N, p) input: ``act(cat_k(A_k x) W + b)``."""
    return O.dense_gcn(stack, x, w, b, relu)


def gcn_u(stack, x, w, b, probe, relu=True):
    """``U_k = dL/dS_k`` of one GCN for the loss ``sum(out * probe)``, node-major (Ks, N, B*p)."""
    ks, p = stack.shape[0], x.shape[-1]
    s = torch.stack([torch.matmul(stack[k], x) for k in range(ks)]).detach().requires_grad_(True)   # (Ks, B, N, p)
    z = sum(torch.matmul(s[k], w[k * p:(k + 1) * p]) for k in range(ks)) + (0 if b is None else b)
    out = torch.relu(z) if relu else z
    (u,) = torch.autograd.grad((out * probe).sum(), [s])
    return u.permute(0, 2, 1, 3).reshape(ks, x.shape[1], -1)


def gcn_formula(stack, x, w, b, probe, relu=True):
    """``dA_k = U_k x^T`` of one GCN, every slice (the kernel's formula)."""
    u = gcn_u(stack, x, w, b, probe, relu)
    xn = x.permute(1, 0, 2).reshape(x.shape[1], -1)
    return torch.einsum("kif,jf->kij", u, xn)


def gcn_autograd(stack, x, w, b, probe, relu=True):
    """Autograd's gradient of the stack for the same loss."""
    leaf = stack.detach().clone().requires_grad_(True)
    (g,) = torch.autograd.grad((gcn_forward(leaf, x, w, b, relu) * probe).sum(), [leaf])
    return g


class DenseStackReference(O.BF16ModeReference):
    """:class:`O.BF16ModeReference` (rounding, forcing with the kernels' tapes, ReLU masks and window chunks as there)
    that also forms every graph convolution's dense-stack gradient from its own backward: ``da[(m, spatial)]`` is
    ``sum over chunks of U_k x^T`` in its dtype, ``U_k = dZ W_k^T`` (``dZ`` the gradient of the pre-activation the
    reference's autograd computes) and ``x`` the reference's own GCN input (the forced ``s[0]`` on the spatial GCN).  A
    stack's gradient is the sum over the GCNs that read it.  Chebyshev chains or ``K = 0`` stacks, as the parent."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.da = {}

    def _gcn(self, m, x, w, b, mask_i, spatial, tape_s=None, windows=None):
        n, bsz, p = x.shape
        used, comp = self._stack(m, x, spatial, tape_s)
        z = sum(used[k].reshape(n, bsz, p) @ w[k * p:(k + 1) * p] for k in range(self.ks))
        if b is not None:
            z = z + b
        if torch.is_grad_enabled():
            x0, wd, key = used[0].detach(), w.detach(), (m, spatial)

            def hook(dz):
                u = torch.stack([(dz @ wd[k * p:(k + 1) * p].t()).reshape(n, -1) for k in range(self.ks)])
                self.da[key] = self.da.get(key, 0) + torch.einsum("kif,jf->kij", u, x0)
            z.register_hook(hook)
        if self.relu and self.masks is not None:
            mask = self.masks[mask_i] if windows is None else self.masks[mask_i][:, windows]
            z = z * mask.to(z.dtype)
        elif self.relu:
            z = torch.relu(z)
        return z, comp

    def stack_grad(self, branches):
        """The gradient of the stack that the graph branches ``branches`` read: both GCNs of each."""
        return sum(self.da[(m, s)] for m in branches for s in (False, True))


def chains_of(stack):
    """The recurrence matrices :class:`O.BF16ModeReference` takes for one branch on a dense Chebyshev stack: ``[L~]``
    as scipy CSR (exact zeros dropped, as the kernels' conversion does), none for ``[I]``."""
    import scipy.sparse as sp
    return [sp.csr_matrix(stack[1].detach().double().cpu().numpy())] if stack.shape[0] > 1 else []
