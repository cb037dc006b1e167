"""Shared model-level cases: the benchmarked workloads with Chebyshev or diffusion supports, the small models of the
input-gradient checks with their dense fp64 gradients, and the recording of the bf16-arithmetic mode's rounding points
for its forced fp64 reference."""
import pytest
import scipy.sparse as sp
import torch
from torch import nn

import stmgcn_oracle as O
from helpers import DEV, rel_err
from lstm_cases import step_local_error


# windows per chunk of the fp64 reference: its autograd tape is ~1 GB per cfg3 window and graph branch, ~8 GB per cfg5
# window (16 384 regions, T = 24)
CHUNK = {"cfg2": 32, "cfg3": 16, "cfg4": 8, "cfg5": 2}


def _csr_of(sup):
    """scipy CSR of L~ from a ChebSupports handle (CPU copy)."""
    rp, ci, va = sup.rowptr.cpu().numpy(), sup.colidx.cpu().numpy(), sup.vals.cpu().numpy()
    return sp.csr_matrix((va, ci, rp), shape=(sup.n, sup.n))


def cheb_workload(w, batch, seed_x=100, relu=True):
    import GCN
    import STMGCN
    from stmgcn_b200 import synth
    pre = GCN.Adj_Preprocessor("chebyshev", w.cheb_order)
    sups_cpu = [pre.process_sparse(a) for a in synth.make_adjacency_list(w)]
    torch.manual_seed(0)
    kw = synth.model_kwargs(w)
    if not relu:
        kw["gconv_activation"] = None
    model = STMGCN.ST_MGCN(**kw)
    params = {k: v.detach().clone().numpy() for k, v in model.state_dict().items()}
    x, y = synth.make_inputs(w, seed=seed_x, batch=batch)
    return model.to(DEV), [s.to(DEV) for s in sups_cpu], [_csr_of(s) for s in sups_cpu], params, x, y


def directed_workload(name, batch):
    """The workload's shapes on directed graphs; in each, region 0 is made a sink and region 1 a source."""
    from stmgcn_b200 import synth
    w = synth.WORKLOADS[name]
    adjs = [synth.make_directed_adjacency(w.n_regions, m, w.density) for m in range(w.n_graphs)]
    for a in adjs:
        a[0, :] = 0.0
        a[:, 1] = 0.0
    return w, adjs


def workload_case(name, batch, relu):
    """Workload ``name`` with Chebyshev supports (:func:`cheb_workload`, inputs of seed 100) -> (model, supports, chains,
    n_supports, params, x, y)."""
    from stmgcn_b200 import synth
    w = synth.WORKLOADS[name]
    model, sups, laps, params, x, y = cheb_workload(w, batch, relu=relu)
    return model, sups, [[lap] for lap in laps], w.n_supports, params, x, y


def diffusion_case(batch, relu, order=2):
    """cfg2 shapes on directed graphs with random_walk_diffusion supports: two chains per graph -> (model, supports,
    chains, n_supports, params, x, y)."""
    import GCN
    import STMGCN
    from stmgcn_b200 import synth
    w, adjs = directed_workload("cfg2", batch)
    sups_cpu = [GCN.Adj_Preprocessor("random_walk_diffusion", order).process_sparse(a) for a in adjs]
    chains = [[sp.csr_matrix(m.numpy()) for m in h.matrices_dense()] for h in sups_cpu]
    torch.manual_seed(0)
    kw = synth.model_kwargs(w)
    kw["sta_kernel_config"] = {"kernel_type": "random_walk_diffusion", "K": order}
    if not relu:
        kw["gconv_activation"] = None
    model = STMGCN.ST_MGCN(**kw)
    params = {k: v.detach().clone() for k, v in model.state_dict().items()}
    x, y = synth.make_inputs(w, seed=100, batch=batch)
    return model.to(DEV), [s.to(DEV) for s in sups_cpu], chains, 2 * order + 1, params, x, y


@pytest.fixture
def bf16_mode(monkeypatch):
    """One-plane tensor-core LSTM and bf16 gather copies: the bf16-arithmetic mode."""
    from stmgcn_b200 import ops
    monkeypatch.setattr(ops, "_PLANES", 1)
    monkeypatch.setattr(ops, "_LSTM_PATH", "tc")
    return ops


def _bits_sum(t):
    """The sum of ``t``'s bit patterns as integers, on the device (no synchronisation): a write to any element moves
    it, barring an exact cancellation."""
    bits = t.reshape(-1).view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype])
    return torch.stack([part.sum(dtype=torch.int64) for part in bits.split(1 << 26)]).sum()


class FullBatchRecorder:
    """Wraps ``ops`` for one training step and keeps, for every row, the kernels' values at the bf16 mode's rounding
    points: per shared LSTM its tape (``hp``, ``cs``, ``h0p``), per spatial GCN its Chebyshev stack ``s`` (graph order).

    These are the very tensors the step saves for its backward, held by reference in the kernels' precision, not
    copied: the tensor-core LSTM backward only reads ``hp`` and ``cs`` (``const`` at the C ABI, so a second backward
    over the same forward is allowed on that path), and ``ChebGCN.backward`` runs its adjoint Clenshaw in the
    projection's fresh ``u``, not in ``s``.  :meth:`check_intact` holds the backward to that: it compares a checksum of
    each tensor, taken as it was recorded, with one taken after the step."""

    def __init__(self):
        self.lstm, self.stacks, self.sums = [], [], []

    def _keep(self, t):
        self.sums.append((t, _bits_sum(t)))

    def __enter__(self):
        from stmgcn_b200 import ops
        self.ops = ops
        self.real = (ops._lstm16_forward, ops.build_stack)
        real_lstm, real_stack = self.real

        def lstm(xo, s_gate, h0c, c0c, n_layers, want_state, weights, planes, keep_tape):
            res = real_lstm(xo, s_gate, h0c, c0c, n_layers, want_state, weights, planes, keep_tape)
            tape = res[3]
            assert tape is not None, "record the forward with autograd on"
            rec = dict(hp=tape["hp"], cs=tape["cs"], h0p=tape["h0p"], rows=xo.shape[0] * xo.shape[1])
            for key in ("hp", "cs", "h0p"):
                if rec[key] is not None:
                    self._keep(rec[key])
            self.lstm.append(rec)
            return res

        def stack(sset, x, gather16=False):
            s = real_stack(sset, x, gather16)
            if gather16:                                # the spatial GCN (ChebGCN); the temporal one passes False
                self._keep(s)
                self.stacks.append(s)
            return s

        ops._lstm16_forward, ops.build_stack = lstm, stack
        return self

    def __exit__(self, *exc):
        self.ops._lstm16_forward, self.ops.build_stack = self.real

    def check_intact(self):
        """Every recorded tensor holds what it held when recorded."""
        for i, (t, before) in enumerate(self.sums):
            assert torch.equal(_bits_sum(t), before), f"recorded tensor {i} {tuple(t.shape)} changed after it was taken"

    def take_tapes(self):
        """Per graph the tape :class:`O.BF16ModeReference` takes, still in the kernels' precision: ``h`` the one bf16
        plane (L, T, R, 64), ``c`` fp32 unblocked (L, T, R, 64), ``h0`` (with an initial state) and ``s``.  The blocked
        cell states are released as each branch's is unblocked, so the recording can be taken once."""
        out = []
        for rec, s in zip(self.lstm, self.stacks):
            assert rec["hp"].shape[2] == 1, "the LSTM ran with two planes: not the bf16 mode"
            tape = dict(h=rec.pop("hp")[:, :, 0], c=self.ops.from_blocked(rec.pop("cs"), rec["rows"]), s=s)
            if rec["h0p"] is not None:
                tape["h0"] = rec["h0p"][:, 0]
            out.append(tape)
        self.lstm, self.stacks, self.sums = [], [], []
        return out


class Recorder:
    """Wraps ``ops`` for one forward and keeps, for the rows of the windows ``picks``, the kernels' values at the
    rounding points: per shared LSTM its tape, per spatial GCN its Chebyshev stack, per GCN its ReLU mask (GCN order
    temporal 0, spatial 0, temporal 1, ...)."""

    def __init__(self, picks):
        self.picks = list(picks)
        self.lstm, self.stacks, self.masks = [], [], []

    def __enter__(self):
        from stmgcn_b200 import ops
        self.ops = ops
        self.real = (ops._lstm16_forward, ops.build_stack, ops._proj_fwd)
        real_lstm, real_stack, real_proj = self.real

        def lstm(xo, s_gate, h0c, c0c, n_layers, want_state, weights, planes, keep_tape):
            res = real_lstm(xo, s_gate, h0c, c0c, n_layers, want_state, weights, planes, keep_tape)
            tape = res[3]
            assert tape is not None, "record the forward with autograd on"
            n, b = xo.shape[:2]
            rows = (torch.arange(n, device=xo.device)[:, None] * b
                    + torch.tensor(self.picks, device=xo.device)[None, :]).reshape(-1)
            lyr, t_len, rows_pad, _ = tape["cs"].shape
            # cs is tile-blocked [tile][unit/4][128][4] (ops.to_blocked): gather the picked rows without unblocking
            cs = tape["cs"].view(lyr, t_len, rows_pad // 128, 16, 128, 4)[:, :, rows // 128, :, rows % 128, :]
            rec = dict(hp=tape["hp"].index_select(3, rows), c=cs.permute(1, 2, 0, 3, 4).reshape(lyr, t_len, -1, 64))
            if tape["h0p"] is not None:
                rec["h0p"] = tape["h0p"].index_select(2, rows)
            self.lstm.append(rec)
            return res

        def stack(sset, x, gather16=False):
            s = real_stack(sset, x, gather16)
            if gather16:                                # the spatial GCN (ChebGCN); the temporal one passes False
                self.stacks.append(s[:, :, self.picks].clone())
            return s

        def proj(*a, **k):
            out = real_proj(*a, **k)
            self.masks.append(out[:, self.picks] > 0)
            return out

        ops._lstm16_forward, ops.build_stack, ops._proj_fwd = lstm, stack, proj
        return self

    def __exit__(self, *exc):
        self.ops._lstm16_forward, self.ops.build_stack, self.ops._proj_fwd = self.real

    def tapes(self):
        """Per graph the tape :class:`O.BF16ModeReference` takes (fp64): h (planes summed), c, h0 and s."""
        out = []
        for m, rec in enumerate(self.lstm):
            assert rec["hp"].shape[2] == 1, "the LSTM ran with two planes: not the bf16 mode"
            tape = dict(h=rec["hp"].double().sum(dim=2), c=rec["c"].double())
            if "h0p" in rec:
                tape["h0"] = rec["h0p"].double().sum(dim=1)
            if m < len(self.stacks):
                tape["s"] = self.stacks[m].double()
            out.append(tape)
        return out


def gpu_run(model, sups, x, y, picks, want_obs=False):
    """One forward (recorded) and backward of ``model`` on the full batch ``x``; the targets of the windows not picked
    are the run's own output.  Returns the picked windows' output, the loss, every parameter gradient, d obs of the
    picked windows (``want_obs``) and the recording."""
    rec = Recorder(picks)
    xd = x.to(DEV).requires_grad_(want_obs)
    with rec:
        out = model(obs_seq=xd, sta_adj_list=sups)
    y2 = out.detach().clone()
    y2[picks] = y[picks].to(DEV)
    loss = nn.MSELoss()(out, y2)
    loss.backward()
    torch.cuda.synchronize()
    return dict(out=out.detach()[picks], loss=loss.item(), rec=rec,
                grads={k: p.grad.detach().clone() for k, p in model.named_parameters()},
                d_obs=xd.grad[picks] if want_obs else None)


def forced_errors(run, params, chains, ks, x, y, picks, relu, rounding=True, want_obs=False):
    """The GPU run against :class:`O.BF16ModeReference` forced with its recording.  Returns (step-local errors: every
    layer-step of each LSTM, its h_top and every spatial S_k; whole-model errors: output, loss, every parameter gradient
    and d obs with ``want_obs``)."""
    rec = run["rec"]
    tapes = rec.tapes()
    ref = O.BF16ModeReference(params, chains, ks, relu=relu, rounding=rounding,
                              relu_masks=rec.masks if relu else None, device=DEV)
    step = {}

    def on_branch(m, br):
        tape = tapes[m]
        n = tape["s"].shape[1]
        step[f"g{m} LSTM layer-steps"] = step_local_error(tape, br["hs"], br["cs"], 1)
        step[f"g{m} h_top"] = rel_err(tape["s"][0].reshape(n, -1), br["hs"][-1][-1].reshape(n, -1))
        for k in range(1, ks):
            step[f"g{m} S_{k}"] = rel_err(tape["s"][k].reshape(n, -1), br["stack"][k])
    batch = x.shape[0]
    out, loss, grads = ref.loss_and_grads(x[picks], y[picks], tapes=tapes, want_obs=want_obs, on_branch=on_branch)
    scale = len(picks) / float(batch)
    errs = {"out": rel_err(run["out"], out), "loss": abs(run["loss"] - float(loss) * scale) / abs(float(loss) * scale)}
    for key, g in run["grads"].items():
        errs["grad " + key] = rel_err(g, grads[key] * scale)
    if want_obs:
        errs["d obs"] = rel_err(run["d_obs"], grads["obs"] * scale)
    del ref, grads
    torch.cuda.empty_cache()
    return step, errs


def small_model(m, c, kernel, relu, seed, hid=64, t=5):
    import STMGCN
    n = 19
    torch.manual_seed(seed)
    cfg = {"kernel_type": kernel, "K": 1 if kernel == "localpool" else 2}
    act = nn.ReLU if relu == "relu" else (nn.Tanh if relu == "tanh" else None)
    model = STMGCN.ST_MGCN(M=m, seq_len=t, n_nodes=n, input_dim=c, lstm_hidden_dim=hid, lstm_num_layers=2,
                           gcn_hidden_dim=24, sta_kernel_config=cfg, gconv_use_bias=True, gconv_activation=act).to(DEV)
    gen = torch.Generator().manual_seed(seed)
    adjs = [(torch.rand(n, n, generator=gen) < 0.3).float() * (0.5 + torch.rand(n, n, generator=gen)) for _ in range(m)]
    if kernel == "localpool":
        sups = []
        for a in adjs:
            a = a + torch.eye(n)
            d = a.sum(1) ** -0.5
            sups.append((d[:, None] * a * d[None, :])[None])
    else:
        sups = [O.chebyshev_supports_dense(a.double(), cfg["K"]).float() for a in adjs]
    return model, sups, n, t


def dense_grads(model, sups, x, y, act):
    params = {k: v.detach().double().cpu().requires_grad_(True) for k, v in model.state_dict().items()}
    xd = x.detach().double().cpu().requires_grad_(True)
    with _gcn_as(_tanh_gcn if act == "tanh" else O.dense_gcn):
        out = O.dense_st_mgcn(params, xd, [s.double() for s in sups], relu=act == "relu")
    loss = torch.mean((out - y.double().cpu()) ** 2)
    g = torch.autograd.grad(loss, [xd] + list(params.values()))
    return g[0], dict(zip(params, g[1:]))


class _gcn_as:
    """Run the dense oracle with another graph convolution in place of ``O.dense_gcn``."""

    def __init__(self, fn):
        self.fn, self.real = fn, O.dense_gcn

    def __enter__(self):
        O.dense_gcn = self.fn

    def __exit__(self, *exc):
        O.dense_gcn = self.real


def _tanh_gcn(supports, x, w, b, relu=True):
    return torch.tanh(_DENSE_GCN(supports, x, w, b, False))


_DENSE_GCN = O.dense_gcn
