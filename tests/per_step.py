"""Per-step parity metric for gradients that decay through time.

``O.max_rel_err`` divides by the maximum over the whole tensor.  The LSTM's gradients shrink going back in time, so the
early steps of ``d_s`` or ``d_xo`` weigh almost nothing in that maximum (at T = 64 the first step's share is ~1e-9): a
backward that dropped them would still pass.  ``per_step_rel_err`` holds every step to its own scale instead.
"""
import numpy as np


def per_step_rel_err(new, ref, axis):
    """For each index ``i`` along ``axis``: ``max|new[i] - ref[i]| / max|ref[i]|`` over the slice, as a float64 array.

    A slice whose reference is exactly zero is judged against ``max|ref|`` over the whole tensor (against 1 if that is
    zero too).  A slice with a NaN or Inf in ``new`` or ``ref`` gives NaN, which fails any ``not err <= bar`` check.
    ``new`` and ``ref`` may be numpy arrays or torch tensors (on any device)."""
    new, ref = _f64(new), _f64(ref)
    if new.shape != ref.shape:
        raise ValueError(f"shapes differ: {new.shape} vs {ref.shape}")
    new, ref = np.moveaxis(new, axis, 0), np.moveaxis(ref, axis, 0)
    n = new.shape[0]
    new, ref = new.reshape(n, -1), ref.reshape(n, -1)
    if new.shape[1] == 0:
        return np.zeros(n)
    finite = np.isfinite(new).all(axis=1) & np.isfinite(ref).all(axis=1)
    with np.errstate(invalid="ignore"):
        diff = np.abs(new - ref).max(axis=1)
    absref = np.abs(ref)
    den = absref.max(axis=1)
    whole = float(np.max(absref, where=np.isfinite(absref), initial=0.0))
    den = np.where(den > 0, den, whole if whole > 0 else 1.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(finite, diff / den, np.nan)


def _f64(v):
    if hasattr(v, "detach"):
        v = v.detach().double().cpu().numpy()
    return np.asarray(v, dtype=np.float64)


def worst_step(new, ref, axis):
    """(largest per-step error, the step where it occurs); NaN (and that step) if any step is not finite."""
    errs = per_step_rel_err(new, ref, axis)
    i = int(np.argmax(np.where(np.isnan(errs), np.inf, errs)))
    return float(errs[i]), i
