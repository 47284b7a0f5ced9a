"""NumPy restatement of filterpy/discrete_bayes/discrete_bayes.py (TEST INFRASTRUCTURE, see oracle/__init__.py),
with every sum written out in the reference's order, for banks of pdfs (one histogram filter per row).

predict      scipy.ndimage.convolve(np.roll(pdf, offset), kernel, mode='wrap') (:124-125), or for any other mode
             convolve(shift(pdf, offset, cval=cval), kernel, mode='constant', cval=cval) (:127-128) with the
             shift taken exact (the reference's order-3 spline equals it up to roundoff for an integer offset).
             scipy correlates with the reversed kernel kr = kernel[::-1] over a window that starts
             c = (K - 1) // 2 bins left of the output bin; that origin rule moves an even kernel's window by
             one against a naive centring, and tests/test_oracle_discrete_bayes.py pins it against the
             reference's output.  The terms are summed in fp64 in window order from 0.0, and a weight with
             |w| <= DBL_EPSILON (NaN included) is left out of the footprint as scipy leaves it out.  The result
             is rounded once to the pdf's dtype.  In constant mode the bins shifted in hold cval rounded to the
             dtype (shift's output array), the bins beyond the row hold cval itself (convolve's extension).
update       prior * likelihood in the arrays' dtype (:88), then normalize.
normalize    p / sum(np.asarray(p, dtype=float)) (:47): the builtin sum, the sequential chain 0 + p0 + p1 + ...
             in fp64, and an fp64 division rounded once to the dtype.
"""
import numpy as np

_EPS = np.finfo(np.float64).eps


def row_sum(p):
    """sum(np.asarray(p, dtype=float)): 0.0 + p0 + p1 + ..., one fp64 add at a time."""
    s = 0.0
    for v in np.asarray(p, dtype=np.float64).tolist():
        s = s + v
    return np.float64(s)


def normalize_row(p):
    p = np.asarray(p)
    s = row_sum(p)
    with np.errstate(divide="ignore", invalid="ignore"):
        return (p.astype(np.float64) / s).astype(p.dtype)


def update_row(likelihood, prior):
    return normalize_row(np.asarray(prior) * np.asarray(likelihood))


def predict_row(pdf, offset, kernel, mode="wrap", cval=0.):
    """The reference's predict for one integer offset, vectorised over the bins and sequential over the window."""
    pdf = np.asarray(pdf)
    dt = pdf.dtype
    M = pdf.shape[0]
    kr = np.asarray(kernel, dtype=np.float64)[::-1]
    K = kr.shape[0]
    c = (K - 1) // 2
    off = int(offset)
    x = pdf.astype(np.float64)
    i = np.arange(M)
    acc = np.zeros(M)
    for j in range(K):
        w = kr[j]
        if not abs(w) > _EPS:
            continue
        q = i + j - c
        if mode == "wrap":
            v = x[(q - off) % M]
        else:
            s = q - off
            inside = (s >= 0) & (s < M)
            v = np.where(inside, x[np.clip(s, 0, M - 1)], np.float64(dt.type(cval)))
            v = np.where((q >= 0) & (q < M), v, np.float64(cval))
        acc = acc + v * w
    return acc.astype(dt)


def _rows(a, B):
    a = np.asarray(a)
    return [a] * B if a.ndim <= 1 else list(a)


def step_bank(pdf, kernel=None, offset=0, likelihood=None, mode="wrap", cval=0., normalize=False):
    """What bke_db_step computes for pdf[B, M]: per row predict (kernel given), update (likelihood given) and
    normalize.  -> (out [B, M], sums [B] or None)."""
    pdf = np.asarray(pdf)
    B = pdf.shape[0]
    offs = [offset] * B if np.ndim(offset) == 0 else list(np.asarray(offset))
    ks = _rows(kernel, B) if kernel is not None else None
    out = np.empty_like(pdf)
    sums = np.zeros(B) if normalize else None
    for b in range(B):
        p = predict_row(pdf[b], offs[b], ks[b], mode, cval) if ks is not None else pdf[b].copy()
        if likelihood is not None:
            p = p * np.asarray(likelihood)[b]
        if normalize:
            sums[b] = row_sum(p)
            p = normalize_row(p)
        out[b] = p
    return out, sums
