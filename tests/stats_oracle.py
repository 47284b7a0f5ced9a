"""fp64 NumPy restatement of bke_score_measurements (csrc/score.cu) with the kernel's rule: S^-1 and log|det S| from
a partially pivoted Gauss-Jordan elimination that fails on an exactly zero pivot (reg_inverse / warp_inverse),
d2 = y' S^-1 y, ll = -0.5 (d2 + log|det S| + m log 2pi), and a missing candidate scored as "z is None"."""
import math
import sys

import numpy as np

LOG_DBL_MIN = math.log(sys.float_info.min)


def inverse(S):
    """(S^-1, log|det S|, ok): Gauss-Jordan with partial pivoting; ok is False on an exactly zero pivot."""
    A = np.array(S, dtype=np.float64)
    m = A.shape[0]
    X = np.eye(m)
    ld = 0.0
    for c in range(m):
        p = c + int(np.argmax(np.abs(A[c:, c])))
        if A[p, c] == 0:
            return None, None, False
        A[[c, p]], X[[c, p]] = A[[p, c]], X[[p, c]]
        piv = A[c, c]
        ld += math.log(abs(piv))
        A[c] /= piv
        X[c] /= piv
        for r in range(m):
            if r != c:
                f = A[r, c]
                A[r] -= f * A[c]
                X[r] -= f * X[c]
    return X, ld, True


def score(z, zhat, S, valid=None):
    """z[N, K, m], zhat[N, m], S[N, m, m], valid[N, K] -> dict y, d2, mahalanobis, log_likelihood, likelihood
    ([N, K]) and status[N].  A singular S gives NaN scores; a missing candidate y = d2 = 0, ll = log(DBL_MIN)."""
    z = np.asarray(z, np.float64)
    N, K, m = z.shape
    y = z - np.asarray(zhat, np.float64)[:, None, :]
    d2, ll = np.zeros((N, K)), np.zeros((N, K))
    status = np.zeros(N, np.int32)
    for f in range(N):
        SI, ld, ok = inverse(S[f])
        if not ok:
            status[f] = 1
            d2[f], ll[f] = np.nan, np.nan
            continue
        d2[f] = np.einsum("ka,ab,kb->k", y[f], SI, y[f])
        ll[f] = -0.5 * (d2[f] + ld + m * math.log(2 * math.pi))
    if valid is not None:
        v = np.asarray(valid, bool)
        y[~v] = 0.0
        d2[~v], ll[~v] = 0.0, LOG_DBL_MIN
    with np.errstate(invalid="ignore"):
        return dict(y=y, d2=d2, mahalanobis=np.sqrt(d2), log_likelihood=ll, likelihood=np.exp(ll), status=status)


def innovation_cov(P, H, R):
    """S = H P H' + R per track (H, R [m, .] shared or [N, m, .])."""
    return np.einsum("...an,...nk,...bk->...ab", H, P, H) + R


def inverse_bank(S):
    """inverse() over a bank S[N, m, m], vectorised: (S^-1 [N, m, m], log|det S| [N], ok [N]); a track with an exactly
    zero pivot has ok False (and meaningless S^-1, log|det S|)."""
    A = np.array(S, dtype=np.float64)
    N, m, _ = A.shape
    X = np.broadcast_to(np.eye(m), A.shape).copy()
    ld, ok, ar = np.zeros(N), np.ones(N, bool), np.arange(N)
    for c in range(m):
        p = c + np.argmax(np.abs(A[:, c:, c]), axis=1)
        for M in (A, X):
            rc, rp = M[ar, c].copy(), M[ar, p].copy()
            M[ar, c], M[ar, p] = rp, rc
        piv = A[:, c, c]
        ok &= piv != 0
        piv = np.where(ok, piv, 1.0)
        ld += np.log(np.abs(piv))
        A[:, c] /= piv[:, None]
        X[:, c] /= piv[:, None]
        f = A[:, :, c].copy()
        f[:, c] = 0.0
        A -= f[:, :, None] * A[:, c][:, None, :]
        X -= f[:, :, None] * X[:, c][:, None, :]
    return X, ld, ok


def score_bank(z, zhat, S, valid=None):
    """score() with inverse_bank: the same outputs, vectorised over the tracks."""
    z = np.asarray(z, np.float64)
    N, K, m = z.shape
    y = z - np.asarray(zhat, np.float64)[:, None, :]
    SI, ld, ok = inverse_bank(S)
    with np.errstate(invalid="ignore", over="ignore"):
        d2 = np.einsum("nka,nab,nkb->nk", y, SI, y)
        ll = -0.5 * (d2 + ld[:, None] + m * math.log(2 * math.pi))
        d2[~ok], ll[~ok] = np.nan, np.nan
        if valid is not None:
            v = np.asarray(valid, bool)
            y[~v] = 0.0
            d2[~v], ll[~v] = 0.0, LOG_DBL_MIN
        return dict(y=y, d2=d2, mahalanobis=np.sqrt(d2), log_likelihood=ll, likelihood=np.exp(ll),
                    status=(~ok).astype(np.int32), SI=SI, logdet=ld)
