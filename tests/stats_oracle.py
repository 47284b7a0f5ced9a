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
