"""Oracle: KalmanFilter.update_correlated and update_sequential (TEST INFRASTRUCTURE).

Restates ``filterpy/kalman/kalman_filter.py`` (reference @ 3b51149):

* ``KalmanFilter.update_correlated`` kalman_filter.py:670-752 (S = HPH' + HM + M'H' + R, K = (PH' + M) S^-1,
  P = P - K (HP + M'), ``np.linalg.inv`` for S)
* ``KalmanFilter.update_sequential`` kalman_filter.py:754-824 (the Joseph update of one block of rows, a
  reciprocal for a one-row block)

``*_single`` is the reference's ``np.dot`` sequence for one filter, ``*_bank`` the same arithmetic vectorised over a
leading N axis with ``np.matmul``.  The predict and the log-likelihoods are ``oracle.kf``'s.  Everything is fp64.
Parity: pinned against the reference by ``tests/golden/kf_forms_*.npz`` (``tests/golden/make_golden_kf_forms.py``).
"""
import numpy as np


def _T(a):
    return np.swapaxes(a, -1, -2)


def kf_update_correlated_single(x, P, z, H, R, M):
    """kalman_filter.py:730-748 (``z is None``: posterior := prior, y = 0, :705-710).

    Returns (x, P, y, K, S, SI)."""
    if z is None:
        return x.copy(), P.copy(), np.zeros(H.shape[0]), None, None, None
    y = z - np.dot(H, x)
    PHT = np.dot(P, H.T)
    S = np.dot(H, PHT) + np.dot(H, M) + np.dot(M.T, H.T) + R
    SI = np.linalg.inv(S)
    K = np.dot(PHT + M, SI)
    x = x + np.dot(K, y)
    P = P - np.dot(K, np.dot(H, P) + M.T)
    return x, P, y, K, S, SI


def kf_update_sequential_single(x, P, start, z_i, H, R, R_i=None, H_i=None):
    """kalman_filter.py:778-819 on the block of rows start .. start+L-1 (``R_i`` / ``H_i`` default to the
    block of R / H; a scalar ``R_i`` is R_i * I).  A reciprocal for L = 1: a zero S_i gives inf/nan.

    Returns (x, P, y_i, K_i)."""
    L = 1 if np.isscalar(z_i) else len(z_i)
    z_i = np.reshape(z_i, [L])
    stop = start + L
    if R_i is None:
        R_i = R[start:stop, start:stop]
    elif np.isscalar(R_i):
        R_i = np.eye(L) * R_i
    if H_i is None:
        H_i = H[start:stop]
    H_i = np.reshape(H_i, [L, x.shape[0]])
    y_i = z_i - np.dot(H_i, x)
    PHT = np.dot(P, H_i.T)
    S_i = np.dot(H_i, PHT) + R_i
    with np.errstate(divide="ignore", invalid="ignore"):
        K_i = PHT * (1.0 / S_i) if L == 1 else np.dot(PHT, np.linalg.inv(S_i))
        I_KH = np.eye(x.shape[0]) - np.dot(K_i, H_i)
        x = x + np.dot(K_i, y_i)
        P = np.dot(np.dot(I_KH, P), I_KH.T) + np.dot(np.dot(K_i, R_i), K_i.T)
    return x, P, y_i, K_i


def zero_pivot(S):
    """bool[N]: S[N,m,m] has an exact zero pivot in elimination with partial pivoting (the largest |entry| of the
    column at or below the diagonal), the kernels' test for a singular S.  An invertible S, however ill-conditioned or
    indefinite, has none; ``np.linalg.matrix_rank``'s SVD tolerance would call the ill-conditioned ones singular."""
    A = np.array(S, np.float64, copy=True).reshape((-1,) + np.shape(S)[-2:])
    N, m = A.shape[0], A.shape[-1]
    sing = np.zeros(N, bool)
    rows = np.arange(N)
    with np.errstate(divide="ignore", invalid="ignore"):
        for c in range(m):
            p = c + np.argmax(np.abs(A[:, c:, c]), axis=1)
            A[rows, [c] * N], A[rows, p] = A[rows, p].copy(), A[rows, [c] * N].copy()
            piv = A[:, c, c]
            sing |= ~(np.abs(piv) > 0)
            f = np.where(sing[:, None], 0.0, A[:, c + 1:, c] / np.where(sing, 1.0, piv)[:, None])
            A[:, c + 1:, :] -= f[:, :, None] * A[:, c, None, :]
    return sing


def status_after(status, failed, sticky):
    """The status word a call leaves: 1 where it failed; elsewhere 0, or the word it started with under
    BKE_STATUS_STICKY (``status`` None: 0)."""
    st = failed.astype(np.int32)
    if sticky and status is not None:
        st = np.where(failed, 1, np.asarray(status, np.int32))
    return st


def kf_update_correlated_bank(x, P, z, H, R, M, valid=None, status=None, sticky=False):
    """``kf_update_correlated_single`` for a bank: H, R, M shared or per filter.  Filters with ``valid`` = False keep
    the prior and get y = 0; those whose S is singular (``zero_pivot``; np.linalg.inv raises there) get status 1, keep
    the prior and have no y (NaN).  K, SI are NaN where S is singular.  ``status`` / ``sticky``: the starting status
    word and BKE_STATUS_STICKY (``status_after``).  Returns dict(x, P, y, K, S, SI, status)."""
    N = x.shape[0]
    y = z - np.matmul(H, x[..., None])[..., 0]
    PHT = np.matmul(P, _T(H))
    HM = np.matmul(H, M)
    S = np.broadcast_to(np.matmul(H, PHT) + HM + _T(HM) + R, (N,) + R.shape[-2:])
    v = np.ones(N, bool) if valid is None else np.asarray(valid, bool)
    zp = zero_pivot(S)
    sing = zp & v
    SI = np.full(S.shape, np.nan)
    SI[~zp] = np.linalg.inv(S[~zp])
    ok = v & ~sing
    K = np.matmul(PHT + M, SI)
    xn = x + np.matmul(K, y[..., None])[..., 0]
    Pn = P - np.matmul(K, np.matmul(H, P) + _T(M))
    xn = np.where(ok[:, None], xn, x)
    Pn = np.where(ok[:, None, None], Pn, P)
    y = np.where(ok[:, None], y, np.where(sing[:, None], np.nan, 0.0))
    return dict(x=xn, P=Pn, y=y, K=K, S=S, SI=SI, status=status_after(status, sing, sticky))


def kf_update_sequential_bank(x, P, start, z_i, H, R, y, K, z, R_i=None, H_i=None, valid=None, status=None,
                              sticky=False):
    """``kf_update_sequential_single`` for a bank: z_i[N,L]; H[.,m,n] and R[.,m,m] (shared or per filter)
    give the block unless ``R_i`` ([.,L,L] or a scalar) / ``H_i`` ([.,L,n]) are given.  ``y[N,m]``,
    ``K[N,n,m]`` and ``z[N,m]`` are the values before the call; their block is replaced where ``valid`` and S_i
    is invertible.  For L > 1 a singular S_i (``zero_pivot``; np.linalg.inv raises there) gives status 1 and the
    filter keeps its prior, y, K and z; for L = 1 the reciprocal gives inf / NaN and status 0.  ``status`` /
    ``sticky``: the starting status word and BKE_STATUS_STICKY (``status_after``).
    Returns dict(x, P, y, K, z, status)."""
    N, n = x.shape
    L = z_i.shape[1]
    stop = start + L
    R_i = R[..., start:stop, start:stop] if R_i is None else (np.eye(L) * R_i if np.isscalar(R_i) else R_i)
    H_i = H[..., start:stop, :] if H_i is None else H_i
    y_i = z_i - np.matmul(H_i, x[..., None])[..., 0]
    PHT = np.matmul(P, _T(H_i))
    S_i = np.broadcast_to(np.matmul(H_i, PHT) + R_i, (N, L, L))
    v = np.ones(N, bool) if valid is None else np.asarray(valid, bool)
    zp = zero_pivot(S_i) if L > 1 else np.zeros(N, bool)
    sing = zp & v
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if L == 1:
            K_i = PHT * (1.0 / S_i)
        else:
            K_i = np.matmul(PHT, np.linalg.inv(np.where(zp[:, None, None], np.eye(L), S_i)))
        I_KH = np.eye(n) - np.matmul(K_i, H_i)
        xn = x + np.matmul(K_i, y_i[..., None])[..., 0]
        Pn = np.matmul(np.matmul(I_KH, P), _T(I_KH)) + np.matmul(np.matmul(K_i, R_i), _T(K_i))
    ok = v & ~sing
    y, K, z = y.copy(), K.copy(), z.copy()
    y[ok, start:stop] = y_i[ok]
    K[ok, :, start:stop] = K_i[ok]
    z[ok, start:stop] = z_i[ok]
    return dict(x=np.where(ok[:, None], xn, x), P=np.where(ok[:, None, None], Pn, P), y=y, K=K, z=z,
                status=status_after(status, sing, sticky))
