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


def kf_update_correlated_bank(x, P, z, H, R, M, valid=None):
    """``kf_update_correlated_single`` for a bank: H, R, M shared or per filter.  Filters with
    ``valid`` = False keep the prior and get y = 0; so do those whose S is singular (``status`` 1, where
    ``np.linalg.inv`` raises LinAlgError).  Returns dict(x, P, y, K, S, SI, status)."""
    N = x.shape[0]
    y = z - np.matmul(H, x[..., None])[..., 0]
    PHT = np.matmul(P, _T(H))
    HM = np.matmul(H, M)
    S = np.broadcast_to(np.matmul(H, PHT) + HM + _T(HM) + R, (N,) + R.shape[-2:])
    sing = np.linalg.matrix_rank(S) < S.shape[-1]
    SI = np.full(S.shape, np.nan)
    SI[~sing] = np.linalg.inv(S[~sing])
    valid = ~sing if valid is None else np.asarray(valid, bool) & ~sing
    K = np.matmul(PHT + M, SI)
    xn = x + np.matmul(K, y[..., None])[..., 0]
    Pn = P - np.matmul(K, np.matmul(H, P) + _T(M))
    v = valid | sing
    xn = np.where(valid[:, None], xn, x)
    Pn = np.where(valid[:, None, None], Pn, P)
    y = np.where(v[:, None], y, 0.0)
    return dict(x=xn, P=Pn, y=y, K=K, S=S, SI=SI, status=sing.astype(int))


def kf_update_sequential_bank(x, P, start, z_i, H, R, y, K, z, R_i=None, H_i=None, valid=None):
    """``kf_update_sequential_single`` for a bank: z_i[N,L]; H[.,m,n] and R[.,m,m] (shared or per filter)
    give the block unless ``R_i`` ([.,L,L] or a scalar) / ``H_i`` ([.,L,n]) are given.  ``y[N,m]``,
    ``K[N,n,m]`` and ``z[N,m]`` are the values before the call; their block is replaced where ``valid``.
    Returns dict(x, P, y, K, z)."""
    N, n = x.shape
    L = z_i.shape[1]
    stop = start + L
    R_i = R[..., start:stop, start:stop] if R_i is None else (np.eye(L) * R_i if np.isscalar(R_i) else R_i)
    H_i = H[..., start:stop, :] if H_i is None else H_i
    y_i = z_i - np.matmul(H_i, x[..., None])[..., 0]
    PHT = np.matmul(P, _T(H_i))
    S_i = np.matmul(H_i, PHT) + R_i
    with np.errstate(divide="ignore", invalid="ignore"):
        K_i = PHT * (1.0 / S_i) if L == 1 else np.matmul(PHT, np.linalg.inv(S_i))
        I_KH = np.eye(n) - np.matmul(K_i, H_i)
        xn = x + np.matmul(K_i, y_i[..., None])[..., 0]
        Pn = np.matmul(np.matmul(I_KH, P), _T(I_KH)) + np.matmul(np.matmul(K_i, R_i), _T(K_i))
    v = np.ones(N, bool) if valid is None else np.asarray(valid, bool)
    y, K, z = y.copy(), K.copy(), z.copy()
    y[v, start:stop] = y_i[v]
    K[v, :, start:stop] = K_i[v]
    z[v, start:stop] = z_i[v]
    return dict(x=np.where(v[:, None], xn, x), P=np.where(v[:, None, None], Pn, P), y=y, K=K, z=z)
