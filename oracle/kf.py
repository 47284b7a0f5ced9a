"""Oracle: linear Kalman filter predict / update / batch_filter (TEST INFRASTRUCTURE).

Restates ``filterpy/kalman/kalman_filter.py`` (reference @ 3b51149):

* ``KalmanFilter.predict``  kalman_filter.py:437-482  (x = Fx [+ Bu], P = a^2 F P F' + Q)
* ``KalmanFilter.update``   kalman_filter.py:485-561  (Joseph-form covariance update,
  ``np.linalg.inv`` for S)
* ``KalmanFilter.batch_filter`` kalman_filter.py:826-993
* ``KalmanFilter.rts_smoother`` kalman_filter.py:995-1074 and procedural ``rts_smoother`` :1792-1858

Two flavours are provided:

``*_single``  one filter, the same ``np.dot`` call sequence as the reference
              (used for small cases and as the "filterpy-shaped" CPU baseline);
``*_bank``    the same arithmetic vectorised over a leading N axis with
              ``np.matmul`` (used for full-size banks).

Everything is fp64, as in the reference (``np.eye`` / ``np.zeros`` defaults,
kalman_filter.py:399-419).  Parity: pinned against the reference by
``tests/golden/kf_*.npz`` (see ``tests/golden/make_golden.py``).
"""
import numpy as np


# --------------------------------------------------------------------------- single filter
def kf_predict_single(x, P, F, Q, alpha_sq=1.0, B=None, u=None):
    """kalman_filter.py:471-478."""
    if B is not None and u is not None:
        x = np.dot(F, x) + np.dot(B, u)
    else:
        x = np.dot(F, x)
    P = alpha_sq * np.dot(np.dot(F, P), F.T) + Q
    return x, P


def kf_update_single(x, P, z, H, R):
    """kalman_filter.py:515-561.  ``z is None`` -> posterior := prior (515-520).

    Returns (x, P, y, K, S, SI)."""
    m = H.shape[0]
    if z is None:
        return x.copy(), P.copy(), np.zeros(m), None, None, None
    y = z - np.dot(H, x)
    PHT = np.dot(P, H.T)
    S = np.dot(H, PHT) + R
    SI = np.linalg.inv(S)
    K = np.dot(PHT, SI)
    x = x + np.dot(K, y)
    I_KH = np.eye(P.shape[0]) - np.dot(K, H)
    P = np.dot(np.dot(I_KH, P), I_KH.T) + np.dot(np.dot(K, R), K.T)
    return x, P, y, K, S, SI


def kf_batch_filter_single(x, P, zs, F, Q, H, R, alpha_sq=1.0, update_first=False):
    """kalman_filter.py:955-993 for one filter with constant models.

    ``zs`` is a length-T sequence whose entries are (m,) arrays or None."""
    T = len(zs)
    n = x.shape[0]
    means = np.zeros((T, n)); means_p = np.zeros((T, n))
    covs = np.zeros((T, n, n)); covs_p = np.zeros((T, n, n))
    for i, z in enumerate(zs):
        if update_first:
            x, P = kf_update_single(x, P, z, H, R)[:2]
            means[i], covs[i] = x, P
            x, P = kf_predict_single(x, P, F, Q, alpha_sq)
            means_p[i], covs_p[i] = x, P
        else:
            x, P = kf_predict_single(x, P, F, Q, alpha_sq)
            means_p[i], covs_p[i] = x, P
            x, P = kf_update_single(x, P, z, H, R)[:2]
            means[i], covs[i] = x, P
    return means, covs, means_p, covs_p


# --------------------------------------------------------------------------- bank (vectorised over N)
def _T(a):
    return np.swapaxes(a, -1, -2)


def kf_predict_bank(x, P, F, Q, alpha_sq=1.0, B=None, u=None):
    """Same arithmetic as ``kf_predict_single`` for x[N,n], P[N,n,n]; F/Q may be
    [N,n,n] or [n,n] (shared)."""
    xn = np.matmul(F, x[..., None])[..., 0]
    if B is not None and u is not None:
        xn = xn + np.matmul(B, u[..., None])[..., 0]
    Pn = alpha_sq * np.matmul(np.matmul(F, P), _T(F)) + Q
    return xn, Pn


def kf_update_bank(x, P, z, H, R, valid=None):
    """Same arithmetic as ``kf_update_single`` for a bank.  ``valid`` (bool[N]) marks
    filters that have a measurement; the others keep the prior (kalman_filter.py:515-520).

    Returns dict(x, P, y, K, S, SI)."""
    N, n = x.shape
    y = z - np.matmul(H, x[..., None])[..., 0]
    PHT = np.matmul(P, _T(H))
    S = np.matmul(H, PHT) + R
    SI = np.linalg.inv(S)
    K = np.matmul(PHT, SI)
    xn = x + np.matmul(K, y[..., None])[..., 0]
    I_KH = np.eye(n) - np.matmul(K, H)
    Rb = R
    Pn = np.matmul(np.matmul(I_KH, P), _T(I_KH)) + np.matmul(np.matmul(K, Rb), _T(K))
    if valid is not None:
        v = np.asarray(valid, bool)
        xn = np.where(v[:, None], xn, x)
        Pn = np.where(v[:, None, None], Pn, P)
        y = np.where(v[:, None], y, 0.0)
    return dict(x=xn, P=Pn, y=y, K=K, S=S, SI=SI)


def kf_step_bank(x, P, z, F, H, Q, R, alpha_sq=1.0, valid=None, B=None, u=None, update_first=False):
    """predict + update for a bank; returns dict with priors as well.  ``B`` [N,n,k] or [n,k] and ``u``
    [N,k] add the control input to the predict; ``update_first`` runs the update on (x, P) and then the
    predict on the posterior (batch_filter's update_first order, kalman_filter.py:963-973), and the
    returned x / P / x_prior / P_prior are that predict's."""
    if update_first:
        out = kf_update_bank(x, P, z, H, R, valid)
        out["x"], out["P"] = kf_predict_bank(out["x"], out["P"], F, Q, alpha_sq, B, u)
        out["x_prior"], out["P_prior"] = out["x"], out["P"]
        return out
    xp, Pp = kf_predict_bank(x, P, F, Q, alpha_sq, B, u)
    out = kf_update_bank(xp, Pp, z, H, R, valid)
    out["x_prior"], out["P_prior"] = xp, Pp
    return out


def kf_batch_filter_bank(x, P, zs, F, H, Q, R, alpha_sq=1.0, valid=None, update_first=False):
    """Bank version of batch_filter: zs[T,N,m] (valid[T,N] optional) ->
    means[T,N,n], covs[T,N,n,n], means_p, covs_p."""
    T = zs.shape[0]
    N, n = x.shape
    means = np.zeros((T, N, n)); means_p = np.zeros((T, N, n))
    covs = np.zeros((T, N, n, n)); covs_p = np.zeros((T, N, n, n))
    for t in range(T):
        v = None if valid is None else valid[t]
        if update_first:
            o = kf_update_bank(x, P, zs[t], H, R, v)
            x, P = o["x"], o["P"]
            means[t], covs[t] = x, P
            x, P = kf_predict_bank(x, P, F, Q, alpha_sq)
            means_p[t], covs_p[t] = x, P
        else:
            x, P = kf_predict_bank(x, P, F, Q, alpha_sq)
            means_p[t], covs_p[t] = x, P
            o = kf_update_bank(x, P, zs[t], H, R, v)
            x, P = o["x"], o["P"]
            means[t], covs[t] = x, P
    return means, covs, means_p, covs_p


def log_likelihood_bank(y, S):
    """log N(y; 0, S) per filter — what ``KalmanFilter.log_likelihood`` evaluates
    (kalman_filter.py:1203-1210 -> stats.py:131-154, scipy multivariate_normal.logpdf)."""
    m = y.shape[-1]
    SI = np.linalg.inv(S)
    q = np.einsum("ni,nij,nj->n", y, SI, y)
    _, logdet = np.linalg.slogdet(S)
    return -0.5 * (q + logdet + m * np.log(2.0 * np.pi))


def missed_log_likelihood_bank(S):
    """log N(0; 0, S) per filter: ``KalmanFilter.log_likelihood`` after ``update(None)``, which keeps the
    last S and sets y = 0 (kalman_filter.py:511-520).  -inf where det S <= 0 (the S = 0 of a filter that
    has never had a measurement: scipy's logpdf with allow_singular gives -inf there)."""
    S = np.asarray(S, float)
    sign, logdet = np.linalg.slogdet(S)
    with np.errstate(invalid="ignore"):
        ll = -0.5 * (logdet + S.shape[-1] * np.log(2.0 * np.pi))
    return np.where(sign > 0, ll, -np.inf)


def rts_smoother(Xs, Ps, Fs, Qs, shift=1):
    """kalman_filter.py:1056-1074 (method, step k uses Fs[k+1]: shift=1) and :1840-1858 (procedural,
    Fs[k]: shift=0), literal; Xs (T,n) or (T,n,1), Ps (T,n,n), Fs/Qs lists of length T."""
    if len(Xs) != len(Ps):
        raise ValueError('length of Xs and Ps must be the same')
    n = Xs.shape[0]
    dim_x = Xs.shape[1]
    K = np.zeros((n, dim_x, dim_x))
    x, P, Pp = Xs.copy(), Ps.copy(), Ps.copy()
    for k in range(n - 2, -1, -1):
        F, Q = Fs[k + shift], Qs[k + shift]
        Pp[k] = np.dot(np.dot(F, P[k]), F.T) + Q
        K[k] = np.dot(np.dot(P[k], F.T), np.linalg.inv(Pp[k]))
        x[k] += np.dot(K[k], x[k + 1] - np.dot(F, x[k]))
        P[k] += np.dot(np.dot(K[k], P[k + 1] - Pp[k]), K[k].T)
    return x, P, K, Pp


def rts_smoother_bank(Xs, Ps, F, Q, shift=1):
    """The same for a bank: Xs (T,N,n), Ps (T,N,n,n), F/Q (n,n) shared, (N,n,n) per filter or
    (T,N,n,n) per epoch and filter; (T,n,n) is NOT accepted here (pass lists through rts_smoother
    per filter)."""
    T, N, n = Xs.shape
    outs = [np.empty_like(Xs), np.empty_like(Ps), np.empty_like(Ps), np.empty_like(Ps)]

    def models(A, i):
        if np.ndim(A) == 4:
            return [A[k, i] for k in range(T)]
        return [A[i] if np.ndim(A) == 3 else A] * T
    for i in range(N):
        r = rts_smoother(Xs[:, i], Ps[:, i], models(F, i), models(Q, i), shift)
        for o, v in zip(outs, r):
            o[:, i] = v
    return tuple(outs)
