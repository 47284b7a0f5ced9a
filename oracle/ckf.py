"""Oracle: cubature Kalman filter (TEST INFRASTRUCTURE).

Restates filterpy/kalman/CubatureKalmanFilter.py (reference @ 3b51149) twice:

* ``ckf_predict_single`` / ``ckf_update_single``: one filter, in the reference's literal call sequence —
  ``spherical_radial_sigmas`` :52-61 (U = cholesky(P) * sqrt(n), upper), ``predict`` :317-327,
  ``update`` :362-379, and ``ckf_transform`` :87-98 with its RAW second moments
  (sum outer(X_k, X_k) - outer(x, x)) / m, ``outer_product_sum`` for Pxz.  Python ``fx(x, dt, *args)`` /
  ``hx(x, *args)`` callables.
* ``ckf_step_bank``: vectorised over N for the closed set of device-side models (the ids of
  ``oracle.ukf``), with the CENTRED sums the CUDA kernel uses.

Parity: pinned by ``tests/golden/ckf_*.npz``.
"""
import numpy as np
import scipy.linalg

from .ukf import FX_LINEAR, FX_CONST_VEL, HX_LINEAR, HX_RANGE_AZ_EL, HX_RANGE_BEARING  # noqa: F401
from .ukf import _chol_upper, fx_apply, hx_apply


# --------------------------------------------------------------------------- single filter, callables
def spherical_radial_sigmas(x, P):
    """CubatureKalmanFilter.py:52-61 -> (2n, n)."""
    n = P.shape[0]
    x = np.asarray(x, float).flatten()
    U = scipy.linalg.cholesky(P) * np.sqrt(n)         # scipy's LAPACK factor: the raw moments amplify its rounding
    return np.concatenate([x + U, x - U], axis=0)


def ckf_transform(Xs, Q):
    """CubatureKalmanFilter.py:87-98: raw second moments; x comes back as a column (n, 1)."""
    m, n = Xs.shape
    x = sum(Xs, 0)[:, None] / m
    P = np.zeros((n, n))
    xf = x.flatten()
    for k in range(m):
        P += np.outer(Xs[k], Xs[k]) - np.outer(xf, xf)
    P *= 1 / m
    P += Q
    return x, P


def ckf_predict_single(x, P, Q, fx, dt, fx_args=()):
    """CubatureKalmanFilter.py:311-327 -> (x_prior (n,1), P_prior, sigmas_f)."""
    if not isinstance(fx_args, tuple):
        fx_args = (fx_args,)
    sigmas = spherical_radial_sigmas(x, P)
    sigmas_f = np.array([fx(s, dt, *fx_args) for s in sigmas])
    xp, Pp = ckf_transform(sigmas_f, Q)
    return xp, Pp, sigmas_f


def ckf_update_single(x, P, sigmas_f, z, R, hx, hx_args=()):
    """CubatureKalmanFilter.py:348-379 -> (x, P, y, K, S, SI); x and z are columns as in the reference."""
    if z is None:
        return x.copy(), P.copy(), None, None, None, None
    if not isinstance(hx_args, tuple):
        hx_args = (hx_args,)
    dim_z = np.size(z)
    if np.isscalar(R):
        R = np.eye(dim_z) * R
    m = sigmas_f.shape[0]
    sigmas_h = np.atleast_2d([hx(s, *hx_args) for s in sigmas_f])
    zp, S = ckf_transform(sigmas_h, R)
    SI = np.linalg.inv(S)
    xf = np.asarray(x).flatten()
    dx, dz = sigmas_f - xf, sigmas_h - zp.flatten()
    Pxz = np.einsum('ij,ik->ijk', dx, dz).sum(axis=0) / m        # outer_product_sum (common/helpers.py:433-438)
    K = np.dot(Pxz, SI)
    y = z - zp
    x = x + np.dot(K, y)
    P = P - np.dot(K, S).dot(K.T)
    return x, P, y, K, S, SI


# --------------------------------------------------------------------------- bank, closed set of models
def _centred(X):
    """mean and centred covariance of points X[..., m, d] (the kernel's form)."""
    mean = X.sum(axis=-2) / X.shape[-2]
    D = X - mean[..., None, :]
    return mean, np.einsum("...ka,...kb->...ab", D, D) * (1.0 / X.shape[-2]), D


def ckf_step_bank(x, P, z, Q, R, dt, fx_model=FX_LINEAR, hx_model=HX_LINEAR, F=None, H=None, valid=None,
                  sigmas_f=None, predict=True):
    """One predict + update (or, ``predict=False``, an update from the given ``sigmas_f[N, 2n, n]``) for a bank
    x[N,n], P[N,n,n], z[N,m]; Q/R [n,n]/[m,m] or per filter.

    Returns dict(x, P, x_prior, P_prior, y, K, S, SI, sigmas_f)."""
    n = x.shape[-1]
    if predict:
        U = _chol_upper(P) * np.sqrt(n)
        sig = np.concatenate([x[:, None, :] + U, x[:, None, :] - U], axis=-2)
        sigmas_f = fx_apply(fx_model, sig, dt, F)
        xp, Pc, _ = _centred(sigmas_f)
        Pp = Pc + Q
    else:
        xp, Pp = x, P
    sig_h = hx_apply(hx_model, sigmas_f, H)
    zp, Sc, Dz = _centred(sig_h)
    S = Sc + R
    SI = np.linalg.inv(S)
    Dx = sigmas_f - xp[:, None, :]
    Pxz = np.einsum("nka,nkb->nab", Dx, Dz) / sigmas_f.shape[-2]
    K = Pxz @ SI
    y = z - zp
    xn = xp + (K @ y[..., None])[..., 0]
    Pn = Pp - (K @ S) @ np.swapaxes(K, -1, -2)
    if valid is not None:
        v = np.asarray(valid, bool)
        xn = np.where(v[:, None], xn, xp)
        Pn = np.where(v[:, None, None], Pn, Pp)
    return dict(x=xn, P=Pn, x_prior=xp, P_prior=Pp, y=y, K=K, S=S, SI=SI, sigmas_f=sigmas_f)
