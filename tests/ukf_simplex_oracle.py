"""Oracle: the UKF on ``SimplexSigmaPoints`` (TEST INFRASTRUCTURE), on top of ``oracle.ukf``.

Restates (reference @ 3b51149):

* ``SimplexSigmaPoints.sigma_points``  sigma_points.py:454-513  (x + (U' sqrt(n) Istar)', U the upper Cholesky
  factor of the UNSCALED P), ``_compute_weights`` :516-522  (Wm = Wc = 1/(n+1), one array);
* ``UnscentedKalmanFilter.predict / update``  UKF.py:393-411, 442-486, and one predict + update for a bank of
  the closed set of device-side models, with these points in place of Merwe's;
* ``rts_smoother``  UKF.py:696-739 with these points (:711).

``simplex_offsets_closed_form`` is the closed form the kernels use for the offsets, checked against the
``Istar`` product.  Parity: pinned by ``tests/golden/ukf_simplex_*.npz``.
"""
import numpy as np

from oracle import ukf as oukf


def simplex_weights(n):
    """sigma_points.py:516-522 (Wc is the same array as Wm)."""
    Wm = np.full(n + 1, 1. / (n + 1))
    return Wm, Wm


def simplex_sigma_points(x, P):
    """sigma_points.py:454-513; x[..., n], P[..., n, n] -> sigmas[..., n+1, n] (Xi_0 .. Xi_n)."""
    n = x.shape[-1]
    U = oukf._chol_upper(P)                                                  # :499
    lambda_ = n / (n + 1)                                                    # :501
    Istar = np.array([[-1 / np.sqrt(2 * lambda_), 1 / np.sqrt(2 * lambda_)]])   # :502
    for d in range(2, n + 1):                                                # :504-507
        row = np.ones((1, Istar.shape[1] + 1)) * 1. / np.sqrt(lambda_ * d * (d + 1))
        row[0, -1] = -d / np.sqrt(lambda_ * d * (d + 1))
        Istar = np.r_[np.c_[Istar, np.zeros((Istar.shape[0]))], row]
    I = np.sqrt(n) * Istar                                                   # :509
    scaled_unitary = np.swapaxes(U, -1, -2) @ I                             # :510
    return x[..., None, :] + np.swapaxes(scaled_unitary, -1, -2)            # :512-513


def simplex_offsets_closed_form(P):
    """The closed form the kernels use for the offsets D = sigmas - x of simplex_sigma_points: with
    c_d = sqrt((n+1) / (d (d+1))) and S_j = sum_{k >= j} c_{k+1} U[k]:
    D_0 = -c_1 U[0] + S_1, D_1 = c_1 U[0] + S_1, D_j = -j c_j U[j-1] + S_j (j >= 2)."""
    U = oukf._chol_upper(P)
    n = U.shape[-1]
    c = [None] + [np.sqrt((n + 1) / (d * (d + 1))) for d in range(1, n + 1)]
    D = np.empty(U.shape[:-2] + (n + 1, n))
    S = np.zeros(U.shape[:-2] + (n,))
    for j in range(n, 1, -1):
        D[..., j, :] = -j * c[j] * U[..., j - 1, :] + S
        S = S + c[j] * U[..., j - 1, :]
    D[..., 0, :] = S - c[1] * U[..., 0, :]
    D[..., 1, :] = S + c[1] * U[..., 0, :]
    return D


def ukf_predict_single(x, P, Q, fx, dt):
    """UKF.py:393-411 -> (x_prior, P_prior, sigmas_f regenerated from the prior)."""
    Wm, Wc = simplex_weights(x.shape[0])
    sig_f = np.array([fx(s, dt) for s in simplex_sigma_points(x, P)])
    x, P = oukf.unscented_transform(sig_f, Wm, Wc, Q)
    return x, P, simplex_sigma_points(x, P)


def ukf_update_single(x, P, sig_f, z, R, hx):
    """UKF.py:442-486 -> (x, P, y, K, S, SI)."""
    if z is None:
        return x.copy(), P.copy(), None, None, None, None
    Wm, Wc = simplex_weights(x.shape[0])
    sig_h = np.atleast_2d([hx(s) for s in sig_f])
    zp, S = oukf.unscented_transform(sig_h, Wm, Wc, R)
    SI = np.linalg.inv(S)
    K = np.einsum("s,sa,sb->ab", Wc, sig_f - x, sig_h - zp) @ SI
    y = z - zp
    return x + K @ y, P - K @ (S @ K.T), y, K, S, SI


def ukf_step_bank(x, P, z, Q, R, dt, fx_model, hx_model, F=None, H=None, valid=None):
    """One predict + update for a bank x[N,n], P[N,n,n], z[N,m] on the simplex points; Q / R [n,n] / [m,m] or per
    filter.  Returns dict(x, P, x_prior, P_prior, y, K, S, SI)."""
    Wm, Wc = simplex_weights(x.shape[-1])
    sig_f = oukf.fx_apply(fx_model, simplex_sigma_points(x, P), dt, F)
    xp, Pp = oukf.unscented_transform(sig_f, Wm, Wc, Q)
    sig_f = simplex_sigma_points(xp, Pp)
    sig_h = oukf.hx_apply(hx_model, sig_f, H)
    zp, S = oukf.unscented_transform(sig_h, Wm, Wc, R)
    SI = np.linalg.inv(S)
    K = np.einsum("s,nsa,nsb->nab", Wc, sig_f - xp[:, None, :], sig_h - zp[:, None, :]) @ SI
    y = z - zp
    xn = xp + (K @ y[..., None])[..., 0]
    Pn = Pp - K @ (S @ np.swapaxes(K, -1, -2))
    if valid is not None:
        v = np.asarray(valid, bool)
        xn = np.where(v[:, None], xn, xp)
        Pn = np.where(v[:, None, None], Pn, Pp)
    return dict(x=xn, P=Pn, x_prior=xp, P_prior=Pp, y=y, K=K, S=S, SI=SI)


def ukf_rts_smoother(Xs, Ps, Q, fx, dts):
    """UnscentedKalmanFilter.rts_smoother, UKF.py:696-739, on the simplex points for ONE filter: Xs (T,n), Ps (T,n,n),
    Q the filter's own Q (:715), fx a callable, dts a list of T time steps -> (xs, Ps, Ks)."""
    T, n = Xs.shape
    Wm, Wc = simplex_weights(n)
    Ks = np.zeros((T, n, n))
    xs, ps = Xs.copy(), Ps.copy()
    for k in reversed(range(T - 1)):
        sigmas = simplex_sigma_points(xs[k], ps[k])                            # :711
        sigmas_f = np.array([fx(s, dts[k]) for s in sigmas])                  # :712-713
        xb, Pb = oukf.unscented_transform(sigmas_f, Wm, Wc, Q)                # :715-717
        Pxb = 0
        for i in range(sigmas.shape[0]):                                      # :720-724
            Pxb = Pxb + Wc[i] * np.outer(sigmas[i] - Xs[k], sigmas_f[i] - xb)
        K = Pxb @ np.linalg.inv(Pb)                                           # :727
        xs[k] += K @ (xs[k + 1] - xb)                                         # :730
        ps[k] += (K @ (ps[k + 1] - Pb)) @ K.T                                 # :731
        Ks[k] = K
    return xs, ps, Ks
