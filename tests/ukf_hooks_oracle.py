"""Oracle: the UKF and CKF with the reference's mean / residual / state-add hooks (TEST INFRASTRUCTURE).

Restates (reference @ 3b51149), on top of ``oracle.ukf`` / ``oracle.ckf``:

* ``ukf_step_single``: one filter in the reference's literal order, with Python hook callables —
  ``predict`` UKF.py:393-411 (``UT(sigmas_f, Wm, Wc, Q, x_mean, residual_x)``), ``update`` :459-481
  (``UT(sigmas_h, Wm, Wc, R, z_mean, residual_z)``, ``cross_variance`` :493-504, ``y = residual_z(z, zp)``,
  ``x = state_add(x, K y)``) and ``unscented_transform`` unscented_transform.py:99-128 with a residual_fn.
* ``ukf_rts_smoother_hooks``: ``rts_smoother`` UKF.py:714-737 with ``x_mean`` / ``residual_x``.
* ``ckf_update_single_hooks``: CubatureKalmanFilter.py:362-379 with ``y = residual_z(z, zp)`` (:376).
* ``ukf_step_bank_hooks`` / ``ckf_step_bank_hooks``: vectorised over N for the built-in models, the hooks
  given as the components that are angles (wrapped residuals, circular means).

Parity: pinned by ``tests/golden/ukf_hooks_*.npz`` / ``ckf_hooks_*.npz``.
"""
import numpy as np
from scipy.stats import multivariate_normal

from oracle import ckf as ockf
from oracle import ukf as oukf


def _wrap(a):
    return np.where(a > np.pi, a - 2 * np.pi, np.where(a <= -np.pi, a + 2 * np.pi, a))


def unscented_transform(sigmas, Wm, Wc, noise_cov, mean_fn=None, residual_fn=None):
    """unscented_transform.py:99-128 for one filter, with its mean_fn / residual_fn."""
    x = np.dot(Wm, sigmas) if mean_fn is None else mean_fn(sigmas, Wm)
    if residual_fn is None or residual_fn is np.subtract:
        y = sigmas - x[np.newaxis, :]
        P = np.dot(y.T, np.dot(np.diag(Wc), y))
    else:
        P = np.zeros((sigmas.shape[1], sigmas.shape[1]))
        for k in range(sigmas.shape[0]):
            y = residual_fn(sigmas[k], x)
            P += Wc[k] * np.outer(y, y)
    return x, P + noise_cov


def ukf_step_single(x, P, z, Q, R, fx, hx, dt, alpha, beta, kappa, hooks, fx_args=None, hx_args=None):
    """predict + update (``z=None``: predict only) of one filter -> dict(x, P, x_prior, P_prior, K, S, y, loglik).
    ``hooks`` maps the reference's keyword names (x_mean_fn, z_mean_fn, residual_x, residual_z, state_add)
    to callables; absent ones are the reference's defaults."""
    res_x = hooks.get("residual_x", np.subtract)
    res_z = hooks.get("residual_z", np.subtract)
    add = hooks.get("state_add", np.add)
    Wm, Wc = oukf.merwe_weights(x.shape[0], alpha, beta, kappa)
    sig = oukf.merwe_sigma_points(x, P, alpha, beta, kappa)
    sf = np.array([fx(s, dt, **(fx_args or {})) for s in sig])
    xp, Pp = unscented_transform(sf, Wm, Wc, Q, hooks.get("x_mean_fn"), res_x)
    out = dict(x=xp, P=Pp, x_prior=xp, P_prior=Pp, K=None, S=None, y=None, loglik=np.nan)
    if z is None:
        return out
    sig = oukf.merwe_sigma_points(xp, Pp, alpha, beta, kappa)
    sh = np.atleast_2d([hx(s, **(hx_args or {})) for s in sig])
    zp, S = unscented_transform(sh, Wm, Wc, R, hooks.get("z_mean_fn"), res_z)
    Pxz = np.zeros((x.shape[0], sh.shape[1]))
    for i in range(sig.shape[0]):
        Pxz += Wc[i] * np.outer(res_x(sig[i], xp), res_z(sh[i], zp))
    K = np.dot(Pxz, np.linalg.inv(S))
    y = res_z(z, zp)
    out.update(x=add(xp, np.dot(K, y)), P=Pp - np.dot(K, np.dot(S, K.T)), K=K, S=S, y=y,
               loglik=multivariate_normal.logpdf(y, cov=S, allow_singular=True))
    return out


def ukf_rts_smoother_hooks(Xs, Ps, Q, fx, dts, alpha, beta, kappa, x_mean_fn=None, residual_x=np.subtract):
    """UKF.py:714-737 for one filter: Xs (T,n), Ps (T,n,n) -> (xs, Ps, Ks).  No state_add (the reference
    adds K residual_x(...) with +=, :735)."""
    T, n = Xs.shape
    Wm, Wc = oukf.merwe_weights(n, alpha, beta, kappa)
    Ks = np.zeros((T, n, n))
    xs, ps = Xs.copy(), Ps.copy()
    for k in reversed(range(T - 1)):
        sigmas = oukf.merwe_sigma_points(xs[k], ps[k], alpha, beta, kappa)
        sigmas_f = np.array([fx(s, dts[k]) for s in sigmas])
        xb, Pb = unscented_transform(sigmas_f, Wm, Wc, Q, x_mean_fn, residual_x)
        Pxb = 0
        for i in range(sigmas.shape[0]):
            Pxb = Pxb + Wc[i] * np.outer(residual_x(sigmas[i], Xs[k]), residual_x(sigmas_f[i], xb))
        K = np.dot(Pxb, np.linalg.inv(Pb))
        xs[k] += np.dot(K, residual_x(xs[k + 1], xb))
        ps[k] += np.dot(K, ps[k + 1] - Pb).dot(K.T)
        Ks[k] = K
    return xs, ps, Ks


def ckf_update_single_hooks(x, P, sigmas_f, z, R, hx, residual_z, hx_args=()):
    """CubatureKalmanFilter.py:362-379 with y = residual_z(z, zp); x and z are columns as in the reference."""
    x0 = x
    x, P, y, K, S, SI = ockf.ckf_update_single(x, P, sigmas_f, z, R, hx, hx_args)
    if y is None:
        return x, P, y, K, S, SI
    y = residual_z(z, z - y)                      # zp = z - (z - zp)
    return x0 + np.dot(K, y), P, y, K, S, SI


# --------------------------------------------------------------------------- banks, built-in models
def _circ_mean(W, X, angles):
    """Weighted mean of points X[N, s, d] with circular means in the ``angles`` components."""
    m = np.einsum("s,nsd->nd", W, X)
    for a in angles:
        m[:, a] = np.arctan2(np.einsum("s,ns->n", W, np.sin(X[:, :, a])), np.einsum("s,ns->n", W, np.cos(X[:, :, a])))
    return m


def _res(a, b, angles):
    d = a - b
    for c in angles:
        d[..., c] = _wrap(d[..., c])
    return d


def ukf_step_bank_hooks(x, P, z, Q, R, dt, alpha, beta, kappa, fx_model, hx_model, angle_x=(), angle_z=(),
                        x_mean=False, z_mean=False, F=None, H=None, valid=None):
    """One predict + update of a bank x[N,n], P[N,n,n], z[N,m].  ``angle_x`` / ``angle_z``: the components
    residual_x / residual_z (and state_add) wrap; ``x_mean`` / ``z_mean``: those components take circular
    means.  Empty tuples and False give the reference's defaults."""
    n = x.shape[-1]
    Wm, Wc = oukf.merwe_weights(n, alpha, beta, kappa)
    sig = oukf.merwe_sigma_points(x, P, alpha, beta, kappa)
    sf = oukf.fx_apply(fx_model, sig, dt, F)
    xp = _circ_mean(Wm, sf, angle_x if x_mean else ())
    D = _res(sf, xp[:, None, :], angle_x)
    Pp = np.einsum("nsa,s,nsb->nab", D, Wc, D) + Q
    sig = oukf.merwe_sigma_points(xp, Pp, alpha, beta, kappa)
    sh = oukf.hx_apply(hx_model, sig, H)
    zp = _circ_mean(Wm, sh, angle_z if z_mean else ())
    Dz = _res(sh, zp[:, None, :], angle_z)
    S = np.einsum("nsa,s,nsb->nab", Dz, Wc, Dz) + R
    Dx = _res(sig, xp[:, None, :], angle_x)
    Pxz = np.einsum("s,nsa,nsb->nab", Wc, Dx, Dz)
    K = Pxz @ np.linalg.inv(S)
    y = _res(z, zp, angle_z)
    xn = _res(xp + (K @ y[..., None])[..., 0], 0.0, angle_x)
    Pn = Pp - K @ (S @ np.swapaxes(K, -1, -2))
    if valid is not None:
        v = np.asarray(valid, bool)
        xn = np.where(v[:, None], xn, xp)
        Pn = np.where(v[:, None, None], Pn, Pp)
    return dict(x=xn, P=Pn, x_prior=xp, P_prior=Pp, y=y, K=K, S=S)


def ckf_step_bank_hooks(x, P, z, Q, R, dt, fx_model, hx_model, angle_z=(), F=None, H=None, valid=None):
    """oracle.ckf.ckf_step_bank (centred sums) with y = residual_z(z, zp) wrapping the ``angle_z`` components."""
    o = ockf.ckf_step_bank(x, P, z, Q, R, dt, fx_model, hx_model, F=F, H=H)
    y = _res(o["y"], 0.0, angle_z)
    xn = o["x_prior"] + (o["K"] @ y[..., None])[..., 0]
    if valid is not None:
        v = np.asarray(valid, bool)
        xn = np.where(v[:, None], xn, o["x_prior"])
        o["P"] = np.where(v[:, None, None], o["P"], o["P_prior"])
    o.update(x=xn, y=y)
    return o
