"""Oracle: the measurement scores of a UKF bank (TEST INFRASTRUCTURE), bke_ukf_score / UnscentedKalmanFilter.score_measurements.

For track i and candidate z_ik, what the reference's UnscentedKalmanFilter reports as ``log_likelihood`` and
``mahalanobis`` right after ``update(z_ik)`` from the track's current (x, P) (UKF.py:459-477, 742-777), composed from
the existing oracles:

* sigma points of (x, P): ``oracle.ukf.merwe_sigma_points`` or ``ukf_simplex_oracle.simplex_sigma_points``;
* hx on every point (``oracle.ukf.hx_apply`` or a per-track callable), then the unscented transform with R and the
  hooks as ``ukf_hooks_oracle`` states them (circular z mean, wrapped residual_z);
* y = residual_z(z_ik, zhat), and the scores by ``stats_oracle``'s rule (its inverse, a missing candidate as
  ``z is None``).  A track whose P has no Cholesky factor gets status 2 and NaN scores.
"""
import numpy as np

import stats_oracle as so
import ukf_hooks_oracle as uho
import ukf_simplex_oracle as uso
from oracle import ukf as oukf


def sigma_points(x, P, pts):
    """(sigmas[N, s, n], Wm, Wc, ok[N]) for pts = ("merwe", alpha, beta, kappa) or ("simplex",); a track whose
    Cholesky fails has ok False (its points are NaN)."""
    N, n = x.shape
    ok = np.ones(N, bool)
    sig = np.full((N, n + 1 if pts[0] == "simplex" else 2 * n + 1, n), np.nan)
    for f in range(N):
        try:
            if pts[0] == "simplex":
                sig[f] = uso.simplex_sigma_points(x[f], P[f])
            else:
                sig[f] = oukf.merwe_sigma_points(x[f], P[f], *pts[1:])
        except np.linalg.LinAlgError:
            ok[f] = False
    Wm, Wc = uso.simplex_weights(n) if pts[0] == "simplex" else oukf.merwe_weights(n, *pts[1:])
    return sig, Wm, Wc, ok


def ukf_score_bank(x, P, z, R, pts, hx_model=oukf.HX_LINEAR, H=None, hx=None, valid=None, angle_z=(), z_mean=False):
    """x[N, n], P[N, n, n], z[N or 1, K, m], R [m, m] or [N, m, m]; ``hx``: a callable hx(s, f) of point s of
    track f (replaces ``hx_model``); ``angle_z``: the components residual_z wraps, circular means there with
    ``z_mean``.  Returns dict zhat[N, m], S[N, m, m], y[N, K, m], d2, mahalanobis, log_likelihood [N, K], status[N]."""
    x, P, z = (np.asarray(a, np.float64) for a in (x, P, z))
    N = x.shape[0]
    z = np.broadcast_to(z, (N,) + z.shape[1:])
    sig, Wm, Wc, ok = sigma_points(x, P, pts)
    if hx is None:
        sh = oukf.hx_apply(hx_model, sig, H)
    else:
        sh = np.array([[hx(s, f) for s in sig[f]] for f in range(N)])
    zhat = uho._circ_mean(Wm, sh, angle_z if z_mean else ())
    Dz = uho._res(sh, zhat[:, None, :], angle_z)
    S = np.einsum("nsa,s,nsb->nab", Dz, Wc, Dz) + R
    y = uho._res(z, zhat[:, None, :], angle_z)
    S_safe = np.where(ok[:, None, None], S, np.eye(S.shape[-1]))
    out = so.score(zhat[:, None, :] + y, zhat, S_safe, valid)
    status = out["status"].copy()
    status[~ok] = 2
    for k in ("d2", "mahalanobis", "log_likelihood"):
        bad = ~ok[:, None] if valid is None else (~ok[:, None] & np.asarray(valid, bool))
        out[k] = np.where(bad, np.nan, out[k])
    return dict(zhat=zhat, S=S, y=out["y"], d2=out["d2"], mahalanobis=out["mahalanobis"],
                log_likelihood=out["log_likelihood"], status=status)
