#!/usr/bin/env python
"""Generate the golden vectors of the UKF measurement scores (tests/golden/ukf_score_*.npz) from the UNMODIFIED
reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_ukf_score.py

Per case: N filters built from x, P, Q, R; ``predict()``; then for every candidate z[f, k] a deepcopy of filter f runs
``update(z)`` and its ``log_likelihood`` and ``mahalanobis`` are recorded (ref_ll, ref_maha [N, K]), next to the prior
(x_prior, P_prior) the scores are taken against.  Cases:
  ukf_score_cv_rae       6/3 CV + range / azimuth / elevation, MerweScaledSigmaPoints
  ukf_score_hooks_rb     4/2 CV + range / bearing behind the sensor with residual_z + z_mean_fn, candidates across
                         +-pi; the script asserts that the hooks move the scores far beyond any tolerance
  ukf_score_simplex_rb   4/2 CV + range / bearing, SimplexSigmaPoints
  ukf_score_julier       6/3 CV + range / azimuth / elevation, JulierSigmaPoints
  ukf_score_user_rb      4/2 CV + a range / bearing sensor hx(x, sx, sy) with a per-filter sensor x
  ukf_score_lin          4/2 CV + a linear H
The tests never import the reference.
"""
import copy
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import save, fx_cv, wl                                                       # noqa: E402
from filterpy.kalman import (UnscentedKalmanFilter, MerweScaledSigmaPoints, JulierSigmaPoints,  # noqa: E402
                             SimplexSigmaPoints)

N, K = 6, 5


def hx_rae(x):
    rho = np.sqrt(x[0] ** 2 + x[2] ** 2)
    return np.array([np.sqrt(rho ** 2 + x[4] ** 2), np.arctan2(x[2], x[0]), np.arctan2(x[4], rho)])


def hx_rb(x):
    return np.array([np.sqrt(x[0] * x[0] + x[2] * x[2]), np.arctan2(x[2], x[0])])


def _run(w, n, m, dt, hx, points, cands, hooks=None, hx_args=None):
    """-> (x_prior [N, n], P_prior, ref_ll [N, K], ref_maha [N, K])."""
    xp, Pp, ll, mh = [], [], np.zeros((N, K)), np.zeros((N, K))
    for f in range(N):
        u = UnscentedKalmanFilter(n, m, dt, hx, fx_cv, points(), **(hooks or {}))
        u.x = w["x"][f].copy(); u.P = w["P"][f].copy(); u.Q = w["Q"][f].copy(); u.R = w["R"][f].copy()
        u.predict()
        xp.append(u.x.copy()); Pp.append(u.P.copy())
        for k in range(K):
            c = copy.deepcopy(u)
            c.update(cands[f, k], **({} if hx_args is None else {a: v[f] for a, v in hx_args.items()}))
            ll[f, k], mh[f, k] = c.log_likelihood, c.mahalanobis
    return np.array(xp), np.array(Pp), ll, mh


def _candidates(rng, z, sd):
    """K candidates per filter around its measurement z[f]: the first is z itself."""
    c = z[:, None, :] + sd * rng.standard_normal((N, K, z.shape[1]))
    c[:, 0] = z
    return c


def _case(name, w, n, m, dt, hx, points, cands, **kw):
    xp, Pp, ll, mh = _run(w, n, m, dt, hx, points, cands, **kw)
    save(name, x=w["x"][:N], P=w["P"][:N], Q=w["Q"][:N], R=w["R"][:N], dt=dt, z=cands, x_prior=xp, P_prior=Pp,
         ref_ll=ll, ref_maha=mh)
    return ll, mh


def main():
    rng = np.random.default_rng(515)
    w = wl.ukf_bank_cv3d(N, seed=31, steps=1)
    _case("ukf_score_cv_rae", w, 6, 3, 0.1, hx_rae, lambda: MerweScaledSigmaPoints(6, .5, 2., 0.),
          _candidates(rng, w["zs"][0], np.array([3.0, 0.02, 0.02])))
    _case("ukf_score_julier", w, 6, 3, 0.1, hx_rae, lambda: JulierSigmaPoints(6, kappa=1.5),
          _candidates(rng, w["zs"][0], np.array([3.0, 0.02, 0.02])))

    w = wl.ukf_bank_rb_behind(N, seed=32, steps=1)
    c = _candidates(rng, w["zs"][0], np.array([1.0, 0.01]))
    c[:, 1:, 1] = -c[:, 1:, 1]                     # the bearing mirrored through the +-pi cut: just across it
    hooks = dict(residual_z=wl.rb_residual_z, z_mean_fn=wl.rb_z_mean)
    pts = lambda: MerweScaledSigmaPoints(4, .8, 2., 0.)                                  # noqa: E731
    ll, _ = _case("ukf_score_hooks_rb", w, 4, 2, 1.0, hx_rb, pts, c, hooks=hooks)
    ll0, _ = _run(w, 4, 2, 1.0, hx_rb, pts, c)[2:]
    assert np.nanmax(np.abs(ll - ll0)) > 100, np.nanmax(np.abs(ll - ll0))
    assert (np.abs(c[:, :, 1]) > 3.0).any() and (c[:, :, 1] > 3.0).any() and (c[:, :, 1] < -3.0).any()

    w = wl.ukf_bank_ct2d(N, seed=33, steps=1)
    _case("ukf_score_simplex_rb", w, 4, 2, 0.5, hx_rb, lambda: SimplexSigmaPoints(4),
          _candidates(rng, w["zs"][0], np.array([2.0, 0.01])))
    sx = w["sensor"][0] + np.arange(N) * 5.0
    sy = np.full(N, w["sensor"][1])
    cu = _candidates(np.random.default_rng(34), w["zs"][0], np.array([2.0, 0.01]))
    xp, Pp, ll, mh = _run(w, 4, 2, 0.5, wl.offset_rb_hx, lambda: MerweScaledSigmaPoints(4, .5, 2., 0.), cu,
                          hx_args=dict(sx=sx, sy=sy))
    save("ukf_score_user_rb", x=w["x"][:N], P=w["P"][:N], Q=w["Q"][:N], R=w["R"][:N], dt=0.5, z=cu, x_prior=xp,
         P_prior=Pp, ref_ll=ll, ref_maha=mh, sx=sx, sy=sy)

    w = wl.ukf_bank_ct2d(N, seed=35, steps=1, linear_hx=True)
    H = w["H"]
    _case("ukf_score_lin", w, 4, 2, 0.5, lambda x: H @ x, lambda: MerweScaledSigmaPoints(4, .5, 2., 0.),
          _candidates(rng, w["zs"][0], np.array([3.0, 3.0])))


if __name__ == "__main__":
    main()
