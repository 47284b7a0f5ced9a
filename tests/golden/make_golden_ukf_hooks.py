#!/usr/bin/env python
"""Generate the golden vectors of the UKF / CKF angle hooks (tests/golden/ukf_hooks_*.npz, ckf_hooks_rb.npz)
from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_ukf_hooks.py

The reference runs the Python hook callables of ``filterpy_b200.common.workloads`` (wrapped residuals,
circular means, a wrapping state_add).  Every case is also run WITHOUT the hooks, and the script asserts
that the two runs differ by more than 1 in some state component: the targets really cross the +-pi cut.
The tests never import the reference.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import save, fx_cv, wl                                                     # noqa: E402
from filterpy.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, CubatureKalmanFilter  # noqa: E402

ALPHA, BETA, KAPPA = 0.8, 2.0, 0.0
KEYS = ["x", "P", "x_prior", "P_prior", "K", "S", "y", "loglik"]
RB_HOOKS = dict(residual_z=wl.rb_residual_z, z_mean_fn=wl.rb_z_mean)
CTRV_HOOKS = dict(residual_z=wl.rb_residual_z, z_mean_fn=wl.rb_z_mean, residual_x=wl.ctrv_residual_x,
                  state_add=wl.ctrv_state_add, x_mean_fn=wl.ctrv_x_mean)


def hx_rb(x):
    return np.array([np.sqrt(x[0] * x[0] + x[2] * x[2]), np.arctan2(x[2], x[0])])


def _record(f, n, m, has_z):
    K = np.zeros((n, m)) if np.isscalar(f.K) else np.array(f.K, float)
    y = np.zeros(m) if np.isscalar(f.y) else np.array(f.y, float).reshape(m)
    return dict(x=np.array(f.x, float).reshape(n), P=np.array(f.P, float), x_prior=np.array(f.x_prior, float).reshape(n),
                P_prior=np.array(f.P_prior, float), K=K, S=np.array(f.S, float), y=y,
                loglik=float(f.log_likelihood) if has_z else np.nan)


def _run(make, w, steps, valid, predict, update):
    """predict / update every filter of the bank for ``steps`` epochs -> {ref_<key>: [T, N, ...]}."""
    N, n = w["x"].shape
    m = w["R"].shape[-1]
    fs = [make(f) for f in range(N)]
    out = {k: [] for k in KEYS}
    for t in range(steps):
        rec = {k: [] for k in KEYS}
        for f, flt in enumerate(fs):
            predict(flt, f)
            update(flt, w["zs"][t, f] if valid[t, f] else None)
            for k, v in _record(flt, n, m, bool(valid[t, f])).items():
                rec[k].append(v)
        for k in KEYS:
            out[k].append(np.array(rec[k]))
    return {"ref_" + k: np.array(v) for k, v in out.items()}


def _crosses(hooked, plain_fn):
    """The run without hooks differs from the hooked one by more than 1 in some state component (or fails)."""
    try:
        plain = plain_fn()
    except np.linalg.LinAlgError:
        return np.inf
    d = np.abs(plain["ref_x"] - hooked["ref_x"])
    return np.inf if not np.all(np.isfinite(d)) else d.max()


def _ukf(w, n, m, dt, fx, hx, hooks):
    def make(f):
        u = UnscentedKalmanFilter(n, m, dt, hx, fx, MerweScaledSigmaPoints(n, ALPHA, BETA, KAPPA), **hooks)
        u.x = w["x"][f].copy(); u.P = w["P"][f].copy(); u.Q = w["Q"][f]; u.R = w["R"][f]
        return u
    return make


def gen_ukf_rb():
    """(a) 4/2 ConstVelFx + RangeBearingHx, targets behind the sensor: residual_z and z_mean_fn."""
    N, steps, dt = 16, 12, 1.0
    w = wl.ukf_bank_rb_behind(N, steps=steps, dt=dt)
    valid = np.random.default_rng(11).random((steps, N)) >= 0.1

    def run(hooks):
        return _run(_ukf(w, 4, 2, dt, fx_cv, hx_rb, hooks), w, steps, valid, lambda u, f: u.predict(), lambda u, z: u.update(z))
    res = run(RB_HOOKS)
    d = _crosses(res, lambda: run({}))
    print("ukf_hooks_rb: the run without hooks differs by %.3g" % d)
    assert d > 1.0
    save("ukf_hooks_rb", **w, valid=valid, dt=dt, alpha=ALPHA, beta=BETA, kappa=KAPPA, **res)


def gen_ukf_ctrv():
    """(b) 5-state CTRV + offset range / bearing, heading across +-pi: all five hooks."""
    N, steps, dt = 16, 12, 0.5
    w = wl.ukf_bank_ctrv(N, steps=steps, dt=dt)
    sx, sy = w["sensor"]
    valid = np.random.default_rng(12).random((steps, N)) >= 0.1

    def run(hooks):
        return _run(_ukf(w, 5, 2, dt, wl.ctrv_fx, wl.ctrv_rb_hx, hooks), w, steps, valid, lambda u, f: u.predict(),
                    lambda u, z: u.update(z, sx=sx, sy=sy))
    res = run(CTRV_HOOKS)
    d = _crosses(res, lambda: run({}))
    print("ukf_hooks_ctrv: the run without hooks differs by %.3g" % d)
    assert d > 1.0
    save("ukf_hooks_ctrv", **w, valid=valid, dt=dt, alpha=ALPHA, beta=BETA, kappa=KAPPA, **res)


def gen_ukf_ctrv_rts():
    """(b) through batch_filter + rts_smoother (x_mean_fn / residual_x in the smoother, UKF.py:720-735)."""
    N, steps, dt = 6, 12, 0.5
    w = wl.ukf_bank_ctrv(N, seed=6161, steps=steps, dt=dt)
    sx, sy = w["sensor"]

    def hx(s):
        return wl.ctrv_rb_hx(s, sx, sy)

    def run(hooks):
        Xs = np.zeros((steps, N, 5)); Ps = np.zeros((steps, N, 5, 5))
        sm = [np.zeros((steps, N, 5)), np.zeros((steps, N, 5, 5)), np.zeros((steps, N, 5, 5))]
        for f in range(N):
            u = _ukf(w, 5, 2, dt, wl.ctrv_fx, hx, hooks)(f)
            mu, cov = u.batch_filter(list(w["zs"][:, f]))
            Xs[:, f] = mu; Ps[:, f] = cov
            for o, v in zip(sm, u.rts_smoother(mu, cov)):
                o[:, f] = v
        return dict(Xs=Xs, Ps=Ps, ref_x=sm[0], ref_P=sm[1], ref_K=sm[2])
    res = run(CTRV_HOOKS)
    d = _crosses(res, lambda: run({}))
    print("ukf_hooks_ctrv_rts: the run without hooks differs by %.3g" % d)
    assert d > 1.0
    save("ukf_hooks_ctrv_rts", **w, dt=dt, alpha=ALPHA, beta=BETA, kappa=KAPPA, **res)


def gen_ckf_rb():
    """(a) through the CKF: residual_z only (CubatureKalmanFilter.py:376)."""
    N, steps, dt = 16, 12, 1.0
    w = wl.ukf_bank_rb_behind(N, seed=8181, steps=steps, dt=dt)
    valid = np.random.default_rng(13).random((steps, N)) >= 0.1

    def run(hooks):
        def make(f):
            c = CubatureKalmanFilter(4, 2, dt, hx_rb, fx_cv, **hooks)
            c.x = w["x"][f].copy()[:, None]; c.P = w["P"][f].copy(); c.Q = w["Q"][f]; c.R = w["R"][f]
            return c
        return _run(make, w, steps, valid, lambda c, f: c.predict(), lambda c, z: c.update(None if z is None else z[:, None]))
    res = run(dict(residual_z=wl.rb_residual_z))
    d = _crosses(res, lambda: run({}))
    print("ckf_hooks_rb: the run without hooks differs by %.3g" % d)
    assert d > 1.0
    save("ckf_hooks_rb", **w, valid=valid, dt=dt, **res)


if __name__ == "__main__":
    gen_ukf_rb()
    gen_ukf_ctrv()
    gen_ukf_ctrv_rts()
    gen_ckf_rb()
