#!/usr/bin/env python
"""Generate the golden vectors of the UKF on SimplexSigmaPoints (tests/golden/ukf_simplex_*.npz) from the
UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_ukf_simplex.py

Cases: the sigma points themselves (n = 1, 2, 3, 4, 6, 9 and a scalar P); banks of 6/3 constant velocity +
range / azimuth / elevation, 4/2 constant velocity + range / bearing and a linear 4/2 model with missing
measurements and an R override; batch_filter + rts_smoother with a built-in and with a user (coordinated
turn) fx; user fx / hx with per-filter arguments; and range / bearing with residual_z / z_mean_fn on targets
crossing behind the sensor (the script asserts that the hooks change the result).  The tests never import
the reference.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import save, fx_cv, hx_rae, wl                                            # noqa: E402
from filterpy.kalman import UnscentedKalmanFilter, SimplexSigmaPoints                    # noqa: E402

KEYS = ["x", "P", "x_prior", "P_prior", "K", "S", "y", "loglik"]
RB_HOOKS = dict(residual_z=wl.rb_residual_z, z_mean_fn=wl.rb_z_mean)


def hx_rb(x):
    return np.array([np.sqrt(x[0] * x[0] + x[2] * x[2]), np.arctan2(x[2], x[0])])


def _record(f, n, m, has_z):
    K = np.zeros((n, m)) if np.isscalar(f.K) else np.array(f.K, float)
    y = np.zeros(m) if np.isscalar(f.y) else np.array(f.y, float).reshape(m)
    return dict(x=np.array(f.x, float).reshape(n), P=np.array(f.P, float), x_prior=np.array(f.x_prior, float).reshape(n),
                P_prior=np.array(f.P_prior, float), K=K, S=np.array(f.S, float), y=y,
                loglik=float(f.log_likelihood) if has_z else np.nan)


def _bank(w, dt, fx, hx, steps, valid, predict=lambda u, f: u.predict(), update=lambda u, f, z, t: u.update(z), **hooks):
    """Per-filter reference UKFs on SimplexSigmaPoints over ``steps`` epochs -> {ref_<key>: [T, N, ...]}."""
    N, n = w["x"].shape
    m = w["R"].shape[-1]
    fs = []
    for f in range(N):
        u = UnscentedKalmanFilter(n, m, dt, hx, fx, SimplexSigmaPoints(n), **hooks)
        u.x = w["x"][f].copy(); u.P = w["P"][f].copy(); u.Q = w["Q"][f]; u.R = w["R"][f]
        fs.append(u)
    out = {k: [] for k in KEYS}
    for t in range(steps):
        rec = {k: [] for k in KEYS}
        for f, u in enumerate(fs):
            predict(u, f)
            update(u, f, w["zs"][t, f] if valid[t, f] else None, t)
            for k, v in _record(u, n, m, bool(valid[t, f])).items():
                rec[k].append(v)
        for k in KEYS:
            out[k].append(np.array(rec[k]))
    return {"ref_" + k: np.array(v) for k, v in out.items()}


def cv2d_bank(N, seed, steps, dt, rb):
    """N constant-velocity targets (x, vx, y, vy) 100-500 m in front of a sensor at the origin (well inside
    (-pi, pi) in bearing), seen in range / bearing (``rb``) or in position; correlated P."""
    rng = np.random.default_rng(seed)
    xt = np.stack([rng.uniform(100, 500, N), rng.uniform(-10, 10, N), rng.uniform(-300, 300, N), rng.uniform(-10, 10, N)], 1)
    x0 = xt + rng.standard_normal((N, 4)) * np.array([2, .5, 2, .5])
    A = rng.standard_normal((N, 4, 4))
    sd = np.array([2.0, 0.5, 2.0, 0.5])
    P0 = (A @ np.swapaxes(A, 1, 2) / 4 + 0.5 * np.eye(4)) * np.outer(sd, sd)
    q = np.exp(rng.uniform(np.log(1e-3), np.log(1e-1), N))
    qb = wl.q_white_noise_block(2, np.full(N, dt), q)
    Q = wl._block_diag([qb, qb])
    sig = np.array([1.0, 0.005]) if rb else np.array([2.5, 2.5])
    R = np.broadcast_to(np.diag(sig ** 2), (N, 2, 2)).copy()
    zs = np.zeros((steps, N, 2))
    for t in range(steps):
        xt = xt.copy()
        xt[:, 0::2] += dt * xt[:, 1::2]
        h = np.stack([hx_rb(s) for s in xt]) if rb else xt[:, [0, 2]]
        zs[t] = h + sig * rng.standard_normal((N, 2))
    F = np.eye(4); F[0, 1] = F[2, 3] = dt
    H = np.zeros((2, 4)); H[0, 0] = H[1, 2] = 1
    return dict(x=x0, P=P0, Q=Q, R=R, zs=zs, F=F, H=H)


def gen_sigma():
    out = {}
    rng = np.random.default_rng(31)
    for n in (1, 2, 3, 4, 6, 9):
        A = rng.standard_normal((n, n))
        P = A @ A.T + n * np.eye(n)
        x = rng.standard_normal(n)
        pts = SimplexSigmaPoints(n)
        out.update({"x%d" % n: x, "P%d" % n: P, "sigmas%d" % n: pts.sigma_points(x, P), "Wm%d" % n: pts.Wm})
    pts = SimplexSigmaPoints(3)
    xs = np.array([1.0, -2.0, 0.5])
    out.update(x_scalar=xs, P_scalar=2.5, sigmas_scalar=pts.sigma_points(xs, 2.5))
    save("ukf_simplex_sigma", **out)


def gen_banks():
    N, steps, dt = 16, 5, 0.1
    w = wl.ukf_bank_cv3d(N, seed=4321, steps=steps, dt=dt)
    valid = np.random.default_rng(41).random((steps, N)) >= 0.2
    save("ukf_simplex_bank_rae", **w, valid=valid, dt=dt, **_bank(w, dt, fx_cv, hx_rae, steps, valid))

    w = cv2d_bank(N, 4242, steps, dt, rb=True)
    valid = np.random.default_rng(42).random((steps, N)) >= 0.2
    save("ukf_simplex_bank_rb", **w, valid=valid, dt=dt, **_bank(w, dt, fx_cv, hx_rb, steps, valid))

    # linear 4/2: missing measurements, and on odd epochs update(z, R=R_override)
    w = cv2d_bank(N, 4343, steps, dt, rb=False)
    F, H = w["F"], w["H"]
    valid = np.random.default_rng(43).random((steps, N)) >= 0.2
    R_override = np.array([[9.0, 1.5], [1.5, 4.0]])
    res = _bank(w, dt, lambda s, dt: F @ s, lambda s: H @ s, steps, valid,
                update=lambda u, f, z, t: u.update(z, R=R_override if t % 2 else None))
    save("ukf_simplex_bank_lin", **w, valid=valid, dt=dt, R_override=R_override, **res)


def gen_user():
    """coordinated turn with a per-filter turn rate (fx_args) and range / bearing from an offset sensor
    (hx_args): the Python callables of workloads.py here, their CUDA text on the GPU."""
    N, steps, dt = 16, 6, 0.5
    w = wl.ukf_bank_ct2d(N, seed=5151, steps=steps, dt=dt)
    sx, sy = w["sensor"]
    valid = np.random.default_rng(51).random((steps, N)) >= 0.1
    res = _bank(w, dt, wl.ct_fx, wl.offset_rb_hx, steps, valid, predict=lambda u, f: u.predict(omega=w["omega"][f]),
                update=lambda u, f, z, t: u.update(z, sx=sx, sy=sy))
    save("ukf_simplex_user_ct_rb", **w, valid=valid, dt=dt, **res)


def gen_rts():
    """batch_filter + rts_smoother: constant velocity (built-in fx) and the coordinated turn (user fx; the
    reference calls fx(sigma, dt) without keyword arguments in the smoother, UKF.py:712, so the turn rate is
    the callable's default), both measured in position."""
    N, steps, dt, om = 6, 10, 0.5, 0.07
    out = {}
    for name in ("cv", "ct"):
        w = wl.ukf_bank_ct2d(N, seed=1133 if name == "cv" else 1144, steps=steps, dt=dt, linear_hx=True)
        Hlin = w["H"]
        fx = fx_cv if name == "cv" else (lambda s, dt, omega=om: wl.ct_fx(s, dt, omega))
        Xs = np.zeros((steps, N, 4)); Ps = np.zeros((steps, N, 4, 4))
        sm = [np.zeros((steps, N, 4)), np.zeros((steps, N, 4, 4)), np.zeros((steps, N, 4, 4))]
        for f in range(N):
            u = UnscentedKalmanFilter(4, 2, dt, lambda s: Hlin @ s, fx, SimplexSigmaPoints(4))
            u.x = w["x"][f].copy(); u.P = w["P"][f].copy(); u.Q = w["Q"][f]; u.R = w["R"][f]
            mu, cov = u.batch_filter(list(w["zs"][:, f]))
            Xs[:, f] = mu; Ps[:, f] = cov
            for o, v in zip(sm, u.rts_smoother(mu, cov)):
                o[:, f] = v
        out.update({name + "_" + k: v for k, v in dict(x0=w["x"], P0=w["P"], Q=w["Q"], R=w["R"], zs=w["zs"], Xs=Xs, Ps=Ps,
                                                       ref_x=sm[0], ref_P=sm[1], ref_K=sm[2]).items()})
    save("ukf_simplex_rts", H=Hlin, dt=dt, omega=om, **out)


def gen_hooks():
    """range / bearing, targets crossing behind the sensor: residual_z and z_mean_fn."""
    N, steps, dt = 16, 12, 1.0
    w = wl.ukf_bank_rb_behind(N, seed=9191, steps=steps, dt=dt)
    valid = np.random.default_rng(61).random((steps, N)) >= 0.1
    res = _bank(w, dt, fx_cv, hx_rb, steps, valid, **RB_HOOKS)
    try:
        plain = _bank(w, dt, fx_cv, hx_rb, steps, valid)
        d = np.abs(plain["ref_x"] - res["ref_x"])
        d = np.inf if not np.all(np.isfinite(d)) else d.max()
    except np.linalg.LinAlgError:
        d = np.inf
    print("ukf_simplex_hooks_rb: the run without hooks differs by %.3g" % d)
    assert d > 1.0
    save("ukf_simplex_hooks_rb", **w, valid=valid, dt=dt, **res)


if __name__ == "__main__":
    gen_sigma()
    gen_banks()
    gen_user()
    gen_rts()
    gen_hooks()
