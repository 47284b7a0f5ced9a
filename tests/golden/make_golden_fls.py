#!/usr/bin/env python
"""Generate the FixedLagSmoother golden vectors (tests/golden/fls_*.npz) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_fls.py

One reference ``FixedLagSmoother`` per filter of each bank runs ``smooth_batch(zs, N, us)``; the generator also
runs the same epochs through ``smooth()`` and asserts that the two agree bit for bit, as the reference's own
test expects.  The online case records the object after selected ``smooth()`` calls.  The tests never import
the reference.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import save, wl                                                          # noqa: E402

from filterpy.kalman import FixedLagSmoother                                             # noqa: E402


def _per(a, f, Nf):
    a = np.asarray(a)
    return a[f] if a.ndim == 3 and a.shape[0] == Nf else a


def _make(w, f, Nf, N, col):
    n, m = w["x"].shape[1], np.shape(w["H"])[-2]
    s = FixedLagSmoother(n, m, N)
    s.x = w["x"][f].copy()[:, None] if col else w["x"][f].copy()
    s.P = _per(w["P"], f, Nf).copy()
    for k in "FHQR":
        setattr(s, k, _per(w[k], f, Nf).copy())
    if "B" in w:
        s.B = w["B"].copy()
    return s


def _z(w, t, f, scalar):
    return float(w["zs"][t, f, 0]) if scalar else w["zs"][t, f].copy()


def run(w, N, col=False, scalar=False):
    """smooth_batch for every filter, checked bit for bit against T smooth() calls; returns the ref_* arrays."""
    Nf, n = w["x"].shape
    T = w["zs"].shape[0]
    xs, xh = np.zeros((T, Nf, n)), np.zeros((T, Nf, n))
    for f in range(Nf):
        s = _make(w, f, Nf, N, col)
        zs = [_z(w, t, f, scalar) for t in range(T)]
        us = None if "us" not in w else w["us"][:, f]
        a, b = s.smooth_batch(zs, N, us=us)
        xs[:, f], xh[:, f] = a.reshape(T, n), b.reshape(T, n)
        if N is not None and T:
            o = _make(w, f, Nf, N, col)
            for t in range(T):
                o.smooth(zs[t], None if us is None else us[t])
            assert np.array_equal(np.array(o.xSmooth).reshape(T, n), xs[:, f]), f
    return dict(ref_xs=xs, ref_xhat=xh, N=N, x_col=col, scalar_z=scalar)


def online(w, N, calls):
    """smooth() calls one by one; after each call in `calls` record xSmooth, x, P, y, S and count."""
    Nf, n = w["x"].shape
    m = np.shape(w["H"])[-2]
    objs = [_make(w, f, Nf, N, False) for f in range(Nf)]
    out = dict(N=N, rec_calls=np.array(calls), x_col=False, scalar_z=False)
    for t in range(w["zs"].shape[0]):
        for f, s in enumerate(objs):
            s.smooth(_z(w, t, f, False))
        c = t + 1
        if c in calls:
            out["ref_xs_%d" % c] = np.stack([np.array(s.xSmooth) for s in objs], 1)
            out["ref_x_%d" % c] = np.stack([s.x for s in objs])
            out["ref_P_%d" % c] = np.stack([s.P for s in objs])
            out["ref_y_%d" % c] = np.stack([np.reshape(s.y, m) for s in objs])
            out["ref_S_%d" % c] = np.stack([s.S for s in objs])
            out["ref_count_%d" % c] = np.array([s.count for s in objs])
            assert all(np.shape(s.y) == (m,) for s in objs)
    return out


def cv_2_1(Nf, T, seed):
    """The reference test's setup (filterpy/kalman/tests/test_fls.py, test_batch_equals_recursive): constant
    velocity, x = [0, .5], P = 200 I, R = 5, Q = 0.001 I, z = t/2 + 1.1 randn, one noise draw per filter."""
    rng = np.random.default_rng(seed)
    nom = np.arange(T) / 2.
    zs = nom[:, None, None] + 1.1 * rng.standard_normal((T, Nf, 1))
    return dict(x=np.tile([0., .5], (Nf, 1)), P=np.tile(200. * np.eye(2), (Nf, 1, 1)), F=np.array([[1., 1.], [0., 1.]]),
                H=np.array([[1., 0.]]), Q=0.001 * np.eye(2), R=5. * np.eye(1), zs=zs)


def gen():
    w = cv_2_1(64, 40, 11)
    save("fls_bank_2_1", **w, **run(w, 4))

    T = 24
    c = wl.kf_bank_cv2d(32, seed=321, steps=T)
    w = dict(x=c["x"], P=c["P"], F=c["F"], H=c["H"], Q=c["Q"], R=c["R"], zs=c["zs"])
    save("fls_bank_4_2", **w, **run(w, 8))

    u = wl.ukf_bank_cv3d(16, seed=654, steps=T, linear_hx=True)
    w = dict(x=u["x"], P=u["P"], F=u["F"], H=u["H"], Q=u["Q"][0], R=u["R"][0], zs=u["zs"])
    save("fls_bank_6_3", **w, **run(w, 5))

    c = wl.kf_bank_ca3d(16, seed=987, steps=T)
    w = dict(x=c["x"], P=c["P"], F=c["F"][0], H=c["H"][0], Q=c["Q"][0], R=c["R"][0], zs=c["zs"])
    save("fls_bank_9_3", **w, **run(w, 6))

    rng = np.random.default_rng(3)
    Nf, T = 16, 20
    A = rng.standard_normal((Nf, 3, 3))
    w = dict(x=rng.standard_normal((Nf, 3)), P=A @ np.swapaxes(A, 1, 2) + np.eye(3),
             F=np.eye(3) + 0.1 * rng.standard_normal((3, 3)), H=rng.standard_normal((2, 3)),
             Q=0.01 * np.eye(3) + 0.005 * np.ones((3, 3)), R=np.array([[0.5, 0.1], [0.1, 0.3]]),
             B=np.array([[0.5], [1.0], [0.2]]), us=rng.standard_normal((T, Nf, 1)), zs=rng.standard_normal((T, Nf, 2)))
    save("fls_ctrl_3_2", **w, **run(w, 3))

    w = cv_2_1(16, 30, 12)
    save("fls_lag_0", **w, **run(w, 0))
    save("fls_lag_1", **w, **run(w, 1))
    save("fls_lag_20", **w, **run(w, 20))          # above the fused kernel's lag cap (BKE_FLS_FUSED_MAX_LAG)
    save("fls_lag_ge_T", **w, **run(w, 30))        # N >= T: every row is that epoch's posterior

    Nf, T = 16, 25                                   # dim_z = 1: scalar z and a column x, a random walk
    w = dict(x=rng.standard_normal((Nf, 1)), P=rng.uniform(0.5, 5.0, (Nf, 1, 1)), F=rng.uniform(0.9, 1.1, (Nf, 1, 1)),
             H=rng.uniform(0.5, 2.0, (Nf, 1, 1)), Q=rng.uniform(0.01, 0.1, (Nf, 1, 1)),
             R=rng.uniform(0.1, 1.0, (Nf, 1, 1)), zs=rng.standard_normal((T, Nf, 1)))
    save("fls_scalar_1_1", **w, **run(w, 5, col=True, scalar=True))

    N, T = 4, 12
    w = cv_2_1(8, T, 13)
    save("fls_online", **w, **online(w, N, [1, N - 1, N, N + 1, T]))


if __name__ == "__main__":
    gen()
