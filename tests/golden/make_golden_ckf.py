#!/usr/bin/env python
"""Generate the CubatureKalmanFilter golden vectors (tests/golden/ckf_*.npz) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_ckf.py

It uses the helpers of ``make_golden.py`` (the reference import, ``save``, the CV / range-az-el callables)
and the seeded workloads of ``filterpy_b200.common.workloads``.  The tests never import the reference.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import save, fx_cv, hx_rae, wl                                          # noqa: E402


# ----------------------------------------------------------------------------- CKF
CKF_KEYS = ["x", "P", "x_prior", "P_prior", "K", "S", "y", "loglik"]
# the update without a predict comes last: it applies the last predict's gain a second time, which can
# leave P indefinite for the next cholesky (CubatureKalmanFilter.py:56)
CKF_OPS = ["update", "predict+update", "predict+none", "predict+update_R", "predict+read+update", "update"]


def _ckf_record(c, n, m, has_z):
    """The reference's attributes after an update; its x / y are columns, K = 0 / y = 0 before the first
    update are stored as zeros of their shapes."""
    K = np.zeros((n, m)) if np.isscalar(c.K) else np.array(c.K, float)
    y = np.zeros(m) if np.isscalar(c.y) else np.array(c.y, float).reshape(m)
    return dict(x=np.array(c.x, float).reshape(n), P=np.array(c.P, float), x_prior=np.array(c.x_prior, float).reshape(n),
                P_prior=np.array(c.P_prior, float), K=K, S=np.array(c.S, float), y=y,
                loglik=float(c.log_likelihood) if has_z else np.nan)


def _ckf_check_centred(c, Q, R, hx, hx_args, predicted, worst):
    """The kernel forms P- (after a predict) and S as centred sums; on the reference's own points they must
    agree with its raw-moment ckf_transform to better than 1e-9 relative."""
    sf = c.sigmas_f
    checks = [(np.atleast_2d([hx(s, *hx_args) for s in sf]), R, c.S)] + ([(sf, Q, c.P_prior)] if predicted else [])
    for pts, noise, ref in checks:
        d = pts - pts.sum(0) / pts.shape[0]
        cen = d.T @ d * (1.0 / pts.shape[0]) + noise
        worst[0] = max(worst[0], np.abs(cen - ref).max() / np.abs(ref).max())


def _ckf_run(w, steps, fx, hx, valid, fx_args=None, hx_args=None, ops=None):
    from filterpy.kalman import CubatureKalmanFilter
    N, n = w["x"].shape
    m = w["R"].shape[-1]
    out = {k: [] for k in CKF_KEYS}
    sig = []
    worst = [0.0]
    ckfs = []
    for f in range(N):
        c = CubatureKalmanFilter(n, m, float(w["dt"]), hx, fx)
        c.x = w["x"][f].copy()[:, None]; c.P = w["P"][f].copy(); c.Q = w["Q"][f]; c.R = w["R"][f]
        ckfs.append(c)
    for t in range(steps):
        rec = {k: [] for k in CKF_KEYS}
        srec = []
        op = ops[t] if ops is not None else "predict+update"
        for f, c in enumerate(ckfs):
            fa = () if fx_args is None else (fx_args[f],)
            ha = () if hx_args is None else tuple(hx_args)
            if op.startswith("predict"):
                c.predict(fx_args=fa)
            z = w["zs"][t, f][:, None] if valid[t, f] and op != "predict+none" else None
            if op == "predict+update_R":
                c.update(z, R=0.5, hx_args=ha)
            else:
                c.update(z, hx_args=ha)
            if z is not None:
                _ckf_check_centred(c, c.Q, 0.5 * np.eye(m) if op == "predict+update_R" else c.R, hx, ha,
                                   op.startswith("predict"), worst)
            for k, v in _ckf_record(c, n, m, z is not None).items():
                rec[k].append(v)
            srec.append(c.sigmas_f.copy())
        for k in CKF_KEYS:
            out[k].append(np.array(rec[k]))
        sig.append(np.array(srec))
    assert worst[0] < 1e-9, worst[0]
    print("  centred vs raw moments, worst relative difference %.2e" % worst[0])
    res = {"ref_" + k: np.array(v) for k, v in out.items()}
    res["ref_sigmas_f"] = np.array(sig)
    res["valid"] = valid
    return res


def gen_ckf():
    """CubatureKalmanFilter (CubatureKalmanFilter.py) banks: CV + range/az/el with missing measurements,
    linear models, user models (coordinated turn with fx_args, offset range/bearing with hx_args) and a
    sequence of split calls (update on a new filter, update without predict, update(None), scalar R)."""
    N, steps, dt = 16, 5, 0.1
    for name, linear in (("ckf_bank_rae", False), ("ckf_bank_lin", True)):
        w = wl.ukf_bank_cv3d(N, seed=2468, steps=steps, dt=dt, linear_hx=linear)
        w["dt"] = dt
        F, Hlin = w["F"], w["H"]
        fx = (lambda s, dt: F @ s) if linear else fx_cv
        hx = (lambda s: Hlin @ s) if linear else hx_rae
        valid = np.random.default_rng(3).random((steps, N)) >= (0.0 if linear else 0.1)
        save(name, **w, **_ckf_run(w, steps, fx, hx, valid))
    N, steps, dt = 16, 6, 0.5
    w = wl.ukf_bank_ct2d(N, steps=steps, dt=dt)
    w["dt"] = dt
    valid = np.random.default_rng(5).random((steps, N)) >= 0.1
    save("ckf_user_ct_rb", **w, **_ckf_run(w, steps, wl.ct_fx, wl.offset_rb_hx, valid, fx_args=w["omega"],
                                           hx_args=w["sensor"]))
    N, steps, dt = 8, len(CKF_OPS), 0.1
    w = wl.ukf_bank_cv3d(N, seed=97, steps=steps, dt=dt, linear_hx=True)
    w["dt"] = dt
    F, Hlin = w["F"], w["H"]
    valid = np.random.default_rng(6).random((steps, N)) >= 0.2
    save("ckf_call_order", **w, ops=np.array(CKF_OPS),
         **_ckf_run(w, steps, lambda s, dt: F @ s, lambda s: Hlin @ s, valid, ops=CKF_OPS))


if __name__ == "__main__":
    gen_ckf()
