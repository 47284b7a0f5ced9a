#!/usr/bin/env python
"""Generate the EnsembleKalmanFilter golden vectors (tests/golden/enkf_*.npz) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_enkf.py

The reference draws from NumPy's global generator through the module attribute
``filterpy.kalman.ensemble_kalman_filter.multivariate_normal``.  That one attribute is replaced by the
replica of the kernel's noise stream (``oracle/enkf.py``): filter f of a bank is one reference object whose
draws are ``mean + xi L'`` from the stream keyed with f, at the bank's draw-call index.  Nothing else of the
reference is touched.  The tests never import the reference.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import ROOT, save, fx_cv, hx_rae, wl                                    # noqa: E402

sys.path.insert(0, ROOT)
import filterpy.kalman.ensemble_kalman_filter as ek                                      # noqa: E402
from oracle.enkf import Stream                                                           # noqa: E402

SEED = 20261016
KEYS = ["x", "P", "x_prior", "P_prior", "K", "S", "SI", "sigmas"]
_cur = {"stream": None, "call": 0}


def _replica_mvn(mean, cov, size):
    return _cur["stream"].draw(_cur["call"], mean, cov, size)


ek.multivariate_normal = _replica_mvn


def _run(w, ops, N, fx, hx, valid, fx_args=None, hx_args=None):
    """Bank-level calls ``ops`` on one reference object per filter.  An op draws at the bank's call index
    (one index per initialize / predict / update of the bank, whether or not a filter's update is skipped
    by ``valid``) and the state of every filter is recorded after it."""
    F = w["x"].shape[0]
    m = w["R"].shape[-1]
    call = 0
    objs = []
    for f in range(F):
        _cur["stream"], _cur["call"] = Stream(SEED, f), call
        fa = (lambda s, dt, f=f: fx(s, dt, fx_args[f])) if fx_args is not None else fx
        ha = (lambda s: hx(s, *hx_args)) if hx_args is not None else hx
        e = ek.EnsembleKalmanFilter(x=w["x"][f].copy(), P=w["P"][f].copy(), dim_z=m, dt=float(w["dt"]), N=N, hx=ha, fx=fa)
        e.Q = w["Q"][f].copy()
        e.R = w["R"][f].copy()
        objs.append(e)
    call += 1
    out = {k: [] for k in KEYS}
    t_z = 0
    for t, op in enumerate(ops):
        if op.startswith("predict"):
            for f, e in enumerate(objs):
                _cur["stream"], _cur["call"] = Stream(SEED, f), call
                e.predict()
            call += 1
        upd = op.split("+")[-1]
        if upd.startswith("update"):
            for f, e in enumerate(objs):
                _cur["stream"], _cur["call"] = Stream(SEED, f), call
                z = w["zs"][t_z, f] if valid[t, f] else None
                R = 0.5 if upd == "update_R" else (w["Rcall"] if upd == "update_Rm" else None)
                e.update(z, R=R)
            call += 1
            t_z = min(t_z + 1, w["zs"].shape[0] - 1)
        elif upd == "none":
            for e in objs:
                e.update(None)
        for k in KEYS:
            out[k].append(np.array([np.array(getattr(e, k), dtype=float) for e in objs]))
    res = {"ref_" + k: np.array(v) for k, v in out.items()}
    res["valid"] = valid
    res["ops"] = np.array(ops)
    res["seed"] = np.uint32(SEED)
    res["n_members"] = N
    return res


def _cv2d(F, steps, seed):
    """4/2 constant velocity with a position sensor (the coordinated-turn workload's geometry)."""
    w = wl.ukf_bank_ct2d(F, seed=seed, steps=steps, dt=0.5, linear_hx=True)
    w["dt"] = 0.5
    return w


def gen_enkf():
    steps = 5
    ops = ["predict+update"] * steps
    lin = lambda H: (lambda s: H @ s)                                                     # noqa: E731

    # ConstVel 4/2 + LinearHx, N = 33, missing measurements
    w = _cv2d(6, steps, 11)
    valid = np.random.default_rng(1).random((steps, 6)) >= 0.2
    save("enkf_cv_lin", **w, **_run(w, ops, 33, fx_cv, lin(w["H"]), valid))

    # 6/3 CV + range / azimuth / elevation, N = 8
    w = wl.ukf_bank_cv3d(6, seed=2468, steps=steps, dt=0.1)
    w["dt"] = 0.1
    valid = np.ones((steps, 6), bool)
    save("enkf_cv_rae", **w, **_run(w, ops, 8, fx_cv, hx_rae, valid))

    # user models: coordinated turn (per-filter omega) + offset range / bearing, N = 33
    w = wl.ukf_bank_ct2d(6, steps=steps, dt=0.5)
    w["dt"] = 0.5
    valid = np.random.default_rng(2).random((steps, 6)) >= 0.1
    save("enkf_user_ct_rb", **w, **_run(w, ops, 33, wl.ct_fx, wl.offset_rb_hx, valid, fx_args=w["omega"], hx_args=w["sensor"]))

    # call order: update right after initialize, two updates in a row, update(None) after a predict,
    # scalar R and a per-call R matrix; N = 8
    co = ["update", "update", "predict+none", "predict+update_R", "predict+update_Rm", "predict+update"]
    w = _cv2d(6, len(co), 13)
    w["Rcall"] = np.array([[2.0, 0.3], [0.3, 1.5]])
    valid = np.random.default_rng(3).random((len(co), 6)) >= 0.2
    save("enkf_call_order", **w, **_run(w, co, 8, fx_cv, lin(w["H"]), valid))

    # rank-deficient Q (one rank-1 block per axis) and Q = 0 on half the filters; N = 2
    w = _cv2d(6, steps, 17)
    w["Q"][3:] = 0.0
    valid = np.ones((steps, 6), bool)
    save("enkf_rank_q", **w, **_run(w, ops, 2, fx_cv, lin(w["H"]), valid))

    # N = 256, 3 epochs
    w = _cv2d(3, 3, 19)
    valid = np.ones((3, 3), bool)
    save("enkf_n256", **w, **_run(w, ["predict+update"] * 3, 256, fx_cv, lin(w["H"]), valid))


if __name__ == "__main__":
    gen_enkf()
