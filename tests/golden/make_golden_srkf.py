#!/usr/bin/env python
"""Generate the SquareRootKalmanFilter golden vectors (tests/golden/srkf_*.npz) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_srkf.py

It uses ``save`` and the reference import of ``make_golden.py`` and the seeded workloads of
``filterpy_b200.common.workloads``.  The reference's own ``qr`` is wrapped (not changed) to assert that no Householder
pivot of any case is within 1e-5 of zero relative to its column's norm, and that no sub-column below a pivot
is either (except in the ill-conditioned case, whose sub-columns are genuinely that small: sqrt(q / p0)), so
that fp32 rounding cannot flip the sign of a row of P1_2.  The tests never import the reference.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import save, wl                                                          # noqa: E402
from oracle import srkf as osr                                                           # noqa: E402

import filterpy.kalman.square_root as _sr                                                # noqa: E402
from filterpy.kalman import SquareRootKalmanFilter                                       # noqa: E402

KEYS = ["x", "P", "P1_2", "x_prior", "P_prior", "P1_2_prior", "P_post", "K", "y", "S1_2", "SI1_2", "S", "SI"]
# the call-order case: what each step does (tests/test_gpu_srkf.py and tests/test_oracle_srkf.py replay it)
CALL_ORDER = ["update_R0", "update", "set_H+predict+update", "update", "predict+predict+update", "predict+none",
              "predict+update_Rs", "predict+update_Rm"]
R2_SCALAR = 0.7
MIN_PIVOT = 1e-5

_qr = _sr.qr
_worst = [1.0, 1.0]          # smallest pivot ratio, smallest sub-column ratio of the current case


def _checked_qr(a, *args, **kw):
    ra, rs = osr.dgeqr2_pivot_ratio(np.asarray(a, np.float64))
    _worst[0], _worst[1] = min(_worst[0], ra), min(_worst[1], rs)
    return _qr(a, *args, **kw)


def _save(name, check_sub=True, **arrs):
    assert _worst[0] > MIN_PIVOT and (_worst[1] > MIN_PIVOT or not check_sub), (name, _worst)
    print("  %s: smallest pivot ratio %.2e, sub-column ratio %.2e" % (name, _worst[0], _worst[1]))
    _worst[:] = [1.0, 1.0]
    save(name, **arrs)


_sr.qr = _checked_qr


def _record(s, n, m):
    return dict(x=np.array(s.x, float).reshape(n), P=s.P, P1_2=s.P1_2, x_prior=np.array(s.x_prior, float).reshape(n),
                P_prior=s.P_prior, P1_2_prior=s._P1_2_prior, P_post=s.P_post, K=s.K, y=np.array(s.y, float).reshape(m),
                S1_2=s.S1_2, SI1_2=s.SI1_2, S=s.S, SI=s.SI)


def _per(a, f, N):
    """filter f's copy of a model given per filter ([N, ...]) or shared."""
    a = np.asarray(a)
    return a[f] if a.ndim == 3 and a.shape[0] == N else a


def run(w, valid, ops=None, rec_steps=None, R2m=None):
    """Drive one reference object per filter through the steps; returns the ref_* arrays."""
    N, n = w["x"].shape
    m = np.shape(w["H"])[-2]
    T = w["zs"].shape[0]
    rec_steps = list(range(T)) if rec_steps is None else list(rec_steps)
    flt = []
    for f in range(N):
        s = SquareRootKalmanFilter(n, m, 0 if "B" not in w else w["B"].shape[-1])
        s.x = w["x"][f].copy()[:, None]
        s.P = w["P"][f].copy(); s.Q = _per(w["Q"], f, N); s.R = _per(w["R"], f, N)
        s.F = _per(w["F"], f, N).copy()
        if ops is None:
            s.H = _per(w["H"], f, N).copy()
        if "B" in w:
            s.B = w["B"].copy()
        flt.append(s)
    out = {k: [] for k in KEYS}
    for t in range(T):
        op = ops[t] if ops is not None else "predict+update"
        rec = {k: [] for k in KEYS}
        for f, s in enumerate(flt):
            if op.startswith("set_H"):
                s.H = _per(w["H"], f, N).copy()
            for _ in range(op.count("predict")):
                if "us" in w:
                    s.predict(w["us"][t, f][:, None])
                else:
                    s.predict()
            z = w["zs"][t, f][:, None] if valid[t, f] and not op.endswith("none") else None
            if op.endswith("R0"):
                s.update(z, R2=0.)
            elif op.endswith("Rs"):
                s.update(z, R2=R2_SCALAR)
            elif op.endswith("Rm"):
                s.update(z, R2=R2m)
            else:
                s.update(z)
            if t in rec_steps:
                for k, v in _record(s, n, m).items():
                    rec[k].append(np.array(v, float))
        if t in rec_steps:
            for k in KEYS:
                out[k].append(np.array(rec[k]))
    res = {"ref_" + k: np.array(v) for k, v in out.items()}
    res["valid"] = valid
    res["rec_steps"] = np.array(rec_steps)
    return res


def gen():
    """The cases of DESIGN.md §4: a 4/2 CV bank with per-filter models and missing measurements, 6/3 and 9/3
    banks with shared models, 3/2 with a control input, 1/1, a call-order sequence and the ill-conditioned
    4/2 bank of the fp32 accuracy contrast."""
    N, T = 16, 8
    w = wl.kf_bank_cv2d(N, seed=321, steps=T)
    w["Q"] = osr.make_pd(w["Q"])
    valid = np.random.default_rng(1).random((T, N)) >= 0.15
    _save("srkf_bank_4_2", **w, **run(w, valid))

    u = wl.ukf_bank_cv3d(N, seed=654, steps=T, linear_hx=True)
    w = dict(x=u["x"], P=u["P"], F=u["F"], H=u["H"], Q=osr.make_pd(u["Q"][0]), R=u["R"][0], zs=u["zs"])
    _save("srkf_bank_6_3", **w, **run(w, np.ones((T, N), bool)))

    c = wl.kf_bank_ca3d(N, seed=987, steps=T)
    w = dict(x=c["x"], P=c["P"], F=c["F"][0], H=c["H"][0], Q=osr.make_pd(c["Q"][0]), R=c["R"][0], zs=c["zs"])
    valid = np.random.default_rng(2).random((T, N)) >= 0.1
    _save("srkf_bank_9_3", **w, **run(w, valid))

    rng = np.random.default_rng(3)
    F = np.eye(3) + 0.1 * rng.standard_normal((3, 3))
    A = rng.standard_normal((N, 3, 3))
    w = dict(x=rng.standard_normal((N, 3)), P=A @ np.swapaxes(A, 1, 2) + np.eye(3), F=F,
             H=rng.standard_normal((2, 3)), Q=0.01 * np.eye(3) + 0.005 * np.ones((3, 3)),
             R=np.array([[0.5, 0.1], [0.1, 0.3]]), B=np.array([[0.5], [1.0], [0.2]]),
             us=rng.standard_normal((T, N, 1)), zs=rng.standard_normal((T, N, 2)))
    _save("srkf_ctrl_3_2", **w, **run(w, np.ones((T, N), bool)))

    w = dict(x=rng.standard_normal((N, 1)), P=rng.uniform(0.5, 5.0, (N, 1, 1)), F=rng.uniform(0.8, 1.2, (N, 1, 1)),
             H=rng.uniform(0.5, 2.0, (N, 1, 1)), Q=rng.uniform(0.01, 0.1, (N, 1, 1)), R=rng.uniform(0.1, 1.0, (N, 1, 1)),
             zs=rng.standard_normal((T, N, 1)))
    _save("srkf_bank_1_1", **w, **run(w, np.random.default_rng(4).random((T, N)) >= 0.2))

    N = 4
    T = len(CALL_ORDER)
    w = wl.kf_bank_cv2d(N, seed=77, steps=T)
    w["Q"] = osr.make_pd(w["Q"])
    R2m = np.array([[0.8, 0.0], [0.0, 0.6]])
    _save("srkf_call_order", **w, ops=np.array(CALL_ORDER), R2m=R2m, R2s=R2_SCALAR,
         **run(w, np.ones((T, N), bool), ops=CALL_ORDER, R2m=R2m))

    w = osr.ill_conditioned_bank()
    T = w["zs"].shape[0]
    rec = [t for t in range(T) if t < 5 or t % 50 == 49]
    _save("srkf_ill_4_2", check_sub=False, **w, **run(w, np.ones((T, w["x"].shape[0]), bool), rec_steps=rec))


if __name__ == "__main__":
    gen()
