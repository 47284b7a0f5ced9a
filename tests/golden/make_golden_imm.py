#!/usr/bin/env python
"""Golden vectors for IMMEstimator.batch_filter (tests/golden/imm_batch_*.npz) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref``:

    python tests/golden/make_golden_imm.py

The reference's IMMEstimator has no batch_filter; each file records its ``predict(); update(z or None)`` loop,
one IMMEstimator per track, so every track may have its own models.  Per case: the inputs (zs[T,N,m],
valid[T,N], trans, mu0, the per-track models F, Q [N,M,n,n] with their own dt, H, R, alpha [M], the initial
states x0 [N,M,n], P0 [N,M,n,n]) and per epoch the estimator's x, P, x_prior (xp), P_prior (Pp), mu, cbar,
omega, likelihood (lik) and every model's x, P (fx, fP).  About 20 % of the measurements are missed, track 0
misses epoch 0 (its models' S is still zero then).  Seeded.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

from filterpy.kalman import IMMEstimator, KalmanFilter  # noqa: E402
import filterpy                                         # noqa: E402

# (name, models, dim_x, dim_z, epochs, tracks, alpha of each model); 5/2 has no fused instance
CASES = [("m2_4_2", 2, 4, 2, 40, 5, (1.0, 1.0)),
         ("m3_4_2", 3, 4, 2, 40, 5, (1.0, 1.0, 1.05)),
         ("m4_4_2", 4, 4, 2, 40, 5, (1.0, 1.0, 1.0, 1.0)),
         ("m3_6_3", 3, 6, 3, 12, 5, (1.0, 1.0, 1.0)),
         ("m2_2_1", 2, 2, 1, 20, 6, (1.0, 1.02)),
         ("m3_3_1", 3, 3, 1, 20, 6, (1.0, 1.0, 1.0)),
         ("m2_5_2", 2, 5, 2, 12, 5, (1.0, 1.0))]
QS = [0.05, 1.0, 8.0, 0.3]


def models(n, m, dt, q):
    """Constant velocity on m axes (n = 2m, H picks the positions), constant acceleration on one axis (3/1), or
    2-D constant velocity with a measured bias on the first axis (5/2)."""
    cv = np.array([[1.0, dt], [0.0, 1.0]])
    qcv = np.array([[dt ** 3 / 3, dt ** 2 / 2], [dt ** 2 / 2, dt]])
    if n == 3:
        F = np.array([[1.0, dt, dt * dt / 2], [0.0, 1.0, dt], [0.0, 0.0, 1.0]])
        H = np.array([[1.0, 0.0, 0.0]])
        Q = np.array([[dt ** 5 / 20, dt ** 4 / 8, dt ** 3 / 6], [dt ** 4 / 8, dt ** 3 / 3, dt ** 2 / 2],
                      [dt ** 3 / 6, dt ** 2 / 2, dt]])
    elif n == 5:
        F = np.eye(5); F[:4, :4] = np.kron(np.eye(2), cv)
        H = np.array([[1.0, 0.0, 0.0, 0.0, 1.0], [0.0, 0.0, 1.0, 0.0, 0.0]])
        Q = np.zeros((5, 5)); Q[:4, :4] = np.kron(np.eye(2), qcv); Q[4, 4] = 0.01 * dt
    else:
        F = np.kron(np.eye(m), cv)
        H = np.kron(np.eye(m), np.array([[1.0, 0.0]]))
        Q = np.kron(np.eye(m), qcv)
    return F, H, Q * q


def gen(ci, name, nm, n, m, T, NT, alphas):
    rng = np.random.default_rng(900 + ci)
    dts = rng.uniform(0.5, 1.5, NT)
    F = np.zeros((NT, nm, n, n)); Q = np.zeros((NT, nm, n, n))
    for i in range(NT):
        for j in range(nm):
            F[i, j], H, Q[i, j] = models(n, m, dts[i], QS[j])
    R = np.eye(m) * 0.5
    x0 = rng.normal(size=(NT, nm, n)) * 3
    P0 = np.array([[np.diag(rng.uniform(1, 5, n)) for _ in range(nm)] for _ in range(NT)])
    zs = rng.normal(size=(T, NT, m)) * 2 + np.cumsum(rng.normal(size=(T, NT, m)), axis=0)
    valid = rng.random((T, NT)) >= 0.2
    valid[0, 0] = False
    trans = np.full((nm, nm), 0.1 / (nm - 1)) + np.eye(nm) * (0.9 - 0.1 / (nm - 1))
    mu0 = np.arange(nm, 0, -1.0) / np.sum(np.arange(nm, 0, -1.0))
    shp = dict(x=(n,), P=(n, n), xp=(n,), Pp=(n, n), mu=(nm,), cbar=(nm,), omega=(nm, nm), lik=(nm,),
               fx=(nm, n), fP=(nm, n, n))
    rec = {k: np.zeros((T, NT) + s) for k, s in shp.items()}
    for i in range(NT):
        fs = []
        for j in range(nm):
            f = KalmanFilter(n, m)
            f.x = x0[i, j].copy(); f.P = P0[i, j].copy()
            f.F, f.H, f.R, f.Q = F[i, j], H, R, Q[i, j]
            f.alpha = alphas[j]
            fs.append(f)
        imm = IMMEstimator(fs, mu0, trans)
        for k in range(T):
            imm.predict()
            rec["xp"][k, i] = imm.x; rec["Pp"][k, i] = imm.P
            imm.update(zs[k, i] if valid[k, i] else None)
            rec["x"][k, i] = imm.x; rec["P"][k, i] = imm.P; rec["mu"][k, i] = imm.mu
            rec["cbar"][k, i] = imm.cbar; rec["omega"][k, i] = imm.omega; rec["lik"][k, i] = imm.likelihood
            for j, f in enumerate(imm.filters):
                rec["fx"][k, i, j] = f.x; rec["fP"][k, i, j] = f.P
    path = os.path.join(HERE, "imm_batch_%s.npz" % name)
    np.savez_compressed(path, reference_version=filterpy.__version__, zs=zs, valid=valid, trans=trans, mu0=mu0,
                        F=F, Q=Q, H=H, R=R, alpha=np.array(alphas), x0=x0, P0=P0, **rec)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    for ci, c in enumerate(CASES):
        gen(ci, *c)
