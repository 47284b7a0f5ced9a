#!/usr/bin/env python
"""Generate the golden vectors of InformationFilter (tests/golden/if_*.npz) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_information.py

Every file is a bank of N reference filters with per-filter x, P_inv, F, F_inv, Q, H, R_inv (optionally B and
us[T,N,du]) and T steps of measurements zs[T,N,m] with valid[T,N] (False: ``update(None)``).  ``order`` is "pu"
(``predict()`` then ``update(z)``) or "up" (update first, as the reference's test_1d), ``compute_ll`` is the
filter's ``compute_log_likelihood``.  ``F_inv`` is the reference's ``_F_inv`` as the steps use it: ``inv(F)``,
or the stale inverse of ``F_set`` where ``F`` was edited in place afterwards.

The outputs are per step, ``out_*[T, N, ...]``: x, P_inv, ni (``_no_information``), ll, y, K, S, x_prior and
P_inv_prior.  Where the reference raises, ``raise_step[f]`` / ``raise_op[f]`` ("p" or "u") / ``raise_type[f]``
record where and what, and the state at the raise is repeated over the remaining steps (``raise_step`` is -1
for a filter that never raises).  The tests never import the reference.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import save                                                            # noqa: E402

from filterpy.kalman import InformationFilter                                            # noqa: E402
from filterpy_b200.common import workloads as wl                                          # noqa: E402

inv = np.linalg.inv


def _state(f, n, m):
    K = np.broadcast_to(np.asarray(f.K, np.float64), (n, m))
    S = np.broadcast_to(np.asarray(f.S, np.float64), (n, n))
    return dict(x=np.asarray(f.x, np.float64).reshape(-1), P_inv=np.asarray(f.P_inv, np.float64),
                ni=np.float64(f._no_information), ll=np.float64(f.log_likelihood),
                y=np.asarray(f.y, np.float64).reshape(-1), K=K.copy(), S=S.copy(),
                x_prior=np.asarray(f.x_prior, np.float64).reshape(-1), P_inv_prior=np.asarray(f.P_inv_prior, np.float64))


def run(name, w, order="pu", compute_ll=False, F_set=None, F_singular=None, **extra):
    """w: x, P_inv, F, Q, H, R_inv (per filter), zs, valid, optionally B, us.  F_set: the F assigned (then edited
    in place to w["F"]); F_singular: a singular F assigned after w["F"] (the setter raises, F_inv stays)."""
    N, n = w["x"].shape
    m = w["H"].shape[1]
    T = w["zs"].shape[0]
    keys = ("x", "P_inv", "ni", "ll", "y", "K", "S", "x_prior", "P_inv_prior")
    out = {k: np.zeros((T, N) + np.shape(_state(InformationFilter(n, m), n, m)[k])) for k in keys}
    raise_step, raise_op, raise_type = np.full(N, -1), np.full(N, "-", dtype="<U1"), np.full(N, "", dtype="<U16")
    F_inv = np.zeros((N, n, n))
    for f in range(N):
        flt = InformationFilter(n, m, dim_u=0 if "B" not in w else w["B"].shape[-1], compute_log_likelihood=compute_ll)
        flt.x = w["x"][f].reshape(n, 1).copy()
        flt.P_inv = w["P_inv"][f].copy()
        flt.Q, flt.H, flt.R_inv = w["Q"][f].copy(), w["H"][f].copy(), w["R_inv"][f].copy()
        if "B" in w:
            flt.B = w["B"][f].copy()
        if F_set is not None:
            flt.F = F_set[f].copy()
            flt.F[...] = w["F"][f]                     # in place: _F_inv stays inv(F_set)
        else:
            flt.F = w["F"][f].copy()
        if F_singular is not None:
            try:
                flt.F = F_singular[f].copy()
            except np.linalg.LinAlgError:
                pass
            else:
                raise AssertionError("F_singular is not singular")
        F_inv[f] = flt._F_inv
        st = None
        for t in range(T):
            if st is None:
                z = w["zs"][t, f].reshape(m, 1) if w["valid"][t, f] else None
                for op in order:
                    try:
                        if op == "p":
                            flt.predict(0 if "us" not in w else w["us"][t, f].reshape(-1, 1))
                        else:
                            flt.update(z)
                    except (np.linalg.LinAlgError, ValueError) as e:
                        raise_step[f], raise_op[f], raise_type[f] = t, op, type(e).__name__
                        st = _state(flt, n, m)
                        break
            s = st if st is not None else _state(flt, n, m)
            for k in keys:
                out[k][t, f] = s[k]
    F_rec = w["F"] if F_singular is None else F_singular
    save(name, order=np.array(order), compute_ll=np.array(compute_ll), F_inv=F_inv,
         raise_step=raise_step, raise_op=raise_op, raise_type=raise_type,
         **dict(w, F=F_rec), **extra, **({} if F_set is None else dict(F_set=F_set)),
         **({} if F_singular is None else dict(F_assigned=w["F"])),
         **{"out_" + k: v for k, v in out.items()})


def _valid(rng, T, N, p=0.2):
    v = rng.random((T, N)) >= p
    return v


def _bank(N, T, n, m, seed, du=0):
    """A random stable bank: F near I, H random, Q and R positive definite, P_inv = inv(P)."""
    rng = np.random.default_rng(seed)
    F = np.eye(n) + 0.1 * rng.standard_normal((N, n, n))
    H = rng.standard_normal((N, m, n))
    a = rng.standard_normal((N, n, n)); Q = 0.05 * (a @ a.transpose(0, 2, 1)) / n + 0.01 * np.eye(n)
    b = rng.standard_normal((N, m, m)); R = 0.5 * (b @ b.transpose(0, 2, 1)) / m + 0.1 * np.eye(m)
    c = rng.standard_normal((N, n, n)); P = (c @ c.transpose(0, 2, 1)) / n + np.eye(n)
    x = rng.standard_normal((N, n))
    zs = rng.standard_normal((T, N, m)) * 2.0
    w = dict(x=x, P_inv=inv(P), F=F, Q=Q, H=H, R_inv=inv(R), zs=zs, valid=_valid(rng, T, N))
    if du:
        w["B"] = rng.standard_normal((N, n, du))
        w["us"] = rng.standard_normal((T, N, du))
    return w


def _one(x, P_inv, F, Q, H, R_inv, zs):
    T = len(zs)
    m = np.shape(H)[0]
    return dict(x=np.array([x], np.float64), P_inv=np.array([P_inv], np.float64), F=np.array([F], np.float64),
                Q=np.array([Q], np.float64), H=np.array([H], np.float64), R_inv=np.array([R_inv], np.float64),
                zs=np.asarray(zs, np.float64).reshape(T, 1, m), valid=np.ones((T, 1), bool))


def _cv(N, T, seed, dt=None):
    c = wl.kf_bank_cv2d(N, seed=seed, steps=T)
    if dt is not None:                                 # a dyadic dt keeps the structural zeros exact
        c["F"][:, 0, 1] = c["F"][:, 2, 3] = dt
    return dict(x=c["x"], P_inv=inv(c["P"]), F=c["F"], Q=c["Q"], H=c["H"], R_inv=inv(c["R"]), zs=c["zs"])


def main():
    rng = np.random.default_rng(7)
    F1 = np.array([[1., 1.], [0., 1.]])
    H1 = np.array([[1., 0.]])
    # the reference tests' 2/1 cases (test_information.py)
    zs = np.arange(100) + rng.standard_normal(100) * 20
    run("if_test_1d", _one([2., 0.], np.eye(2), F1, np.eye(2) * 1e-4, H1, np.eye(1) / 5, zs), order="up", compute_ll=True)
    zs = np.arange(50) + rng.standard_normal(50) * np.sqrt(5)
    run("if_test_1d_0P", _one([2., 0.], np.eye(2) * 1e-21, F1, np.eye(2) * 1e-4, H1, np.eye(1) / 5, zs), compute_ll=True)
    zs = np.arange(1, 50) + rng.random(49) * .2
    run("if_test_against_kf", _one([0., 0.], np.eye(2), F1, np.array([[.25, .5], [.5, 1.]]), H1,
                                   inv(np.array([[.04]])), zs), compute_ll=True)
    # seeded constant-velocity banks with missing measurements
    w = _cv(64, 10, seed=11)
    w["valid"] = _valid(rng, 10, 64)
    run("if_cv_4_2", w)
    # the log-likelihood: m == n, and m == 1 (y broadcast over n)
    run("if_ll_2_2", _bank(32, 8, 2, 2, seed=21), compute_ll=True)
    run("if_ll_4_4", _bank(32, 8, 4, 4, seed=22), compute_ll=True)
    run("if_ll_2_1", _bank(32, 8, 2, 1, seed=23), compute_ll=True)
    run("if_bank_6_3", _bank(32, 6, 6, 3, seed=24))
    run("if_bank_9_3", _bank(16, 6, 9, 3, seed=25))
    run("if_ctrl_3_2", _bank(32, 6, 3, 2, seed=26, du=2))
    # no information: a 2/2 bank from P_inv = 0 with H = I (one step in the branch, informed from the next)
    w = _bank(16, 5, 2, 2, seed=27)
    w["P_inv"][:] = 0.
    w["H"][:] = np.eye(2)
    w["valid"][:] = True
    run("if_noinfo_2_2", w, compute_ll=True)
    # a 4/2 constant-velocity bank whose second axis starts with no information, H observing positions: that axis'
    # block of A stays rank-deficient, so every step takes the branch (and x grows)
    w = _cv(16, 5, seed=28, dt=0.5)
    w["P_inv"][:, 2:, :] = 0.
    w["P_inv"][:, :, 2:] = 0.
    w["R_inv"][:] = 4. * np.eye(2)
    w["Q"] = w["Q"] + 1e-3 * np.eye(4)                # full rank: A + Q stays invertible
    w["valid"] = np.ones((5, 16), bool)
    run("if_noinfo_4_2", w)
    # a stale F_inv: F assigned, then edited in place
    w = _cv(16, 5, seed=29)
    F_set = w["F"].copy()
    w["F"] = w["F"].copy()
    w["F"][:, 0, 1] *= 1.5
    w["F"][:, 2, 3] *= 1.5
    w["valid"] = _valid(rng, 5, 16)
    run("if_stale_F_inv", w, F_set=F_set)
    # the raising cases
    w = _cv(4, 4, seed=30)
    w["valid"] = np.ones((4, 4), bool)
    Fs = w["F"].copy()
    Fs[:, 1, :] = 0.                                   # singular F: the setter raises and keeps the old F_inv
    run("if_raise_F", w, F_singular=Fs)
    w = _one([1., 2.], np.eye(2), np.eye(2), -np.eye(2), H1, np.eye(1), [[3.], [4.]])
    run("if_raise_AIQ", w)                             # inv(AI + Q) = inv(0)
    w = _one([1., 2.], np.diag([0., 1.]), F1, np.eye(2), np.array([[0., 1.]]), np.eye(1), [[3.], [4.]])
    run("if_raise_S", w, order="up")                   # S = diag(0, 2)
    w = _cv(1, 2, seed=31)
    w["valid"] = np.ones((2, 1), bool)
    run("if_raise_ll_4_2", w, compute_ll=True)         # scipy cannot broadcast y (2) against the mean (4)


if __name__ == "__main__":
    main()
