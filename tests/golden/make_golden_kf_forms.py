#!/usr/bin/env python
"""Generate the golden vectors of KalmanFilter.update_sequential and update_correlated
(tests/golden/kf_forms_*.npz) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_kf_forms.py

Every file is a bank of N reference filters with per-filter models x, P, F, Q, H, R (and M) and T steps of
measurements zs[T,N,m] with valid[T,N]: each step is ``predict()`` followed by

* ``seq`` files: ``update_sequential(starts[k], z[starts[k]:starts[k]+lens[k]], R_i, H_i)`` for each block k,
  where ``Ri_k`` / ``Hi_k`` (when present) are the caller's R_i (a scalar or [N,L,L]) and H_i ([N,L,n]); a filter
  without a measurement (valid = False) skips the blocks;
* ``corr`` files: ``update_correlated(z or None)`` with the cross-correlation ``M``.

The outputs are the final ``out_*`` attributes; ``out_status`` is 1 where the reference raised LinAlgError
(the state is then the prior of that step); ``out_ll`` is NaN there and where scipy refuses the S.
``upd_x`` / ``upd_P`` are the same bank stepped with ``update``.  The tests never import the reference.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import save                                                            # noqa: E402

from filterpy.kalman import KalmanFilter                                                 # noqa: E402
from filterpy.common import Q_discrete_white_noise                                       # noqa: E402
from scipy.linalg import block_diag                                                      # noqa: E402


def _filter(w, f):
    n, m = w["x"].shape[1], w["H"].shape[1]
    kf = KalmanFilter(n, m)
    kf.x = w["x"][f].reshape(n, 1).copy(); kf.P = w["P"][f].copy()
    kf.F, kf.Q, kf.H, kf.R = w["F"][f], w["Q"][f], w["H"][f], w["R"][f]
    if "M" in w:
        kf.M = w["M"][f]
    return kf


def _z_rec(z):
    return np.array([np.nan if v is None else float(v) for v in np.asarray(z).reshape(-1)])


def run_seq(name, w, starts, lens, blocks=None, with_update=False):
    blocks = blocks or {}
    N, n = w["x"].shape
    m = w["H"].shape[1]
    T = w["zs"].shape[0]
    out = {k: [] for k in ("x", "P", "y", "K", "z")}
    upd_x, upd_P = [], []
    for f in range(N):
        kf = _filter(w, f)
        for t in range(T):
            kf.predict()
            if not w["valid"][t, f]:
                continue
            z = w["zs"][t, f]
            for k, (s, L) in enumerate(zip(starts, lens)):
                Ri = blocks.get("Ri_%d" % k)
                Hi = blocks.get("Hi_%d" % k)
                Ri = None if Ri is None else (float(Ri) if np.ndim(Ri) == 0 else Ri[f])
                Hi = None if Hi is None else Hi[f]
                kf.update_sequential(s, z[s:s + L], R_i=Ri, H_i=Hi)
        for k, v in (("x", kf.x.reshape(-1)), ("P", kf.P), ("y", kf.y.reshape(-1)), ("K", kf.K), ("z", _z_rec(kf.z))):
            out[k].append(np.array(v, dtype=np.float64))
        if with_update:
            ku = _filter(w, f)
            for t in range(T):
                ku.predict()
                ku.update(w["zs"][t, f] if w["valid"][t, f] else None)
            upd_x.append(ku.x.reshape(-1).copy()); upd_P.append(ku.P.copy())
    extra = dict(upd_x=np.array(upd_x), upd_P=np.array(upd_P)) if with_update else {}
    save(name, kind="seq", starts=np.array(starts), lens=np.array(lens), **w, **blocks,
         **{"out_" + k: np.array(v) for k, v in out.items()}, **extra)


def run_corr(name, w):
    N, n = w["x"].shape
    T = w["zs"].shape[0]
    out = {k: [] for k in ("x", "P", "y", "K", "S", "SI", "ll", "status")}
    for f in range(N):
        kf = _filter(w, f)
        status = 0
        for t in range(T):
            kf.predict()
            try:
                kf.update_correlated(w["zs"][t, f] if w["valid"][t, f] else None)
            except np.linalg.LinAlgError:
                status = 1
        try:
            ll = kf.log_likelihood if status == 0 else np.nan
        except ValueError:          # scipy's logpdf refuses an S that is not positive semidefinite
            ll = np.nan
        for k, v in (("x", kf.x.reshape(-1)), ("P", kf.P), ("y", kf.y.reshape(-1)), ("K", kf.K), ("S", kf.S),
                     ("SI", kf.SI), ("ll", ll), ("status", status)):
            out[k].append(np.array(v, dtype=np.float64))
    save(name, kind="corr", **w, **{"out_" + k: np.array(v) for k, v in out.items()})


def _spd(rng, N, k, scale):
    A = rng.normal(size=(N, k, k)) * scale
    return np.matmul(A, np.swapaxes(A, 1, 2)) + scale * scale * np.eye(k)


def random_bank(n, m, N, T, seed, none_frac=0.0):
    """Per-filter models: a constant-velocity-like F with per-filter dt, random SPD P, Q, R, a random H."""
    rng = np.random.default_rng(seed)
    dt = rng.uniform(0.05, 0.5, size=N)
    F = np.repeat(np.eye(n)[None], N, 0)
    for i in range(n - 1):
        F[:, i, i + 1] = dt
    w = dict(x=rng.normal(size=(N, n)), P=_spd(rng, N, n, 1.0), F=F, Q=_spd(rng, N, n, 0.1),
             H=rng.normal(size=(N, m, n)), R=_spd(rng, N, m, 0.5))
    w["zs"] = rng.normal(size=(T, N, m)) * 2.0
    w["valid"] = rng.random((T, N)) >= none_frac
    return w


def cv63_bank(N=16, T=12, seed=7, R_std=1.0, dt=0.5):
    """The 6/3 constant-velocity bank of the reference's test_kf.py:255-343 (three independent axes)."""
    rng = np.random.default_rng(seed)
    F1 = np.array([[1., dt], [0., 1.]])
    q = Q_discrete_white_noise(dim=2, dt=dt, var=0.0001)
    h = np.array([[1., 0.]])
    rep = lambda a: np.repeat(np.asarray(a, np.float64)[None], N, 0)          # noqa: E731
    w = dict(x=np.zeros((N, 6)), P=rep(np.eye(6)), F=rep(block_diag(F1, F1, F1)), Q=rep(block_diag(q, q, q)),
             H=rep(block_diag(h, h, h)), R=rep(np.eye(3) * R_std ** 2))
    v = np.array([3.0, 4.0, 5.0])
    t = np.arange(T)[:, None, None]
    w["zs"] = v * t + rng.normal(size=(T, N, 3)) * 20
    w["valid"] = np.ones((T, N), bool)
    return w


def main():
    # the reference test's splittings against update()
    for tag, starts, lens in (("111", [0, 1, 2], [1, 1, 1]), ("12", [0, 1], [1, 2]), ("21", [0, 2], [2, 1])):
        run_seq("kf_forms_seq_cv63_" + tag, cv63_bank(), starts, lens, with_update=True)
    # seeded per-filter banks with missing measurements
    run_seq("kf_forms_seq_4_2", random_bank(4, 2, 24, 5, seed=11, none_frac=0.25), [0, 1], [1, 1])
    run_seq("kf_forms_seq_6_3", random_bank(6, 3, 24, 4, seed=12, none_frac=0.25), [0, 2], [2, 1])
    # caller-supplied R_i / H_i: a scalar R_i, per-filter H_i and R_i
    w = random_bank(4, 2, 16, 3, seed=13)
    rng = np.random.default_rng(14)
    blocks = dict(Ri_0=np.array(0.7), Hi_1=rng.normal(size=(16, 1, 4)), Ri_1=_spd(rng, 16, 1, 0.5))
    run_seq("kf_forms_seq_given", w, [0, 1], [1, 1], blocks)
    w = random_bank(4, 4, 16, 2, seed=15)
    blocks = dict(Hi_0=rng.normal(size=(16, 3, 4)), Ri_0=_spd(rng, 16, 3, 0.5), Ri_1=np.array(0.3))
    run_seq("kf_forms_seq_given_4_4", w, [0, 3], [3, 1], blocks)
    # an L = 1 block with S_i = 0: a zero row of H and a zero R_i give inf / nan, no LinAlgError
    w = random_bank(2, 2, 4, 1, seed=16)
    blocks = dict(Hi_0=np.zeros((4, 1, 2)), Ri_0=np.array(0.0))
    run_seq("kf_forms_seq_s0", w, [0], [1], blocks)

    # the reference's test_update_correlated (test_kf.py:720-726): 2/1, M = [[1], [0]], z = 3
    dt = 1.0
    w = dict(x=np.array([[2., 0.]]), P=np.eye(2)[None].copy(), F=np.array([[[1., dt], [0., 1.]]]),
             Q=Q_discrete_white_noise(2, dt, 5.1)[None], H=np.array([[[1., 0.]]]), R=np.eye(1)[None].copy(),
             M=np.array([[[1.], [0.]]]), zs=np.full((10, 1, 1), 3.), valid=np.ones((10, 1), bool))
    run_corr("kf_forms_corr_2_1", w)
    # a per-filter 4/2 bank with per-filter M and missing measurements
    w = random_bank(4, 2, 24, 5, seed=21, none_frac=0.25)
    w["M"] = np.random.default_rng(22).normal(size=(24, 4, 2)) * 0.1
    run_corr("kf_forms_corr_4_2", w)
    # a singular S: H = 0 and a singular R in the even filters
    w = random_bank(2, 2, 8, 1, seed=23)
    w["H"][::2] = 0.0
    w["R"][::2] = np.array([[1., 1.], [1., 1.]])
    w["M"] = np.random.default_rng(24).normal(size=(8, 2, 2)) * 0.1
    run_corr("kf_forms_corr_singular", w)


if __name__ == "__main__":
    main()
