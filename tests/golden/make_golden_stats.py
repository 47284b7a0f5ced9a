#!/usr/bin/env python
"""Generate the golden vectors of the stats evaluators (tests/golden/stats_*.npz) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_stats.py

Files (every value is one call of the reference):
  stats_mahalanobis      the inputs of the reference's test_stats.py::test_mahalanobis (its seeded random part with
                         S = A A' + I), its three docstring examples; c{i}_x / _mean / _cov / _out
  stats_bank_{n}_{m}     N tracks x[N, n], P, H[N, m, n], R and K candidates per track (z_own[N, K, m]) and one scan
                         shared by all (z_scan[K, m]); per pair log_likelihood, likelihood, mahalanobis(z, Hx, S) and
                         logpdf(z, Hx, S)
  stats_kf_methods       a KalmanFilter(4, 2) run: log_likelihood_of on candidates after predict (the stale S) and
                         after update, residual_of and measurement_of_state
  stats_nees             NEES over a batch_filter run against its ground truth
  stats_deviations       what scipy returns or raises where the kernel's rule differs: a singular S, S = 0 (before
                         the first update), an eigenvalue under scipy's cutoff, an indefinite S; and the raises of
                         mahalanobis (length mismatch, singular inv) and NEES (singular inv)
The tests never import the reference.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import save                                                            # noqa: E402

from filterpy.kalman import KalmanFilter                                                  # noqa: E402
from filterpy.stats import NEES, likelihood, log_likelihood, logpdf, mahalanobis          # noqa: E402


def _raises(fn):
    try:
        fn()
    except Exception as e:          # noqa: BLE001 - the type is the record
        return type(e).__name__
    return ""


def gen_mahalanobis():
    cases = [(3, 1, 2), ([3], [1], [2]), ([3], 1, 2), (3.123, 3.235235, .01234), ([3.123], [3.235235], [.01234]),
             ([3.123], 3.235235, .01234), (np.array([3.123]), 3.235235, .01234),
             (np.array([1., 2.]), np.array([1.4, 1.2]), np.array([[1., 2.], [2., 4.001]])),
             (np.array([[1., 2.]]), np.array([[1.4, 1.2]]), np.array([[1., 2.], [2., 4.001]])),
             (np.array([[1., 2.]]).T, np.array([[1.4, 1.2]]), np.array([[1., 2.], [2., 4.001]])),
             (3., 3.5, 4. ** 2), (3., 6, 1), ([1., 2], [1.1, 3.5], [[1., .1], [.1, 13]])]
    rng = np.random.default_rng(11)
    for _ in range(20):
        n = int(rng.integers(1, 20))
        A = rng.standard_normal((n, n))
        cases.append((rng.standard_normal(n), rng.standard_normal(n), A @ A.T + np.eye(n)))
    out = {"n_cases": len(cases)}
    for i, (x, mean, cov) in enumerate(cases):
        out["c%d_x" % i], out["c%d_mean" % i], out["c%d_cov" % i] = np.asarray(x, float), np.asarray(mean, float), \
            np.asarray(cov, float)
        out["c%d_out" % i] = mahalanobis(x, mean, cov)
    save("stats_mahalanobis", **out)


def _bank(n, m, N=48, K=7, seed=0):
    rng = np.random.default_rng(seed + 100 * n + m)
    x = rng.standard_normal((N, n))
    A = rng.standard_normal((N, n, n))
    P = A @ A.transpose(0, 2, 1) / n + np.eye(n)
    H = rng.standard_normal((N, m, n))
    B = rng.standard_normal((N, m, m))
    R = B @ B.transpose(0, 2, 1) / m + 0.5 * np.eye(m)
    z_own = np.einsum("fmn,fn->fm", H, x)[:, None, :] + rng.standard_normal((N, K, m)) * 2
    z_scan = rng.standard_normal((K, m)) * 3
    res = {}
    for lay, Z in (("own", z_own), ("scan", np.broadcast_to(z_scan, (N, K, m)))):
        ll, lk, ma, lp = (np.zeros((N, K)) for _ in range(4))
        for f in range(N):
            S = H[f] @ P[f] @ H[f].T + R[f]
            for k in range(K):
                z = Z[f, k]
                ll[f, k] = log_likelihood(z, x[f], P[f], H[f], R[f])
                lk[f, k] = likelihood(z, x[f], P[f], H[f], R[f])
                ma[f, k] = mahalanobis(z, H[f] @ x[f], S)
                lp[f, k] = logpdf(z, H[f] @ x[f], S)
        res.update({"ll_" + lay: ll, "lk_" + lay: lk, "maha_" + lay: ma, "logpdf_" + lay: lp})
    save("stats_bank_%d_%d" % (n, m), x=x, P=P, H=H, R=R, z_own=z_own, z_scan=z_scan, **res)


def gen_kf_methods(T=12, C=5):
    rng = np.random.default_rng(7)
    dt = 1.
    F = np.array([[1, dt, 0, 0], [0, 1, 0, 0], [0, 0, 1, dt], [0, 0, 0, 1.]])
    H = np.array([[1., 0, 0, 0], [0, 0, 1., 0]])
    Q = np.eye(4) * .02
    R = np.array([[.5, .1], [.1, .8]])
    kf = KalmanFilter(4, 2)
    kf.x = np.array([[0.], [1.], [0.], [-1.]])
    kf.P = np.eye(4) * 10.
    kf.F, kf.H, kf.Q, kf.R = F, H, Q, R
    x0, P0 = kf.x.copy(), kf.P.copy()
    zs = np.stack([np.array([t * 1., -t * 1.]) + rng.standard_normal(2) for t in range(1, T + 1)])
    cands = zs[:, None, :] + rng.standard_normal((T, C, 2)) * 1.5
    ll_pred, ll_upd = np.zeros((T, C)), np.zeros((T, C))
    res_pred, res_upd, mos = np.zeros((T, 2, 1)), np.zeros((T, 2, 1)), np.zeros((T, 2, 1))
    ll_before = kf.log_likelihood_of(cands[0, 0])          # S = 0 before the first update: -inf
    for t in range(T):
        kf.predict()
        ll_pred[t] = [kf.log_likelihood_of(c) for c in cands[t]]
        res_pred[t] = kf.residual_of(zs[t])
        mos[t] = kf.measurement_of_state(kf.x)
        kf.update(zs[t])
        ll_upd[t] = [kf.log_likelihood_of(c) for c in cands[t]]
        res_upd[t] = kf.residual_of(zs[t])
    save("stats_kf_methods", x0=x0, P0=P0, F=F, H=H, Q=Q, R=R, zs=zs, cands=cands, ll_pred=ll_pred, ll_upd=ll_upd,
         res_pred=res_pred, res_upd=res_upd, mos=mos, ll_before=ll_before, ll_none=kf.log_likelihood_of(None))


def gen_nees(T=40):
    rng = np.random.default_rng(8)
    kf = KalmanFilter(4, 2)
    kf.F = np.array([[1, 1., 0, 0], [0, 1, 0, 0], [0, 0, 1, 1.], [0, 0, 0, 1.]])
    kf.H = np.array([[1., 0, 0, 0], [0, 0, 1., 0]])
    kf.Q = np.eye(4) * .01
    kf.R = np.eye(2) * .3
    kf.P = np.eye(4) * 5.
    truth = np.zeros((T, 4))
    s = np.array([0., 1., 0., .5])
    for t in range(T):
        s = kf.F @ s + rng.standard_normal(4) * .1
        truth[t] = s
    zs = truth[:, [0, 2]] + rng.standard_normal((T, 2)) * .5
    mu, cov, _, _ = kf.batch_filter(list(zs[:, :, None]))
    xs = truth[:, :, None]
    nees = np.array(NEES(xs, mu, cov)).reshape(T)
    save("stats_nees", xs=xs, est_xs=mu, ps=cov, nees=nees)


def gen_deviations():
    z, mean = np.array([.3, -.2]), np.array([0., 0.])
    S_sing = np.array([[1., 1.], [1., 1.]])
    S_cut = np.diag([1., 1e-14])                 # under scipy's 1e6 * eps * max|lambda| cutoff
    S_indef = np.array([[1., 0.], [0., -2.]])
    save("stats_deviations", z=z, mean=mean, S_sing=S_sing, S_cut=S_cut, S_indef=S_indef,
         logpdf_sing=logpdf(z, mean, S_sing), logpdf_cut=logpdf(z, mean, S_cut),
         raise_indef=_raises(lambda: logpdf(z, mean, S_indef)),
         raise_len=_raises(lambda: mahalanobis([1], [1.4, 1.2], [[1., 2.], [2., 4.001]])),
         raise_maha_sing=_raises(lambda: mahalanobis(z, mean, S_sing)),
         raise_nees_sing=_raises(lambda: NEES(np.ones((2, 2)), np.zeros((2, 2)), np.stack([np.eye(2), S_sing]))))


if __name__ == "__main__":
    gen_mahalanobis()
    for n, m in ((1, 1), (2, 1), (4, 2), (6, 3), (9, 3)):
        _bank(n, m)
    gen_kf_methods()
    gen_nees()
    gen_deviations()
