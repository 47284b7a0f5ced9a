"""Oracle: multiple-model estimators over a list of linear Kalman filters (TEST INFRASTRUCTURE).

Restates, for ONE track (reference @ 3b51149):

* ``IMMEstimator``   filterpy/kalman/IMM.py:133-158 (init), :160-184 (update), :186-226 (predict),
  :228-237 (_compute_state_estimate), :239-247 (_compute_mixing_probabilities)
* ``MMAEFilterBank`` filterpy/kalman/mmae.py:140-153 (predict), :155-206 (update) — including the
  element-wise ``zip(self.x, self.filters, self.p)`` of :197-199, which pairs COMPONENT i of the
  mixed state with filter i.

Filters are plain dicts ``{x, P, F, H, Q, R}`` advanced with ``oracle.kf``; each also carries the S of
its last real update (zero before the first), because ``update(None)`` leaves it and the likelihood of
a missed measurement is ``logpdf(0; 0, S)`` of that S (kalman_filter.py:511-520, :1203-1210).
Everything fp64.

The ``*_bank`` functions restate the same three steps vectorised over N tracks — what ``csrc/mix.cu``
computes per launch: ``mm_probabilities_bank`` (IMM, MMAE and from-mu forms), ``mm_mix_bank`` and
``mm_estimate_bank`` (IMM and the MMAE ``zip``), with per-track or shared weights.

Parity: pinned by ``tests/golden/mm.npz`` and ``tests/golden/mm_missing.npz`` (generated from the
reference's own classes).
"""
import sys

import numpy as np

from . import kf as okf

FLOAT_MIN = sys.float_info.min


def likelihood(y, S):
    """kalman_filter.py:1203-1223: exp(logpdf(y; 0, S)), floored at float min.  ``y = None`` is the
    likelihood after ``update(None)``: y = 0 with the kept S, which may still be the zero matrix."""
    S = np.asarray(S, float)
    if y is None:
        ll = okf.missed_log_likelihood_bank(S[None])[0]
    else:
        ll = okf.log_likelihood_bank(np.asarray(y, float).reshape(1, -1), S[None])[0]
    lk = np.exp(ll)
    return lk if lk != 0 else FLOAT_MIN


def _with_kept_S(filters):
    for f in filters:
        m = np.shape(f["H"])[0]
        f.setdefault("S", np.zeros((m, m)))
    return filters


def _update_filter(f, z):
    """KalmanFilter.update(z) on one filter dict; returns the filter's likelihood."""
    if z is None:                                                              # kalman_filter.py:515-520
        return likelihood(None, f["S"])
    x, P, y, K, S, SI = okf.kf_update_single(f["x"], f["P"], np.asarray(z, float), f["H"], f["R"])
    f["x"], f["P"], f["S"] = x, P, S
    return likelihood(y, S)


class Imm(object):
    def __init__(self, filters, mu, M):
        self.filters = _with_kept_S(filters)
        self.mu = np.asarray(mu, float) / np.sum(mu)
        self.M = np.asarray(M, float)
        self.N = len(filters)
        self.likelihood = np.zeros(self.N)
        self.omega = np.zeros((self.N, self.N))
        self._mixing_probabilities()
        self._state_estimate()

    def _mixing_probabilities(self):
        self.cbar = np.dot(self.mu, self.M)                                    # IMM.py:244
        for i in range(self.N):
            for j in range(self.N):
                self.omega[i, j] = (self.M[i, j] * self.mu[i]) / self.cbar[j]  # :247

    def _state_estimate(self):
        self.x = np.zeros_like(self.filters[0]["x"])
        for f, mu in zip(self.filters, self.mu):
            self.x += f["x"] * mu                                              # :232-233
        self.P = np.zeros_like(self.filters[0]["P"])
        for f, mu in zip(self.filters, self.mu):
            y = f["x"] - self.x
            self.P += mu * (np.outer(y, y) + f["P"])                           # :235-237

    def update(self, z):
        for i, f in enumerate(self.filters):
            self.likelihood[i] = _update_filter(f, z)                          # :174-176
        self.mu = self.cbar * self.likelihood                                  # :179
        self.mu /= np.sum(self.mu)
        self._mixing_probabilities()
        self._state_estimate()

    def predict(self):
        xs, Ps = [], []
        for i, (f, w) in enumerate(zip(self.filters, self.omega.T)):           # :201
            x = np.zeros_like(self.x)
            for kf, wj in zip(self.filters, w):
                x += kf["x"] * wj
            xs.append(x)
            P = np.zeros_like(self.P)
            for kf, wj in zip(self.filters, w):
                y = kf["x"] - x
                P += wj * (np.outer(y, y) + kf["P"])
            Ps.append(P)
        for i, f in enumerate(self.filters):                                   # :215-220
            f["x"], f["P"] = okf.kf_predict_single(xs[i].copy(), Ps[i].copy(), f["F"], f["Q"])
        self._state_estimate()


class Mmae(object):
    def __init__(self, filters, p):
        self.filters = _with_kept_S(filters)
        self.p = np.asarray(p, float).copy()
        self.likelihood = np.zeros(len(filters))
        self.x = filters[0]["x"].copy()
        self.P = filters[0]["P"].copy()

    def predict(self):
        for f in self.filters:
            f["x"], f["P"] = okf.kf_predict_single(f["x"], f["P"], f["F"], f["Q"])

    def update(self, z):
        for i, f in enumerate(self.filters):
            self.likelihood[i] = _update_filter(f, z)
            self.p[i] *= self.likelihood[i]                                    # mmae.py:182
        self.p /= sum(self.p)
        self.P = np.zeros(self.filters[0]["P"].shape)
        self.x = np.zeros(self.filters[0]["x"].shape)
        for f, p in zip(self.filters, self.p):
            self.x += np.dot(f["x"], p)                                        # :191-192
        for x, f, p in zip(self.x, self.filters, self.p):                      # :197 (components of x!)
            y = f["x"] - x
            self.P += p * (np.outer(y, y) + f["P"])


# --------------------------------------------------------------------------- bank forms
def _weights(w, N, shape):
    """per-track weights (N, *shape), or one set shared by the bank (*shape) -> (N, *shape)."""
    w = np.asarray(w, float)
    return np.broadcast_to(w, (N,) + shape) if w.shape == shape else w


def mm_probabilities_bank(mu, ll=None, cbar=None, trans=None, mmae=False):
    """Mode probabilities for N tracks of M models.  ``mu``, ``cbar`` (N, M), ``ll`` (N, M) log-likelihoods
    (None: keep ``mu``, the ``from_mu`` form), ``trans`` (M, M).
    IMM:  mu = cbar L / sum(cbar L) (IMM.py:178-180), then cbar = mu . trans and
          omega[i, j] = trans[i, j] mu[i] / cbar[j] (:239-247).  Returns (mu, cbar, omega).
    MMAE: mu = mu L / sum(mu L) (mmae.py:180-184).  Returns mu.
    L = exp(ll) floored at float min (kalman_filter.py:1213-1223)."""
    mu = np.asarray(mu, float)
    if ll is not None:
        L = np.exp(np.asarray(ll, float))
        L = np.where(L == 0.0, FLOAT_MIN, L)
        mu = (mu if mmae else np.asarray(cbar, float)) * L
        mu = mu / np.sum(mu, axis=1, keepdims=True)
    if mmae:
        return mu
    trans = np.asarray(trans, float)
    cb = mu @ trans
    omega = trans[None] * mu[:, :, None] / cb[:, None, :]
    return mu, cb, omega


def mm_mix_bank(xs, Ps, omega):
    """Mixed initial conditions (IMM.py:201-213) for N tracks: ``xs`` (M, N, n), ``Ps`` (M, N, n, n),
    ``omega`` (N, M, M) or shared (M, M).  Returns x0 (M, N, n), P0 (M, N, n, n):
    x0_i = sum_j omega[j, i] x_j,  P0_i = sum_j omega[j, i] ((x_j - x0_i)(x_j - x0_i)' + P_j)."""
    xs, Ps = np.asarray(xs, float), np.asarray(Ps, float)
    M, N, n = xs.shape
    w = _weights(omega, N, (M, M))
    x0 = np.einsum("nji,jnc->inc", w, xs)
    d = xs[None] - x0[:, None]                                   # [i, j, N, n]
    P0 = np.einsum("nji,ijnr,ijnc->inrc", w, d, d) + np.einsum("nji,jnrc->inrc", w, Ps)
    return x0, P0


def mm_estimate_bank(xs, Ps, mu, mmae=False):
    """Combined estimate for N tracks: ``xs`` (M, N, n), ``Ps`` (M, N, n, n), ``mu`` (N, M) or shared (M,).
    IMM (IMM.py:228-237): x = sum_j mu_j x_j, P = sum_j mu_j ((x_j - x)(x_j - x)' + P_j).
    MMAE (mmae.py:186-199): the same x; P sums over the reference's ``zip(self.x, self.filters, self.p)``,
    so term j (j < min(n, M)) uses y = x_j - x[j], component j of the combined state, a scalar."""
    xs, Ps = np.asarray(xs, float), np.asarray(Ps, float)
    M, N, n = xs.shape
    w = _weights(mu, N, (M,))
    x = np.einsum("nj,jnc->nc", w, xs)
    if not mmae:
        d = xs - x[None]
        P = np.einsum("nj,jnr,jnc->nrc", w, d, d) + np.einsum("nj,jnrc->nrc", w, Ps)
        return x, P
    P = np.zeros((N, n, n))
    for j in range(min(n, M)):
        d = xs[j] - x[:, j:j + 1]
        P += w[:, j, None, None] * (d[:, :, None] * d[:, None, :] + Ps[j])
    return x, P
