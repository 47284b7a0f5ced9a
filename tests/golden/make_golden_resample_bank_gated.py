#!/usr/bin/env python
"""Golden vectors of the gated bank resampler (``BankResamplePlan.resample_if_degenerate``,
``systematic_resample_bank_if_degenerate`` / ``stratified_resample_bank_if_degenerate``) from the
UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_resample_bank_gated.py

For each case it seeds NumPy and runs a particle filter's resampling step over the rows of a bank with the
reference's ``systematic_resample`` (then, reseeded, ``stratified_resample``)::

    w = w / np.sum(w); neff = 1. / np.sum(np.square(w))
    if neff < M / 2: particles[:] = particles[fn(w)]; w = np.full(M, 1. / M)

and stores the weights and particles before and after, neff, the mask, the indexes of resampled rows
(-1 elsewhere) and the next ``random()``, or the row the reference raised IndexError at.  The failing row
is the last row of its bank, so the stored state is the whole bank's.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

from filterpy.monte_carlo import systematic_resample, stratified_resample  # noqa: E402
import filterpy                                                            # noqa: E402

from filterpy_b200.common import workloads as wl                          # noqa: E402

KINDS = ["heavy", "uniform", "random", "zeros", "degenerate", "dyadic"]


def kinds_bank(B, M, seed):
    return np.stack([wl.resample_weights(M, KINDS[b % len(KINDS)], seed=seed * 1000 + b) for b in range(B)])


def special_bank(M, seed):
    """Rows of every kind, rows around the threshold M / 2 (M = 128: exactly at it too) and special values."""
    rng = np.random.default_rng(seed)
    rows = list(kinds_bank(len(KINDS), M, seed))
    for ones in (M // 2 - 1, M // 2, M // 2 + 1):        # neff = 63 (resamples), 64 (exactly M / 2: not), 65
        r = np.zeros(M)
        r[rng.permutation(M)[:ones]] = 1.0
        rows.append(r)
    rows.append(np.zeros(M))                             # 0 / 0: NaN weights and neff, not resampled
    r = rng.random(M); r[5] = np.nan; rows.append(r)
    r = rng.random(M); r[7] = np.inf; rows.append(r)     # inf / inf = NaN
    r = rng.random(M); r[2] = np.inf; r[9] = -np.inf; rows.append(r)
    r = np.full(M, -0.0); r[M // 2] = 1.0; rows.append(r)   # -0.0 / 1 = -0.0; neff = 1
    r = rng.random(M) ** 4; rows.append(2.0 * r / r.sum())    # sums to 2
    r = rng.random(M) ** 4; rows.append(1e-300 * r / r.sum())  # sums to 1e-300
    return np.stack(rows)


def failing_row(M):
    """A row whose np.sum-normalised sequential cumsum ends below (M - 1) / M, so that every u makes the
    reference raise: [-2^k, 2^k, p...].  The pairwise sum adds the p in the accumulators of -2^k and 2^k with
    the rounding of 2^k and comes out larger than the p's sum; the cumsum cancels the pair exactly first."""
    for seed in range(10000):
        rng = np.random.default_rng(seed)
        p = 2.0 * rng.random(M - 2)
        for k in range(50, 57):
            row = np.concatenate([[-2.0 ** k, 2.0 ** k], p])
            S = np.sum(row)
            if not (np.isfinite(S) and S > 0):
                continue
            w = row / S
            if np.cumsum(w)[-1] < (M - 1) / M - 1e-3 and 1. / np.sum(np.square(w)) < M / 2:
                return row
    raise RuntimeError("no failing row found")


def particles_for(B, M):
    base = (np.arange(B)[:, None] * 1000 + np.arange(M)[None, :]).astype(np.float32)
    return np.stack([base, base + 0.5], axis=-1)         # (B, M, 2) float32, every particle distinct


def loop(fn, w, particles, seed):
    """The reference's step over the rows: (weights, particles, neff, mask, indexes, next draw, failing row)."""
    np.random.seed(seed)
    w = w.copy()
    p = particles.copy()
    B, M = w.shape
    neff = np.zeros(B)
    mask = np.zeros(B, bool)
    idx = np.full((B, M), -1, np.int32)
    with np.errstate(all="ignore"):
        for b in range(B):
            w[b] = w[b] / np.sum(w[b])
            neff[b] = 1. / np.sum(np.square(w[b]))
            if neff[b] < M / 2:
                mask[b] = True
                try:
                    idx[b] = fn(w[b])
                except IndexError:
                    return w, p, neff, mask, idx, np.nan, b
                p[b] = p[b][idx[b]]
                w[b] = np.full(M, 1. / M)
    return w, p, neff, mask, idx, np.random.random(), -1


def main():
    cases = [(kinds_bank(1, 1, 3), 3), (kinds_bank(3, 7, 5), 5), (special_bank(128, 7), 7),
             (kinds_bank(3, 1000, 12), 12), (kinds_bank(3, 300, 13), 13)]
    w_fail = kinds_bank(5, 64, 17)
    w_fail[-1] = failing_row(64)
    cases.append((w_fail, 17))
    out, meta = {}, []
    for k, (w, seed) in enumerate(cases):
        B, M = w.shape
        p = particles_for(B, M)
        out["w%d" % k], out["p%d" % k] = w, p
        fails = []
        for kind, fn in (("sys", systematic_resample), ("str", stratified_resample)):
            wa, pa, neff, mask, idx, nxt, fail = loop(fn, w, p, seed)
            out["%s_w%d" % (kind, k)], out["%s_p%d" % (kind, k)] = wa, pa
            out["%s_neff%d" % (kind, k)], out["%s_mask%d" % (kind, k)] = neff, mask
            out["%s_idx%d" % (kind, k)], out["%s_next%d" % (kind, k)] = idx, np.float64(nxt)
            fails.append(fail)
        if k == len(cases) - 1:
            assert fails == [B - 1, B - 1], fails           # the reference raises IndexError at the built row
        else:
            assert fails == [-1, -1], (k, fails)
        meta.append((k, B, M, seed, fails[0], fails[1]))
    path = os.path.join(HERE, "resample_bank_gated.npz")
    np.savez_compressed(path, reference_version=filterpy.__version__, meta=np.array(meta, np.int64), **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
