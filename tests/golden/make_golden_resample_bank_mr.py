#!/usr/bin/env python
"""Golden vectors of the multinomial / residual bank resamplers (``multinomial_resample_bank`` /
``residual_resample_bank``) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_resample_bank_mr.py

For each case (n_sets, n_particles, seed, special rows) it seeds NumPy, loops the reference's
``multinomial_resample`` (then, reseeded, ``residual_resample``) over the rows of a bank whose rows mix the
weight kinds of ``workloads.resample_weights`` with special rows, and stores the weights, the indexes of
every row, and the next draw ``random()`` after the loop.  Where the reference raises IndexError (residual:
a row with more than M deterministic copies) the row it raised at is stored instead of the next draw.
Special rows: negative, NaN, +inf, -inf, signed-zero and subnormal weights, a row summing to 2 (its
cumulative sum passes 1 before the last element), and a row scaled by 1.5 (k > M for residual).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

from filterpy.monte_carlo import multinomial_resample, residual_resample  # noqa: E402
import filterpy                                                            # noqa: E402

from filterpy_b200.common import workloads as wl                          # noqa: E402

KINDS = ["heavy", "uniform", "zeros", "degenerate", "dyadic"]
# (n_sets, n_particles, seed, {row: special kind})
CASES = [(1, 1, 3, {}), (3, 7, 5, {}), (5, 64, 11, {}), (8, 1000, 12, {}), (40, 33, 13, {}),
         (10, 64, 17, {1: "neg", 3: "nan", 4: "inf", 6: "neginf", 8: "zeros", 9: "subnormal"}),
         (7, 37, 19, {2: "neg", 5: "nan", 6: "inf"}),
         (6, 64, 23, {2: "sum2"}),
         (6, 50, 29, {1: "neg", 4: "x1.5"})]


def special_row(kind, M, rng):
    r = rng.random(M)
    if kind == "neg":
        r[::5] *= -1
        return r / np.abs(r).sum()
    r = r / r.sum()
    if kind == "nan":
        r[M // 2] = np.nan
    elif kind == "inf":
        r[3] = np.inf
    elif kind == "neginf":
        r[1] = -np.inf
    elif kind == "zeros":
        r = np.full(M, -0.0)
        r[-1] = 1.0
    elif kind == "subnormal":
        r = np.full(M, 5e-324)
        r[M // 3] = 1.0
    elif kind == "sum2":
        r = 2.0 * r
    elif kind == "x1.5":
        r = 1.5 * r
    return r


def bank(B, M, seed, specials):
    w = np.empty((B, M))
    rng = np.random.default_rng(seed)
    for b in range(B):
        w[b] = wl.resample_weights(M, KINDS[b % len(KINDS)], seed=seed * 1000 + b)
        if b in specials:
            w[b] = special_row(specials[b], M, rng)
    return w


def loop(fn, w, seed):
    """The reference over the rows: (indexes, next draw, failing row or -1)."""
    np.random.seed(seed)
    idx = np.zeros(w.shape, np.int64)
    for b in range(w.shape[0]):
        try:
            with np.errstate(all="ignore"):
                idx[b] = fn(w[b])
        except IndexError:
            return idx, np.nan, b
    return idx, np.random.random(), -1


def main():
    out = {}
    meta = []
    for k, (B, M, seed, specials) in enumerate(CASES):
        w = bank(B, M, seed, specials)
        mul_idx, mul_next, mul_fail = loop(multinomial_resample, w, seed)
        res_idx, res_next, res_fail = loop(residual_resample, w, seed)
        out["w%d" % k] = w
        out["mul%d" % k], out["res%d" % k] = mul_idx, res_idx.astype(np.int32)
        out["mul_next%d" % k], out["res_next%d" % k] = np.float64(mul_next), np.float64(res_next)
        meta.append((k, B, M, seed, mul_fail, res_fail))
        print(k, (B, M), "multinomial fails at", mul_fail, "residual fails at", res_fail)
    path = os.path.join(HERE, "resample_bank_mr.npz")
    np.savez_compressed(path, reference_version=filterpy.__version__, meta=np.array(meta, np.int64), **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
