#!/usr/bin/env python
"""Golden vectors of the bank resamplers (``systematic_resample_bank`` / ``stratified_resample_bank``)
from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_resample_bank.py

For each case (n_sets, n_particles, seed) it seeds NumPy, loops the reference's ``systematic_resample``
(then, reseeded, ``stratified_resample``) over the rows of a bank whose rows mix the weight kinds of
``workloads.resample_weights``, and stores the weights, the indexes of every row, and the next draw
``random()`` after the loop.  One bank is unnormalised (a row sums to less than 1): there the reference
raises IndexError, and the row it raised at is stored instead of the next draw.
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

KINDS = ["heavy", "uniform", "zeros", "degenerate", "dyadic"]
# (n_sets, n_particles, seed, unnormalised row or -1)
CASES = [(1, 1, 3, -1), (3, 7, 5, -1), (5, 64, 11, -1), (8, 1000, 12, -1), (40, 33, 13, -1), (6, 64, 17, 2)]


def bank(B, M, seed, short_row):
    w = np.empty((B, M))
    for b in range(B):
        w[b] = wl.resample_weights(M, KINDS[b % len(KINDS)], seed=seed * 1000 + b)
    if short_row >= 0:
        w[short_row] *= 0.9                  # sums to 0.9: the last positions lie beyond cumsum[-1]
    return w


def loop(fn, w, seed):
    """The reference over the rows: (indexes, next draw, failing row or -1)."""
    np.random.seed(seed)
    idx = np.zeros(w.shape, np.int32)
    for b in range(w.shape[0]):
        try:
            idx[b] = fn(w[b])
        except IndexError:
            return idx, np.nan, b
    return idx, np.random.random(), -1


def main():
    out = {}
    meta = []
    for k, (B, M, seed, short_row) in enumerate(CASES):
        w = bank(B, M, seed, short_row)
        sys_idx, sys_next, sys_fail = loop(systematic_resample, w, seed)
        str_idx, str_next, str_fail = loop(stratified_resample, w, seed)
        out["w%d" % k] = w
        out["sys%d" % k], out["str%d" % k] = sys_idx, str_idx
        out["sys_next%d" % k], out["str_next%d" % k] = np.float64(sys_next), np.float64(str_next)
        meta.append((k, B, M, seed, sys_fail, str_fail))
    path = os.path.join(HERE, "resample_bank.npz")
    np.savez_compressed(path, reference_version=filterpy.__version__, meta=np.array(meta, np.int64), **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
