"""Oracle: multinomial_resample / residual_resample over the rows of a bank (TEST INFRASTRUCTURE).

The reference's own NumPy calls (filterpy/monte_carlo/resampling.py:153-176 and :27-76), vectorised
over the rows where that keeps every row's arithmetic in the reference's order, so that checks at
millions of particles stay fast:

* ``np.cumsum(.., axis=1)`` accumulates each row strictly left to right, as ``np.cumsum`` of one row;
* the builtin ``sum(residual)`` (:70) is one column added at a time to the running row sums;
* the bisection is ``np.searchsorted`` itself, per row, with NumPy's carried bracket.

``oracle.resample.binsearch_left`` restates that bisection; the CPU tests check it against the golden
vectors of the unmodified reference.
"""
import numpy as np


def multinomial_bank(w, U):
    """resampling.py:173-176 per row for the uniforms ``U[b]``: int64 (B, M)."""
    with np.errstate(all="ignore"):
        c = np.cumsum(w, axis=1)
    c[:, -1] = 1.
    return np.stack([np.searchsorted(c[b], U[b]) for b in range(w.shape[0])]).reshape(w.shape)


def residual_prepare_bank(w):
    """resampling.py:52-72 per row: (indexes with the first k_b entries filled, k (saturated at M + 1),
    cumulative sums with [-1] = 1)."""
    B, M = w.shape
    with np.errstate(all="ignore"):
        num_copies = np.floor(M * w).astype(int)
        copies = np.maximum(num_copies, 0)
        k = np.minimum(copies, M + 1).sum(axis=1)
        residual = w - num_copies
        s = np.zeros(B)
        for j in range(M):                    # builtin sum(): 0 + r0 + r1 + ... per row
            s = s + residual[:, j]
        c = np.cumsum(residual / s[:, None], axis=1)
    c[:, -1] = 1.
    idx = np.zeros((B, M), np.int32)
    for b in range(B):
        if k[b] <= M:
            idx[b, :k[b]] = np.repeat(np.arange(M), copies[b])
    return idx, k, c


def residual_bank(w, U):
    """resampling.py:27-76 per row, row b drawing ``U[b, :M - k_b]``: (int32 (B, M), k, failing rows)."""
    idx, k, c = residual_prepare_bank(w)
    M = w.shape[1]
    for b in range(w.shape[0]):
        if k[b] <= M:
            idx[b, k[b]:] = np.searchsorted(c[b], U[b, :M - k[b]])
    return idx, k, np.flatnonzero(k > M)
