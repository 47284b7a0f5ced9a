"""Oracle: a particle filter's resampling step over the rows of a bank, resampling only the degenerate sets
(TEST INFRASTRUCTURE).

Every particle filter built on filterpy's resamplers runs, per set,

    w = w / np.sum(w)
    neff = 1. / np.sum(np.square(w))
    if neff < threshold:
        idx = systematic_resample(w)          # or stratified_resample(w)
        particles[:] = particles[idx]
        w = np.full(M, 1. / M)

``np_pairwise_sum`` restates how NumPy sums a contiguous float64 vector, which decides the last bits of the
normalised weights, of ``neff`` and so of the gate.  ``resample_if_degenerate_loop`` is the loop above on
the oracle's restatements of the two resamplers (``oracle.resample``).
"""
import numpy as np

from oracle import resample as ors

PW_BLOCKSIZE = 128


def _pairwise(a, off, n):
    """``pairwise_sum`` of numpy/_core/src/umath/loops_utils.h.src (NumPy 2.x), literally."""
    if n < 8:
        res = 0.
        for i in range(n):
            res = res + a[off + i]
        return res
    if n <= PW_BLOCKSIZE:
        r = [a[off + k] for k in range(8)]
        i = 8
        while i < n - (n % 8):
            for k in range(8):
                r[k] = r[k] + a[off + i + k]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        while i < n:                               # the n % 8 rest, in order
            res = res + a[off + i]
            i += 1
        return res
    n2 = n // 2
    n2 -= n2 % 8                                   # split at a multiple of the unroll factor
    return _pairwise(a, off, n2) + _pairwise(a, off + n2, n - n2)


def np_pairwise_sum(a):
    """``np.sum(a)`` of a 1-D float64 vector, bit for bit: the add reduction starts from its identity +0.0
    and adds the pairwise sum of the whole vector to it, so the result is ``fl(+0.0 + pairwise_sum(a))``
    (a sum of -0.0s is +0.0).  Python floats are IEEE doubles with round-to-nearest, as NumPy's are."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    return np.float64(0. + _pairwise(a.tolist(), 0, a.shape[0]))


def resample_if_degenerate_loop(w, particles, draws, threshold=None, method="systematic", resample=None):
    """The loop above over the rows of ``w[B, M]`` and ``particles[B, M, ...]`` (copies are returned).

    ``draws`` are the uniforms the resampled sets take, in row order: ``draws[k]`` is the k-th resampled
    set's ``random()`` (stratified: ``random(M)``).  ``resample(w_b, draw)`` defaults to the oracle's literal
    merge; ``oracle.resample.*_c`` gives the same result faster.  A set whose positions run past its
    cumulative sum (the reference's IndexError) keeps its particles and its normalised weights and is listed
    in ``failed``.  The reference's loop stops at the first failing set; this one goes on, as the bank does.

    Returns dict(weights, particles, neff, resampled, indexes (rows of unresampled sets are -1), failed,
    n_draws)."""
    w = np.array(w, dtype=np.float64)
    p = np.array(particles)
    B, M = w.shape
    thr = M / 2 if threshold is None else threshold
    if resample is None:
        resample = ors.systematic_resample_loop if method == "systematic" else ors.stratified_resample_loop
    neff = np.zeros(B)
    mask = np.zeros(B, bool)
    idx = np.full((B, M), -1, np.int32)
    failed = []
    k = 0
    with np.errstate(all="ignore"):
        for b in range(B):
            w[b] = w[b] / np.sum(w[b])
            neff[b] = 1. / np.sum(np.square(w[b]))
            if not neff[b] < thr:
                continue
            mask[b] = True
            d = draws[k]
            k += 1
            try:
                ix = resample(w[b], d)
            except IndexError:
                failed.append(b)
                continue
            idx[b] = ix
            p[b] = p[b][ix]
            w[b] = np.full(M, 1. / M)
    return dict(weights=w, particles=p, neff=neff, resampled=mask, indexes=idx, failed=failed, n_draws=k)
