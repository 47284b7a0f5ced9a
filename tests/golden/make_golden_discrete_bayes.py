#!/usr/bin/env python
"""Golden vectors of the discrete Bayes filter (tests/golden/db_*.npz) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_discrete_bayes.py

Per case: a bank pdf[B, M] (fp32 or fp64), one kernel per row (kernel[B, K]), one offset per row, and a likelihood
per row.  The reference runs on every row in turn:
  prior[b] = predict(pdf[b], offsets[b], kernel[b], mode, cval)
  post[b]  = update(lik[b], prior[b])
  norm[b]  = normalize(pdf[b].copy())
Cases:
  db_wrap_k3_f64     K = 3, offsets negative, zero and beyond M, an all-zero row (0 / 0 = NaN)
  db_wrap_k4_f32     even K (scipy's origin rule moves the window by one), fp32
  db_wrap_klong_f64  K > M, weights 0, +-1e-17 and NaN (scipy leaves them out of the footprint)
  db_const_k5_f64    constant mode, cval = 0.05, offsets within and beyond the row
  db_const_k2_f32    constant mode, even K, fp32, cval = 0
  db_onebin_f64      a one-bin pdf (M = 1), wrap and constant alike
The tests never import the reference.
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

warnings.filterwarnings("ignore", category=DeprecationWarning)   # scipy.ndimage.filters / .interpolation
from filterpy.discrete_bayes import predict, update, normalize  # noqa: E402
import filterpy                                                  # noqa: E402


def save(name, **arrs):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, reference_version=filterpy.__version__, **arrs)
    print("wrote", path, os.path.getsize(path), "bytes")


def case(name, B, M, K, dtype, mode, cval, offsets, seed, zero_row=-1, kernel_edit=None):
    rng = np.random.default_rng(seed)
    pdf = rng.random((B, M)).astype(dtype)
    pdf /= pdf.sum(axis=1, keepdims=True)
    if zero_row >= 0:
        pdf[zero_row] = 0
    kernel = rng.random((B, K))
    if kernel_edit is not None:
        kernel_edit(kernel)
    lik = (rng.random((B, M)) + 0.05).astype(dtype)
    prior = np.empty_like(pdf)
    post = np.empty_like(pdf)
    norm = np.empty_like(pdf)
    with np.errstate(divide="ignore", invalid="ignore"):
        for b in range(B):
            prior[b] = predict(pdf[b], int(offsets[b]), kernel[b], mode=mode, cval=cval)
            post[b] = update(lik[b], prior[b])
            p = pdf[b].copy()
            assert normalize(p) is p
            norm[b] = p
    save(name, pdf=pdf, kernel=kernel, offsets=np.asarray(offsets, np.int64), lik=lik, wrap=np.int32(mode == "wrap"),
         cval=np.float64(cval), prior=prior, post=post, norm=norm)


def _klong(k):
    k[:, 1] = 0.0
    k[:, 3] = 1e-17
    k[0, 4] = -1e-17
    k[1, 5] = np.nan


def main():
    case("db_wrap_k3_f64", 8, 50, 3, np.float64, "wrap", 0., [0, 1, -1, 7, -23, 50, 1000001, -77], 1, zero_row=5)
    case("db_wrap_k4_f32", 6, 33, 4, np.float32, "wrap", 0., [2, -3, 0, 40, -66, 5], 2)
    case("db_wrap_klong_f64", 4, 5, 9, np.float64, "wrap", 0., [1, -2, 11, 0], 3, kernel_edit=_klong)
    case("db_const_k5_f64", 6, 40, 5, np.float64, "constant", 0.05, [3, -4, 0, 39, -45, 100], 4)
    case("db_const_k2_f32", 5, 17, 2, np.float32, "constant", 0., [1, -1, 0, 16, -3], 5)
    case("db_onebin_f64", 3, 1, 3, np.float64, "wrap", 0., [0, 4, -9], 6)


if __name__ == "__main__":
    main()
