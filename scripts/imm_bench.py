#!/usr/bin/env python
"""IMMEstimator.batch_filter against the predict(); update(z) loop it replaces, on one GPU.

Workload: 2^20 tracks x 3 constant-velocity models at dim_x = 4, dim_z = 2, per-track F and Q (each track its own
dt), shared H and R, T = 32 epochs, every track measured, in fp32 and fp64.  Variants, alternated in one run and
repeated (median of the repeats, CUDA events after warm-up):
  batch_filter   the T epochs in one call (one launch where the shape has a fused instance)
  loop           T x (predict(); update(z)) on the same estimator, ~14 launches per epoch; its outputs are not
                 copied anywhere (less work than batch_filter, which writes the five outputs of every epoch)
  graph          the loop replayed as IMMEstimator.capture's CUDA graph of 3 epochs (the model filters' buffers
                 rotate with period 3), 32 / 3 replays per 32 epochs
Prints one JSON line per dtype: ms per epoch of each variant, the algorithmic bytes per track-epoch of
batch_filter's fused kernel (z in, the five outputs out: state, models and probabilities stay on chip), that
traffic over its time as a share of the data sheet's 3.35 TB/s, the largest relative difference between
batch_filter's and the loop's outputs on the timed inputs, and the card's name and power limit.
"""
import argparse
import json
import subprocess
import sys
import os

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from filterpy_b200.kalman import IMMEstimator, KalmanFilter  # noqa: E402

PEAK_BPS = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def make(N, dtype, seed=0):
    rng = np.random.default_rng(seed)
    dt = rng.uniform(0.5, 1.5, N)
    F = np.zeros((N, 4, 4)); F[:] = np.eye(4); F[:, 0, 1] = F[:, 2, 3] = dt
    Q1 = np.zeros((N, 4, 4))
    Q1[:, 0, 0] = Q1[:, 2, 2] = dt ** 3 / 3
    Q1[:, 0, 1] = Q1[:, 1, 0] = Q1[:, 2, 3] = Q1[:, 3, 2] = dt ** 2 / 2
    Q1[:, 1, 1] = Q1[:, 3, 3] = dt
    H = np.kron(np.eye(2), np.array([[1.0, 0.0]]))
    x0 = rng.normal(size=(N, 4)) * 3
    fs = []
    for j, q in enumerate((0.05, 1.0, 8.0)):
        f = KalmanFilter(4, 2, n_filters=N, dtype=dtype)
        f.x, f.P, f.F, f.Q, f.H, f.R = x0 + j, np.eye(4) * 2.0, F, Q1 * q, H, np.eye(2) * 0.5
        fs.append(f)
    trans = np.array([[.9, .05, .05], [.1, .8, .1], [.05, .15, .8]])
    return IMMEstimator(fs, [0.5, 0.3, 0.2], trans)


def timed(fn, reps):
    out = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); e.synchronize()
        out.append(s.elapsed_time(e))
    return out


def bench(N, T, dtype, reps):
    es = np.dtype(dtype).itemsize
    rng = np.random.default_rng(1)
    zs = torch.from_numpy((rng.normal(size=(T, N, 2)) * 2 + np.cumsum(rng.normal(size=(T, N, 2)), axis=0)).astype(dtype)).cuda()

    # the outputs of batch_filter and of the loop from the same initial state
    a, b = make(N, dtype), make(N, dtype)
    means, covs, means_p, covs_p, mus = a.batch_filter(zs)
    diff = 0.0
    for k in range(T):
        b.predict()
        for got, want in ((means_p[k], b.x), (covs_p[k], b.P)):
            diff = max(diff, float(((got - want).abs().max() / want.abs().max().clamp_min(1.0)).item()))
        b.update(zs[k])
        for got, want in ((means[k], b.x), (covs[k], b.P), (mus[k], b.mu)):
            diff = max(diff, float(((got - want).abs().max() / want.abs().max().clamp_min(1.0)).item()))
    del a, b, means, covs, means_p, covs_p, mus

    imm_b, imm_l, imm_g = make(N, dtype), make(N, dtype), make(N, dtype)
    zbuf = [zs[k].clone() for k in range(3)]

    def loop():
        for k in range(T):
            imm_l.predict(); imm_l.update(zs[k])

    def ring():
        for k in range(3):
            imm_g.predict(); imm_g.update(zbuf[k])
    g = imm_g.capture(ring)
    n_replay = -(-T // 3)

    def graph():
        for _ in range(n_replay):
            g.replay()
    variants = {"batch_filter": lambda: imm_b.batch_filter(zs), "loop": loop, "graph": graph}
    epochs = {"batch_filter": T, "loop": T, "graph": 3 * n_replay}
    for fn in variants.values():                                # warm-up
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(reps):                                       # alternated
        for k, fn in variants.items():
            times[k] += timed(fn, 1)
    ms = {k: float(np.median(v)) / epochs[k] for k, v in times.items()}
    spread = {k: [round(min(v) / epochs[k], 4), round(max(v) / epochs[k], 4)] for k, v in times.items()}
    M, n, m = 3, 4, 2
    bytes_te = m * es + (2 * n + 2 * n * n) * es + M * 8
    fused = imm_b.filters[0]._dtype == torch.float32            # 4/2 has a fused instance in fp32 only
    return {
        "dtype": np.dtype(dtype).name, "tracks": N, "models": M, "dim_x": n, "dim_z": m, "epochs": T, "repeats": reps,
        "fused_kernel": fused,
        "ms_per_epoch": {k: round(v, 4) for k, v in ms.items()},
        "ms_per_epoch_min_max": spread,
        "speedup_vs_graph": round(ms["graph"] / ms["batch_filter"], 2),
        "speedup_vs_loop": round(ms["loop"] / ms["batch_filter"], 2),
        "fused_bytes_per_track_epoch": bytes_te,
        "fused_share_of_3.35TBps": round(bytes_te * N / (ms["batch_filter"] * 1e-3) / PEAK_BPS, 3) if fused else None,
        "max_rel_diff_vs_loop": diff,
        "card": card(),
    }


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--tracks", type=int, default=1 << 20)
    p.add_argument("--epochs", type=int, default=32)
    p.add_argument("--repeats", type=int, default=5)
    p.add_argument("--dtypes", default="float32,float64")
    args = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("imm_bench.py needs a GPU")
    for d in args.dtypes.split(","):
        print(json.dumps(bench(args.tracks, args.epochs, np.dtype(d).type, args.repeats)), flush=True)


if __name__ == "__main__":
    main()
