#!/usr/bin/env python
"""Time EnsembleKalmanFilter banks on one GPU.

    python scripts/enkf_bench.py [--filters 65536] [--steps 20] [--warmup 5] [--repeats 3]

Legs: 4/2 constant-velocity banks (per-filter F, H, Q, R through LinearFx / LinearHx), fp32 and fp64, with
N = 32 and 256 members; each step is one fused predict + update launch, diagnostics off.  Times are CUDA
events around `steps` steps after `warmup` steps, median over repeats.

Bytes per filter-step are what the algorithm must move: the ensemble read and written once
(2 N n), the per-filter F, H, Q, R, z, and x and P in and out, times sizeof(T), over the H100 SXM data-sheet
3.35 TB/s.  The other floor is the noise: N (n + m) normals per filter-step, each pair a Philox4x32-10
block and one log / sqrt / sincos (Box-Muller).  The leg is named bytes-bound when the byte floor is at
least half the measured time, else bound by that arithmetic (fp64 transcendentals in the fp64 legs).  One
JSON line per leg goes to stdout, with the GPU name, power limit and max SM clock of the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from filterpy_b200.common import workloads as wl                                              # noqa: E402
from filterpy_b200.kalman import EnsembleKalmanFilter, LinearFx, LinearHx                      # noqa: E402

PEAK_BPS = 3.35e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def leg(w, dtype, N, steps, warmup, repeats):
    F = w["x"].shape[0]
    n, m = 4, 2
    e = EnsembleKalmanFilter(w["x"], w["P"], m, 0.1, N, LinearHx(w["H"]), LinearFx(w["F"]), n_filters=F, dtype=dtype,
                             diagnostics=False, seed=1)
    e.Q, e.R = w["Q"], w["R"]
    td = torch.float32 if dtype == np.float32 else torch.float64
    z = torch.as_tensor(w["zs"][0], dtype=td, device="cuda").contiguous()
    for _ in range(warmup):
        e.predict(); e.update(z)
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            e.predict(); e.update(z)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) / steps)
    assert torch.isfinite(e.x).all().item()
    ms = float(np.median(times))
    T = 4 if dtype == np.float32 else 8
    per_filter = (2 * N * n + n * n + m * n + n * n + m * m + m + 2 * (n + n * n)) * T
    byte_floor_ms = F * per_filter / PEAK_BPS * 1e3
    normals = F * N * (n + m)
    return dict(leg="enkf_4_2_%s_N%d" % ("fp32" if T == 4 else "fp64", N), n_filters=F, members=N,
                ms_per_epoch=round(ms, 4), bytes_per_filter_step=per_filter,
                achieved_TBps=round(F * per_filter / (ms * 1e-3) / 1e12, 3),
                frac_hbm_peak=round(byte_floor_ms / ms, 3),
                normals_per_s=float("%.3g" % (normals / (ms * 1e-3))),
                bound="bytes" if byte_floor_ms >= 0.5 * ms else
                      ("fp64 transcendental / Philox arithmetic" if T == 8 else "fp32 Philox / Box-Muller arithmetic"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--filters", type=int, default=1 << 16)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("enkf_bench.py needs a CUDA device")
    info = gpu_info()
    w = wl.kf_bank_cv2d(a.filters, seed=7, steps=1)
    for dtype in (np.float32, np.float64):
        for N in (32, 256):
            r = leg(w, dtype, N, a.steps, a.warmup, a.repeats)
            r.update(info)
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
