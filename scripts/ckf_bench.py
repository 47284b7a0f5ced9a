#!/usr/bin/env python
"""Time CubatureKalmanFilter banks against the UKF at the same shapes, in one run on one GPU.

    python scripts/ckf_bench.py [--N 262144] [--steps 50] [--warmup 10] [--repeats 5]

Legs (each a fused predict + update per step, diagnostics off, per-filter Q and R):
  c4    6/3 CV + range/azimuth/elevation (bench.py's ukf_c4 shape), fp64 and fp32
  rb    4/2 CV + range/bearing, fp64
  user  4/2 coordinated turn + offset range/bearing compiled from CUDA text (DeviceFx / DeviceHx), fp64
The CKF and UKF arms of a leg alternate, repeat by repeat.  Times are CUDA events around `steps` steps
after `warmup` steps; the median over repeats is reported.  Bytes per filter-step are the algorithmic
(2n + 3n^2 + m + m^2) * sizeof(T): x and P in and out, Q, z and R (as bench.py counts the UKF leg), over
the H100 SXM data-sheet 3.35 TB/s.  Each CKF bank's outputs are checked against the oracle once.  One JSON
line per leg and arm goes to stdout, with the GPU name, power limit and max SM clock.
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
from filterpy_b200.kalman import (CubatureKalmanFilter, UnscentedKalmanFilter, MerweScaledSigmaPoints,  # noqa: E402
                                  ConstVelFx, RangeAzElHx, RangeBearingHx, DeviceFx, DeviceHx)
from oracle import ckf as ockf                                                                  # noqa: E402

PEAK_BPS = 3.35e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def cv_bank(N, n, dtype):
    """x, P, Q, R, z for a CV bank: the C4 workload for n = 6, its first two axes for n = 4."""
    w = wl.ukf_bank_cv3d(N, seed=2468, steps=1, dtype=np.float64)
    if n == 6:
        return w, w["zs"][0]
    idx = [0, 1, 2, 3]
    x, P, Q = w["x"][:, idx], w["P"][:, idx][:, :, idx], w["Q"][:, idx][:, :, idx]
    px, py = x[:, 0], x[:, 2]
    z = np.stack([np.hypot(px, py), np.arctan2(py, px)], 1) + np.random.default_rng(1).normal(size=(N, 2)) * [1.0, 0.005]
    R = np.broadcast_to(np.diag([1.0, 0.005 ** 2]), (N, 2, 2)).copy()
    return dict(x=x, P=P, Q=Q, R=R), z


def make(kind, leg, N, dtype):
    if leg == "user":
        w = wl.ukf_bank_ct2d(N, steps=1)
        # the argument values are given once, as the models' defaults: no per-step host-to-device copy
        fx = DeviceFx(wl.CT_FX_SOURCE, arg_names=("omega",), omega=torch.from_numpy(w["omega"]).cuda())
        hx = DeviceHx(wl.OFFSET_RB_HX_SOURCE, arg_names=("sx", "sy"), sx=float(w["sensor"][0]), sy=float(w["sensor"][1]))
        n, m = 4, 2
        z, dt = w["zs"][0], 0.5
    else:
        n, m = (6, 3) if leg == "c4" else (4, 2)
        w, z = cv_bank(N, n, dtype)
        fx, hx, dt = ConstVelFx(), (RangeAzElHx() if n == 6 else RangeBearingHx()), 0.1
    if kind == "ckf":
        f = CubatureKalmanFilter(n, m, dt, hx, fx, n_filters=N, dtype=dtype, diagnostics=False)
    else:
        f = UnscentedKalmanFilter(n, m, dt, hx, fx, MerweScaledSigmaPoints(n, .5, 2., 0.), n_filters=N, dtype=dtype,
                                  diagnostics=False)
    f.x = w["x"]; f.P = w["P"]; f.Q = w["Q"]; f.R = w["R"]
    zt = torch.from_numpy(np.ascontiguousarray(z)).to("cuda", dtype=f._dtype)
    step = lambda: (f.predict(), f.update(zt))                                                  # noqa: E731
    return f, step, w, z, n, m


def timed(step, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def check(leg, f, w, z):
    """one CKF step on the timed bank's inputs against the fp64 centred oracle, on a 4096-filter subset"""
    if leg == "user":
        return None
    sel = np.random.default_rng(0).choice(f.n_filters, 4096, replace=False)
    f.x = w["x"]; f.P = w["P"]
    f.predict(); f.update(torch.from_numpy(np.ascontiguousarray(z)).to("cuda", dtype=f._dtype))
    hx = ockf.HX_RANGE_AZ_EL if w["x"].shape[1] == 6 else ockf.HX_RANGE_BEARING
    o = ockf.ckf_step_bank(w["x"][sel], w["P"][sel], z[sel], w["Q"][sel], w["R"][sel], 0.1, ockf.FX_CONST_VEL, hx)
    ex = np.abs(f.x.cpu().numpy()[sel] - o["x"]).max() / np.abs(o["x"]).max()
    eP = np.abs(f.P.cpu().numpy()[sel] - o["P"]).max() / np.abs(o["P"]).max()
    return max(float(ex), float(eP))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=1 << 18)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ckf_bench.py needs a GPU")
    info = gpu_info()
    for leg, dtype in (("c4", np.float64), ("c4", np.float32), ("rb", np.float64), ("user", np.float64)):
        arms = {k: make(k, leg, args.N, dtype) for k in ("ckf", "ukf")}
        for k in arms:
            for _ in range(args.warmup):
                arms[k][1]()
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        for _ in range(args.repeats):
            for k in arms:
                ms[k].append(timed(arms[k][1], args.steps))
        f, _, w, z, n, m = arms["ckf"]
        err = check(leg, f, w, z)
        s = np.dtype(dtype).itemsize
        nbytes = (2 * n + 3 * n * n + m + m * m) * s
        for k in arms:
            med = float(np.median(ms[k]))
            rec = dict(leg=leg, filter=k, dtype=np.dtype(dtype).name, n_filters=args.N, dim_x=n, dim_z=m,
                       ms_per_step=med, ms_all=ms[k], filter_steps_per_s=args.N / (med * 1e-3),
                       bytes_per_filter_step=nbytes, frac_of_3_35_TBps=args.N * nbytes / (med * 1e-3) / PEAK_BPS, **info)
            if k == "ckf" and err is not None:
                rec["max_rel_err_vs_oracle"] = err
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
