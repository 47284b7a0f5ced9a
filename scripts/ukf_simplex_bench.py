#!/usr/bin/env python
"""Merwe against simplex sigma points in the fused UKF step: 2^18 filters of 6/3 ConstVelFx + RangeAzElHx
(config 4, ``workloads.ukf_bank_cv3d``) and of 4/2 ConstVelFx + RangeBearingHx (its first four components), fp64
and fp32, the two point sets alternating in one process, the median of 5 runs of ``--steps`` steps each (CUDA
events).  Prints the card, ms per fused predict + update, the registers of each pre-built instance (from
``cuobjdump -res-usage`` of libbke.so) and the bytes per filter-step, which are the same for both sets.

    python scripts/ukf_simplex_bench.py [--filters 262144] [--steps 200] [--reps 5]
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from filterpy_b200 import _lib                                                         # noqa: E402
from filterpy_b200.common import workloads as wl                                      # noqa: E402
from filterpy_b200.kalman import (UnscentedKalmanFilter, MerweScaledSigmaPoints, SimplexSigmaPoints,  # noqa: E402
                                  ConstVelFx, RangeAzElHx, RangeBearingHx)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def registers():
    """{(dtype, n, m, fx, hx, simplex): registers} of the plain (no optional outputs) pre-built instances."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    r = subprocess.run([exe, "-res-usage", _lib.lib_path()], capture_output=True, text=True)
    out, name = {}, None
    for ln in r.stdout.splitlines():
        m = re.search(r"Function (_ZN3bke4ukfk10ukf_kernelI([df])Li(\d)ELi(\d)ELi(\d)ELi(\d)ELi\dELb0E(Lb([01])E)?EEv\S*):", ln)
        if m:
            name = (m.group(2), int(m.group(3)), int(m.group(4)), int(m.group(5)), int(m.group(6)), m.group(8) == "1")
            continue
        m = re.search(r"REG:(\d+)", ln)
        if m and name:
            out[name] = int(m.group(1))
            name = None
    return out


def bank(kind, N, dtype):
    w = wl.ukf_bank_cv3d(N, seed=2468, steps=16)
    if kind == "6/3":
        return {k: w[k] for k in ("x", "P", "Q", "R", "zs")}, 6, 3, RangeAzElHx()
    x = w["x"][:, :4]
    rng = np.random.default_rng(5)
    zs = np.stack([np.stack([np.hypot(x[:, 0], x[:, 2]), np.arctan2(x[:, 2], x[:, 0])], 1)
                   + rng.normal(size=(N, 2)) * np.array([0.5, 0.002]) for _ in range(16)])
    return dict(x=x, P=w["P"][:, :4, :4], Q=w["Q"][:, :4, :4], R=w["R"][:, :2, :2], zs=zs), 4, 2, RangeBearingHx()


def make(w, n, m, hx, N, dtype, simplex):
    pts = SimplexSigmaPoints(n) if simplex else MerweScaledSigmaPoints(n, .5, 2., 0.)
    u = UnscentedKalmanFilter(n, m, 0.1, hx, ConstVelFx(), pts, n_filters=N, dtype=dtype, device="cuda:0", diagnostics=False)
    u.x = w["x"]; u.P = w["P"]; u.Q = w["Q"]; u.R = w["R"]
    return u


def time_steps(u, zt, steps):
    for t in range(3):                                       # warm-up
        u.predict(); u.update(zt[t % zt.shape[0]])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(steps):
        u.predict(); u.update(zt[t % zt.shape[0]])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--filters", type=int, default=1 << 18)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ukf_simplex_bench.py needs a GPU")
    N = a.filters
    regs = registers()
    res = dict(card=card(), filters=N, steps=a.steps, reps=a.reps)
    for kind in ("6/3", "4/2"):
        for dtype, dn in ((np.float64, "fp64"), (np.float32, "fp32")):
            w, n, m, hx = bank(kind, N, dtype)
            w = {k: np.ascontiguousarray(v, dtype=dtype) for k, v in w.items()}
            hxm = hx.model
            arms = {"merwe": make(w, n, m, hx, N, dtype, False), "simplex": make(w, n, m, hx, N, dtype, True)}
            zt = torch.as_tensor(w["zs"], device="cuda:0")
            times = {k: [] for k in arms}
            for _ in range(a.reps):
                for k, u in arms.items():                    # alternate the arms
                    times[k].append(time_steps(u, zt, a.steps))
            e = np.dtype(dtype).itemsize
            # per filter-step: x, P read and written, per-filter Q and R, z read
            nbytes = e * (2 * (n + n * n) + n * n + m * m + m)
            key = "%s_%s" % (kind.replace("/", "_"), dn)
            res[key + "_bytes_per_filter_step"] = nbytes
            for k, ts in times.items():
                ms = float(np.median(ts))
                res["%s_%s_ms_per_step" % (key, k)] = round(ms, 5)
                res["%s_%s_spread_ms" % (key, k)] = [round(min(ts), 5), round(max(ts), 5)]
                res["%s_%s_GBps" % (key, k)] = round(nbytes * N / (ms * 1e-3) / 1e9, 1)
                res["%s_%s_registers" % (key, k)] = regs.get(("d" if dtype == np.float64 else "f", n, m, 1, hxm, k == "simplex"))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
