#!/usr/bin/env python
"""Cost of the angle hooks: the pre-built 4/2 ConstVelFx + RangeBearingHx UKF step against the run-time
compiled instance with residual_z and z_mean_fn (workload (a), ``workloads.ukf_bank_rb_behind``), 2^18 filters,
fp64 and fp32, the two arms alternating in one process.  Reports ms per fused predict + update (CUDA events),
the registers of the hooked instance and the bytes per filter-step the step moves over its time.

    python scripts/ukf_hooks_bench.py [--filters 262144] [--steps 200] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from filterpy_b200.common import workloads as wl                                      # noqa: E402
from filterpy_b200.kalman import (UnscentedKalmanFilter, MerweScaledSigmaPoints, ConstVelFx, RangeBearingHx,  # noqa: E402
                                  DeviceFn)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def make(w, N, dtype, hooked):
    rb = DeviceFn(wl.RB_HOOKS_SOURCE)
    u = UnscentedKalmanFilter(4, 2, 1.0, RangeBearingHx(), ConstVelFx(), MerweScaledSigmaPoints(4, .8, 2., 0.),
                              n_filters=N, dtype=dtype, device="cuda:0", diagnostics=False,
                              **(dict(residual_z=rb, z_mean_fn=rb) if hooked else {}))
    u.x = w["x"]; u.P = w["P"]; u.Q = w["Q"]; u.R = w["R"]
    return u


def time_steps(u, zs, steps):
    zt = torch.as_tensor(zs, device="cuda:0").to(u._dtype)
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
        raise SystemExit("ukf_hooks_bench.py needs a GPU")
    N = a.filters
    w = wl.ukf_bank_rb_behind(N, seed=77, steps=16)
    res = dict(card=card(), filters=N, steps=a.steps)
    for dtype, name in ((np.float64, "fp64"), (np.float32, "fp32")):
        ww = {k: v.astype(dtype) for k, v in w.items()}
        arms = {"builtin": make(ww, N, dtype, False), "hooked": make(ww, N, dtype, True)}
        times = {k: [] for k in arms}
        for _ in range(a.reps):
            for k, u in arms.items():                        # alternate the arms
                times[k].append(time_steps(u, ww["zs"], a.steps))
        e = np.dtype(dtype).itemsize
        # per filter-step: x, P read and written, per-filter Q and R, z read
        nbytes = e * (2 * (4 + 16) + 16 + 4 + 2)
        h = arms["hooked"]
        regs = [h._lib.bke_ukf_model_registers(h._user_model, x) for x in (0, 1)]
        for k, ts in times.items():
            ms = float(np.median(ts))
            res["%s_%s_ms_per_step" % (name, k)] = round(ms, 5)
            res["%s_%s_spread_ms" % (name, k)] = [round(min(ts), 5), round(max(ts), 5)]
            res["%s_%s_GBps" % (name, k)] = round(nbytes * N / (ms * 1e-3) / 1e9, 1)
        res["%s_bytes_per_filter_step" % name] = nbytes
        res["%s_hooked_registers_plain_extras" % name] = regs
    print(json.dumps(res))


if __name__ == "__main__":
    main()
