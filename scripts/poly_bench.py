#!/usr/bin/env python
"""Time the polynomial tracker banks (bke_poly_filter) on one GPU, with the reference's CPU form beside them.

    python scripts/poly_bench.py [--n 1048576] [--T 64] [--repeats 5] [--warmup 3]

Arms, each at N filters with per-filter parameters, in fp64 and fp32: GHFilter, GHKFilter, LeastSquaresFilter order 2
and FadingMemoryFilter order 2, as batch_filter over T epochs (one launch; results[T+1, N, W] written) and as T
update() calls (one launch each).  The arms alternate within each repeat; times are CUDA events around the call after
warm-up, and the median over repeats is reported per epoch.  Algorithmic bytes per filter-epoch are computed from the
shapes (below) and reported as a share of the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s.
CPU comparison: the reference's own vectorised GHFilter.update over an (N,) array, and a loop of reference
LeastSquaresFilter objects (order 2) on a subsample, per epoch and scaled to N; the reference is imported from
oracle/_ref when build() staged it, and the CPU arms are skipped otherwise.  One JSON line per arm, with the GPU name,
power limit and max SM clock.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from filterpy_b200.gh import GHFilter, GHKFilter                                                 # noqa: E402
from filterpy_b200.leastsq import LeastSquaresFilter                                             # noqa: E402
from filterpy_b200.memory import FadingMemoryFilter                                              # noqa: E402

PEAK_BPS = 3.35e12
DEV = "cuda:0"


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def bytes_per_filter_epoch(arm, mode, T, itemsize):
    """z in, results out (batch) or the state in and out per launch (update), plus the per-filter parameters once per
    launch: GH g, h, dt; GHK g, h, k, dt, dt2; LSQ dt, dt2, hdt2 and the int64 counter; Fading g, h, k, dt, dt2"""
    state = {"gh": 2, "ghk": 3, "lsq": 3, "fm": 3}[arm]
    params = {"gh": 3, "ghk": 5, "lsq": 3, "fm": 5}[arm] * itemsize + (16 if arm == "lsq" else 0)
    if mode == "batch":
        W = 2 if arm in ("gh", "ghk") else 3
        return itemsize * (1 + W) + (itemsize * (state + W) + params) / T
    out = {"gh": 2 + 3, "ghk": 3 + 4, "lsq": 3 + 3, "fm": 3}[arm]           # + y and predictions / K
    return itemsize * (1 + state + out) + params


def make(arm, N, dtype, rng):
    dt = rng.uniform(.1, 1., N)
    if arm == "gh":
        return GHFilter(rng.standard_normal(N), rng.standard_normal(N), dt, rng.uniform(.1, .8, N),
                        rng.uniform(.01, .1, N), n_filters=N, dtype=dtype, device=DEV)
    if arm == "ghk":
        return GHKFilter(rng.standard_normal(N), rng.standard_normal(N), rng.standard_normal(N), dt,
                         rng.uniform(.1, .8, N), rng.uniform(.01, .1, N), rng.uniform(.001, .01, N),
                         n_filters=N, dtype=dtype, device=DEV)
    if arm == "lsq":
        return LeastSquaresFilter(dt, 2, n_filters=N, dtype=dtype, device=DEV)
    return FadingMemoryFilter(rng.standard_normal((N, 3)), dt, 2, rng.uniform(.1, .9, N), n_filters=N, dtype=dtype,
                              device=DEV)


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e)


def cpu_arms(N, T, rng):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    try:
        from filterpy.gh import GHFilter as RefGH
        from filterpy.leastsq import LeastSquaresFilter as RefLSQ
    except ImportError:
        return []
    z = rng.standard_normal((T, N))
    f = RefGH(np.zeros(N), np.zeros(N), .5, np.full(N, .4), np.full(N, .05))
    t0 = time.perf_counter()
    for t in range(T):
        f.update(z[t])
    gh_ms = (time.perf_counter() - t0) * 1e3 / T
    sub = 2000
    objs = [RefLSQ(.5, 2) for _ in range(sub)]
    t0 = time.perf_counter()
    for t in range(8):
        for i, o in enumerate(objs):
            o.update(z[t, i])
    lsq_ms = (time.perf_counter() - t0) * 1e3 / 8 * (N / sub)
    return [dict(arm="reference_GHFilter_update_vectorised", n_filters=N, ms_per_epoch=round(gh_ms, 4)),
            dict(arm="reference_LeastSquaresFilter_loop", n_filters=N, sampled=sub, ms_per_epoch_scaled=round(lsq_ms, 1))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--T", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("poly_bench.py needs a GPU")
    info = gpu_info()
    N, T = args.n, args.T
    rng = np.random.default_rng(0)
    for dtype in (np.float64, np.float32):
        itemsize = np.dtype(dtype).itemsize
        td = torch.float64 if dtype == np.float64 else torch.float32
        z = torch.as_tensor(rng.standard_normal((T, N)), device=DEV).to(td)
        arms = {a: make(a, N, dtype, rng) for a in ("gh", "ghk", "lsq", "fm")}
        calls = {}
        for a, f in arms.items():
            calls[(a, "batch")] = (lambda f=f: f.batch_filter(z))
            calls[(a, "update")] = (lambda f=f: [f.update(z[t]) for t in range(T)])
        for fn in calls.values():
            for _ in range(args.warmup):
                fn()
        times = {k: [] for k in calls}
        for _ in range(args.repeats):
            for k, fn in calls.items():
                times[k].append(timed(fn) / T)
        for (a, mode), ts in times.items():
            ms = float(np.median(ts))
            b = bytes_per_filter_epoch(a, mode, T, itemsize)
            print(json.dumps(dict(arm=a, mode=mode, dtype=np.dtype(dtype).name, n_filters=N, T=T,
                                  ms_per_epoch=round(ms, 5), spread=[round(min(ts), 5), round(max(ts), 5)],
                                  bytes_per_filter_epoch=round(b, 2), hbm_share=round(b * N / (ms * 1e-3) / PEAK_BPS, 3),
                                  **info)), flush=True)
        del arms, calls, z
        torch.cuda.empty_cache()
    if not args.no_cpu:
        for r in cpu_arms(N, 8, rng):
            print(json.dumps(dict(r, **info)), flush=True)


if __name__ == "__main__":
    main()
