#!/usr/bin/env python
"""Time KalmanFilter.update_correlated and update_sequential's row block against bke_kf_step on one bank.

For 2^20 filters with per-filter models, on one GPU:
  * 4/2 fp32 and 6/3 fp32 run on the register tiles, 6/3 fp64 on the warp-per-filter catch-all;
  * ``step``        bke_kf_step, predict + update (the bank's usual call);
  * ``correlated``  bke_kf_step_correlated, predict + update_correlated;
  * ``rows``        two bke_kf_update_rows calls of one row each (update only: the two blocks of a 2-row z).
Each call steps x and P in place and writes no optional output.  Times are CUDA events over ``--iters`` calls
after ``--warmup``; the bytes are the algorithmic ones, computed from the shapes (every array read or written
once per call): a predict + update reads x, P, F, Q, H, R, z and writes x, P (344 B per 4/2 fp32 filter), the
correlated step reads M as well (376 B), a one-row block reads x, P, its row of H, its entry of R and of z and
writes x, P (184 B).  The share is of the H100 SXM's 3.35 TB/s HBM3 data-sheet bandwidth.

    python scripts/kf_update_forms_bench.py [--filters 1048576] [--iters 50] [--warmup 5]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from filterpy_b200 import _lib                                                           # noqa: E402
from filterpy_b200._dev import ptr                                                        # noqa: E402

HBM_BPS = 3.35e12


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                       "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        out = torch.cuda.get_device_name(0) + ", power limit unknown"
    return out


def bytes_per_filter(kind, n, m, es):
    xP = 2 * (n + n * n)
    if kind == "rows":                  # two blocks of one row, each: x, P in and out, a row of H, R_ii, z_i
        return 2 * es * (xP + n + 1 + 1)
    b = es * (xP + 2 * n * n + m * n + m * m + m)
    return b + (es * n * m if kind == "correlated" else 0)


def bank(N, n, m, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    kw = dict(dtype=dtype, device="cuda")

    def spd(k, s):
        A = torch.randn(N, k, k, generator=g, **kw) * s
        return A @ A.transpose(1, 2) + s * s * torch.eye(k, **kw)
    F = torch.eye(n, **kw).repeat(N, 1, 1) + 0.05 * torch.randn(N, n, n, generator=g, **kw)
    return dict(x=torch.randn(N, n, generator=g, **kw), P=spd(n, 1.0), F=F, Q=spd(n, 0.1),
                H=torch.randn(N, m, n, generator=g, **kw), R=spd(m, 0.5),
                M=0.01 * torch.randn(N, n, m, generator=g, **kw), z=torch.randn(N, m, generator=g, **kw),
                z1=torch.randn(N, 1, generator=g, **kw))


def args(w, n, m, dtype, flags):
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z = w["x"].shape[0], n, m
    a.dtype = _lib.BKE_F32 if dtype == torch.float32 else _lib.BKE_F64
    a.flags, a.alpha_sq = flags, 1.0
    a.x = a.x_out = ptr(w["x"]); a.P = a.P_out = ptr(w["P"])
    a.F, a.F_stride = ptr(w["F"]), n * n
    a.Q, a.Q_stride = ptr(w["Q"]), n * n
    a.H, a.H_stride = ptr(w["H"]), m * n
    a.R, a.R_stride = ptr(w["R"]), m * m
    a.z = ptr(w["z"])
    return a


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--filters", type=int, default=1 << 20)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    opt = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("kf_update_forms_bench.py needs a CUDA device")
    lib = _lib.load()
    N = opt.filters
    print(json.dumps({"card": card(), "filters": N}))
    for n, m, dtype, path in ((4, 2, torch.float32, "register tile"), (6, 3, torch.float32, "register tile"),
                              (6, 3, torch.float64, "catch-all")):
        w = bank(N, n, m, dtype, seed=n * 10 + m)
        es = 4 if dtype == torch.float32 else 8
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        both = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
        a_step = args(w, n, m, dtype, both)
        a_corr = args(w, n, m, dtype, both)
        rows = []
        for start in (0, 1):
            r = _lib.KfRowsArgs()
            r.step = args(w, n, m, dtype, _lib.BKE_DO_UPDATE)
            r.step.z = ptr(w["z1"])
            r.start, r.rows = start, 1
            rows.append(r)
        Mp = ptr(w["M"])
        calls = {
            "step": lambda: _lib.check(lib.bke_kf_step(a_step, s)),
            "correlated": lambda: _lib.check(lib.bke_kf_step_correlated(a_corr, Mp, n * m, s)),
            "rows": lambda: [_lib.check(lib.bke_kf_update_rows(r, s)) for r in rows],
        }
        res = {}
        for kind, fn in calls.items():
            ms = time_ms(fn, opt.iters, opt.warmup)
            b = bytes_per_filter(kind, n, m, es)
            res[kind] = dict(ms=round(ms, 4), bytes_per_filter=b, hbm_share=round(b * N / (ms * 1e-3) / HBM_BPS, 3))
        ratio = {k: round((res[k]["ms"] / res[k]["bytes_per_filter"]) / (res["step"]["ms"] / res["step"]["bytes_per_filter"]), 2)
                 for k in ("correlated", "rows")}
        print(json.dumps({"shape": "%d/%d" % (n, m), "dtype": str(dtype).replace("torch.", ""), "path": path,
                          **res, "time_per_byte_vs_step": ratio}))
        del w
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
