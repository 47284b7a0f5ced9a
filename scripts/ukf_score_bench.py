#!/usr/bin/env python
"""Time UnscentedKalmanFilter.score_measurements (bke_ukf_score, csrc/ukf_score_kernel.cuh) on one GPU, beside the
linear score of the same shape and the chain a user would otherwise build from the public pieces.

    python scripts/ukf_score_bench.py [--repeats 7] [--warmup 3] [--out FILE]

Workloads, each in fp32 and fp64:
  rae_scan  N = 2^17 tracks x K = 1024 candidates of one scan shared by every track, 6/3 CV + range / azimuth /
            elevation (the benchmark's radar tracker)
  rb_own    N = 2^20 tracks x K = 8 candidates of their own [N, K, m], 4/2 CV + range / bearing
Arms, alternated in every repeat; each timed window holds --calls back-to-back calls between two CUDA events (after
warm-up) and gives ms per call; the median over repeats:
  ukf     (a) the new call, bke_ukf_score through the C-ABI on a struct filled once: kernel-bound, its share of HBM
              below is the kernel's
  lin     (b) bke_score_measurements the same way, on a linear bank of the same shape (x, P, a shared H and R): the
              same phase B
  chain   (c) MerweScaledSigmaPoints.sigma_points -> hx in torch -> unscented_transform -> score with mean and S,
              end to end from Python (host work included)
  method  UnscentedKalmanFilter.score_measurements end to end from Python: (a) plus the method's host work
The outputs of (a) and (c) are compared (log-likelihood relative to max(|ll|, 1), tolerance 1e-6 fp64 / 1e-2 fp32).
Algorithmic bytes: x and P once per track, R shared, the candidates once (a shared scan is K m words) and two
outputs of N K words; over the time per call as a share of the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s
(``hbm_share`` for the C-ABI arms; ``hbm_share_end_to_end`` for the Python arms, which includes their host work).  One
JSON line per workload and arm, with the GPU name, power limit and SM clock read in the same run.
"""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from filterpy_b200.kalman import (UnscentedKalmanFilter, MerweScaledSigmaPoints, ConstVelFx,  # noqa: E402
                                  RangeAzElHx, RangeBearingHx, unscented_transform)
from filterpy_b200 import _lib                                                                  # noqa: E402
from filterpy_b200._dev import bke_dtype, ptr                                                    # noqa: E402
from filterpy_b200.stats.stats import score                                                    # noqa: E402

HBM = 3.35e12
TOL = {torch.float32: 1e-2, torch.float64: 1e-6}
WORKLOADS = {"rae_scan": (1 << 17, 1024, 6, 3, True), "rb_own": (1 << 20, 8, 4, 2, False)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock, max_clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, sm_clock=clock, max_sm_clock=max_clock)


def inputs(N, K, n, m, dtype, shared, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    kw = dict(device="cuda", dtype=dtype)
    x = torch.zeros(N, n, **kw)
    x[:, 1::2] = (torch.rand(N, n // 2, generator=g, **kw) - 0.5) * 20
    x[:, 0] = 100 + 400 * torch.rand(N, generator=g, **kw)
    x[:, 2] = (torch.rand(N, generator=g, **kw) - 0.5) * 600
    if n == 6:
        x[:, 4] = 20 + 180 * torch.rand(N, generator=g, **kw)
    P = torch.diag_embed(1 + 8 * torch.rand(N, n, generator=g, **kw))
    sd = torch.tensor([1.0, 0.005, 0.005][:m], **kw)
    R = torch.diag(sd ** 2)
    rho = torch.sqrt(x[:, 0] ** 2 + x[:, 2] ** 2)
    h = [torch.sqrt(rho ** 2 + (x[:, 4] ** 2 if n == 6 else 0)), torch.atan2(x[:, 2], x[:, 0])]
    if n == 6:
        h.append(torch.atan2(x[:, 4], rho))
    zh = torch.stack(h, 1)
    z = zh[:1 if shared else N, None, :] + 3 * sd * torch.randn(1 if shared else N, K, m, generator=g, **kw)
    return x, P, R, z.contiguous()


def hx_torch(s, m):
    px, py = s[..., 0], s[..., 2]
    rho2 = px * px + py * py
    if m == 2:
        return torch.stack([torch.sqrt(rho2), torch.atan2(py, px)], -1)
    pz = s[..., 4]
    return torch.stack([torch.sqrt(rho2 + pz * pz), torch.atan2(py, px), torch.atan2(pz, torch.sqrt(rho2))], -1)


def algo_bytes(N, K, n, m, itemsize, shared):
    return itemsize * (N * (n + n * n) + m * m + (K * m if shared else N * K * m) + 2 * N * K)


def time_window(fn, calls):
    """ms per call over `calls` back-to-back calls between two CUDA events."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(calls):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / calls


def abi_args(N, K, n, m, dtype, hx_model, x, P, R, z, ll, maha):
    """bke_ukf_score_args for the bank, filled once."""
    a = _lib.UkfScoreArgs()
    a.n_filters, a.n_candidates, a.dim_x, a.dim_z = N, K, n, m
    a.dtype, a.flags, a.hx_model = bke_dtype(dtype), 0, hx_model
    a.alpha, a.beta, a.kappa = 0.5, 2.0, 0.0
    a.x, a.P, a.R, a.R_stride = ptr(x), ptr(P), ptr(R), 0
    a.z, a.z_track_stride, a.z_cand_stride = ptr(z), (0 if z.shape[0] == 1 else K * m), m
    a.log_likelihood, a.mahalanobis = ptr(ll), ptr(maha)
    return a


def lin_args(N, K, n, m, dtype, x, P, H, R, z, ll, maha):
    """bke_score_args of the linear bank of the same shape, filled once."""
    a = _lib.ScoreArgs()
    a.n_tracks, a.n_candidates, a.dim_x, a.dim_z, a.dtype = N, K, n, m, bke_dtype(dtype)
    a.x, a.P, a.H, a.R = ptr(x), ptr(P), ptr(H), ptr(R)
    a.z, a.z_track_stride, a.z_cand_stride = ptr(z), (0 if z.shape[0] == 1 else K * m), m
    a.log_likelihood, a.mahalanobis = ptr(ll), ptr(maha)
    return a


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    rows = []
    for name, (N, K, n, m, shared) in WORKLOADS.items():
        for dtype in (torch.float32, torch.float64):
            x, P, R, z = inputs(N, K, n, m, dtype, shared)
            pts = MerweScaledSigmaPoints(n, 0.5, 2.0, 0.0)
            u = UnscentedKalmanFilter(n, m, 0.1, RangeAzElHx() if m == 3 else RangeBearingHx(), ConstVelFx(), pts,
                                      n_filters=N, dtype=dtype, device="cuda", diagnostics=False)
            u.x = x; u.P = P; u.R = R
            H = torch.zeros(m, n, device="cuda", dtype=dtype)
            H[torch.arange(m), 2 * torch.arange(m)] = 1
            Wm = torch.as_tensor(pts.Wm, device="cuda", dtype=dtype)
            Wc = torch.as_tensor(pts.Wc, device="cuda", dtype=dtype)

            ll_a, mh_a = torch.empty(N, K, device="cuda", dtype=dtype), torch.empty(N, K, device="cuda", dtype=dtype)
            ll_b, mh_b = torch.empty_like(ll_a), torch.empty_like(mh_a)
            a_ukf = abi_args(N, K, n, m, dtype, u.hx.model, x, P, R, z, ll_a, mh_a)
            a_lin = lin_args(N, K, n, m, dtype, x, P, H, R, z, ll_b, mh_b)

            def arm_ukf():
                _lib.check(lib.bke_ukf_score(ctypes.byref(a_ukf), stream))

            def arm_lin():
                _lib.check(lib.bke_score_measurements(ctypes.byref(a_lin), stream))

            def arm_method():
                return u.score_measurements(z)

            def arm_chain():
                sig = pts.sigma_points(x, P)
                zh, S = unscented_transform(hx_torch(sig, m), Wm, Wc, R)
                o = score(z, mean=zh.contiguous(), S=S.contiguous(), want=("log_likelihood", "mahalanobis"))
                return o["log_likelihood"], o["mahalanobis"]
            arms = {"ukf": arm_ukf, "lin": arm_lin, "chain": arm_chain, "method": arm_method}
            for fn in arms.values():
                for _ in range(args.warmup):
                    fn()
            torch.cuda.synchronize()
            arm_ukf()
            la, _ = arm_method()
            lc, _ = arm_chain()
            torch.cuda.synchronize()
            assert torch.equal(la, ll_a)                       # the method is the C-ABI call
            err = ((la.double() - lc.double()).abs() / lc.double().abs().clamp(min=1.0)).max().item()
            times = {k: [] for k in arms}
            for _ in range(args.repeats):
                for k, fn in arms.items():
                    times[k].append(time_window(fn, args.calls))
            nbytes = algo_bytes(N, K, n, m, torch.finfo(dtype).bits // 8, shared)
            info = gpu_info()                                  # the SM clock just after the timed repeats
            for k in arms:
                ms = sorted(times[k])[len(times[k]) // 2]
                row = dict(workload=name, dtype=str(dtype).split(".")[1], arm=k, N=N, K=K, n=n, m=m, ms=round(ms, 4),
                           spread_ms=[round(min(times[k]), 4), round(max(times[k]), 4)], algo_bytes=nbytes,
                           ukf_vs_chain_err=err, calls_per_window=args.calls,
                           agrees=err <= TOL[dtype], **info)
                share = round(nbytes / (ms * 1e-3) / HBM, 4)
                row["hbm_share" if k in ("ukf", "lin") else "hbm_share_end_to_end"] = share
                rows.append(row)
                print(json.dumps(row), flush=True)
            del u, x, P, z
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as fh:
            for r in rows:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
