#!/usr/bin/env python
"""Time bke_score_measurements (csrc/score.cu) on one GPU, with the torch chain a user would otherwise write beside it.

    python scripts/score_bench.py [--repeats 10] [--warmup 3] [--out FILE]

Configurations, each in fp32 and fp64, per-track x, P and shared H, R:
  scan   N = 2^17 tracks x K = 1024 candidates of one scan shared by every track, at 4/2 and 6/3
  own    N = 2^20 tracks x K = 8 candidates of their own [N, K, m], at 4/2
Arms: "ll" (log_likelihood alone) and "score" (log_likelihood + mahalanobis, score_measurements), and "torch": batched
S = H P H' + R, torch.linalg.inv and slogdet, and einsum over y[N, K, m], on the same inputs.  The arms alternate in
each repeat; times are CUDA events around the call after warm-up, the median over repeats.  Algorithmic bytes come
from the shapes: x and P once per track, the candidates once (a shared scan is K m words), and the requested outputs
N K words each; they are reported over the time as a share of the H100 SXM data-sheet HBM3 bandwidth, 3.35 TB/s.  The
kernel's outputs are compared with the torch chain's at the compute type's tolerance.  One JSON line per arm, with the
GPU name, power limit and max SM clock.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from filterpy_b200.stats.stats import score                                                     # noqa: E402

HBM = 3.35e12
TOL = {torch.float32: 1e-3, torch.float64: 1e-6}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def inputs(N, K, n, m, dtype, shared_scan, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    kw = dict(device="cuda", dtype=dtype, generator=g)
    x = torch.randn(N, n, **kw)
    A = torch.randn(N, n, n, **kw)
    P = A @ A.transpose(1, 2) / n + torch.eye(n, device="cuda", dtype=dtype)
    H = torch.randn(m, n, **kw)
    R = torch.eye(m, device="cuda", dtype=dtype) * 0.5
    z = torch.randn(1 if shared_scan else N, K, m, **kw) * 2
    return x, P, H, R, z


def torch_chain(x, P, H, R, z):
    S = H @ P @ H.T + R
    SI = torch.linalg.inv(S)
    logdet = torch.linalg.slogdet(S)[1]
    y = z - (x @ H.T)[:, None, :]
    d2 = torch.einsum("nka,nab,nkb->nk", y, SI, y)
    m = S.shape[-1]
    return -0.5 * (d2 + logdet[:, None] + m * math.log(2 * math.pi)), torch.sqrt(d2)


def algo_bytes(N, K, n, m, itemsize, shared_scan, outs):
    return itemsize * (N * (n + n * n) + (K * m if shared_scan else N * K * m) + N * K * outs)


def time_it(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "score_bench.py needs a GPU"
    info = gpu_info()
    configs = [("scan", 1 << 17, 1024, 4, 2), ("scan", 1 << 17, 1024, 6, 3), ("own", 1 << 20, 8, 4, 2)]
    lines = []
    for layout, N, K, n, m in configs:
        for dtype in (torch.float32, torch.float64):
            x, P, H, R, z = inputs(N, K, n, m, dtype, layout == "scan")
            arms = {
                "ll": lambda: score(z, x=x, P=P, H=H, R=R, want=("log_likelihood",)),
                "score": lambda: score(z, x=x, P=P, H=H, R=R, want=("log_likelihood", "mahalanobis")),
                "torch": lambda: torch_chain(x, P, H, R, z),
            }
            for fn in arms.values():
                for _ in range(args.warmup):
                    fn()
            torch.cuda.synchronize()
            times = {k: [] for k in arms}
            for _ in range(args.repeats):
                for k, fn in arms.items():
                    times[k].append(time_it(fn, 1))
            out = arms["score"]()
            ll_t, d_t = arms["torch"]()
            scale = max(ll_t.abs().max().item(), 1.0)
            err_ll = (out["log_likelihood"] - ll_t).abs().max().item() / scale
            err_d = (out["mahalanobis"] - d_t).abs().max().item() / max(d_t.abs().max().item(), 1.0)
            agree = err_ll < TOL[dtype] and err_d < TOL[dtype]
            itemsize = 4 if dtype == torch.float32 else 8
            for k in arms:
                ms = sorted(times[k])[len(times[k]) // 2]
                rec = dict(layout=layout, N=N, K=K, n=n, m=m, dtype=str(dtype).replace("torch.", ""), arm=k, ms=ms,
                           pairs_per_s=N * K / (ms * 1e-3), **info)
                if k != "torch":
                    nb = algo_bytes(N, K, n, m, itemsize, layout == "scan", 1 if k == "ll" else 2)
                    rec.update(bytes=nb, hbm_fraction=nb / (ms * 1e-3) / HBM)
                else:
                    rec.update(max_rel_err_ll=err_ll, max_rel_err_maha=err_d, agree=agree)
                print(json.dumps(rec), flush=True)
                lines.append(rec)
            del x, P, H, R, z, out, ll_t, d_t
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")
    if not all(r.get("agree", True) for r in lines):
        sys.exit("the kernel and the torch chain disagree beyond the tolerance")


if __name__ == "__main__":
    main()
