#!/usr/bin/env python
"""The gated bank epoch (BankResamplePlan.resample_if_degenerate, csrc/resample_bank.cu) on the GPU, against
the route a bank had before it: a torch row sum, a division, a squared sum and a compare, the bank
systematic resample and gather of every set, a torch.where that keeps the healthy sets and a masked fill of
the weights.

    python scripts/resample_bank_gated_bench.py [--iters 10] [--warmup 2]

For each bank (4 x fp32 particles) and each fraction f of degenerate sets, the weights are built so that
exactly round(f B) chosen sets have neff < M / 2: rand^8 rows (neff ~ 0.21 M) among rand + 0.5 rows
(neff ~ 0.92 M).  Both routes update weights and particles in place, so each call gets fresh copies, made
outside the timed window.  The two alternate within one run; times are CUDA-event medians.  The gated
statistics launch is timed on its own too, so that resample + gather = gated - statistics.

Algorithmic bytes of the gated call: 16 B per particle for the statistics (weight read, normalised weight
written) and, per particle of a resampled set, 12 B for the resample (weight read, index written) and
2 * 16 + 4 B for the gather (particle read and written, index read); the share is of the data sheet's
3.35 TB/s (H100 SXM).  A seeded sample of rows is checked against the per-set loop in the same run.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from filterpy_b200.monte_carlo import BankResamplePlan                  # noqa: E402
from oracle import resample as ors                                      # noqa: E402
import resample_bank_gated_oracle as rgo                                # noqa: E402

PEAK_BPS = 3.35e12
SHAPES = [(1 << 16, 1024), (1 << 20, 64), (1 << 12, 4096)]
FRACTIONS = [0.0, 0.05, 0.25, 1.0]


def power_limit():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:      # the number is reported without it, but says so
        return "unknown (%s)" % e


def bank(B, M, f, gen):
    """weights with exactly round(f B) sets below M / 2, and those sets' rows"""
    n_deg = int(round(f * B))
    rows = torch.randperm(B, generator=gen, device="cuda")[:n_deg]
    w = torch.rand((B, M), generator=gen, device="cuda", dtype=torch.float64) + 0.5
    w[rows] = torch.rand((n_deg, M), generator=gen, device="cuda", dtype=torch.float64) ** 8
    return w, rows


def timed_pair(fns, reset, iters, warmup):
    """CUDA-event medians of each fn, alternating them, each call on fresh inputs"""
    for _ in range(warmup):
        for fn in fns:
            reset()
            fn()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(iters):
        for k, fn in enumerate(fns):
            reset()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts[k].append(a.elapsed_time(b) * 1e-3)
    return [float(np.median(t)) for t in ts]


def check_rows(w0, p0, u, w, p, plan, rows):
    """rows of the gated result against the per-set loop on the same draws"""
    M = w0.shape[1]
    for b in rows:
        wb = w0[b:b + 1].cpu().numpy()
        o = rgo.resample_if_degenerate_loop(wb, p0[b:b + 1].cpu().numpy(), [float(u[b])],
                                            resample=ors.systematic_resample_c)
        assert bool(plan._resampled[b]) == bool(o["resampled"][0]), ("mask", b)
        assert np.array_equal(w[b].cpu().numpy().view(np.uint64), o["weights"][0].view(np.uint64)), ("weights", b)
        assert np.array_equal(p[b].cpu().numpy(), o["particles"][0]), ("particles", b)
        assert float(plan._neff[b]) == o["neff"][0], ("neff", b)
    assert M > 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    print("device: %s; power limit, max SM clock: %s" % (torch.cuda.get_device_name(), power_limit()), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(1)
    for B, M in SHAPES:
        n = B * M
        p0 = torch.rand((B, M, 4), generator=gen, device="cuda", dtype=torch.float32)
        u = torch.rand(B, generator=gen, device="cuda", dtype=torch.float64)
        w = torch.empty((B, M), dtype=torch.float64, device="cuda")
        p = torch.empty_like(p0)
        scratch = torch.empty_like(p0)
        plan = BankResamplePlan(B, M)
        chain_plan = BankResamplePlan(B, M)
        thr = M / 2
        for f in FRACTIONS:
            w0, deg = bank(B, M, f, gen)

            def reset():
                w.copy_(w0)
                p.copy_(p0)

            def gated():
                plan.resample_if_degenerate(w, p, u=u)

            def stats():
                plan._gated(plan._lib.bke_resample_bank_gated_stats, w, p, None, None, None)

            def chain():
                w.div_(w.sum(dim=1, keepdim=True))
                mask = (1.0 / (w * w).sum(dim=1)) < thr
                chain_plan.systematic(w, u)
                chain_plan.gather(p, out=scratch)
                torch.where(mask[:, None, None], scratch, p, out=p)
                w.masked_fill_(mask[:, None], 1.0 / M)

            t_gated, t_chain, t_stats = timed_pair([gated, chain, stats], reset, args.iters, args.warmup)
            reset()
            gated()
            torch.cuda.synchronize()
            n_res = int(plan._resampled.sum())
            assert n_res == deg.numel(), (n_res, deg.numel())
            fails = int(plan.status.sum())
            rng = np.random.default_rng(B + int(100 * f))
            rows = sorted(set(rng.integers(0, B, size=6).tolist()) | set(deg[:4].tolist()))
            check_rows(w0, p0, u, w, p, plan, rows)
            moved = n_res * M
            nbytes = 16 * n + moved * (12 + 2 * 16 + 4)
            r = {"shape": [B, M], "degenerate_fraction": f, "resampled_sets": n_res, "failed_sets": fails,
                 "gated_ms": t_gated * 1e3, "stats_ms": t_stats * 1e3, "resample_gather_ms": (t_gated - t_stats) * 1e3,
                 "chain_ms": t_chain * 1e3, "gated_over_chain": t_gated / t_chain,
                 "gated_bytes": nbytes, "gated_TBps": nbytes / t_gated / 1e12,
                 "gated_peak_share": nbytes / t_gated / PEAK_BPS, "stats_peak_share": 16 * n / t_stats / PEAK_BPS,
                 "rows_checked": len(rows)}
            print(json.dumps(r), flush=True)
            del w0
        del p0, w, p, scratch, plan, chain_plan
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
