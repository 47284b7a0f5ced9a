#!/usr/bin/env python
"""Bank resampling (csrc/resample_bank.cu) on the GPU: time per call of systematic, stratified, multinomial,
residual and the per-set gather of a 4-float state, for banks from many small sets to a few huge ones,
against the route a bank had before (one single-set call per set).

    python scripts/resample_bank_bench.py [--iters 20] [--warmup 3]

Times are CUDA-event medians over --iters calls after --warmup calls.  Algorithmic bytes: 12 B per
particle systematic (8 B weight read, 4 B index written), 20 B stratified (+ 8 B uniform), and
2 * 16 + 4 B gather (row read and written, index read), 24 B multinomial (weight, uniform, int64 index)
and at most 20 B residual (weight, index, a uniform for each of the M - k searched particles); the share
is of the data sheet's 3.35 TB/s (H100 SXM).  The multinomial and residual legs run on the first three
shapes (a few huge sets are the single-set path's ground).  A seeded sample of rows is checked against
the C / NumPy oracles in the same run.
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

from filterpy_b200.monte_carlo import BankResamplePlan, ResamplePlan, residual_resample_with_uniforms  # noqa: E402
from oracle import resample as ors                                     # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "tests"))
import resample_bank_mr_oracle as mro                                   # noqa: E402

PEAK_BPS = 3.35e12
SHAPES = [(1 << 16, 1024), (1 << 20, 64), (1 << 12, 1 << 14), (16, 1 << 22)]


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return float(np.median(ts))


def power_limit():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[torch.cuda.current_device()]
    except Exception as e:      # the number is reported without it, but says so
        return "unknown (%s)" % e


def heavy_bank(B, M, gen):
    w = torch.rand((B, M), generator=gen, device="cuda", dtype=torch.float64) ** 4
    w = w / w.sum(dim=1, keepdim=True)
    # the sequential cumsum of a row normalised with a pairwise sum can end a few ulps below 1, under the last
    # positions of a u close to 1 (the reference's IndexError); 1e-9 on the last weight keeps every row valid
    w[:, -1] += 1e-9
    return w


def check_rows(w, u, U, idx_s, idx_t, rows):
    for b in rows:
        wb = w[b].cpu().numpy()
        assert np.array_equal(idx_s[b].cpu().numpy(), ors.systematic_resample_c(wb, float(u[b]))), ("systematic", b)
        assert np.array_equal(idx_t[b].cpu().numpy(), ors.stratified_resample_c(wb, U[b].cpu().numpy())), ("stratified", b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    print("device: %s; power limit, max SM clock: %s" % (torch.cuda.get_device_name(), power_limit()), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(1)
    results = []
    for B, M in SHAPES:
        w = heavy_bank(B, M, gen)
        u = torch.rand(B, generator=gen, device="cuda", dtype=torch.float64)
        U = torch.rand((B, M), generator=gen, device="cuda", dtype=torch.float64)
        parts = torch.rand((B, M, 4), generator=gen, device="cuda", dtype=torch.float32)
        out = torch.empty_like(parts)
        plan = BankResamplePlan(B, M)
        idx_t = torch.empty((B, M), dtype=torch.int32, device="cuda")
        t_sys = timed(lambda: plan.systematic(w, u), args.iters, args.warmup)
        plan.raise_if_overflow()
        t_str = timed(lambda: plan.stratified(w, U, out=idx_t), args.iters, args.warmup)
        plan.raise_if_overflow()
        t_gat = timed(lambda: plan.gather(parts, idx_t, out=out), args.iters, args.warmup)
        plan.raise_if_bad_index()
        rows = sorted(set(np.random.default_rng(B).integers(0, B, size=8).tolist()) | {0, B - 1})
        check_rows(w, u, U, plan.indexes, idx_t, rows)
        n = B * M
        r = {"shape": [B, M], "particles": n,
             "systematic_ms": t_sys * 1e3, "systematic_TBps": 12 * n / t_sys / 1e12,
             "stratified_ms": t_str * 1e3, "stratified_TBps": 20 * n / t_str / 1e12,
             "gather_ms": t_gat * 1e3, "gather_TBps": 36 * n / t_gat / 1e12, "rows_checked": len(rows)}
        if M < (1 << 22):
            idx64 = torch.empty((B, M), dtype=torch.int64, device="cuda")
            t_mul = timed(lambda: plan.multinomial(w, U, out=idx64), args.iters, args.warmup)
            t_res = timed(lambda: plan.residual(w, U), args.iters, args.warmup)
            exact = int(((plan.status & 2) != 0).sum())
            plan.raise_if_overflow()
            wr, Ur = w[rows].cpu().numpy(), U[rows].cpu().numpy()
            assert np.array_equal(idx64[rows].cpu().numpy(), mro.multinomial_bank(wr, Ur)), "multinomial"
            assert np.array_equal(plan.indexes[rows].cpu().numpy(), mro.residual_bank(wr, Ur)[0]), "residual"
            r.update({"multinomial_ms": t_mul * 1e3, "multinomial_TBps": 24 * n / t_mul / 1e12,
                      "residual_ms": t_res * 1e3, "residual_TBps": 20 * n / t_res / 1e12,
                      "residual_exact_sets": exact})
            del idx64
        for k in ("systematic", "stratified", "gather", "multinomial", "residual"):
            if k + "_TBps" in r:
                r[k + "_peak_share"] = r[k + "_TBps"] * 1e12 / PEAK_BPS
        results.append(r)
        print(json.dumps(r), flush=True)
        del w, U, parts, out, plan, idx_t
        torch.cuda.empty_cache()

    # the route before the bank call: one single-set ResamplePlan call per set
    for B, M, label in ((1 << 12, 1024, "per_set_loop"), (16, 1 << 22, "single_set_calls")):
        w = heavy_bank(B, M, gen)
        u = torch.rand(B, generator=gen, device="cuda", dtype=torch.float64)
        one = ResamplePlan(M)
        outs = torch.empty((B, M), dtype=torch.int32, device="cuda")
        uh = u.cpu().numpy().tolist()

        def loop():
            for b in range(B):
                one.systematic(w[b], uh[b], out=outs[b])
        t_loop = timed(loop, max(3, args.iters // 4), 1)
        plan = BankResamplePlan(B, M)
        t_bank = timed(lambda: plan.systematic(w, u), args.iters, args.warmup)
        torch.cuda.synchronize()
        assert torch.equal(outs, plan.indexes), label
        r = {"compare": label, "shape": [B, M], "loop_ms": t_loop * 1e3, "bank_ms": t_bank * 1e3,
             "bank_speedup": t_loop / t_bank}
        results.append(r)
        print(json.dumps(r), flush=True)

    # multinomial / residual: a loop of the single-set calls (residual reads k back per set) against the bank
    B, M = 1 << 12, 1024
    w = heavy_bank(B, M, gen)
    U = torch.rand((B, M), generator=gen, device="cuda", dtype=torch.float64)
    one = ResamplePlan(M)
    plan = BankResamplePlan(B, M)
    mul_loop = torch.empty((B, M), dtype=torch.int64, device="cuda")
    res_loop = torch.empty((B, M), dtype=torch.int32, device="cuda")

    def mloop():
        for b in range(B):
            one.multinomial(w[b], U[b], out=mul_loop[b])

    def rloop():
        for b in range(B):
            res_loop[b] = residual_resample_with_uniforms(w[b], lambda m: U[b, :m].cpu().numpy())[0]
    for label, loop, bank, check in (
            ("multinomial_loop", mloop, lambda: plan.multinomial(w, U), lambda out: torch.equal(out, mul_loop)),
            ("residual_loop", rloop, lambda: plan.residual(w, U), lambda out: torch.equal(out, res_loop))):
        t_loop = timed(loop, 3, 1)
        t_bank = timed(bank, args.iters, args.warmup)
        torch.cuda.synchronize()
        assert check(bank()), label
        r = {"compare": label, "shape": [B, M], "loop_ms": t_loop * 1e3, "bank_ms": t_bank * 1e3,
             "bank_speedup": t_loop / t_bank}
        results.append(r)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
