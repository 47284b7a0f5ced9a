#!/usr/bin/env python
"""Time one discrete Bayes epoch over a bank of histogram filters: ``predict_update_bank`` (csrc/discrete_bayes.cu)
against the same epoch as a torch chain (a gather for the per-row roll, ``conv1d`` on circular padding, multiply,
sum, divide) in the same run, alternating the two, and against the reference looped over a subsample of rows on
the host CPU.

Workloads: 2^16 x 1024 bins (the single-pass path, a row per CTA) and 2^10 x 2^16 bins (rows too long to stage:
the multi-pass path, one row at a time) in fp32 and fp64 with K = 3 and 15 and per-row offsets, and one row of
2^24 bins.  The epoch must move the pdf read, the likelihood read and the posterior written: 12 B per bin in fp32,
24 in fp64; the HBM fraction is those bytes over the kernel time against the data sheet's 3.35 TB/s.  Prints one
JSON line per workload, with the card's name and power limit read in the same run, and writes them all to
``--out`` when given.

    python scripts/discrete_bayes_bench.py [--iters N] [--out FILE] [--quick]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                       # the measurement still stands; say what is unknown
        import torch
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown (%s)" % e}


def torch_chain(torch, pdf, lik, kr, offs):
    """predict (roll + circular conv1d), multiply, sum, divide: the epoch written with torch ops."""
    B, M = pdf.shape
    K = kr.shape[-1]
    c = (K - 1) // 2
    idx = (torch.arange(M, device=pdf.device)[None, :] - offs[:, None]) % M
    rolled = torch.gather(pdf, 1, idx)
    x = torch.nn.functional.pad(rolled[:, None, :], (c, K - 1 - c), mode="circular")
    prior = torch.nn.functional.conv1d(x, kr.to(pdf.dtype).reshape(1, 1, K))[:, 0, :]
    post = prior * lik
    return post / post.sum(dim=1, keepdim=True)


def time_pair(torch, f_a, f_b, iters):
    """Alternate a and b, CUDA events around each call: -> (median ms of a, median ms of b)."""
    ta, tb = [], []
    for _ in range(iters):
        for f, acc in ((f_a, ta), (f_b, tb)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            e1.synchronize()
            acc.append(e0.elapsed_time(e1))
    return float(np.median(ta)), float(np.median(tb))


def reference_ms_per_row(pdf, lik, kernel, offs, n_rows):
    """The unmodified reference (staged in oracle/_ref by build()) looped over the first n_rows rows on the host."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "filterpy", "discrete_bayes")):
        return None
    sys.path.insert(0, ref)
    import warnings
    warnings.filterwarnings("ignore", category=DeprecationWarning)
    from filterpy.discrete_bayes import predict, update
    n = min(n_rows, pdf.shape[0])
    t0 = time.perf_counter()
    for b in range(n):
        update(lik[b], predict(pdf[b], int(offs[b]), kernel, mode="wrap"))
    return (time.perf_counter() - t0) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="small shapes: a rehearsal of the script, not a measurement")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("discrete_bayes_bench.py needs a CUDA device; a CPU run measures nothing")
    from filterpy_b200.discrete_bayes.discrete_bayes import _step
    from filterpy_b200 import _lib
    dev = torch.device("cuda")
    info = card()
    shapes = [(1 << 16, 1024), (1 << 10, 1 << 16)]
    if args.quick:
        shapes = [(256, 1024), (4, 1 << 16)]
    work = [(B, M, dt, K) for (B, M) in shapes for dt in (np.float32, np.float64) for K in (3, 15)]
    work += [(1, 1 << 24, np.float32, 3), (1, 1 << 24, np.float64, 3)]
    rows = []
    for B, M, dt, K in work:
        rng = np.random.default_rng(B + M + K)
        tdt = torch.float32 if dt == np.float32 else torch.float64
        pdf = torch.rand(B, M, device=dev, dtype=torch.float64).to(tdt)
        pdf /= pdf.sum(1, keepdim=True)
        lik = (torch.rand(B, M, device=dev, dtype=torch.float64) + 0.01).to(tdt)
        kernel = rng.random(K)
        kernel /= kernel.sum()
        kr = torch.from_numpy(kernel).to(dev)
        offs = torch.from_numpy(rng.integers(-M, M, B)).to(dev)
        out = torch.empty_like(pdf)
        multi = _lib.load().bke_db_workspace_bytes(M, _lib.BKE_F32 if dt == np.float32 else _lib.BKE_F64) > 0

        def ours():
            _step(pdf, out, kernel=kr, offset=offs, likelihood=lik, normalize=True)

        def chain():
            torch_chain(torch, pdf, lik, kr.flip(0), offs)

        ours(); chain(); torch.cuda.synchronize()                     # warm both (attributes, cuDNN algorithms)
        iters = args.iters if not multi else max(3, args.iters // 4)
        t_ours, t_chain = time_pair(torch, ours, chain, iters)
        ours()
        diff = float((out.double() - torch_chain(torch, pdf, lik, kr.flip(0), offs).double()).abs().max())
        nbytes = 3 * B * M * pdf.element_size()
        ref_rows = 64 if M <= 1024 else (2 if M <= (1 << 16) else 1)
        if args.quick:
            ref_rows = 2
        ref_ms = reference_ms_per_row(pdf[:ref_rows].cpu().numpy(), lik[:ref_rows].cpu().numpy(), kernel,
                                      offs[:ref_rows].cpu().numpy(), ref_rows)
        r = dict(workload="%d x %d" % (B, M), dtype=np.dtype(dt).name, K=K, path="multi-pass" if multi else "single-pass",
                 kernel_ms=round(t_ours, 4), torch_chain_ms=round(t_chain, 4), speedup=round(t_chain / t_ours, 2),
                 bytes_per_bin=3 * pdf.element_size(), hbm_fraction=round(nbytes / (t_ours * 1e-3) / HBM, 3),
                 max_abs_diff_vs_chain=diff,
                 reference_cpu_ms_per_row=None if ref_ms is None else round(ref_ms, 4),
                 reference_cpu_s_per_epoch=None if ref_ms is None else round(ref_ms * B / 1e3, 3),
                 reference_rows_timed=ref_rows if ref_ms is not None else 0, **info)
        rows.append(r)
        print(json.dumps(r), flush=True)
        del pdf, lik, out
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
