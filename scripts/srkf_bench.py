#!/usr/bin/env python
"""Time the square-root filter step (bke_srkf_step) against the dense linear filter step (bke_kf_step) on the
same banks, in one run on one GPU.

    python scripts/srkf_bench.py [--steps 50] [--warmup 10] [--repeats 5]

Legs (one fused predict + update per step, in place, per-filter models, no optional outputs):
  cv2d_f32  kf_bank_cv2d, 2^20 filters, 4/2, fp32     (the register tile)
  cv2d_f64  kf_bank_cv2d, 2^20 filters, 4/2, fp64     (the register tile)
  ca3d_f64  kf_bank_ca3d, 2^18 filters, 9/3, fp64     (config C3's shape, the warp-per-filter kernel)
The workloads' discrete white-noise Q is rank-deficient, so cholesky refuses it: both arms step the bank with
Q + 1e-3 max|Q| I (oracle.srkf.make_pd), the square-root arm with Lq = chol(that Q) and Lr = chol(R).  The two
arms of a leg alternate, repeat by repeat.  Times are CUDA events around `steps` steps after `warmup` steps;
the median over repeats is reported.  Bytes per filter-step are computed from the shapes: x and L (P) in and
out, F, Lq (Q), H, Lr (R) and z in, the same count for both arms, over the H100 SXM data-sheet 3.35 TB/s.
Each leg's square-root outputs are checked once, after one step, against the dgeqr2 oracle on a 4096-filter
subset.  One JSON line per leg and arm goes to stdout, with the GPU name, power limit and max SM clock.
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

from filterpy_b200 import _lib                                                                   # noqa: E402
from filterpy_b200.common import workloads as wl                                                 # noqa: E402
from oracle import srkf as osr                                                                   # noqa: E402

PEAK_BPS = 3.35e12
LEGS = [("cv2d_f32", wl.kf_bank_cv2d, 1 << 20, np.float32), ("cv2d_f64", wl.kf_bank_cv2d, 1 << 20, np.float64),
        ("ca3d_f64", wl.kf_bank_ca3d, 1 << 18, np.float64)]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def bytes_per_filter_step(n, m, itemsize):
    return (2 * n + 2 * n * n + n * n + n * n + m * n + m * m + m) * itemsize


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("srkf_bench.py needs a GPU")
    lib = _lib.load()
    info = gpu_info()
    stream = torch.cuda.current_stream().cuda_stream
    for leg, make, N, dtype in LEGS:
        w = make(N, steps=1)
        w["Q"] = osr.make_pd(w["Q"])
        n, m = w["x"].shape[1], w["H"].shape[1]
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()       # noqa: E731
        x0, P0 = dev(w["x"]), dev(w["P"])
        L0 = dev(np.linalg.cholesky(w["P"]))
        F, H, Q, R, z = dev(w["F"]), dev(w["H"]), dev(w["Q"]), dev(w["R"]), dev(w["zs"][0])
        Lq, Lr = dev(np.linalg.cholesky(w["Q"])), dev(np.linalg.cholesky(w["R"]))
        bt = _lib.BKE_F32 if dtype == np.float32 else _lib.BKE_F64

        xs, Ls = x0.clone(), L0.clone()
        sa = _lib.SrkfArgs()
        sa.n_filters, sa.dim_x, sa.dim_z, sa.dtype = N, n, m, bt
        sa.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
        sa.x = sa.x_out = xs.data_ptr(); sa.L = sa.L_out = Ls.data_ptr()
        sa.F, sa.F_stride, sa.H, sa.H_stride = F.data_ptr(), n * n, H.data_ptr(), m * n
        sa.Lq, sa.Lq_stride, sa.Lr, sa.Lr_stride = Lq.data_ptr(), n * n, Lr.data_ptr(), m * m
        sa.z = z.data_ptr()
        xk, Pk = x0.clone(), P0.clone()
        ka = _lib.KfArgs()
        ka.n_filters, ka.dim_x, ka.dim_z, ka.dtype, ka.alpha_sq = N, n, m, bt, 1.0
        ka.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
        ka.x = ka.x_out = xk.data_ptr(); ka.P = ka.P_out = Pk.data_ptr()
        ka.F, ka.F_stride, ka.H, ka.H_stride = F.data_ptr(), n * n, H.data_ptr(), m * n
        ka.Q, ka.Q_stride, ka.R, ka.R_stride = Q.data_ptr(), n * n, R.data_ptr(), m * m
        ka.z = z.data_ptr()
        arms = {"srkf": lambda: _lib.check(lib.bke_srkf_step(sa, stream)),
                "kf": lambda: _lib.check(lib.bke_kf_step(ka, stream))}

        # the output check: one step from the initial state against the oracle
        arms["srkf"]()
        torch.cuda.synchronize()
        sel = np.sort(np.random.default_rng(0).choice(N, 4096, replace=False))
        o = osr.srkf_step_bank(w["x"][sel], np.linalg.cholesky(w["P"][sel]), w["zs"][0][sel], w["F"][sel], w["H"][sel],
                               np.linalg.cholesky(w["Q"][sel]), np.linalg.cholesky(w["R"][sel]))
        err = max(float(np.abs(xs.cpu().numpy()[sel] - o["x"]).max() / np.abs(o["x"]).max()),
                  float(np.abs(Ls.cpu().numpy()[sel] - o["L"]).max() / np.abs(o["L"]).max()))

        times = {k: [] for k in arms}
        for _ in range(args.repeats):
            for name, fn in arms.items():
                for _ in range(args.warmup):
                    fn()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / args.steps)
        nbytes = bytes_per_filter_step(n, m, np.dtype(dtype).itemsize)
        for name in arms:
            ms = float(np.median(times[name]))
            res = dict(leg=leg, arm=name, n_filters=N, dim_x=n, dim_z=m, dtype=np.dtype(dtype).name,
                       ms_per_step=round(ms, 5), ms_all=[round(t, 5) for t in times[name]],
                       bytes_per_filter_step=nbytes, share_of_hbm_peak=round(nbytes * N / (ms * 1e-3) / PEAK_BPS, 3),
                       **info)
            if name == "srkf":
                res["max_rel_err_vs_oracle_4096"] = err
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
