#!/usr/bin/env python
"""Time the fixed-lag smoother (bke_fls_smooth) on a 2^20-filter 4/2 fp32 bank with per-filter models
(kf_bank_cv2d), in one run on one GPU.

    python scripts/fls_bench.py [--steps 20] [--warmup 3] [--repeats 5]

Legs:
  batch_N{1,4,16}  smooth_batch at T = 32 epochs per call (count = 0, history = the [T, N, n] output, xhat
                   written): the fused kernel, one launch per call.  Reported per epoch.
  online_N4        smooth() per epoch: T = 1 per call, continuing the history (count = 0 .. steps-1 in each
                   repeat), against bke_kf_step on the same bank; the two arms alternate, repeat by repeat.
Times are CUDA events around `steps` calls after `warmup` calls; the median over repeats is reported.

Bytes per filter-step are what the algorithm must move, computed from the shapes:
  batch:  z in, the finished row and xhat out, (m + 2n) words, plus x, P, F, Q, H, R in and x, P out once per call
          (divided by T);
  online: the KF step's x, P in and out, F, Q, H, R and z in, plus the window: N-1 live rows in, N rows out;
  kf:     the KF step's words alone.
FMAs per filter-step count the KF step (Joseph form, as kf_regtile.cuh computes it) and the correction
(g = H' SI y, A = (F - K H)', then P v and A v per lag row).  The least times the hardware could take are
bytes / 3.35 TB/s (H100 SXM HBM3) and FMAs / 33.5 T FMA/s (the data sheet's 67 TFLOP/s fp32); `bound` names the
larger, `share_of_bound` is that least time over the measured time.  Each batch leg's output is checked once
against the fp64 oracle on a 4096-filter subset.  One JSON line per leg and arm goes to stdout, with the GPU name,
power limit and max SM clock.
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
from oracle import fls as ofl                                                                    # noqa: E402

PEAK_BPS = 3.35e12
PEAK_FMA = 67e12 / 2
NF, T_BATCH, LAGS = 1 << 20, 32, (1, 4, 16)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def kf_words(n, m):
    return 2 * (n + n * n) + 2 * n * n + m * n + m * m + m


def kf_fmas(n, m):
    pred = n * n + 2 * n ** 3
    upd = m * n + n * n * m + m * m * n + n * m * m + n * m + n * n * m + n ** 3 + n * m * m + n ** 3 + n * n * m
    return pred + upd


def corr_fmas(n, m, lag):
    if lag == 0:
        return 0
    return m * m + n * m + n * n * m + lag * n * n + (lag - 1) * n * n


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def report(leg, arm, ms_all, per, nbytes, fmas, info, **extra):
    ms = float(np.median(ms_all)) / per
    t_hbm, t_fma = nbytes * NF / PEAK_BPS * 1e3, fmas * NF / PEAK_FMA * 1e3
    bound = "hbm" if t_hbm >= t_fma else "fma"
    print(json.dumps(dict(leg=leg, arm=arm, n_filters=NF, dim_x=4, dim_z=2, dtype="float32",
                          ms_per_epoch=round(ms, 5), ms_all=[round(t / per, 5) for t in ms_all],
                          bytes_per_filter_step=round(nbytes, 2), fmas_per_filter_step=fmas,
                          share_of_hbm_peak=round(nbytes * NF / (ms * 1e-3) / PEAK_BPS, 3),
                          hbm_bound_ms=round(t_hbm, 5), fma_bound_ms=round(t_fma, 5), bound=bound,
                          share_of_bound=round(max(t_hbm, t_fma) / ms, 3), **extra, **info)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fls_bench.py needs a GPU")
    lib = _lib.load()
    info = gpu_info()
    stream = torch.cuda.current_stream().cuda_stream
    n, m, es = 4, 2, 4
    w = wl.kf_bank_cv2d(NF, seed=1234, steps=T_BATCH)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()       # noqa: E731
    x0, P0, F, H, Q, R, zs = (dev(w[k]) for k in ("x", "P", "F", "H", "Q", "R", "zs"))
    x_out, P_out = torch.empty_like(x0), torch.empty_like(P0)

    def fls_args(lag, count, T, xs, xhat, x, P, xo, Po, z):
        a = _lib.FlsArgs()
        k = a.step
        k.n_filters, k.dim_x, k.dim_z, k.dtype, k.alpha_sq = NF, n, m, _lib.BKE_F32, 1.0
        k.x, k.P, k.x_out, k.P_out = x.data_ptr(), P.data_ptr(), xo.data_ptr(), Po.data_ptr()
        k.F, k.F_stride, k.H, k.H_stride = F.data_ptr(), n * n, H.data_ptr(), m * n
        k.Q, k.Q_stride, k.R, k.R_stride = Q.data_ptr(), n * n, R.data_ptr(), m * m
        a.n_steps, a.lag, a.count = T, lag, count
        a.zs, a.xs_smooth, a.xhat = z.data_ptr(), xs.data_ptr(), None if xhat is None else xhat.data_ptr()
        assert lib.bke_fls_workspace_bytes(NF, n, m, 0, _lib.BKE_F32, lag) == 0
        return a

    xs = torch.empty(T_BATCH, NF, n, dtype=torch.float32, device="cuda")
    xhat = torch.empty_like(xs)
    sel = np.sort(np.random.default_rng(0).choice(NF, 4096, replace=False))
    for lag in LAGS:
        a = fls_args(lag, 0, T_BATCH, xs, xhat, x0, P0, x_out, P_out, zs)
        fn = lambda: _lib.check(lib.bke_fls_smooth(a, stream))                             # noqa: E731
        fn()
        torch.cuda.synchronize()
        o = ofl.fls_bank(w["x"][sel], w["P"][sel], w["F"][sel], w["H"][sel], w["Q"][sel], w["R"][sel], w["zs"][:, sel], lag)
        err = float(np.abs(xs.cpu().numpy()[:, sel] - o["xs"]).max() / np.abs(o["xs"]).max())
        ms_all = [timed(fn, args.steps, args.warmup) for _ in range(args.repeats)]
        once = 2 * (n + n * n) + 2 * n * n + m * n + m * m
        nbytes = ((m + 2 * n) + once / T_BATCH) * es
        report("batch_N%d" % lag, "fls", ms_all, T_BATCH, nbytes, kf_fmas(n, m) + corr_fmas(n, m, lag), info,
               T=T_BATCH, lag=lag, max_rel_err_vs_oracle_4096=err)

    # smooth() per epoch at N = 4 against bke_kf_step on the same bank, in place, alternating
    lag = 4
    rows = args.warmup + args.steps
    hist = torch.zeros(rows, NF, n, dtype=torch.float32, device="cuda")
    xf, Pf = x0.clone(), P0.clone()
    calls = [fls_args(lag, c, 1, hist, None, xf, Pf, xf, Pf, zs[c % T_BATCH]) for c in range(rows)]
    xk, Pk = x0.clone(), P0.clone()
    ka = _lib.KfArgs()
    ka.n_filters, ka.dim_x, ka.dim_z, ka.dtype, ka.alpha_sq = NF, n, m, _lib.BKE_F32, 1.0
    ka.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
    ka.x = ka.x_out = xk.data_ptr(); ka.P = ka.P_out = Pk.data_ptr()
    ka.F, ka.F_stride, ka.H, ka.H_stride = F.data_ptr(), n * n, H.data_ptr(), m * n
    ka.Q, ka.Q_stride, ka.R, ka.R_stride = Q.data_ptr(), n * n, R.data_ptr(), m * m
    ka.z = zs[0].data_ptr()
    times = {"fls": [], "kf": []}
    for _ in range(args.repeats):
        it = iter(calls)
        times["fls"].append(timed(lambda: _lib.check(lib.bke_fls_smooth(next(it), stream)), args.steps, args.warmup))
        times["kf"].append(timed(lambda: _lib.check(lib.bke_kf_step(ka, stream)), args.steps, args.warmup))
    report("online_N4", "fls", times["fls"], 1, (kf_words(n, m) + (2 * lag - 1) * n) * es,
           kf_fmas(n, m) + corr_fmas(n, m, lag), info, T=1, lag=lag)
    report("online_N4", "kf", times["kf"], 1, kf_words(n, m) * es, kf_fmas(n, m), info, T=1)


if __name__ == "__main__":
    main()
