#!/usr/bin/env python
"""Time the information filter step (bke_if_step) against the linear filter step (bke_kf_step) on the same bank,
in one run on one GPU.

    python scripts/information_bench.py [--steps 50] [--warmup 10] [--repeats 5]

Legs: kf_bank_cv2d, 2^20 filters, 4/2, per-filter models, fp32 and fp64 (the register tile), one fused predict +
update per step, in place, no optional outputs.  The information arm starts from P_inv = inv(P) and
R_inv = inv(R) with F_inv = inv(F), so every filter stays in the informed branch.  The two arms of a leg alternate,
repeat by repeat.  Times are CUDA events around `steps` steps after `warmup` steps; the median over repeats is
reported.  Bytes per filter-step are computed from the shapes (information arm: x, P_inv and the no-information
flag in and out, F, F_inv, Q, H, R_inv and z in; KF arm: x and P in and out, F, Q, H, R and z in), over the H100
SXM data-sheet 3.35 TB/s.  The information arm's outputs are checked once, after one step, against the fp64 oracle
on a 2048-filter subset (max relative error of x and P_inv below 1e-3 in fp32, 1e-9 in fp64, or the script fails
before timing anything).  One JSON line per leg and arm goes to stdout, with the GPU name, power limit and max SM
clock.
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

from filterpy_b200 import _lib                                                                   # noqa: E402
from filterpy_b200.common import workloads as wl                                                 # noqa: E402
import information_oracle as io                                                                  # noqa: E402

PEAK_BPS = 3.35e12
LEGS = [("cv2d_f32", 1 << 20, np.float32), ("cv2d_f64", 1 << 20, np.float64)]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def bytes_if(n, m, itemsize):
    return (2 * n + 2 * n * n + 3 * n * n + m * n + m * m + m) * itemsize + 2


def bytes_kf(n, m, itemsize):
    return (2 * n + 2 * n * n + 2 * n * n + m * n + m * m + m) * itemsize


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("information_bench.py needs a GPU")
    lib = _lib.load()
    info = gpu_info()
    stream = torch.cuda.current_stream().cuda_stream
    for leg, N, dtype in LEGS:
        w = wl.kf_bank_cv2d(N, steps=1)
        n, m = w["x"].shape[1], w["H"].shape[1]
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()       # noqa: E731
        Pi0, Fi0, Ri0 = np.linalg.inv(w["P"]), np.linalg.inv(w["F"]), np.linalg.inv(w["R"])
        F, Fi, H, Q, R, Ri, z = (dev(w["F"]), dev(Fi0), dev(w["H"]), dev(w["Q"]), dev(w["R"]), dev(Ri0),
                                 dev(w["zs"][0]))
        bt = _lib.BKE_F32 if dtype == np.float32 else _lib.BKE_F64

        xi, Pi = dev(w["x"]), dev(Pi0)
        ni = torch.zeros(N, dtype=torch.uint8, device="cuda")
        ia = _lib.IfArgs()
        ia.n_filters, ia.dim_x, ia.dim_z, ia.dtype = N, n, m, bt
        ia.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
        ia.x = ia.x_out = xi.data_ptr(); ia.P_inv = ia.P_inv_out = Pi.data_ptr(); ia.no_information = ni.data_ptr()
        ia.F, ia.F_stride, ia.F_inv, ia.F_inv_stride = F.data_ptr(), n * n, Fi.data_ptr(), n * n
        ia.Q, ia.Q_stride, ia.H, ia.H_stride = Q.data_ptr(), n * n, H.data_ptr(), m * n
        ia.R_inv, ia.R_inv_stride = Ri.data_ptr(), m * m
        ia.z = z.data_ptr()
        xk, Pk = dev(w["x"]), dev(w["P"])
        ka = _lib.KfArgs()
        ka.n_filters, ka.dim_x, ka.dim_z, ka.dtype, ka.alpha_sq = N, n, m, bt, 1.0
        ka.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
        ka.x = ka.x_out = xk.data_ptr(); ka.P = ka.P_out = Pk.data_ptr()
        ka.F, ka.F_stride, ka.H, ka.H_stride = F.data_ptr(), n * n, H.data_ptr(), m * n
        ka.Q, ka.Q_stride, ka.R, ka.R_stride = Q.data_ptr(), n * n, R.data_ptr(), m * m
        ka.z = z.data_ptr()
        arms = {"information": lambda: _lib.check(lib.bke_if_step(ia, stream)),
                "kf": lambda: _lib.check(lib.bke_kf_step(ka, stream))}

        # the output check: one step from the initial state against the oracle
        arms["information"]()
        torch.cuda.synchronize()
        sel = np.sort(np.random.default_rng(0).choice(N, 2048, replace=False))
        xs, Ps = xi.double().cpu().numpy()[sel], Pi.double().cpu().numpy()[sel]
        err = 0.
        for j, f in enumerate(sel):
            o = io.Filter(w["x"][f], Pi0[f], w["F"][f], Fi0[f], w["Q"][f], w["H"][f], Ri0[f])
            o.predict(); o.update(w["zs"][0][f])
            err = max(err, float(np.abs(xs[j] - o.x).max() / np.abs(o.x).max()),
                      float(np.abs(Ps[j] - o.P_inv).max() / np.abs(o.P_inv).max()))
        assert int(ni.sum().item()) == 0, "a filter left the informed branch"
        bound = 1e-3 if dtype == np.float32 else 1e-9
        assert err < bound, "%s: the step is %.2e away from the oracle (bound %.0e)" % (leg, err, bound)

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
        for name in arms:
            nbytes = (bytes_if if name == "information" else bytes_kf)(n, m, np.dtype(dtype).itemsize)
            ms = float(np.median(times[name]))
            res = dict(leg=leg, arm=name, n_filters=N, dim_x=n, dim_z=m, dtype=np.dtype(dtype).name,
                       ms_per_step=round(ms, 5), ms_all=[round(t, 5) for t in times[name]],
                       bytes_per_filter_step=nbytes, share_of_hbm_peak=round(nbytes * N / (ms * 1e-3) / PEAK_BPS, 3),
                       **info)
            if name == "information":
                res["max_rel_err_vs_oracle_2048"] = err
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
