"""wgmma covariance propagation (csrc/kf_tc.cu) against NumPy fp64: errors and timings.
python scripts/tc_check.py [check|time]"""
import json
import os
import sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from filterpy_b200.kalman import KalmanFilter

PEAK = 3350.0            # GB/s: H100 SXM data-sheet HBM3 bandwidth (not measured)


def make(n, m, N, seed=0):
    rng = np.random.default_rng(seed)

    def spd(k, cnt, scale):
        a = rng.normal(size=(cnt, k, k))
        return scale * (a @ np.swapaxes(a, -1, -2) / k + np.eye(k))
    F = np.eye(n) + 0.1 * rng.normal(size=(n, n))
    H = rng.normal(size=(m, n))
    Q, R, P0 = spd(n, 1, 0.05)[0], spd(m, 1, 0.5)[0], spd(n, N, 2.0)
    x0 = rng.normal(size=(N, n))
    z = rng.normal(size=(N, m))
    return F, H, Q, R, P0, x0, z


def check():
    worst = 0.0
    for n, m in [(16, 4), (32, 4)]:
        for N in [1, 7, 8, 9, 1037, 40003]:
            for alpha in [1.0, 1.02]:
                F, H, Q, R, P0, x0, z = make(n, m, N, seed=n + N)
                kf = KalmanFilter(n, m, n_filters=N, dtype=np.float32, diagnostics=False)
                kf.x, kf.P, kf.F, kf.H, kf.Q, kf.R = x0, P0, F, H, Q, R
                kf.alpha = alpha
                kf.predict()
                Pg = kf.P.cpu().numpy().astype(np.float64); xg = kf.x.cpu().numpy().astype(np.float64)
                F32, Q32, P32, x32 = [a.astype(np.float32).astype(np.float64) for a in (F, Q, P0, x0)]
                Pr = alpha * alpha * (F32 @ P32 @ F32.T) + Q32
                xr = x32 @ F32.T
                eP = np.abs(Pg - Pr).max() / np.abs(Pr).max(); ex = np.abs(xg - xr).max() / np.abs(xr).max()
                asym = np.abs(Pg - np.swapaxes(Pg, -1, -2)).max() / np.abs(Pr).max()
                worst = max(worst, eP, ex)
                print(json.dumps({"n": n, "N": N, "alpha": alpha, "err_P": eP, "err_x": ex, "asym": asym}), flush=True)
    print("worst", worst, "OK" if worst < 5e-5 else "FAIL", flush=True)


def timeit(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    return float(np.median([ev[i].elapsed_time(ev[i + 1]) for i in range(reps)]))


def time_():
    for n, m, N in [(16, 4, 1 << 19), (32, 4, 1 << 17)]:
        F, H, Q, R, P0, x0, z = make(n, m, N)
        kf = KalmanFilter(n, m, n_filters=N, dtype=np.float32, diagnostics=False)
        kf.x, kf.P, kf.F, kf.H, kf.Q, kf.R = x0, P0, F, H, Q, R
        zd = torch.from_numpy(z.astype(np.float32)).cuda()

        def pred():
            kf.predict(); kf._flush()
        ms = timeit(pred)
        bpu = (2 * n + 2 * n * n) * 4
        print(json.dumps({"case": "predict %d shared f32 N=%d" % (n, N), "ms": round(ms, 4),
                          "GBps": round(N * bpu / ms / 1e6, 1), "frac": round(N * bpu / ms / 1e6 / PEAK, 4)}), flush=True)

        def step():
            kf.predict(); kf.update(zd)
        ms = timeit(step)
        bpu = (2 * n + 2 * n * n + m) * 4
        print(json.dumps({"case": "predict+update %d/%d shared f32 N=%d" % (n, m, N), "ms": round(ms, 4),
                          "GBps": round(N * bpu / ms / 1e6, 1), "frac": round(N * bpu / ms / 1e6 / PEAK, 4)}), flush=True)


if __name__ == "__main__":
    (check if (len(sys.argv) < 2 or sys.argv[1] == "check") else time_)()
