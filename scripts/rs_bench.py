"""Stand-alone driver for timing and profiling the resample passes:
python scripts/rs_bench.py [log2N] [reps] [kind] [systematic|stratified|normalized]
`normalized` times ResamplePlan.normalized twice, systematic and with uniforms (the weight sum included)."""
import os
import sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from filterpy_b200.common import workloads as wl
from filterpy_b200.monte_carlo import ResamplePlan

lg = int(sys.argv[1]) if len(sys.argv) > 1 else 26
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
kind = sys.argv[3] if len(sys.argv) > 3 else "heavy"
mode = sys.argv[4] if len(sys.argv) > 4 else "systematic"
N = 1 << lg
w = torch.from_numpy(wl.resample_weights(N, kind, seed=97)).cuda()
U = torch.from_numpy(np.random.default_rng(98).random(N)).cuda()
plan = ResamplePlan(N)
calls = {
    "systematic": [("systematic", lambda: plan.systematic(w, 0.0763))],
    "stratified": [("stratified", lambda: plan.stratified(w, U))],
    "normalized": [("normalized", lambda: plan.normalized(w, u=0.0763)),
                   ("normalized.stratified", lambda: plan.normalized(w, uniforms=U))],
}
if mode not in calls:
    sys.exit("mode must be one of %s" % ", ".join(calls))
for name, call in calls[mode]:
    for _ in range(2):
        call()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        call()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(reps)]
    print("%s N=2^%d kind=%s median_ms=%.3f ms=%s  info=%s  GB/s(12B)=%.0f" % (
        name, lg, kind, float(np.median(ms)), ["%.3f" % m for m in ms], plan.info().tolist(),
        12.0 * N / (min(ms) * 1e-3) / 1e9))
