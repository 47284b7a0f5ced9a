"""A/B of the 4/2 fp32 bank step with Q and R read dense (344 B per filter-step) or as the packed
upper triangles of a symmetric bank (316 B), and the one-time cost of packing them.

    python scripts/kf42_sym_ab.py [--out DIR] [--rounds R] [--steps 400,50] [--diag-rounds D]
                                  [--baseline-tree DIR]

Prints JSON lines (and writes them to DIR/kf42_sym_ab.jsonl with --out):

  card     name, power limit and maximum SM clock (read-only nvidia-smi query)
  pack     device time of bke_kf_pack_sym_models for the 2^20-filter bench bank (CUDA events, median of
           rounds of 20 calls), with the bytes it moves (80 B read, 52 B written per filter) and the
           number of steps the saving of 28 B per step takes to repay it
  run      one `bench.py --no-cpu --no-extra --no-resample --steps K` per arm and round: ms_per_step
           and the kernel time of the headline
  diag     one `bench.py --no-cpu --no-resample --steps 50` per arm and round: the ms_per_step of the
           kf_c2_diagnostics leg (the same kernel with its optional outputs)
  summary  per arm and step count: the median ms_per_step, and the change against the dense arm

Arms, alternated inside every round, each in its own process: `dense` (BKE_KF_SYM=0) and `packed`
(the default) of this tree, and `baseline` (bench.py of another checkout, e.g. the parent commit
built in place) when --baseline-tree is given.
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

N = 1 << 20


def card():
    # by path: a plain import would find the ceiling kernel's kf42_ceiling.so next to the script first
    spec = importlib.util.spec_from_file_location("kf42_ceiling_py", os.path.join(HERE, "kf42_ceiling.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.card()


def pack_cost(rounds):
    import torch
    from filterpy_b200 import _lib
    from filterpy_b200.common import workloads as wl
    lib = _lib.load()
    w = wl.kf_bank_cv2d(N, seed=1234, steps=1, dtype=np.float32)
    Q = torch.from_numpy(w["Q"]).cuda()
    R = torch.from_numpy(w["R"]).cuda()
    rec = torch.empty(lib.bke_kf_sym_models_bytes(N) // 4, dtype=torch.float32, device="cuda")
    flag = torch.empty(1, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream

    def pack():
        _lib.check(lib.bke_kf_pack_sym_models(N, 4, 2, _lib.BKE_F32, Q.data_ptr(), R.data_ptr(), rec.data_ptr(),
                                              flag.data_ptr(), s))
    for _ in range(3):
        pack()
    torch.cuda.synchronize()
    reps, ms = 20, []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            pack()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / reps)
    med = float(np.median(ms))
    moved = N * (80 + 52)
    return {"what": "pack", "n_filters": N, "symmetric": int(flag.item()) == 0, "ms": med, "ms_rounds": ms,
            "bytes": moved, "GBps": moved / (med * 1e-3) / 1e9}


def bench(cwd, env_extra, argv):
    env = dict(os.environ)
    env.update(env_extra)
    r = subprocess.run([sys.executable, "bench.py", "--gpus", "1"] + argv, cwd=cwd, env=env,
                       capture_output=True, text=True, timeout=1800)
    if r.returncode != 0:
        raise RuntimeError("bench.py failed in %s:\n%s\n%s" % (cwd, r.stdout[-3000:], r.stderr[-3000:]))
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON lines to OUT/kf42_sym_ab.jsonl")
    ap.add_argument("--rounds", type=int, default=5, help="rounds per step count (each runs every arm once)")
    ap.add_argument("--steps", default="400,50", help="comma-separated --steps values")
    ap.add_argument("--diag-rounds", type=int, default=2, help="rounds of the bench run with the diagnostics leg (0: none)")
    ap.add_argument("--baseline-tree", default=None, help="a checkout whose bench.py is the third arm")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "kf42_sym_ab.py measures on a GPU"
    out_f = None
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        out_f = open(os.path.join(args.out, "kf42_sym_ab.jsonl"), "a")

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if out_f:
            out_f.write(line + "\n"); out_f.flush()
    emit(dict(what="card", **card()))
    emit(pack_cost(args.rounds))
    torch.cuda.empty_cache()
    arms = [("dense", ROOT, {"BKE_KF_SYM": "0"}), ("packed", ROOT, {})]
    if args.baseline_tree:
        arms.append(("baseline", os.path.abspath(args.baseline_tree), {}))
    res = {}
    for K in [int(k) for k in args.steps.split(",")]:
        for r in range(args.rounds):
            order = arms if r % 2 == 0 else arms[::-1]
            for name, cwd, env in order:
                j = bench(cwd, env, ["--steps", str(K), "--warmup", "5", "--no-cpu", "--no-extra", "--no-resample"])
                res.setdefault((name, K), []).append(j["ms_per_step"])
                emit({"what": "run", "arm": name, "steps": K, "round": r, "ms_per_step": j["ms_per_step"],
                      "kernel_ms": j["roofline"]["kernel_ms"], "value": j["value"]})
    diag = {}
    for r in range(args.diag_rounds):
        order = arms if r % 2 == 0 else arms[::-1]
        for name, cwd, env in order:
            j = bench(cwd, env, ["--steps", "50", "--warmup", "5", "--no-cpu", "--no-resample"])
            diag.setdefault(name, []).append(j["kf_c2_diagnostics"]["ms_per_step"])
            emit({"what": "diag", "arm": name, "round": r, "kf_c2_diagnostics_ms": j["kf_c2_diagnostics"]["ms_per_step"]})
    summary = {}
    for (name, K), v in sorted(res.items()):
        med = float(np.median(v))
        dense = float(np.median(res[("dense", K)]))
        summary["%s_%d" % (name, K)] = {"median_ms": med, "min_ms": min(v), "max_ms": max(v),
                                        "gain_vs_dense": dense / med - 1.0}
    for name, v in diag.items():
        summary["diag_%s" % name] = {"median_ms": float(np.median(v)), "all_ms": v}
    emit({"what": "summary", **summary})


if __name__ == "__main__":
    main()
