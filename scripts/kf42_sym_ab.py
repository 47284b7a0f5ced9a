"""A/B of the 4/2 fp32 bank step, which reads the packed model words that differ between the filters,
each distinct plane once (188 B per filter-step on the bench bank, whose 10 varying words hold 5
distinct planes), against another checkout (e.g. the parent commit), and the one-time cost of scanning
and packing the models.

    python scripts/kf42_sym_ab.py --baseline-tree DIR [--out DIR] [--rounds R] [--steps 400,50]
                                  [--diag-rounds D]

Prints JSON lines (and writes them to DIR/kf42_sym_ab.jsonl with --out):

  card     name, power limit and maximum SM clock (read-only nvidia-smi query)
  pack     device time of bke_kf_scan_models + bke_kf_pack_models for the 2^20-filter bench bank (CUDA
           events, median of rounds of 20 calls), with the bytes they move (176 B read three times:
           the two scan passes and the pack; 40 B written per filter)
  all_words  device time of one step of a 2^20-filter bank whose 37 model words all vary (316 B either
           way): bke_kf_step_packed against bke_kf_step_sym, alternated (the cost of the per-word select)
  run      one `bench.py --no-cpu --no-extra --no-resample --steps K` per arm and round: ms_per_step
           and the kernel time of the headline
  diag     one `bench.py --no-cpu --no-resample --steps 50` per arm and round: the ms_per_step of the
           kf_c2_diagnostics leg (the same kernel with its optional outputs)
  summary  per arm and step count: the median ms_per_step, and the change against the baseline arm

Arms, alternated inside every round, each in its own process: `tree` (bench.py of this tree) and
`baseline` (bench.py of the checkout at --baseline-tree, e.g. the parent commit built in place).  The
summary's `repay_steps` is the scan + pack time over the per-step saving against the baseline at 400
steps.
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


def _dev(w):
    import torch
    return {k: torch.from_numpy(np.ascontiguousarray(w[k])).cuda() for k in "FQHR"}


def pack_cost(rounds):
    import ctypes
    import torch
    from filterpy_b200 import _lib
    from filterpy_b200.common import workloads as wl
    lib = _lib.load()
    w = wl.kf_bank_cv2d(N, seed=1234, steps=1, dtype=np.float32)
    d = _dev(w)
    dmap = torch.empty(ctypes.sizeof(_lib.KfModelMap), dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    m = [ptr.data_ptr() for ptr in (d["F"], d["Q"], d["H"], d["R"])]
    _lib.check(lib.bke_kf_scan_models(N, 4, 2, _lib.BKE_F32, *m, dmap.data_ptr(), s))
    hmap = _lib.KfModelMap.from_buffer_copy(dmap.cpu().numpy().tobytes())
    k = bin(hmap.varying).count("1")
    rec = torch.empty(lib.bke_kf_packed_models_bytes(N, hmap.varying) // 4, dtype=torch.float32, device="cuda")

    def pack():
        _lib.check(lib.bke_kf_scan_models(N, 4, 2, _lib.BKE_F32, *m, dmap.data_ptr(), s))
        _lib.check(lib.bke_kf_pack_models(N, 4, 2, _lib.BKE_F32, *m, hmap.varying, rec.data_ptr(), s))
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
    moved = N * (3 * 176 + 4 * k)
    return {"what": "pack", "n_filters": N, "varying_words": k, "symmetric": hmap.asymmetric == 0, "ms": med,
            "ms_rounds": ms, "bytes": moved, "GBps": moved / (med * 1e-3) / 1e9}


def all_words(rounds):
    """One step of a bank whose 37 model words all vary: the packed words (bke_kf_step_packed, k = 37)
    against the packed Q / R (bke_kf_step_sym); both move 316 B per filter."""
    import ctypes
    import torch
    from filterpy_b200 import _lib
    from filterpy_b200.common import workloads as wl
    lib = _lib.load()
    w = wl.kf_bank_cv2d(N, seed=1234, steps=1, dtype=np.float32)
    rng = np.random.default_rng(5)
    for k, n in (("F", (4, 4)), ("H", (2, 4)), ("Q", (4, 4)), ("R", (2, 2))):
        a = w[k] + np.float32(1e-3) * rng.standard_normal((N,) + n).astype(np.float32)
        if k in "QR":
            a = np.triu(a) + np.swapaxes(np.triu(a, 1), 1, 2)
        w[k] = np.ascontiguousarray(a)
    d = _dev(w)
    m = [d[k].data_ptr() for k in "FQHR"]
    s = torch.cuda.current_stream().cuda_stream
    dmap = torch.empty(ctypes.sizeof(_lib.KfModelMap), dtype=torch.uint8, device="cuda")
    _lib.check(lib.bke_kf_scan_models(N, 4, 2, _lib.BKE_F32, *m, dmap.data_ptr(), s))
    hmap = _lib.KfModelMap.from_buffer_copy(dmap.cpu().numpy().tobytes())
    assert bin(hmap.varying).count("1") == 37 and hmap.asymmetric == 0
    rec = torch.empty(lib.bke_kf_packed_models_bytes(N, hmap.varying) // 4, dtype=torch.float32, device="cuda")
    _lib.check(lib.bke_kf_pack_models(N, 4, 2, _lib.BKE_F32, *m, hmap.varying, rec.data_ptr(), s))
    srec = torch.empty(lib.bke_kf_sym_models_bytes(N) // 4, dtype=torch.float32, device="cuda")
    flag = torch.empty(1, dtype=torch.int32, device="cuda")
    _lib.check(lib.bke_kf_pack_sym_models(N, 4, 2, _lib.BKE_F32, m[1], m[3], srec.data_ptr(), flag.data_ptr(), s))
    x = torch.from_numpy(w["x"]).cuda(); P = torch.from_numpy(w["P"]).cuda(); z = torch.from_numpy(w["zs"][0]).cuda()
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags, a.alpha_sq = N, 4, 2, _lib.BKE_F32, 3, 1.0
    a.x = a.x_out = x.data_ptr(); a.P = a.P_out = P.data_ptr()
    a.F, a.F_stride, a.Q, a.Q_stride = m[0], 16, m[1], 16
    a.H, a.H_stride, a.R, a.R_stride = m[2], 8, m[3], 4
    a.z = z.data_ptr()
    calls = {"packed_words": lambda: lib.bke_kf_step_packed(a, rec.data_ptr(), hmap, s),
             "packed_QR": lambda: lib.bke_kf_step_sym(a, srec.data_ptr(), s)}
    reps, ms = 100, {k: [] for k in calls}
    for r in range(2 * rounds):
        for name in (list(calls) if r % 2 == 0 else list(calls)[::-1]):
            for _ in range(10):
                _lib.check(calls[name]())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                calls[name]()
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / reps)
    return {"what": "all_words", "n_filters": N, "bytes_per_filter": 316,
            **{k: {"median_ms": float(np.median(v)), "ms_rounds": v} for k, v in ms.items()}}


def bench(cwd, argv):
    r = subprocess.run([sys.executable, "bench.py", "--gpus", "1"] + argv, cwd=cwd,
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
    ap.add_argument("--baseline-tree", required=True, help="the checkout whose bench.py is the baseline arm")
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
    pack = pack_cost(args.rounds)
    emit(pack)
    torch.cuda.empty_cache()
    emit(all_words(args.rounds))
    torch.cuda.empty_cache()
    arms = [("tree", ROOT), ("baseline", os.path.abspath(args.baseline_tree))]
    res = {}
    for K in [int(k) for k in args.steps.split(",")]:
        for r in range(args.rounds):
            order = arms if r % 2 == 0 else arms[::-1]
            for name, cwd in order:
                j = bench(cwd, ["--steps", str(K), "--warmup", "5", "--no-cpu", "--no-extra", "--no-resample"])
                res.setdefault((name, K), []).append(j["ms_per_step"])
                emit({"what": "run", "arm": name, "steps": K, "round": r, "ms_per_step": j["ms_per_step"],
                      "kernel_ms": j["roofline"]["kernel_ms"], "value": j["value"]})
    diag = {}
    for r in range(args.diag_rounds):
        order = arms if r % 2 == 0 else arms[::-1]
        for name, cwd in order:
            j = bench(cwd, ["--steps", "50", "--warmup", "5", "--no-cpu", "--no-resample"])
            diag.setdefault(name, []).append(j["kf_c2_diagnostics"]["ms_per_step"])
            emit({"what": "diag", "arm": name, "round": r, "kf_c2_diagnostics_ms": j["kf_c2_diagnostics"]["ms_per_step"]})
    summary = {}
    for (name, K), v in sorted(res.items()):
        med = float(np.median(v))
        base = float(np.median(res[("baseline", K)]))
        summary["%s_%d" % (name, K)] = {"median_ms": med, "min_ms": min(v), "max_ms": max(v),
                                        "gain_vs_baseline": base / med - 1.0}
    if ("baseline", 400) in res:
        saved = float(np.median(res[("baseline", 400)])) - float(np.median(res[("tree", 400)]))
        summary["repay_steps"] = pack["ms"] / saved if saved > 0 else None
    for name, v in diag.items():
        summary["diag_%s" % name] = {"median_ms": float(np.median(v)), "all_ms": v}
    emit({"what": "summary", **summary})


if __name__ == "__main__":
    main()
