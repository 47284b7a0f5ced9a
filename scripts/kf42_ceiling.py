"""Where the time of the 4/2 fp32 bank step goes: the card's ceiling for its traffic, and the step's
fixed cost and streaming rate.

    python scripts/kf42_ceiling.py [--out DIR] [--rounds R] [--ring]

Prints JSON lines (and writes them to DIR/kf42_ceiling.jsonl with --out):

  card       name, power limit and maximum SM clock (nvidia-smi query)
  ceiling    scripts/kf42_ceiling.cu: a memory-only kernel that moves exactly the dense step's 344 B
             per filter (264 B read, 80 B written in place) with flat coalesced 16-byte accesses, 2^20
             filters; GB/s and its share of the data sheet's 3.35 TB/s
  ceiling_sym  the same twin with Q and R replaced by the packed 52 B-per-filter stream a symmetric
             bank's step reads instead (bke_kf_pack_sym_models): 316 B per filter
  ceiling_words  the same twin with F, Q, H and R replaced by one 40 B-per-filter stream, the 10 model
             words that differ between the filters of the bench bank (bke_kf_pack_models): 208 B
  ceiling_distinct  the same twin with that stream cut to 20 B per filter, the 5 distinct planes
             among those 10 words (the step does not read a plane the scan flags as a copy): 188 B
  ceiling_alternating  the 188 B twin at N = 2^19 .. 2^22, with a ring of 4 measurement buffers (z is
             a different buffer every step, as in bench.py): `forward` launches every step in the same
             tile order (as the shipped step did), the other arms in forward / reverse pairs, so that a
             launch starts on the tiles the previous one finished: `alt` with the default L2 policy,
             `alt_zfirst` with z read evict_first, `alt_tail_<W>MB` with, on top, the last W MB of a
             launch's order (100 B per filter: x, P and the model planes) read and written evict_last
             and demoted (evict_first) by the next launch.  ms per launch (best grid of 4 or 8 CTAs per
             SM, median of rounds, the arms alternated inside every round) and the gain over `forward`
  step       the shipped step (KalmanFilter.predict + update, per-filter F/H/Q/R) replayed as CUDA
             graphs of 4 separate steps, at N = 2^19 .. 2^22 (all above the bound under which
             the L2 hints are used); per-step time and GB/s for every N, counted with the bytes the
             step moves (168 + 4 per distinct plane of the packed model words, i.e. per varying word
             not flagged in the map's `duplicate`: 188 for the bench bank)
  fit        t(N) = a + b N over those sizes: a is the fixed cost of a step, bytes / b its
             streaming rate
  shared     the same graph of 4 steps for a 2^20-filter bank whose F/H/Q/R are shared (one model
             for the bank, carried in the launch parameters)
  ring       the fused ring (bke_kf_steps_packed, what KalmanFilter.capture returns for a ring of plain
             steps) at N = 2^19 .. 2^22 and K = 2, 4, 8 steps per launch, the arms alternated inside every
             round: `twin`, the memory-only kernel moving the ring's 180 + 8 K B per filter; `steps`, the
             graph of K separate steps; `fused`, a graph of one fused launch that takes its tile order from
             a bank-owned order word (bke_kf_args.tile_order), so consecutive replays alternate forward and
             reverse, as KalmanFilter.capture runs it; `fused_forward`, the same graph with tile_order
             cleared, so every replay walks the bank first to last.  ms per step (median of rounds), for twin
             and fused GB/s of the ring's bytes, and alt_gain = fused_forward / fused - 1.  --ring prints
             only the card and these lines.

The ceiling kernel is compiled with nvcc into scripts/kf42_ceiling.so (git-ignored) when that file
is missing or older than its source.  BKE_LIB_PATH selects the engine library as everywhere else.
"""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

SRC = os.path.join(HERE, "kf42_ceiling.cu")
LIB = os.path.join(HERE, "kf42_ceiling.so")
BYTES = 344                 # per filter-step: x, P, F, Q, H, R, z read (264 B), x, P written (80 B)
BYTES_SYM = 316             # the same with Q and R read as their packed upper triangles (52 B instead of 80)
BYTES_WORDS = 208           # the same with F, Q, H, R read as the 10 varying words of the bench bank (40 B instead of 176)
BYTES_DISTINCT = 188        # the same with only the 5 distinct planes among those words read (20 B)
PEAK_GBS = 3350.0           # H100 SXM data sheet, HBM3
RING = 4                    # steps per graph replay, as in bench.py


def build_lib():
    if os.path.exists(LIB) and os.path.getmtime(LIB) >= os.path.getmtime(SRC):
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-shared", "-Xcompiler", "-fPIC",
                    SRC, "-o", LIB + ".tmp"], check=True)
    os.replace(LIB + ".tmp", LIB)
    return LIB


def traffic_lib():
    lib = ctypes.CDLL(build_lib())
    lib.kf42_ring_traffic.restype = ctypes.c_int
    lib.kf42_ring_traffic.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.kf42_traffic.restype = ctypes.c_int
    lib.kf42_traffic.argtypes = [ctypes.c_void_p] * 7 + [ctypes.c_int64, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                         ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int64,
                                                         ctypes.c_int64]
    return lib


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        name, power, sm = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": sm}
    except Exception as e:
        return {"error": "%s: %s" % (type(e).__name__, e)}


def time_ms(fn, reps, torch):
    """Device time of `reps` calls of fn (CUDA events), in ms per call."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def reps_for(n_filters, seconds=0.3):
    return max(8, int(seconds / (n_filters * BYTES / 2.5e12)))


def ceiling(torch, rounds, mode=0):
    lib = traffic_lib()
    N = 1 << 20
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(5)
    arr = {k: torch.randn(N * e, device=dev, generator=g) for k, e in
           (("x", 4), ("P", 16), ("F", 16), ("Q", 16), ("H", 8), ("R", 4), ("z", 2))}
    nbytes = (BYTES, BYTES_SYM, BYTES_WORDS, BYTES_DISTINCT)[mode]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    stream = torch.cuda.current_stream().cuda_stream
    out = {}
    for per_sm in (4, 8):
        grid = sms * per_sm

        def run():
            rc = lib.kf42_traffic(*[arr[k].data_ptr() for k in "xPFQHRz"], N, grid, mode, stream, 0, 0, 0, 0, 0)
            assert rc == 0, rc
        for _ in range(5):
            run()
        torch.cuda.synchronize()
        ms = float(np.median([time_ms(run, reps_for(N), torch) for _ in range(rounds)]))
        gbs = nbytes * N / (ms * 1e-3) / 1e9
        out["ctas_per_sm_%d" % per_sm] = {"ms": ms, "GBps": gbs, "frac_of_3350": gbs / PEAK_GBS}
    best = max(out.values(), key=lambda v: v["GBps"])
    return {"what": ("ceiling", "ceiling_sym", "ceiling_words", "ceiling_distinct")[mode], "n_filters": N, "bytes_per_filter": nbytes, "ms": best["ms"],
            "GBps": best["GBps"],
            "frac_of_3350": best["frac_of_3350"], "by_grid": out}


TAIL_MB = (8, 16, 24, 32)   # the tail windows of the alternating sweep
REUSED = 100                # bytes per filter a launch can take over from the previous one: x, P, the model planes


def alternating(torch, rounds):
    """The 188 B twin launched every step in one tile order, or in forward / reverse pairs (with and
    without L2 hints); one line per bank size."""
    lib = traffic_lib()
    dev = torch.device("cuda")
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    stream = torch.cuda.current_stream().cuda_stream
    arms = [("forward", False, 0, 0, 0), ("alt", True, 0, 0, 0), ("alt_zfirst", True, 1, 1, 0)]
    arms += [("alt_tail_%dMB" % w, True, 1, 1, (w << 20) // REUSED) for w in TAIL_MB]
    lines = []
    for lg in (19, 20, 21, 22):
        N = 1 << lg
        g = torch.Generator(device=dev).manual_seed(5)
        arr = {k: torch.randn(N * e, device=dev, generator=g) for k, e in
               (("x", 4), ("P", 16), ("Q", 5), ("z", 2 * RING))}
        ptr = {k: v.data_ptr() for k, v in arr.items()}
        reps = reps_for(N) // 2 * 2
        res = {}
        ms = {}
        for r in range(rounds):
            for per_sm in (4, 8):
                grid = sms * per_sm
                for name, alt, hints, z_first, tail in (arms if r % 2 == 0 else arms[::-1]):
                    state = {"i": 0}

                    def run(alt=alt, hints=hints, z_first=z_first, tail=tail, grid=grid):
                        i = state["i"]
                        state["i"] = i + 1
                        rc = lib.kf42_traffic(ptr["x"], ptr["P"], None, ptr["Q"], None, None,
                                              ptr["z"] + (i % RING) * N * 8, N, grid, 3, stream,
                                              i % 2 if alt else 0, hints, z_first, tail, tail)
                        assert rc == 0, rc
                    for _ in range(4):
                        run()
                    ms.setdefault((name, per_sm), []).append(time_ms(run, reps, torch))
                    if tail:
                        # one more launch (untimed) demotes the last launch's evict_last tail, so no line
                        # keeps that priority once the sequence stops
                        i = state["i"]
                        rc = lib.kf42_traffic(ptr["x"], ptr["P"], None, ptr["Q"], None, None,
                                              ptr["z"] + (i % RING) * N * 8, N, grid, 3, stream,
                                              i % 2, hints, z_first, tail, 0)
                        assert rc == 0, rc
        for name, *_ in arms:
            best = min((float(np.median(ms[(name, s)])), s) for s in (4, 8))
            res[name] = {"ms": best[0], "ctas_per_sm": best[1],
                         "GBps": BYTES_DISTINCT * N / (best[0] * 1e-3) / 1e9}
        fwd = res["forward"]["ms"]
        for v in res.values():
            v["gain_vs_forward"] = fwd / v["ms"] - 1.0
        lines.append({"what": "ceiling_alternating", "n_filters": N, "bytes_per_filter": BYTES_DISTINCT,
                      "tail_filters_per_MB": (1 << 20) // REUSED, "arms": res})
        del arr
        torch.cuda.empty_cache()
    return lines


def bank(torch, N, shared=False):
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.common import workloads as wl
    base = 1 << 19
    w = wl.kf_bank_cv2d(base, seed=1234, steps=RING, dtype=np.float32)
    r = N // base
    kf = KalmanFilter(4, 2, n_filters=N, dtype=np.float32, device="cuda", diagnostics=False)
    kf.x = np.tile(w["x"], (r, 1))
    kf.P = np.tile(w["P"], (r, 1, 1))
    for k in "FHQR":
        setattr(kf, k, w[k][0] if shared else np.tile(w[k], (r, 1, 1)))
    zs = [torch.from_numpy(np.tile(w["zs"][i], (r, 1))).cuda() for i in range(RING)]

    def ring():
        for i in range(RING):
            kf.predict()
            kf.update(zs[i])
    # the graph of separate steps: kf.capture would return this ring fused (the `ring` lines measure that)
    from filterpy_b200._dev import StepGraph
    return kf, StepGraph(ring, kf._device)


def ring(torch, rounds):
    """The fused ring against its memory-only twin and against the graph of separate steps."""
    from filterpy_b200 import _lib
    from filterpy_b200._dev import StepGraph
    lib, tlib = _lib.load(), traffic_lib()
    dev = torch.device("cuda")
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    lines = []
    for lg in (19, 20, 21, 22):
        N = 1 << lg
        kf, _ = bank(torch, N)
        assert kf._sym_buf is not None, "the bank does not step from the packed model words"
        zs = torch.randn(8, N, 2, device=dev)
        tw = {k: torch.randn(N * e, device=dev) for k, e in (("x", 4), ("P", 16), ("Q", 5))}
        a_fwd = _lib.KfArgs.from_buffer_copy(next(iter(kf._args_cache.values()))[1])
        a_fwd.z_valid, a_fwd.flags, a_fwd.tile_order = None, 3, None
        order = torch.zeros(2, dtype=torch.int32, device=dev)
        a_word = _lib.KfArgs.from_buffer_copy(a_fwd)
        a_word.tile_order = order.data_ptr()
        for K in (2, 4, 8):
            arr = (ctypes.c_void_p * K)(*[zs[k].data_ptr() for k in range(K)])

            def fused(a):
                _lib.check(lib.bke_kf_steps_packed(a, kf._sym_buf.data_ptr(), kf._sym_host_map, arr, K,
                                                   torch.cuda.current_stream().cuda_stream))

            def steps():
                for k in range(K):
                    kf.predict(); kf.update(zs[k])
            fused(a_fwd)                                # the one-time function attribute, outside capture
            g_word = StepGraph(lambda: fused(a_word), dev, warmup=1)
            g_fwd = StepGraph(lambda: fused(a_fwd), dev, warmup=1)
            g_steps = StepGraph(steps, dev)
            assert g_word.nodes == 1 and g_fwd.nodes == 1 and g_steps.nodes == K

            def twin(grid):
                rc = tlib.kf42_ring_traffic(tw["x"].data_ptr(), tw["P"].data_ptr(), tw["Q"].data_ptr(), zs.data_ptr(), N,
                                            grid, K, torch.cuda.current_stream().cuda_stream)
                assert rc == 0, rc
            arms = [("twin_4", lambda: twin(4 * sms)), ("twin_8", lambda: twin(8 * sms)), ("steps", g_steps.replay),
                    ("fused", g_word.replay), ("fused_forward", g_fwd.replay)]
            reps = max(4, reps_for(N) // K) // 2 * 2
            ms = {}
            for r in range(rounds):
                for name, fn in (arms if r % 2 == 0 else arms[::-1]):
                    for _ in range(4):
                        fn()
                    ms.setdefault(name, []).append(time_ms(fn, reps, torch) / K)
            med = {k: float(np.median(v)) for k, v in ms.items()}
            moved = 180 + 8 * K
            twin_ms = min(med["twin_4"], med["twin_8"])
            gbs = lambda t: moved * N / (t * K * 1e-3) / 1e9
            lines.append({"what": "ring", "n_filters": N, "steps_per_launch": K, "bytes_per_filter_launch": moved,
                          "ms_per_step": {"twin": twin_ms, "steps": med["steps"], "fused": med["fused"],
                                          "fused_forward": med["fused_forward"]},
                          "GBps": {"twin": gbs(twin_ms), "fused": gbs(med["fused"])},
                          "fused_over_twin": med["fused"] / twin_ms, "steps_over_fused": med["steps"] / med["fused"],
                          "alt_gain": med["fused_forward"] / med["fused"] - 1.0})
        del kf, zs, tw, order
        torch.cuda.empty_cache()
    return lines


def step_ms(torch, graph, N, rounds):
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    reps = max(4, reps_for(N) // RING)
    return [time_ms(graph.replay, reps, torch) / RING for _ in range(rounds)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON lines to OUT/kf42_ceiling.jsonl")
    ap.add_argument("--rounds", type=int, default=5, help="timed rounds per measurement (the median is reported)")
    ap.add_argument("--ring", action="store_true", help="only the fused-ring lines")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "kf42_ceiling.py measures on a GPU"
    lines = [dict(what="card", **card()), dict(what="library", path=os.environ.get("BKE_LIB_PATH") or "in-tree")]
    if args.ring:
        return emit(lines + ring(torch, args.rounds), args.out)
    lines.append(ceiling(torch, args.rounds))
    lines.append(ceiling(torch, args.rounds, mode=1))
    lines.append(ceiling(torch, args.rounds, mode=2))
    lines.append(ceiling(torch, args.rounds, mode=3))
    lines += alternating(torch, args.rounds)
    sizes, times = [], []
    moved = BYTES
    for lg in (19, 20, 21, 22):
        N = 1 << lg
        kf, graph = bank(torch, N)
        t = step_ms(torch, graph, N, args.rounds)
        ms = float(np.median(t))
        sizes.append(N); times.append(ms)
        packed = kf._sym_state is not None and kf._sym_state[1]
        if packed:
            hm = kf._sym_host_map
            moved = 168 + 4 * (bin(hm.varying).count("1") - bin(hm.duplicate).count("1"))
        else:
            moved = BYTES
        lines.append({"what": "step", "n_filters": N, "packed_words": packed, "bytes_per_filter": moved, "ms": ms,
                      "ms_rounds": t, "GBps": moved * N / (ms * 1e-3) / 1e9})
        del kf, graph
        torch.cuda.empty_cache()
    b, a = np.polyfit(np.array(sizes, dtype=np.float64), np.array(times, dtype=np.float64), 1)
    resid = np.array(times) - (a + b * np.array(sizes))
    lines.append({"what": "fit", "fixed_us": a * 1e3, "stream_GBps": moved / (b * 1e-3) / 1e9,
                  "stream_frac_of_3350": moved / (b * 1e-3) / 1e9 / PEAK_GBS,
                  "max_abs_residual_us": float(np.abs(resid).max() * 1e3)})
    N = 1 << 20
    kf, graph = bank(torch, N, shared=True)
    t = step_ms(torch, graph, N, args.rounds)
    lines.append({"what": "shared", "n_filters": N, "ms": float(np.median(t)), "ms_rounds": t})
    emit(lines + ring(torch, args.rounds), args.out)


def emit(lines, out):
    text = "\n".join(json.dumps(l) for l in lines)
    print(text, flush=True)
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "kf42_ceiling.jsonl"), "a") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
