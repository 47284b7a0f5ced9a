"""Every kernel instance behind bke_kf_step, bke_kf_batch_filter and bke_kf_rts_smoother against the fp64 oracle
(oracle/kf.py), through the C-ABI, with a table that names the kernel(s) each case launches.

bke_kf_step tries, in order, the tensor-core tile kf_cov_tc_kernel<NX, M> (csrc/kf_tc.cu), the TMA 4/2 fp32 kernels
(csrc/kf_fast.cu), the register tiles kf_direct_kernel<T, N, M, EX> (csrc/kf_direct.cu), the row blocks
kf_rowblock_kernel<T, N, M, RPL, EX, MODE, SHARED> (csrc/kf_rowblock.cu, a ragged tail goes to the catch-all) and the
catch-all kf_generic_kernel<T> (csrc/kf_generic.cu).  bke_kf_batch_filter runs kf_batch_kernel<T, N, M, STAGED>
(csrc/kf_batch.cu) or a host loop of bke_kf_step epochs; bke_kf_rts_smoother runs rts_reg_kernel<T, N> or
rts_generic_kernel<T> (csrc/kf_rts.cu).  CASES reaches every instance these dispatches can launch.

Inputs are rounded to the kernel's dtype before the oracle sees them, so only the kernel's own arithmetic is measured.
Each error is taken relative to the filter's own scale (the largest |entry| of the same quantity of that filter, the
state's scale for y) and divided by the condition number of the filter's S (of Pp for the smoother, the largest over
the epochs for batch_filter; 1 where nothing is inverted), so a well-conditioned bank is held tightly and an
ill-conditioned one is not given a pass.  Worst cases measured on an H100 80GB HBM3 (700 W power limit) with BKE_TEST_ERRLOG, as
error / (scale * cond) over every case, output and bank size of the family, and the bound set from each:

    family                            fp64 worst  bound     fp32 worst  bound
    direct    kf_direct_kernel         1.0e-15    4e-15     4.8e-7      2e-6
    rowblock  kf_rowblock_kernel       6.1e-16    3e-15     5.7e-7      2e-6
    tc        kf_cov_tc_kernel            -         -       7.8e-7      3e-6
    fast      kf42_f32_kernel             -         -       2.8e-7      1e-6
    generic   kf_generic_kernel        6.7e-16    3e-15     4.1e-7      2e-6
    batch     kf_batch_kernel          5.8e-15    2e-14     3.1e-6      1e-5   (up to 4 epochs)
    host      batch host loop          2.3e-15    1e-14     1.9e-6      8e-6   (3 epochs)
    rts       rts_*_kernel             6.1e-16    3e-15     5.3e-7      2e-6
"""
import ctypes
import re

import numpy as np
import pytest

from gpu_harness import (F32, F64, TNAME, Bufs, b, body, call_ok, check_launch_order, close, k_direct, k_fast, k_gen,
                         k_rb, mag, profiled_names, ptr, rb_fpw, rd, spd, src)

ALPHA_SQ = 1.01 ** 2

TOL = {
    "direct": {F64: 4e-15, F32: 2e-6},
    "rowblock": {F64: 3e-15, F32: 2e-6},
    "tc": {F32: 3e-6},
    "fast": {F32: 1e-6},
    "generic": {F64: 3e-15, F32: 2e-6},
    "batch": {F64: 2e-14, F32: 1e-5},
    "host": {F64: 1e-14, F32: 8e-6},
    "rts": {F64: 3e-15, F32: 2e-6},
}


def _bound(c):
    """Case c's tolerance and the label of its BKE_TEST_ERRLOG lines."""
    return TOL[c.family][c.dt], "test_gpu_kf_instances %s %s" % (c.family, np.dtype(c.dt).name)


# ------------------------------------------------------------------------------------------ kernel names
def k_tc(nx, M):
    return "kf_cov_tc_kernel<%d, %d>" % (nx, M)


def k_batch(dt, n, m, staged):
    return "kf_batch_kernel<%s, %d, %d, %s>" % (TNAME[dt], n, m, b(staged))


def k_rts(dt, n=None):
    return "rts_generic_kernel<%s>" % TNAME[dt] if n is None else "rts_reg_kernel<%s, %d>" % (TNAME[dt], n)


# ------------------------------------------------------------------------------------------ the instance table
class Case:
    """One call of an entry point ("step", "batch", "rts") and the kernels it launches at N = Np (in launch order;
    a batch host loop repeats them once per epoch).  Layout:
      models   "per" (stride = the matrix size), "shared" (stride 0), "mixed" (F, Q shared; H, R per filter),
               "FH" (F, H shared; Q, R per filter), "epoch" (smoother: per-epoch per-filter F, Q)
      mis      None, "F" (the shared F one element past a 16-byte boundary), "bank" (x, P and their outputs one element
               off), "means" (batch_filter's outputs one element off)
      inplace  x_out / P_out are x / P;  ex: the optional outputs (x_prior, P_prior, K, y, S, SI, log_likelihood;
               smoother: K, Pp) are passed;  mode: BKE_DO_PREDICT | BKE_DO_UPDATE bits;  uf: BKE_UPDATE_FIRST;
               ctrl: B u;  T: epochs;  shift: the smoother's model_shift
    Ns are the bank sizes of the oracle runs: N = 1, one below and one above the family's tile and a ragged N near 1037
    (below a row-block tile the whole bank runs on the catch-all kernel)."""

    def __init__(self, entry, family, dt, n, m, kernels, Np, Ns, models="per", mis=None, inplace=False, ex=True,
                 mode=3, uf=False, ctrl=False, T=1, shift=1):
        self.entry, self.family, self.dt, self.n, self.m = entry, family, dt, n, m
        self.kernels, self.Np, self.Ns = list(kernels), Np, tuple(Ns)
        self.models, self.mis, self.inplace, self.ex, self.mode = models, mis, inplace, ex, mode
        self.uf, self.ctrl, self.T, self.shift = uf, ctrl, T, shift

    @property
    def id(self):
        s = "%s-%s-%s-%d_%d-%s" % (self.entry, self.family, "f32" if self.dt == F32 else "f64", self.n, self.m, self.models)
        if self.entry == "step":
            s += "-mode%d" % self.mode
        s += "" if self.ex else "-noex"
        for flag, name in ((self.mis, "mis" + str(self.mis)), (self.inplace, "inplace"), (self.uf, "uf"),
                           (self.ctrl, "ctrl")):
            if flag:
                s += "-" + name
        if self.entry != "step":
            s += "-T%d" % self.T
        if self.entry == "rts":
            s += "-shift%d" % self.shift
        return s + "-N%d" % self.Np


def _sweep(tile):
    return tuple(sorted({1, max(tile - 1, 1), tile + 1, 1037}))


DIRECT = {F64: [(4, 2), (2, 1), (1, 1), (2, 2), (3, 1), (4, 1), (4, 4)],
          F32: [(4, 2), (2, 1), (1, 1), (2, 2), (3, 1), (4, 1), (4, 4), (6, 3), (6, 2)]}
ROWBLOCK = {F64: [(9, 3, 3), (6, 3, 3), (16, 4, 1), (16, 2, 1)],
            F32: [(16, 4, 2), (16, 2, 2), (32, 4, 1), (9, 3, 3)]}
TC_DIMS = (16, 32)


def _cases():
    out = []
    # kf_direct: every shape x EX x mode.  4/2 fp32 runs there only when the TMA 4/2 kernel refuses the call: a bank
    # with F and H shared but Q and R per filter.
    for dt in (F64, F32):
        for n, m in DIRECT[dt]:
            mod = "FH" if (dt == F32 and (n, m) == (4, 2)) else None
            for mode in (3, 1, 2):
                for ex in (True, False):
                    models = mod or (("per", "shared")[(mode + ex) % 2])
                    out.append(Case("step", "direct", dt, n, m, [k_direct(dt, n, m, ex)], 129, _sweep(128),
                                    models=models, ex=ex, mode=mode, inplace=(mode == 2 and not ex)))
    # the row blocks: every shape x MODE x SHARED (x EX for the fused per-filter instance), except the shared-model
    # predicts of fp32 dim_x = 16 / 32, which the tensor-core kernel takes (alone or fused)
    for dt in (F64, F32):
        for n, m, rpl in ROWBLOCK[dt]:
            fpw = rb_fpw(dt, n, m, rpl)
            Np = 3 * fpw
            for mode in (3, 1, 2):
                for shared in (False, True):
                    if shared and mode != 2 and dt == F32 and n in TC_DIMS:
                        continue
                    exs = (True, False) if (mode == 3 and not shared) else ((mode == 1,) if not shared else (mode != 3,))
                    for ex in exs:
                        kern_ex = ex or mode != 3 or shared
                        out.append(Case("step", "rowblock", dt, n, m, [k_rb(dt, n, m, rpl, kern_ex, mode, shared)], Np,
                                        _sweep(fpw), models="shared" if shared else "per", ex=ex, mode=mode,
                                        inplace=(mode == 1 and shared)))
            # a ragged bank: the whole warp tiles on the row block, the tail on the catch-all kernel
            if fpw > 1:
                out.append(Case("step", "rowblock", dt, n, m, [k_rb(dt, n, m, rpl, True, 3, False), k_gen(dt)],
                                3 * fpw + 1, (fpw + 1, 2 * fpw - 1, 1037)))
    # the tensor cores: NX x M (M = dim_z of a fused step with shared H, R; 0 = the predict alone)
    for nx in TC_DIMS:
        tile = 128 // nx
        for M in range(5):
            if M == 0:
                out.append(Case("step", "tc", F32, nx, 4, [k_tc(nx, 0)], tile + 1, _sweep(tile), models="shared", mode=1,
                                inplace=(nx == 16)))
            else:
                out.append(Case("step", "tc", F32, nx, M, [k_tc(nx, M)], tile + 1, _sweep(tile), models="shared",
                                inplace=(M == 2)))
        out.append(Case("step", "tc", F32, nx, 2, [k_tc(nx, 2)], tile + 1, _sweep(tile), models="shared", ex=False))
        # two launches: the predict here, the update (per-filter H and R, or dim_z > 4) on the row block / catch-all
    out.append(Case("step", "tc", F32, 32, 4, [k_tc(32, 0), k_rb(F32, 32, 4, 1, True, 2, False)], 5, _sweep(4),
                    models="mixed"))
    out.append(Case("step", "tc", F32, 32, 6, [k_tc(32, 0), k_gen(F32)], 5, _sweep(4), models="shared", ex=False))
    # the TMA 4/2 fp32 kernel: the plain per-filter and shared calls (its own suites test the rest)
    out.append(Case("step", "fast", F32, 4, 2, [k_fast(3, 0, True)], 129, _sweep(128)))
    out.append(Case("step", "fast", F32, 4, 2, [k_fast(3, 1, True)], 129, _sweep(128), models="shared"))
    # the catch-all kernel
    G = (1, 3, 5, 1037)
    for dt in (F64, F32):
        out += [
            Case("step", "generic", dt, 4, 2, [k_gen(dt)], 5, G, uf=True),                         # update, then predict
            Case("step", "generic", dt, 9, 3, [k_gen(dt)], 5, G, models="shared", uf=True, ex=False),
            Case("step", "generic", dt, 4, 2, [k_gen(dt)], 5, G, ctrl=True),                       # B u
            Case("step", "generic", dt, 6, 3, [k_gen(dt)], 5, G, models="shared", ctrl=True, mode=1),
            Case("step", "generic", dt, 9, 3, [k_gen(dt)], 5, G, models="mixed"),                  # F, Q shared; H, R not
            Case("step", "generic", dt, 16, 4, [k_gen(dt)], 5, G, models="mixed", ex=False),
            Case("step", "generic", dt, 12, 3, [k_gen(dt)], 5, G),                                 # no specialisation
            Case("step", "generic", dt, 12, 3, [k_gen(dt)], 5, G, mode=1, inplace=True),
            Case("step", "generic", dt, 12, 3, [k_gen(dt)], 5, G, models="shared", mode=2, ex=False),
            Case("step", "generic", dt, 9, 3, [k_gen(dt)], 5, G, mis="bank"),                      # a misaligned bank
            Case("step", "generic", dt, 4, 4, [k_gen(dt)], 5, G, mis="bank", inplace=True),
        ]
    # a shared F one element off a 16-byte boundary at a kf_direct shape: kf_direct refuses it, and the row block has
    # no instance of these shapes
    for dt, (n, m) in ((F64, (4, 2)), (F32, (6, 3))):
        for mode in (3, 1, 2):
            out.append(Case("step", "generic", dt, n, m, [k_gen(dt)], 48, _sweep(16), models="shared", mis="F",
                            ex=(mode != 3), mode=mode, inplace=(mode == 1)))
    # batch_filter: the four register instances, staged (bulk copies, N >= 32 and an epoch's slice 16-byte aligned)
    # and unstaged, then the host loop of bke_kf_step epochs
    out += [
        Case("batch", "batch", F32, 4, 2, [k_batch(F32, 4, 2, True)], 33, (32, 33, 1057), T=4, models="shared", uf=True),
        Case("batch", "batch", F32, 4, 2, [k_batch(F32, 4, 2, False)], 31, (1, 31), T=3),
        Case("batch", "batch", F32, 2, 1, [k_batch(F32, 2, 1, True)], 34, (32, 34, 1058), T=1, inplace=True),
        Case("batch", "batch", F32, 2, 1, [k_batch(F32, 2, 1, False)], 33, (1, 33, 1037), T=3, models="shared", uf=True),
        Case("batch", "batch", F64, 2, 1, [k_batch(F64, 2, 1, True)], 33, (32, 33, 1057), T=4, ex=False),
        Case("batch", "batch", F64, 2, 1, [k_batch(F64, 2, 1, False)], 31, (1, 31), T=3, models="shared", uf=True),
        Case("batch", "batch", F64, 4, 2, [k_batch(F64, 4, 2, True)], 33, (32, 33, 1057), T=4, models="shared", uf=True),
        Case("batch", "batch", F64, 4, 2, [k_batch(F64, 4, 2, False)], 31, (1, 31), T=3, ex=False, inplace=True),
    ]
    H_ = (1, 20, 1037)
    out += [
        Case("batch", "host", F64, 3, 2, [k_gen(F64)], 5, H_, T=3),
        Case("batch", "host", F64, 3, 2, [k_gen(F64)], 5, H_, T=3, ex=False, inplace=True),      # NULL outputs
        Case("batch", "host", F32, 4, 2, [k_gen(F32)], 5, H_, T=3, ctrl=True),
        Case("batch", "host", F64, 4, 2, [k_gen(F64)], 5, H_, T=3, mis="means"),
        Case("batch", "host", F64, 4, 4, [k_direct(F64, 4, 4, False)] * 2, 6, (2, 20, 1036), T=3, uf=True),
        Case("batch", "host", F64, 9, 3, [k_rb(F64, 9, 3, 3, True, 2, False), k_rb(F64, 9, 3, 3, True, 1, False)], 20,
             (10, 20, 1030), T=3, uf=True),
        Case("batch", "host", F32, 16, 4, [k_rb(F32, 16, 4, 2, True, 2, True), k_tc(16, 0)], 8, (8, 32, 1036), T=3,
             uf=True, models="shared"),
    ]
    # the RTS smoother
    R_ = (1, 127, 129, 1037)
    RG = (1, 63, 65, 1037)
    for dt in (F64, F32):
        out += [
            Case("rts", "rts", dt, 4, 0, [k_rts(dt, 4)], 129, R_, T=5),
            Case("rts", "rts", dt, 4, 0, [k_rts(dt, 4)], 129, R_, T=4, models="shared", ex=False, shift=0),
            Case("rts", "rts", dt, 2, 0, [k_rts(dt, 2)], 129, R_, T=5, models="shared"),
            Case("rts", "rts", dt, 2, 0, [k_rts(dt, 2)], 129, R_, T=2, shift=0),
            Case("rts", "rts", dt, 4, 0, [k_rts(dt)], 65, RG, T=5, models="epoch"),
            Case("rts", "rts", dt, 4, 0, [k_rts(dt)], 65, RG, T=5, models="epoch", shift=0),
            Case("rts", "rts", dt, 3, 0, [k_rts(dt)], 65, RG, T=4),
            Case("rts", "rts", dt, 1, 0, [k_rts(dt)], 65, RG, T=4, models="shared", ex=False),
            Case("rts", "rts", dt, 12, 0, [k_rts(dt)], 65, RG, T=3, models="epoch"),
            Case("rts", "rts", dt, 4, 0, [k_rts(dt)], 65, RG, T=4, mis="bank"),
            Case("rts", "rts", dt, 3, 0, [k_rts(dt)], 65, RG, T=1),
        ]
    return out


CASES = _cases()
CASE_IDS = [c.id for c in CASES]


def _dispatched():
    """Every kernel instance the five dispatch functions can launch, parsed from the source."""
    inst = set()
    # kf_direct.cu dispatch(): the shapes (those after `if constexpr (sizeof(T) == 4)` are fp32 only), EX both ways
    d = body(src("kf_direct.cu"), "int dispatch(const bke_kf_args &a, cudaStream_t s)")
    both, f32only = d.split("if constexpr (sizeof(T) == 4)") if "if constexpr" in d else (d, "")
    pat = r"a\.dim_x == (\d+) && a\.dim_z == (\d+)\) return launch_inst<T, (\d+), (\d+)>"
    direct = {F64: [], F32: []}
    for part, dts in ((both, (F64, F32)), (f32only, (F32,))):
        for a, b, c, e in re.findall(pat, part):
            assert (a, b) == (c, e)
            for dt in dts:
                direct[dt].append((int(a), int(b)))
    li = body(src("kf_direct.cu"), "int launch_inst(const bke_kf_args &a, cudaStream_t s, const DirP<T> *form")
    exs = set(re.findall(r"kf_direct_kernel<T, N, M, (true|false), FORM>", li))
    assert exs == {"true", "false"}
    for dt, shapes in direct.items():
        for n, m in shapes:
            for ex in (True, False):
                inst.add(k_direct(dt, n, m, ex))
    # kf_rowblock.cu launch_kf_rowblock: shapes and RPL per dtype; launch_rb: the (EX, MODE, SHARED) instances, where
    # the fp32 shapes its `if constexpr` names take the first branch's shared-model instances instead of the second's
    rbsrc = src("kf_rowblock.cu")
    lr = body(rbsrc, "int launch_kf_rowblock(const bke_kf_args &a, cudaStream_t s)")
    f64part, f32part = lr.split("} else {")
    rows = {F64: [], F32: []}
    for part, dt in ((f64part, F64), (f32part, F32)):
        for a, b, t, c, e, rpl in re.findall(r"n == (\d+) && m == (\d+)\) return launch_rb<(\w+), (\d+), (\d+), (\d+)>", part):
            assert (a, b) == (c, e) and t == TNAME[dt]
            rows[dt].append((int(a), int(b), int(rpl)))
    lrb = body(rbsrc, "int launch_rb(const bke_kf_args &a, cudaStream_t s)")
    guard = re.search(r"if constexpr \(sizeof\(T\) == 4 && \(N == (\d+) \|\| N == (\d+)\)\) \{([^{}]*)\} else \{([^{}]*)\}",
                      lrb)
    vpat = r"kf_rowblock_kernel<T, N, M, RPL, (true|false), (\d), (true|false)>"
    variants = set(re.findall(vpat, lrb.replace(guard.group(0), "")))
    guarded, unguarded = (set(re.findall(vpat, guard.group(i))) for i in (3, 4))
    assert len(variants | unguarded) == 7 and guarded < unguarded
    guarded_n = {int(guard.group(1)), int(guard.group(2))}
    for dt, shapes in rows.items():
        for n, m, rpl in shapes:
            for ex, mode, sh in variants | (guarded if dt == F32 and n in guarded_n else unguarded):
                inst.add(k_rb(dt, n, m, rpl, ex == "true", int(mode), sh == "true"))
    # kf_tc.cu: the NX of launch_kf_tc and the M of launch_m (its default is M = 4)
    tcsrc = src("kf_tc.cu")
    nxs = sorted(int(v) for v in re.findall(r"tc::launch_m<(\d+)>\(p, m_here, s\)", tcsrc))
    lm = body(tcsrc, "int launch_m(const TcP &p, int m, cudaStream_t s)")
    ms = [(c, v) for c, v in re.findall(r"case (\d+): return launch_t<NX, (\d+)>", lm)]
    assert all(c == v for c, v in ms)
    ms = sorted({int(v) for _, v in ms} | {int(v) for v in re.findall(r"default: return launch_t<NX, (\d+)>", lm)})
    inst |= {k_tc(nx, M) for nx in nxs for M in ms}
    # kf_batch.cu launch_kf_batch: the register shapes, staged and unstaged; everything else is the host loop
    bsrc = src("kf_batch.cu")
    lb = body(bsrc, "int launch_kf_batch(const bke_kf_batch_args &a, cudaStream_t s)")
    stg = set(re.findall(r"kf_batch_kernel<T, N, M, (true|false)>", body(bsrc, "int launch_reg(const bke_kf_batch_args &a")))
    assert stg == {"true", "false"}
    for d_, a, b, t, c, e in re.findall(r"k\.dtype == BKE_(F32|F64) && k\.dim_x == (\d+) && k\.dim_z == (\d+)\) "
                                        r"return launch_reg<(\w+), (\d+), (\d+)>", lb):
        dt = F32 if d_ == "F32" else F64
        assert (a, b) == (c, e) and t == TNAME[dt]
        for s in (True, False):
            inst.add(k_batch(dt, int(a), int(b), s))
    assert "return launch_host_loop(a, s);" in lb
    # kf_rts.cu launch_t: the register dims and the generic kernel, both dtypes
    lt = body(src("kf_rts.cu"), "int launch_t(const bke_rts_args &a, cudaStream_t s)")
    for dt in (F32, F64):
        inst |= {k_rts(dt, int(v)) for v in re.findall(r"a\.dim_x == (\d+)\) \{ rts_reg_kernel<T, \1>", lt)}
        assert "rts_generic_kernel<T><<<" in lt
        inst.add(k_rts(dt))
        inst.add(k_gen(dt))
    return inst, direct, rows, nxs


def test_instance_table_matches_dispatch():
    """CASES launches every instance the dispatch code can reach (and no other): a new shape, mode, staging or tensor-core
    M in the dispatch, or a removed one, fails here, on a machine without a GPU too."""
    inst, direct, rows, nxs = _dispatched()
    assert direct == DIRECT and rows == ROWBLOCK and tuple(nxs) == TC_DIMS
    table = {k for c in CASES for k in c.kernels if not k.startswith("kf42_")}
    assert table == inst, (sorted(inst - table), sorted(table - inst))
    # every kf_direct shape x EX x mode
    got = {(c.dt, c.n, c.m, c.ex, c.mode) for c in CASES if c.family == "direct"}
    assert got == {(dt, n, m, ex, mode) for dt in (F32, F64) for n, m in DIRECT[dt] for ex in (True, False)
                   for mode in (1, 2, 3)}
    # the catch-all's features, both dtypes (mis="F": a shared model kf_direct refuses at one of its shapes)
    gen = [c for c in CASES if c.family == "generic"]
    for dt in (F32, F64):
        g = [c for c in gen if c.dt == dt]
        assert any(c.uf for c in g) and any(c.ctrl for c in g) and any(c.models == "mixed" for c in g)
        assert any(c.mis == "bank" for c in g) and any((c.n, c.m) == (12, 3) for c in g)
        assert any(c.mis == "F" and (c.n, c.m) in DIRECT[dt] for c in g)
    # both plain TMA 4/2 calls, the two-launch steps, the host loop with update_first on each kind of epoch kernel
    assert {c.models for c in CASES if c.family == "fast"} == {"per", "shared"}
    assert any(c.kernels[0].startswith("kf_cov_tc") and c.kernels[1].startswith("kf_rowblock") for c in CASES
               if len(c.kernels) == 2 and c.entry == "step")
    assert any(c.kernels[0].startswith("kf_rowblock") and c.kernels[1].startswith("kf_generic") for c in CASES
               if len(c.kernels) == 2 and c.entry == "step")
    host_uf = {c.kernels[0].split("<")[0] for c in CASES if c.family == "host" and c.uf}
    assert {"kf_direct_kernel", "kf_rowblock_kernel"} <= host_uf
    assert any(c.family == "host" and c.uf and any(k.startswith("kf_cov_tc") for k in c.kernels) for c in CASES)
    # the dispatch conditions the table relies on
    assert "if (a.flags & BKE_UPDATE_FIRST) return BKE_ERR_UNSUPPORTED;" in src("kf_direct.cu")
    assert "if (dense && shared) return BKE_ERR_UNSUPPORTED;" in src("kf_rowblock.cu")
    assert "const bool staged = ((size_t)p.N * N * sizeof(T)) % 16 == 0 && p.N >= 32;" in src("kf_batch.cu")


def _inputs(c, N, seed, singular):
    """The arrays of one call, rounded to the case's dtype (a shared model is one matrix).  singular: P = 0 for every
    7th filter, and Q = 0 and R's last row and column 0 there (in every filter where the model is shared), so those
    filters' S = R is singular and the others' is not."""
    rng = np.random.default_rng(seed)
    n, m, dt = c.n, c.m, c.dt
    shared = {"per": "", "shared": "FQHR", "mixed": "FQ", "FH": "FH"}[c.models]
    cnt = lambda k: () if k in shared else (N,)
    d = dict(x=rng.normal(size=(N, n)) * 3, P=spd(rng, (N,), n, 2.0),
             F=np.eye(n) + 0.1 * rng.normal(size=cnt("F") + (n, n)), Q=spd(rng, cnt("Q"), n, 0.05),
             H=rng.normal(size=cnt("H") + (m, n)), R=spd(rng, cnt("R"), m, 0.5), z=rng.normal(size=(N, m)) * 3)
    if c.ctrl:
        d["B"] = rng.normal(size=(N, n, 2)) if c.models == "per" else rng.normal(size=(n, 2))
        d["u"] = rng.normal(size=(N, 2))
    sing = np.zeros(N, bool)
    if singular:
        sing[::7] = True
        Q, R = d["Q"].copy(), d["R"].copy()
        if Q.ndim == 3:
            Q[sing] = 0
        else:
            Q[:] = 0
        if R.ndim == 3:
            R[sing, -1, :] = 0; R[sing, :, -1] = 0
        else:
            R[-1, :] = 0; R[:, -1] = 0
        d["Q"], d["R"] = Q, R
        d["P"][sing] = 0
    d = {k: rd(v, dt) for k, v in d.items()}
    return d, sing


def _full(a, N):
    return np.broadcast_to(a, (N,) + a.shape[-2:]) if a.ndim == 2 else a


# ------------------------------------------------------------------------------------------ the step oracle
def _oracle_step(d, N, do_p, do_u, uf, valid, sing, alpha_sq):
    """One bke_kf_step in fp64: the oracle's predict / update on the filters that update, the prior kept where z is
    missing or S is singular.  Returns the outputs, the filters whose update ran, those with S singular and cond(S)."""
    from oracle import kf as okf
    F, Q, H, R = (_full(d[k], N) for k in "FQHR")
    B = _full(d["B"], N) if "B" in d else None
    u = d.get("u")
    o = dict(status=np.zeros(N, np.int32), cond=np.ones(N))
    upd = np.zeros(N, bool); bad = np.zeros(N, bool)

    def predict(x, P):
        xp, Pp = okf.kf_predict_bank(x, P, F, Q, alpha_sq, B, u)
        o["x_prior"], o["P_prior"] = xp, Pp
        return xp, Pp

    def update(x, P):
        v = np.ones(N, bool) if valid is None else valid.copy()
        b = v & sing
        g = v & ~sing
        x, P = x.copy(), P.copy()
        o["y"] = np.zeros((N, H.shape[1]))
        for k, shp in (("K", H.shape[1:][::-1]), ("S", R.shape[1:]), ("SI", R.shape[1:]), ("ll", ())):
            o[k] = np.full((N,) + tuple(shp), np.nan)
        if g.any():
            r = okf.kf_update_bank(x[g], P[g], d["z"][g], H[g], R[g])
            x[g], P[g] = r["x"], r["P"]
            o["y"][g], o["K"][g], o["S"][g], o["SI"][g] = r["y"], r["K"], r["S"], r["SI"]
            o["ll"][g] = okf.log_likelihood_bank(r["y"], r["S"])
            o["cond"][g] = np.linalg.cond(r["S"])
        o["status"][b] = 1
        upd[:] = g; bad[:] = b
        return x, P

    x, P = d["x"], d["P"]
    if uf:
        x, P = update(x, P)
        x, P = predict(x, P)
    else:
        if do_p:
            x, P = predict(x, P)
        if do_u:
            x, P = update(x, P)
    o["x"], o["P"] = x, P
    return o, upd, bad


# ------------------------------------------------------------------------------------------ running a case
def run_step(c, N, seed=0, variant="plain"):
    """One bke_kf_step call of case c on N filters: (got, want, masks) with every output host-side."""
    from filterpy_b200 import _lib
    dt, n, m = c.dt, c.n, c.m
    do_p, do_u = bool(c.mode & 1), bool(c.mode & 2)
    singular = "singular" in variant and do_u
    sticky = "sticky" in variant
    d, sing = _inputs(c, N, seed, singular)
    rng = np.random.default_rng(seed + 1)
    valid = (rng.random(N) > 0.2) if do_u else None
    if valid is not None and N > 1:
        valid[1] = False
    bf = Bufs(dt)
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z = N, n, m
    a.dtype = _lib.BKE_F32 if dt == F32 else _lib.BKE_F64
    a.flags = c.mode | (_lib.BKE_UPDATE_FIRST if c.uf else 0) | (_lib.BKE_STATUS_STICKY if sticky else 0)
    a.alpha_sq = ALPHA_SQ
    bank_mis = c.mis == "bank"
    xv = bf.put(d["x"], bank_mis, out=c.inplace); Pv = bf.put(d["P"], bank_mis, out=c.inplace)
    a.x, a.P = ptr(xv), ptr(Pv)
    if c.inplace:
        xo, Po = xv, Pv
    else:
        xo, Po = bf.out((N, n), bank_mis), bf.out((N, n, n), bank_mis)
    a.x_out, a.P_out = ptr(xo), ptr(Po)
    for k in "FQHR":
        arr = d[k]
        v = bf.put(arr, c.mis == "F" and k == "F")
        setattr(a, k, ptr(v))
        setattr(a, k + "_stride", 0 if arr.ndim == 2 else arr.shape[-1] * arr.shape[-2])
    if c.ctrl:
        a.dim_u = 2
        a.B = ptr(bf.put(d["B"])); a.B_stride = 0 if d["B"].ndim == 2 else 2 * n
        a.u = ptr(bf.put(d["u"])); a.u_stride = 2
    a.z = ptr(bf.put(d["z"]))
    if valid is not None:
        a.z_valid = ptr(bf.put(valid.astype(np.uint8), dtype=np.uint8))
    outs = {}
    if c.ex:
        shapes = dict(x_prior=(N, n), P_prior=(N, n, n), K=(N, n, m), y=(N, m), S=(N, m, m), SI=(N, m, m),
                      log_likelihood=(N,))
        for k, s in shapes.items():
            outs[k] = bf.out(s)
            setattr(a, k, ptr(outs[k]))
    st = bf.out((N,), dtype=np.int32, fill=5)
    a.status = ptr(st)
    call_ok("bke_kf_step", ctypes.byref(a))
    bf.check_guards()
    want, upd, bad = _oracle_step(d, N, do_p, do_u, c.uf, valid, sing, ALPHA_SQ)
    got = dict(x=xo.cpu().numpy().reshape(N, n), P=Po.cpu().numpy().reshape(N, n, n),
               status=st.cpu().numpy())
    for k, v in outs.items():
        got[k] = v.cpu().numpy().reshape(dict(x_prior=(N, n), P_prior=(N, n, n), K=(N, n, m), y=(N, m),
                                              S=(N, m, m), SI=(N, m, m), log_likelihood=(N,))[k])
    return got, want, d, upd, bad, valid, sticky


def check_step(c, N, seed, variant):
    got, want, d, upd, bad, valid, sticky = run_step(c, N, seed, variant)
    do_p, do_u = bool(c.mode & 1), bool(c.mode & 2)
    what = "%s N=%d %s" % (c.id, N, variant)
    tol, label = _bound(c)
    cond = want["cond"]
    prior_x = want.get("x_prior", d["x"]); prior_P = want.get("P_prior", d["P"])
    sx = mag(d["x"], prior_x, want["x"])
    sP = mag(d["P"], prior_P, want["P"])
    close(got["x"], want["x"], sx, cond, tol, what + " x", label)
    close(got["P"], want["P"], sP, cond, tol, what + " P", label)
    st_want = want["status"].copy()
    if sticky:
        st_want[st_want == 0] = 5                   # BKE_STATUS_STICKY: written only where the step failed
    assert np.array_equal(got["status"], st_want), what + " status"
    if not c.ex:
        return
    S = Bufs.SENT
    if do_p:                                        # (update first: the prior is predicted from the posterior)
        pc = cond if c.uf else np.ones(N)
        close(got["x_prior"], want["x_prior"], sx, pc, tol, what + " x_prior", label)
        close(got["P_prior"], want["P_prior"], sP, pc, tol, what + " P_prior", label)
    else:
        assert np.all(got["x_prior"] == S) and np.all(got["P_prior"] == S), what + " prior written without a predict"
    if not do_u:
        for k in ("K", "y", "S", "SI", "log_likelihood"):
            assert np.all(got[k] == S), what + " %s written without an update" % k
        return
    # the state that entered the update: x_prior after a predict, x otherwise (update first: the input)
    ux = d["x"] if (c.uf or not do_p) else prior_x
    H = _full(d["H"], N)
    sy = np.abs(H).max(axis=(1, 2)) * np.abs(ux).sum(axis=1) + np.abs(d["z"]).max(axis=1)
    close(got["y"], want["y"], sy, cond, tol, what + " y", label, upd)
    miss = ~valid if valid is not None else np.zeros(N, bool)
    assert np.all(got["y"][miss] == 0), what + " y of a missed measurement"
    for k, w in (("K", "K"), ("S", "S"), ("SI", "SI")):
        close(got[k], want[w], mag(np.nan_to_num(want[w])), cond, tol, what + " " + k, label, upd)
        assert np.all(got[k][miss] == S), what + " %s written for a missed measurement" % k
    close(got["log_likelihood"], want["ll"], np.maximum(np.abs(np.nan_to_num(want["ll"])), 1.0), cond, tol,
          what + " log_likelihood", label, upd)
    assert np.all(got["log_likelihood"][miss] == S), what + " log_likelihood written for a missed measurement"


STEP_CASES = [c for c in CASES if c.entry == "step"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEP_CASES, ids=[c.id for c in STEP_CASES])
def test_step_instance_vs_oracle(case):
    """bke_kf_step: x, P, x_prior, P_prior, K, y, S, SI, log_likelihood and status against the fp64 oracle, over the
    family's bank sizes, with a z_valid mask, alpha^2 != 1, BKE_STATUS_STICKY and singular S."""
    for i, N in enumerate(case.Ns):
        check_step(case, N, seed=N + 7 * i, variant="sticky" if i % 2 else "plain")
    if case.mode & 2:
        check_step(case, case.Ns[-1], seed=3, variant="singular-sticky")
        check_step(case, 1, seed=4, variant="singular")


# ------------------------------------------------------------------------------------------ batch_filter
def run_batch(c, N, seed=0, singular=False):
    from filterpy_b200 import _lib
    dt, n, m, T = c.dt, c.n, c.m, c.T
    if singular and c.models != "per":
        T = 1                     # a shared Q = 0 and a singular R would make every filter's S degenerate over the epochs
    d, sing = _inputs(c, N, seed, singular)
    rng = np.random.default_rng(seed + 2)
    zs = rd(rng.normal(size=(T, N, m)) * 3, dt)
    valid = rng.random((T, N)) > 0.2
    bf = Bufs(dt)
    ba = _lib.KfBatchArgs()
    a = ba.step
    a.n_filters, a.dim_x, a.dim_z = N, n, m
    a.dtype = _lib.BKE_F32 if dt == F32 else _lib.BKE_F64
    a.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE | (_lib.BKE_UPDATE_FIRST if c.uf else 0)
    a.alpha_sq = ALPHA_SQ
    xv = bf.put(d["x"], out=c.inplace); Pv = bf.put(d["P"], out=c.inplace)
    a.x, a.P = ptr(xv), ptr(Pv)
    xo, Po = (xv, Pv) if c.inplace else (bf.out((N, n)), bf.out((N, n, n)))
    a.x_out, a.P_out = ptr(xo), ptr(Po)
    for k in "FQHR":
        arr = d[k]
        setattr(a, k, ptr(bf.put(arr)))
        setattr(a, k + "_stride", 0 if arr.ndim == 2 else arr.shape[-1] * arr.shape[-2])
    if c.ctrl:
        a.dim_u = 2
        a.B = ptr(bf.put(d["B"])); a.B_stride = 0 if d["B"].ndim == 2 else 2 * n
        a.u = ptr(bf.put(d["u"])); a.u_stride = 2
    st = bf.out((N,), dtype=np.int32, fill=5)
    a.status = ptr(st)
    ba.n_steps = T
    ba.zs = ptr(bf.put(zs))
    ba.zs_valid = ptr(bf.put(valid.astype(np.uint8), dtype=np.uint8))
    outs = {}
    if c.ex:
        mis = c.mis == "means"
        for k, s in (("means", (T, N, n)), ("covariances", (T, N, n, n)), ("means_p", (T, N, n)),
                     ("covariances_p", (T, N, n, n))):
            outs[k] = bf.out(s, mis)
            setattr(ba, k, ptr(outs[k]))
    call_ok("bke_kf_batch_filter", ctypes.byref(ba))
    bf.check_guards()
    # the oracle: epoch by epoch
    want = dict(means=np.zeros((T, N, n)), covariances=np.zeros((T, N, n, n)), means_p=np.zeros((T, N, n)),
                covariances_p=np.zeros((T, N, n, n)))
    cond = np.ones(N); status = np.zeros(N, np.int32)
    dd = dict(d)
    for t in range(T):
        dd["z"] = zs[t]
        if c.uf:                                        # update -> means[t], then predict -> means_p[t]
            o = _oracle_step(dd, N, False, True, False, valid[t], sing, ALPHA_SQ)[0]
            want["means"][t], want["covariances"][t] = o["x"], o["P"]
            p = _oracle_step(dict(dd, x=o["x"], P=o["P"]), N, True, False, False, None, sing, ALPHA_SQ)[0]
            want["means_p"][t], want["covariances_p"][t] = p["x"], p["P"]
            dd["x"], dd["P"] = p["x"], p["P"]
        else:
            o = _oracle_step(dd, N, True, True, False, valid[t], sing, ALPHA_SQ)[0]
            want["means_p"][t], want["covariances_p"][t] = o["x_prior"], o["P_prior"]
            want["means"][t], want["covariances"][t] = o["x"], o["P"]
            dd["x"], dd["P"] = o["x"], o["P"]
        cond = np.maximum(cond, o["cond"]); status |= o["status"]
    got = {k: v.cpu().numpy().reshape(want[k].shape) for k, v in outs.items()}
    got["x"], got["P"], got["status"] = xo.cpu().numpy().reshape(N, n), Po.cpu().numpy().reshape(N, n, n), st.cpu().numpy()
    return got, want, dd, cond, status


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if c.entry == "batch"],
                         ids=[c.id for c in CASES if c.entry == "batch"])
def test_batch_instance_vs_oracle(case):
    """bke_kf_batch_filter: means, covariances, means_p, covariances_p, the final x / P and status against the fp64
    oracle, with a z_valid mask, alpha^2 != 1 and filters whose S is singular every epoch."""
    tol, label = _bound(case)
    for i, N in enumerate(case.Ns):
        for singular in ((False, True) if N == case.Ns[-1] else (False,)):
            got, want, last, cond, status = run_batch(case, N, seed=N + i, singular=singular)
            what = "%s N=%d%s" % (case.id, N, " singular" if singular else "")
            sx = np.maximum(mag(*[np.swapaxes(want[k], 0, 1) for k in ("means", "means_p")]), 1e-300)
            sP = np.maximum(mag(*[np.swapaxes(want[k], 0, 1) for k in ("covariances", "covariances_p")]), 1e-300)
            for k, sc in (("means", sx), ("means_p", sx), ("covariances", sP), ("covariances_p", sP)):
                if k in got:
                    close(np.swapaxes(got[k], 0, 1), np.swapaxes(want[k], 0, 1), sc, cond, tol, what + " " + k, label)
            close(got["x"], last["x"], sx, cond, tol, what + " x", label)
            close(got["P"], last["P"], sP, cond, tol, what + " P", label)
            assert np.array_equal(got["status"], status), what + " status"


# ------------------------------------------------------------------------------------------ RTS smoother
def run_rts(c, N, seed=0, singular=False):
    from filterpy_b200 import _lib
    from oracle import kf as okf
    dt, n, T = c.dt, c.n, c.T
    rng = np.random.default_rng(seed)
    Xs = rng.normal(size=(T, N, n)) * 3
    Ps = spd(rng, (T, N), n, 1.0)
    shape = {"shared": (), "per": (N,), "epoch": (T, N)}[c.models]
    F = np.eye(n) + 0.2 * rng.normal(size=shape + (n, n))
    Q = spd(rng, shape, n, 0.1)
    sing = np.zeros(N, bool)
    if singular and T > 1:
        sing[::7] = True
        Q = Q * 0
        Ps[T - 2, sing] = 0                            # Pp[T-2] = F 0 F' + 0
    Xs, Ps, F, Q = (rd(v, dt) for v in (Xs, Ps, F, Q))
    bf = Bufs(dt)
    a = _lib.RtsArgs()
    a.n_filters, a.n_steps, a.dim_x = N, T, n
    a.dtype = _lib.BKE_F32 if dt == F32 else _lib.BKE_F64
    a.model_shift = c.shift
    mis = c.mis == "bank"
    a.Xs, a.Ps = ptr(bf.put(Xs, mis)), ptr(bf.put(Ps, mis))
    a.F, a.Q = ptr(bf.put(F)), ptr(bf.put(Q))
    a.F_stride = a.Q_stride = 0 if c.models == "shared" else n * n
    a.F_step_stride = a.Q_step_stride = N * n * n if c.models == "epoch" else 0
    xo, Po = bf.out((T, N, n), mis), bf.out((T, N, n, n), mis)
    a.x_out, a.P_out = ptr(xo), ptr(Po)
    K = Pp = None
    if c.ex:
        K, Pp = bf.out((T, N, n, n), mis), bf.out((T, N, n, n), mis)
        a.K, a.Pp = ptr(K), ptr(Pp)
    st = bf.out((N,), dtype=np.int32, fill=5)
    a.status = ptr(st)
    call_ok("bke_kf_rts_smoother", ctypes.byref(a))
    bf.check_guards()
    g = ~sing
    want = [v for v in okf.rts_smoother_bank(Xs[:, g], Ps[:, g], F[:, g] if c.models == "epoch" else
                                                  (F[g] if c.models == "per" else F),
                                                  Q[:, g] if c.models == "epoch" else (Q[g] if c.models == "per" else Q),
                                                  c.shift)] if g.any() else None
    got = [xo.cpu().numpy().reshape(T, N, n), Po.cpu().numpy().reshape(T, N, n, n)]
    got += [None if v is None else v.cpu().numpy().reshape(T, N, n, n) for v in (K, Pp)]
    got = [None if v is None else v[:, g] for v in got]
    return got, want, st.cpu().numpy(), sing, (Xs[:, g], Ps[:, g])


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if c.entry == "rts"], ids=[c.id for c in CASES if c.entry == "rts"])
def test_rts_instance_vs_oracle(case):
    """bke_kf_rts_smoother: smoothed x, P, K, Pp and status against the fp64 oracle; a filter whose Pp is singular
    reports it."""
    tol, label = _bound(case)
    for i, N in enumerate(case.Ns):
        for singular in ((False, True) if (N == case.Ns[-1] and case.T > 1) else (False,)):
            got, want, status, sing, (Xs, Ps) = run_rts(case, N, seed=N + i, singular=singular)
            what = "%s N=%d%s" % (case.id, N, " singular" if singular else "")
            assert np.array_equal(status, sing.astype(np.int32)), what + " status"
            if want is None:
                continue
            wx, wP, wK, wPp = want
            cond = np.ones(wx.shape[1])
            if case.T > 1:
                cond = np.linalg.cond(wPp[:-1].reshape(-1, case.n, case.n)).reshape(case.T - 1, -1).max(axis=0)
            sw = lambda v: np.swapaxes(v, 0, 1)
            sx = mag(sw(Xs), sw(wx)); sP = mag(sw(Ps), sw(wP), sw(wPp))
            close(sw(got[0]), sw(wx), sx, cond, tol, what + " x", label)
            close(sw(got[1]), sw(wP), sP, cond, tol, what + " P", label)
            if case.ex:
                close(sw(got[2]), sw(wK), np.maximum(mag(sw(wK)), 1.0), cond, tol, what + " K", label)
                close(sw(got[3]), sw(wPp), sP, cond, tol, what + " Pp", label)


# ------------------------------------------------------------------------------------------ which kernel runs
def run_case(c, N):
    if c.entry == "step":
        return run_step(c, N)
    if c.entry == "batch":
        return run_batch(c, N)
    return run_rts(c, N)


def _profiled_names():
    """The kernel names of every CASES entry run once at its N, in launch order."""
    return profiled_names(lambda: [run_case(c, c.Np) for c in CASES], r"kf\w*_kernel|rts_\w+_kernel")


@pytest.mark.gpu
def test_dispatch_runs_the_kernels_of_the_table():
    """Each CASES entry, run once at its N, launches the kernels the table names, in order, template arguments included
    (a batch host loop once per epoch)."""
    check_launch_order("test_gpu_kf_instances",
                       [(c.id, c.kernels * (c.T if c.family == "host" else 1)) for c in CASES])
