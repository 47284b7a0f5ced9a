"""Every kernel instance behind bke_if_step and bke_inverse against the fp64 oracle, through the C-ABI, with a table that
names the kernel each case launches.

bke_if_step (csrc/information.cu) runs the register tile if_reg_kernel<T, N, M, EX> (one thread per filter) for the
shapes of dispatch() without a control input (6/3 in fp32 only), when every 16-byte row it loads or stores is aligned;
every other call runs if_warp_kernel<T> (one warp per filter, 4, 2 or 1 warps per block, refused above 200 KB per
warp).  bke_inverse runs inverse_kernel<T> (one warp per matrix, the same launch shape).  CASES reaches every one of
these instances.

Inputs are rounded to the kernel's dtype before the oracle (tests/information_oracle.py, np.linalg.inv) sees them, so
only the kernel's own arithmetic is measured.  Each bank mixes, in every block: informed filters, filters without
information whose P_inv is invertible, and filters with P_inv = 0 (the A-singular predict); with per-filter models, also
the four failures that set status (inv(AI + Q), inv(F'), inv(A + Q), inv(S)) and, at n = 2, S = [[a, -a], [-a, a]].
Each error is taken relative to the filter's own scale of that quantity (the state's for y) and divided by the product
of the condition numbers of the matrices the filter inverts on the way to it (predict: A, P_inv, AI + Q or F', A + Q;
update: S), or of the inverted matrix.  Worst cases measured on an H100 80GB HBM3 (700 W power limit) with
BKE_TEST_ERRLOG, as error / (scale * cond) over every case, output and bank size of the family, and the bound set from
each:

    family                            fp64 worst  bound     fp32 worst  bound
    reg   if_reg_kernel                5.5e-16    2e-15     4.5e-7      2e-6
    warp  if_warp_kernel               1.0e-15    4e-15     4.6e-7      2e-6
    inv   inverse_kernel               2.4e-16    1e-15     7.7e-8      4e-7
"""
import ctypes
import re
from fractions import Fraction

import numpy as np
import pytest

from gpu_harness import (BUDGET, F32, F64, TNAME, Bufs, b, body, call, check_launch_order, close, mag, profiled_names,
                         ptr, rd, src)

LL_NONE, LL_FULL, LL_BROADCAST = 0, 1, 2

TOL = {
    "reg": {F64: 2e-15, F32: 2e-6},
    "warp": {F64: 4e-15, F32: 2e-6},
    "inv": {F64: 1e-15, F32: 4e-7},
}


def _bound(c):
    """Case c's tolerance and the label of its BKE_TEST_ERRLOG lines."""
    return TOL[c.family][c.dt], "test_gpu_if_instances %s %s" % (c.family, np.dtype(c.dt).name)


# ------------------------------------------------------------------------------------------ kernel names

def k_reg(dt, n, m, ex):
    return "if_reg_kernel<%s, %d, %d, %s>" % (TNAME[dt], n, m, b(ex))


def k_warp(dt):
    return "if_warp_kernel<%s>" % TNAME[dt]


def k_inv(dt):
    return "inverse_kernel<%s>" % TNAME[dt]


# ------------------------------------------------------------------------------------------ the launch shape
def if_per_warp(n, m):
    """information.cu if_per_warp, rounded up to 4 as launch_warp does."""
    return (4 * n + 2 * m + 6 * n * n + 4 * m * n + m * m + 3) & ~3


def inv_per_warp(k):
    """information.cu launch_inv: the matrix, its inverse and a column."""
    return (2 * k * k + k + 3) & ~3


def _wpb(elems, dt):
    b = elems * np.dtype(dt).itemsize
    for w in (4, 2, 1):
        if b * w <= BUDGET:
            return w
    return 0


def warps_per_block(c):
    return _wpb(inv_per_warp(c.n) if c.family == "inv" else if_per_warp(c.n, c.m), c.dt)


def _firsts(per_warp, dt):
    """(first size with 2 warps per block, first with 1, the largest accepted, the first refused)."""
    n, out = 1, {}
    while True:
        w = _wpb(per_warp(n), dt)
        out.setdefault(w, n)
        if w == 0:
            return out[2], out[1], n - 1, n
        n += 1


REG = {F64: [(4, 2), (1, 1), (2, 1), (2, 2), (3, 1), (4, 1), (4, 4)],
       F32: [(4, 2), (1, 1), (2, 1), (2, 2), (3, 1), (4, 1), (4, 4), (6, 3)]}


def vec_operands(dt, n, m):
    """kf_rowio.cuh vec_ok: the arrays information.cu launch_reg loads or stores as 16-byte vectors."""
    v = 16 // np.dtype(dt).itemsize
    rows = [("x", n), ("P_inv", n * n), ("F", n * n), ("F_inv", n * n), ("Q", n * n), ("H", m * n), ("R_inv", m * m),
            ("z", m), ("x_out", n), ("P_inv_out", n * n), ("x_prior", n), ("P_inv_prior", n * n), ("K", n * m),
            ("y", m), ("S", n * n)]
    return [k for k, c in rows if c % v == 0]


OUT_SHAPES = lambda n, m: dict(x_prior=(n,), P_inv_prior=(n, n), K=(n, m), y=(m,), S=(n, n))  # noqa: E731


# ------------------------------------------------------------------------------------------ the instance table
class Case:
    """One call and the kernels it launches at N = Np.  family "reg" / "warp" (bke_if_step) or "inv" (bke_inverse,
    n = k).  models: "per" or "shared" (stride 0); mis: the array placed one element past a 16-byte boundary; inplace:
    x_out / P_inv_out are x / P_inv; ex: x_prior, P_inv_prior, K, y and S are passed; mode: BKE_DO_PREDICT |
    BKE_DO_UPDATE; ctrl: B u; refused: BKE_ERR_UNSUPPORTED (no kernel runs); grid: one more bank, large enough for the
    warp kernel's grid-stride loop.  log_likelihood is always passed: ll_mode FULL where m == n, BROADCAST where m == 1."""

    def __init__(self, family, dt, n, m, kernels, Np, Ns, models="per", mis=None, inplace=False, ex=True, mode=3,
                 ctrl=False, refused=False, grid=False):
        self.family, self.dt, self.n, self.m = family, dt, n, m
        self.kernels, self.Np, self.Ns = list(kernels), Np, tuple(Ns)
        self.models, self.mis, self.inplace, self.ex, self.mode = models, mis, inplace, ex, mode
        self.ctrl, self.refused, self.grid = ctrl, refused, grid

    @property
    def ll_mode(self):
        return LL_FULL if self.m == self.n else (LL_BROADCAST if self.m == 1 else LL_NONE)

    @property
    def id(self):
        s = "%s-%s-%d_%d-%s" % (self.family, "f32" if self.dt == F32 else "f64", self.n, self.m, self.models)
        if self.family != "inv":
            s += "-mode%d" % self.mode + ("" if self.ex else "-noex")
        for flag, name in ((self.mis, "mis_%s" % self.mis), (self.inplace, "inplace"), (self.ctrl, "ctrl"),
                           (self.refused, "refused"), (self.grid, "grid")):
            if flag:
                s += "-" + name
        return s + "-N%d" % self.Np


TILE_NS = (1, 127, 129, 1037)
WARP_NS = (1, 5, 37)


def _cases():
    out = []
    for dt in (F64, F32):
        for n, m in REG[dt]:
            for mode in (3, 1, 2):
                for ex in (True, False):
                    out.append(Case("reg", dt, n, m, [k_reg(dt, n, m, ex)], 129, TILE_NS,
                                    models=("per", "shared")[(mode + ex) % 2], ex=ex, mode=mode,
                                    inplace=(mode != 3 and ex) or (mode == 3 and not ex)))
            vec = vec_operands(dt, n, m)
            if vec:
                for i, k in enumerate(vec[::3] if len(vec) > 3 else vec):
                    out.append(Case("reg", dt, n, m, [k_warp(dt)], 33, (1, 33), mis=k,
                                    ex=(i % 2 == 0) or k in OUT_SHAPES(n, m)))
            else:                                   # nothing is loaded as vectors: the tile runs on any address
                out.append(Case("reg", dt, n, m, [k_reg(dt, n, m, True)], 129, (1, 129), mis="x"))
        two, one, top, refused = _firsts(lambda n: if_per_warp(n, 3), dt)
        out += [
            Case("warp", dt, 4, 2, [k_warp(dt)], 37, WARP_NS, ctrl=True),
            Case("warp", dt, 3, 2, [k_warp(dt)], 37, WARP_NS, ctrl=True, models="shared", ex=False),
            Case("warp", dt, 1, 1, [k_warp(dt)], 37, WARP_NS, ctrl=True, mode=1, inplace=True),
            Case("warp", dt, 5, 3, [k_warp(dt)], 37, (1, 5, 37, 1037), grid=True),
            Case("warp", dt, 9, 3, [k_warp(dt)], 37, WARP_NS, models="shared", mode=2, inplace=True),
            Case("warp", dt, 5, 5, [k_warp(dt)], 37, WARP_NS, mode=1, ex=False),
            Case("warp", dt, 3, 4, [k_warp(dt)], 37, WARP_NS, ex=False),
            Case("warp", dt, 2, 3, [k_warp(dt)], 37, WARP_NS, mode=2),
            Case("warp", dt, 5, 5, [k_warp(dt)], 37, WARP_NS),                       # ll_mode FULL
            Case("warp", dt, 7, 1, [k_warp(dt)], 37, WARP_NS, models="shared"),      # ll_mode BROADCAST
            Case("warp", dt, 33, 2, [k_warp(dt)], 9, (1, 9)),
            Case("warp", dt, 20, 14, [k_warp(dt)], 9, (1, 9), models="shared"),
            Case("warp", dt, two, 3, [k_warp(dt)], 5, (1, 5), mode=2),
            Case("warp", dt, one, 3, [k_warp(dt)], 3, (3,), inplace=True),
            Case("warp", dt, top, 3, [k_warp(dt)], 3, (3,), models="shared"),
            Case("warp", dt, refused, 3, [], 3, (3,), refused=True),
        ]
        if dt == F64:                               # 6/3 is a register tile in fp32 only
            out += [Case("warp", dt, 6, 3, [k_warp(dt)], 129, TILE_NS, mode=m_, ex=e_)
                    for m_, e_ in ((3, True), (3, False), (1, True), (2, False))]
    for dt in (F64, F32):
        two, one, top, refused = _firsts(inv_per_warp, dt)
        for k in list(range(1, 9)) + [31, 32, 33, 64, two, one]:
            out.append(Case("inv", dt, k, 0, [k_inv(dt)], 37, (1, 37) if k < 64 else (3,),
                            models="shared" if k in (3, 32) else "per"))
        out += [Case("inv", dt, 4, 0, [k_inv(dt)], 37, (37,), grid=True),
                Case("inv", dt, top, 0, [k_inv(dt)], 2, (2,)),
                Case("inv", dt, refused, 0, [], 2, (2,), refused=True)]
    return out


CASES = _cases()


# ------------------------------------------------------------------------------------------ the table vs the source
def _dispatched():
    """Every kernel instance information.cu's dispatch() and launch_inv can launch, parsed from the source."""
    text = src("information.cu")
    d = body(text, "int dispatch(const bke_if_args &a, cudaStream_t s)")
    assert d.count("if constexpr (sizeof(T) == 4)") == 1, "the fp32-only register shapes are not where they were"
    both, f32only = d.split("if constexpr (sizeof(T) == 4)")
    pat = r"n == (\d+) && m == (\d+)\) rc = launch_reg<T, (\d+), (\d+)>"
    reg = {F64: [], F32: []}
    for part, dts in ((both, (F64, F32)), (f32only, (F32,))):
        for a, b, c, e in re.findall(pat, part):
            assert (a, b) == (c, e)
            for dt in dts:
                reg[dt].append((int(a), int(b)))
    assert "return rc == BKE_ERR_UNSUPPORTED ? launch_warp<T>(a, s) : rc;" in d
    assert "if (a.B == nullptr || a.u == nullptr) {" in d
    lr = body(text, "int launch_reg(const bke_if_args &a, cudaStream_t s)")
    assert set(re.findall(r"if_reg_kernel<T, N, M, (true|false)><<<", lr)) == {"true", "false"}
    inst = {k_reg(dt, n, m, ex) for dt, shapes in reg.items() for n, m in shapes for ex in (True, False)}
    inst |= {k_warp(dt) for dt in (F32, F64)} | {k_inv(dt) for dt in (F32, F64)}
    assert "inverse_kernel<T><<<" in body(text, "int launch_inv(int64_t N, int k, const void *A, int64_t stride, "
                                                "void *Ai, int32_t *status, cudaStream_t s)")
    return inst, reg


def test_instance_table_matches_dispatch():
    """CASES launches every instance information.cu's dispatch() and launch_inv can reach, and no other: a new register
    shape (or a dtype condition changed) without a case fails here, on a machine without a GPU too."""
    inst, reg = _dispatched()
    assert reg == REG
    table = {k for c in CASES for k in c.kernels}
    assert table == inst, (sorted(inst - table), sorted(table - inst))
    got = {(c.dt, c.n, c.m, c.ex, c.mode) for c in CASES if c.family == "reg" and not c.mis}
    assert got == {(dt, n, m, ex, mode) for dt in (F32, F64) for n, m in REG[dt] for ex in (True, False)
                   for mode in (1, 2, 3)}
    # fp64 6/3 runs the warp kernel
    assert any(c.dt == F64 and (c.n, c.m) == (6, 3) and c.kernels == [k_warp(F64)] for c in CASES)
    for dt in (F32, F64):
        for n, m in REG[dt]:
            mis = [c for c in CASES if c.family == "reg" and c.mis and (c.dt, c.n, c.m) == (dt, n, m)]
            assert mis and all(c.kernels == ([k_warp(dt)] if vec_operands(dt, n, m) else [k_reg(dt, n, m, True)])
                               for c in mis)
        for fam in ("warp", "inv"):
            w = [c for c in CASES if c.family == fam and c.dt == dt]
            assert {warps_per_block(c) for c in w} == {0, 1, 2, 4}
            assert any(c.n > 32 for c in w if not c.refused) and any(c.grid for c in w)
            top = max(c.n for c in w if not c.refused and c.m == (3 if fam == "warp" else 0))
            assert any(c.refused and c.n == top + 1 for c in w)
            assert {c.models for c in w} == {"per", "shared"}
        assert any(c.ctrl for c in CASES if c.dt == dt)
        assert {c.n for c in CASES if c.family == "inv" and c.dt == dt} >= set(range(1, 9)) | {31, 32, 33, 64}
    text = src("information.cu")
    assert "return 4 * n + 2 * m + 6 * n * n + 4 * m * n + m * m;" in body(text, "inline int if_per_warp(int n, int m)")
    assert "const int per_warp = (2 * k * k + k + 3) & ~3;" in text and "budget = 200 * 1024" in text


# ------------------------------------------------------------------------------------------ inputs
EDGE_A = 0.1


def edge_is_exact(dt):
    """S = [[a, -a], [-a, a]] with a = EDGE_A in dtype dt: dgetrf2's l = -a * (1 / a) rounds to -1 (so u = 0 and S is
    singular, as the oracle's elimination finds it), while a * a is inexact, so a determinant that fuses a * a - a * a
    into an FMA is not zero."""
    a = dt(EDGE_A)
    ra = dt(1) / a
    return bool(a * ra == 1) and Fraction(float(a)) ** 2 != Fraction(float(a * a))


def _spd(rng, shape, k, scale, eye):
    a = rng.normal(size=shape + (k, k))
    return scale * (a @ np.swapaxes(a, -1, -2) / k) + eye * np.eye(k)


def if_inputs(c, N, seed):
    """The arrays of one bke_if_step call, rounded to the dtype, with the kinds of filter of the module docstring
    (kind[f]: 0 informed, 1 no information, 2 P_inv = 0, 3 informed; failures "AIQ", "FT", "AQ", "S", "edge")."""
    rng = np.random.default_rng(seed)
    n, m = c.n, c.m
    cnt = () if c.models == "shared" else (N,)
    s = 1 / np.sqrt(n)
    F = np.eye(n) + 0.2 * s * rng.normal(size=cnt + (n, n))
    d = dict(x=rng.normal(size=(N, n)) * 3, P_inv=np.linalg.inv(_spd(rng, (N,), n, 1.0, 1.0)), F=F,
             F_inv=np.linalg.inv(F), Q=_spd(rng, cnt, n, 0.05, 0.5), H=np.eye(m, n) + 0.3 * rng.normal(size=cnt + (m, n)),
             R_inv=np.linalg.inv(_spd(rng, cnt, m, 1.0, 0.5)), z=rng.normal(size=(N, m)) * 3)
    if c.ctrl:
        d["B"] = rng.normal(size=cnt + (n, 2))
        d["u"] = rng.normal(size=(N, 2))
    f = np.arange(N)
    kind = f % 4
    ni = kind == 1
    d["P_inv"][kind == 2] = 0
    if c.mode == 2:
        ni = ni | (kind == 2)                      # update only: P_inv = 0 without information
    fail = np.array([""] * N, dtype=object)
    if c.models == "per" and N >= 11:
        for k, v in d.items():
            d[k] = np.array(v, copy=True)
        I = np.eye(n)
        if c.mode & 1:
            sel = f % 11 == 3                      # inv(AI + Q): A = I, Q = -I
            d["F"][sel] = I; d["F_inv"][sel] = I; d["P_inv"][sel] = I; d["Q"][sel] = -I; ni[sel] = False
            sel = f % 11 == 6                      # inv(F'): A = 0, F singular
            d["F"][sel] = 0; d["F_inv"][sel] = I; d["P_inv"][sel] = 0; ni[sel] = False
            fail[f % 11 == 3], fail[sel] = "AIQ", "FT"
            sel = f % 11 == 9                      # inv(A + Q): A = 0, Q = 0
            d["P_inv"][sel] = 0; d["Q"][sel] = 0; ni[sel] = False
            fail[sel] = "AQ"
        else:
            sel = f % 11 == 3                      # inv(S): S = P_inv = 0
            d["P_inv"][sel] = 0; d["H"][sel] = 0; ni[sel] = False
            fail[sel] = "S"
            if n == 2:                             # S = [[a, -a], [-a, a]]: singular by dgetrf2's rule
                sel = f % 11 == 6
                d["P_inv"][sel] = np.array([[1, -1], [-1, 1]]) * EDGE_A; d["H"][sel] = 0; ni[sel] = False
                fail[sel] = "edge"
    d = {k: rd(v, c.dt) for k, v in d.items()}
    d["ni"] = ni
    return d, fail


# ------------------------------------------------------------------------------------------ the oracle
def if_oracle(c, d, valid):
    """information_oracle.Filter per filter, with what the kernel writes: the prior (a predict that succeeded), y and
    S (an informed update), K (one whose inv(S) succeeded), log_likelihood (that or a no-information update); and the
    product of the condition numbers of what each filter inverted, in the predict and in all."""
    import information_oracle as io
    N, n = d["x"].shape
    m = c.m
    full = lambda k: np.broadcast_to(d[k], (N,) + d[k].shape[-2:]) if k in d else None   # noqa: E731
    F, Fi, Q, H, Ri, B = (full(k) for k in ("F", "F_inv", "Q", "H", "R_inv", "B"))
    keys = ("x", "P_inv", "ni", "status", "x_prior", "P_inv_prior", "y", "S", "K", "ll")
    o = {k: [] for k in keys}
    w = {k: np.zeros(N, bool) for k in ("prior", "yS", "K", "ll")}
    cp, ct = np.ones(N), np.ones(N)
    conds = []
    real_inv = io.inv

    def rec_inv(A):
        r = real_inv(A)
        if r is not None:
            conds.append(np.linalg.cond(A))
        return r

    io.inv = rec_inv
    try:
        for f in range(N):
            flt = io.Filter(d["x"][f], d["P_inv"][f], F[f], Fi[f], Q[f], H[f], Ri[f], None if B is None else B[f],
                            c.ll_mode)
            flt.ni = bool(d["ni"][f])
            del conds[:]
            ok = True
            if c.mode & 1:
                ok = flt.predict(d["u"][f] if "u" in d else None)
                w["prior"][f] = ok
            cp[f] = np.prod(conds)
            if ok and c.mode & 2 and valid[f]:
                informed = not flt.ni
                ok = flt.update(d["z"][f])
                w["yS"][f] = informed
                w["K"][f] = informed and ok
                w["ll"][f] = (not informed) or (ok and c.ll_mode != LL_NONE)
            ct[f] = np.prod(conds)
            for k in keys:
                o[k].append(np.array(getattr(flt, k), np.float64))
    finally:
        io.inv = real_inv
    o = {k: np.array(v) for k, v in o.items()}
    o["y"] = o["y"].reshape(N, m)
    return o, w, cp, ct


def test_oracle_kinds_and_edge():
    """The inputs reach what the docstring lists: each kind of filter and each failure, in the oracle, and the
    [[a, -a], [-a, a]] edge is exact in both dtypes."""
    for dt in (F64, F32):
        assert edge_is_exact(dt)
        for mode in (3, 2):
            c = Case("reg", dt, 2, 2, [], 1, (1,), mode=mode)
            N = 44
            d, fail = if_inputs(c, N, 0)
            valid = np.ones(N, bool)
            o, w, cp, ct = if_oracle(c, d, valid)
            st = o["status"] != 0
            assert np.array_equal(st, fail != ""), (mode, st, fail)
            if mode == 3:
                assert set(fail[st]) == {"AIQ", "FT", "AQ"}
                kind = np.where(fail == "", np.arange(N) % 4, -1)
                assert o["ni"][kind == 2].all() and not o["ni"][kind == 1].any() and not o["ni"][kind == 0].any()
                assert not w["prior"][st].any() and not w["yS"][st].any()
            else:
                assert set(fail[st]) == {"S", "edge"}
                assert w["yS"][st].all() and not w["K"][st].any()
            assert w["ll"][~st].all() and np.all(np.isfinite(cp)) and np.all(np.isfinite(ct))


# ------------------------------------------------------------------------------------------ running a step
def run_step(c, N, seed=0, sticky=False):
    """One bke_if_step call of case c on N filters: (rc, error text, got, d, fail, valid)."""
    from filterpy_b200 import _lib
    dt, n, m = c.dt, c.n, c.m
    d, fail = if_inputs(c, N, seed)
    rng = np.random.default_rng(seed + 1)
    valid = (rng.random(N) > 0.2) if c.mode & 2 else np.ones(N, bool)
    valid[fail != ""] = True
    if c.mode & 2 and N > 1:
        valid[1] = False
    bf = Bufs(dt)
    a = _lib.IfArgs()
    a.n_filters, a.dim_x, a.dim_z = N, n, m
    a.dtype = _lib.BKE_F32 if dt == F32 else _lib.BKE_F64
    a.flags = c.mode | (_lib.BKE_STATUS_STICKY if sticky else 0)
    a.ll_mode = c.ll_mode
    xv, Pv = bf.put(d["x"], c.mis == "x", out=c.inplace), bf.put(d["P_inv"], c.mis == "P_inv", out=c.inplace)
    a.x, a.P_inv = ptr(xv), ptr(Pv)
    xo, Po = (xv, Pv) if c.inplace else (bf.out((N, n), c.mis == "x_out"), bf.out((N, n, n), c.mis == "P_inv_out"))
    a.x_out, a.P_inv_out = ptr(xo), ptr(Po)
    niv = bf.put(d["ni"].astype(np.uint8), dtype=np.uint8)
    a.no_information = ptr(niv)
    for k in ("F", "F_inv", "Q", "H", "R_inv"):
        arr = d[k]
        setattr(a, k, ptr(bf.put(arr, c.mis == k)))
        setattr(a, k + "_stride", 0 if arr.ndim == 2 else arr.shape[-1] * arr.shape[-2])
    if c.ctrl:
        a.dim_u = 2
        a.B = ptr(bf.put(d["B"])); a.B_stride = 0 if d["B"].ndim == 2 else 2 * n
        a.u = ptr(bf.put(d["u"])); a.u_stride = 2
    a.z = ptr(bf.put(d["z"], c.mis == "z"))
    if c.mode & 2:
        a.z_valid = ptr(bf.put(valid.astype(np.uint8), dtype=np.uint8))
    outs = {}
    if c.ex:
        for k, s in OUT_SHAPES(n, m).items():
            outs[k] = bf.out((N,) + s, c.mis == k)
            setattr(a, k, ptr(outs[k]))
    ll = bf.out((N,))
    a.log_likelihood = ptr(ll)
    st = bf.out((N,), dtype=np.int32, fill=5)
    a.status = ptr(st)
    rc, err = call("bke_if_step", ctypes.byref(a))
    if rc:
        return rc, err, None, d, fail, valid
    bf.check_guards()
    got = dict(x=xo.cpu().numpy().reshape(N, n), P_inv=Po.cpu().numpy().reshape(N, n, n), status=st.cpu().numpy(),
               ni=niv.cpu().numpy(), ll=ll.cpu().numpy())
    for k, v in outs.items():
        got[k] = v.cpu().numpy().reshape((N,) + OUT_SHAPES(n, m)[k])
    return rc, err, got, d, fail, valid


def check_step(c, N, seed, sticky):
    rc, err, got, d, fail, valid = run_step(c, N, seed, sticky)
    assert rc == 0, err
    want, w, cp, ct = if_oracle(c, d, valid)
    what = "%s N=%d seed=%d%s" % (c.id, N, seed, " sticky" if sticky else "")
    tol, label = _bound(c)
    st_want = want["status"].astype(np.int32)
    if sticky:
        st_want[st_want == 0] = 5                   # BKE_STATUS_STICKY: written only where the step failed
    assert np.array_equal(got["status"], st_want), (what + " status", np.nonzero(got["status"] != st_want))
    assert np.array_equal(got["ni"], want["ni"].astype(np.uint8)), what + " no_information"
    pw = w["prior"]
    sx = mag(d["x"], np.where(pw[:, None], want["x_prior"], 0), want["x"])
    sP = mag(d["P_inv"], np.where(pw[:, None, None], want["P_inv_prior"], 0), want["P_inv"])
    close(got["x"], want["x"], sx, ct, tol, what + " x", label)
    close(got["P_inv"], want["P_inv"], sP, ct, tol, what + " P_inv", label)
    S = Bufs.SENT
    close(got["ll"], want["ll"], np.maximum(np.abs(want["ll"]), 1.0), ct, tol, what + " log_likelihood", label, w["ll"])
    assert np.all(got["ll"][~w["ll"]] == S), what + " log_likelihood written"
    if not c.ex:
        return
    close(got["x_prior"], want["x_prior"], sx, cp, tol, what + " x_prior", label, pw)
    close(got["P_inv_prior"], want["P_inv_prior"], sP, cp, tol, what + " P_inv_prior", label, pw)
    assert np.all(got["x_prior"][~pw] == S) and np.all(got["P_inv_prior"][~pw] == S), what + " prior written"
    ys, kw = w["yS"], w["K"]
    ux = np.where(pw[:, None], want["x_prior"], d["x"])
    H = np.broadcast_to(d["H"], (N,) + d["H"].shape[-2:])
    sy = np.abs(H).max(axis=(1, 2)) * np.abs(ux).sum(axis=1) + np.abs(d["z"]).max(axis=1)
    close(got["y"], want["y"], sy, cp, tol, what + " y", label, ys)
    close(got["S"], want["S"], mag(want["S"]), cp, tol, what + " S", label, ys)
    close(got["K"], want["K"], mag(want["K"]), ct, tol, what + " K", label, kw)
    for k, m_ in (("y", ys), ("S", ys), ("K", kw)):
        assert np.all(got[k][~m_] == S), what + " %s written" % k
    if N >= 11 and c.models == "per":
        assert (st_want == 1).sum() >= 1


def _grid_N(c):
    import torch
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count * warps_per_block(c) + 37


STEP_CASES = [c for c in CASES if c.family != "inv"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEP_CASES, ids=[c.id for c in STEP_CASES])
def test_step_instance_vs_oracle(case):
    """bke_if_step: x, P_inv, no_information, x_prior, P_inv_prior, K, y, S, log_likelihood and status against the
    fp64 oracle, over the family's bank sizes, with both branches in every block, a z_valid mask, BKE_STATUS_STICKY,
    each failure that sets status (a failed predict writes no prior and skips the update, a failed update writes y and
    S but not K), guard elements around every output; a refused shape returns BKE_ERR_UNSUPPORTED and says why."""
    from filterpy_b200 import _lib
    c = case
    if c.refused:
        rc, err = run_step(c, c.Ns[0], seed=1)[:2]
        assert rc == _lib.BKE_ERR_UNSUPPORTED, rc
        assert err == ("bke_if_step: dim_x=%d dim_z=%d needs %d B of shared memory per filter (> %d)"
                       % (c.n, c.m, if_per_warp(c.n, c.m) * np.dtype(c.dt).itemsize, BUDGET)), err
        return
    Ns = c.Ns + ((_grid_N(c),) if c.grid else ())
    for i, N in enumerate(Ns):
        check_step(c, N, seed=N + 13 * i, sticky=bool(i % 2))


# ------------------------------------------------------------------------------------------ bke_inverse
def run_inv(c, N, seed=0):
    """bke_inverse on N random k x k matrices (stride 0: one), every 7th (per filter) with a zero row."""
    dt, k = c.dt, c.n
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(() if c.models == "shared" else (N,)) + (k, k)) + 0.5 * np.eye(k)
    sing = np.zeros(N, bool)
    if c.models == "per" and N > 1:
        sing[3::7] = True
        A[sing, rng.integers(0, k), :] = 0
    A = rd(A, dt)
    bf = Bufs(dt)
    Av = bf.put(A)
    Ao = bf.out((N, k, k))
    st = bf.out((N,), dtype=np.int32, fill=5)
    rc, err = call("bke_inverse", ctypes.c_int64(N), ctypes.c_int32(k), ctypes.c_int32(0 if dt == F32 else 1),
                   ctypes.c_void_p(ptr(Av)), ctypes.c_int64(0 if c.models == "shared" else k * k),
                   ctypes.c_void_p(ptr(Ao)), ctypes.c_void_p(ptr(st)))
    if rc:
        return rc, err, None, None, None, None
    bf.check_guards()
    return rc, err, Ao.cpu().numpy().reshape(N, k, k), st.cpu().numpy(), np.broadcast_to(A, (N, k, k)), sing


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if c.family == "inv"], ids=[c.id for c in CASES if c.family == "inv"])
def test_inverse_instance_vs_numpy(case):
    """bke_inverse: the inverse against np.linalg.inv, status 1 exactly on the matrices with a zero row, guard elements
    around the outputs; a k above one warp's slice returns BKE_ERR_UNSUPPORTED and says why."""
    from filterpy_b200 import _lib
    c = case
    if c.refused:
        rc, err = run_inv(c, 2)[:2]
        assert rc == _lib.BKE_ERR_UNSUPPORTED, rc
        assert err == ("bke_inverse: k=%d needs %d B of shared memory per matrix (> %d)"
                       % (c.n, inv_per_warp(c.n) * np.dtype(c.dt).itemsize, BUDGET)), err
        return
    Ns = c.Ns + ((_grid_N(c),) if c.grid else ())
    tol, label = _bound(c)
    for N in Ns:
        rc, err, Ai, st, A, sing = run_inv(c, N, seed=N)
        assert rc == 0, err
        what = "%s N=%d" % (c.id, N)
        assert np.array_equal(st, sing.astype(np.int32)), what + " status"
        ok = ~sing
        want = np.linalg.inv(A[ok])
        close(Ai[ok], want, mag(want), np.linalg.cond(A[ok]), tol, what + " inverse", label)


# ------------------------------------------------------------------------------------------ which kernel runs
def _run_cases():
    for c in CASES:
        rc, err = (run_inv(c, c.Np) if c.family == "inv" else run_step(c, c.Np))[:2]
        assert (rc != 0) == c.refused, (c.id, err)


def _profiled_names():
    """The kernel names of every CASES entry run once at its N, in launch order."""
    return profiled_names(_run_cases, r"if_\w+_kernel|inverse_kernel")


@pytest.mark.gpu
def test_dispatch_runs_the_kernels_of_the_table():
    """Each CASES entry, run once at its N, launches the kernels the table names, in order, template arguments included
    (a refused shape launches none)."""
    check_launch_order("test_gpu_if_instances", [(c.id, c.kernels) for c in CASES])
