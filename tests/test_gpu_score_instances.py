"""Every kernel instance behind bke_score_measurements against the fp64 oracle (tests/stats_oracle.py), through the
C-ABI, with a table that names the kernel each case launches.

csrc/score.cu runs score_kernel<T, N, M>: phase A (each track's zhat, S^-1 and log|det S|) in registers at n = N for
the shapes dispatch_m lists, by a warp per track for N = 0; phase B (the pairs) at m = M, or any m for M = 0.  That
is 14 instances per dtype.  The warp path's tile shrinks from 128 tracks to 4 until a CTA's shared memory fits 64 KB,
opts in above 48 KB and refuses more than 200 KB (launch()'s rule, restated in warp_smem()).

Every call runs on guarded sentinel buffers (tests/gpu_harness.py).  The cases cover each source combination an
instance can take (x or mean; P with R, S or no covariance; H or the identity), H, R and S each shared or per track,
K from 1 to 300 (K >= 128 walks the pairs on dk alone, K = 64 and 128 on di alone), per-track candidates and one scan
shared by the bank, candidate strides 0 and m + 3, a ~20 % z_valid mask, each output alone, all and the minimal
sets, n < m, and one periodic bank per path past the grid-stride cap, whose every period must equal the first bit for
bit.

Exact comparisons where the arithmetic allows one: status; zhat = mean or x and y = z - zhat (one rounded
subtraction in the dtype) where zhat is not computed; mahalanobis == sqrt(d2); an invalid pair's 0 and
(T) log(DBL_MIN); likelihood within 2 ulps of exp(log_likelihood).  The rest is compared with the oracle in fp64 on
the inputs rounded to the dtype, per track: |error| / (scale * cond(S_i)) with scale = (max |y| + |zhat| terms)^2
||S^-1|| + |log det S| + m for d2 and log_likelihood, and the terms of H x for zhat and y.  Edge tracks (an exactly
singular S, an indefinite S, an ill-conditioned S and a NaN candidate) sit inside healthy tiles of a register and a
warp instance, and every other track must equal a clean run bit for bit.

Worst cases measured on an H100 80GB HBM3 (700 W power limit) with BKE_TEST_ERRLOG, as error / (scale * cond), and
the bounds set from them (about 4x):

    family                             fp64 worst  bound     fp32 worst  bound
    reg   score_kernel<T, N > 0, M>     5.6e-16    2.5e-15    2.1e-7     8e-7
    warp  score_kernel<T, 0, M>         3.8e-16    1.5e-15    1.9e-7     8e-7
"""
import ctypes
import math
import re
import sys

import numpy as np
import pytest

from gpu_harness import (F32, F64, TNAME, Bufs, body, call, check_launch_order, close, profiled_names, ptr, rd, spd,
                         src)

import stats_oracle as so

SENT = Bufs.SENT
THREADS = 128
LOG_DBL_MIN = math.log(sys.float_info.min)
TOL = {"reg": {F64: 2.5e-15, F32: 8e-7}, "warp": {F64: 1.5e-15, F32: 8e-7}}
OUTS = ("zhat", "y", "d2", "mahalanobis", "log_likelihood", "likelihood", "status")
SCORES = ("d2", "mahalanobis", "log_likelihood", "likelihood")
KS = (1, 3, 37, 64, 127, 128, 129, 300)
EDGE_OK, SINGULAR, INDEFINITE, ILLCOND, NANCAND = 0, 1, 2, 3, 4
ILLCOND_COND = {F32: 1e3, F64: 1e9}


def k_score(dt, n, m):
    return "score_kernel<%s, %d, %d>" % (TNAME[dt], n, m)


# ------------------------------------------------------------------------------------------ the dispatch, in Python
REG = {1: (1, 2, 3, 4), 2: (2, 4), 3: (3, 6), 4: (4,)}        # dispatch_m: the register (n, M) shapes


def route(n, m):
    """dispatch / dispatch_m: the (N, M) of the instance a call with phase-A width n (dim_x with x or P, else dim_z)
    and dim_z m runs."""
    if m in REG:
        return (n, m) if n in REG[m] else (0, m)
    return 0, 0


def warp_smem(n, m, es):
    """launch() for N = 0: (tracks per tile, shared-memory bytes); the tile halves from 128 while it is above 4
    tracks and the CTA needs more than 64 KB.  Refused (BKE_ERR_UNSUPPORTED) above 200 KB."""
    per = m + m * m + 1
    scratch = (m * m + m + n * m + 1) & ~1
    scr = (THREADS // 32) * scratch * es
    tile = THREADS
    while tile > THREADS // 32 and tile * per * es + scr > 64 * 1024:
        tile >>= 1
    return tile, tile * per * es + scr


def warp_shapes(dt):
    """At n = m: {tile: the first m >= 5 on that tile} for 128 .. 4, the first m above 48 KB, the largest accepted
    m and the first refused one."""
    es = np.dtype(dt).itemsize
    tiles, big, top = {}, None, None
    for m in range(5, 400):
        tile, smem = warp_smem(m, m, es)
        if smem > 200 * 1024:
            return tiles, big, top, m
        tiles.setdefault(tile, m)
        if big is None and smem > 48 * 1024:
            big = m
        top = m
    raise AssertionError("no refused shape")


# ------------------------------------------------------------------------------------------ the instance table
class Case:
    """One bke_score_measurements call and the kernel it launches.
      n, m        dim_x (0: not given) and dim_z;  mean: "x" or "mean";  cov: "P", "S" or None;  H: H given
      shared      which of H, R, S are one matrix for the bank (stride 0)
      K, zlay     candidates per track; "own" z[N, K, .] or "scan" z[K, .] shared by the bank (z_track_stride 0)
      zc          "dense" (z_cand_stride m), "zero" (0: every candidate the same) or "pad" (m + 3)
      mask        a z_valid mask;  outs: the outputs passed;  Ns: bank sizes
      grid        one more periodic bank past the grid-stride cap;  refused: BKE_ERR_UNSUPPORTED, nothing written"""

    def __init__(self, dt, n, m, mean, cov, H, Ns=(1, 1037), shared="", K=3, zlay="own", zc="dense", mask=True,
                 outs=OUTS, grid=False, refused=False, tag=""):
        self.dt, self.n, self.m, self.mean, self.cov, self.H = dt, n, m, mean, cov, H
        self.shared, self.K, self.zlay, self.zc, self.mask = shared, K, zlay, zc, mask
        self.outs, self.Ns, self.grid, self.refused, self.tag = tuple(outs), tuple(Ns), grid, refused, tag
        self.width = n if (mean == "x" or cov == "P") else m
        N_, M_ = route(self.width, m)
        self.path = "reg" if N_ > 0 else "warp"
        self.kernels = [] if refused else [k_score(dt, N_, M_)]

    @property
    def id(self):
        s = "%s-%s-%d_%d-%s-%s%s" % (self.path, "f32" if self.dt == F32 else "f64", self.width, self.m, self.mean,
                                     self.cov or "nocov", "-H" if self.H else "-I")
        s += "-sh" + self.shared if self.shared else ""
        s += "-K%d-%s-%s" % (self.K, self.zlay, self.zc)
        s += "-all" if set(self.outs) == set(OUTS) else "-" + "+".join(self.outs)
        for flag, name in ((not self.mask, "nomask"), (self.grid, "grid"), (self.refused, "refused"),
                           (self.tag, self.tag)):
            if flag:
                s += "-" + name
        return s


# the (n, m) per instance: the register shapes, and warp shapes with n > m, n < m and (any m) n = m
WARP_SHAPES = [(7, 1), (5, 2), (1, 2), (9, 3), (2, 3), (8, 4), (6, 6), (12, 5), (3, 5)]


def _sources(n, m):
    """(mean, cov, H) an instance at (n, m) can take: H may be the identity only where n == m; with mean and S (or
    no covariance) the phase-A width is m."""
    out = []
    for mean in ("x", "mean"):
        for cov in ("P", "S", None):
            uses_n = mean == "x" or cov == "P"
            for H in ((True, False) if uses_n else (False,)):
                if uses_n and not H and n != m:
                    continue
                if not uses_n and n != m:
                    continue
                out.append((mean, cov, H))
    return out


SHARED_SETS = ("", "H", "R", "S", "HR", "HRS", "RS", "HS")
OUT_SETS_COV = [OUTS] + [(o,) for o in OUTS] + [("zhat", "status"), ("y", "d2"), ("mahalanobis", "likelihood")]
OUT_SETS_NOCOV = [("zhat", "y"), ("zhat",), ("y",)]


def _cases():
    out = []
    for dt in (F64, F32):
        shapes = [(n, m) for m, ns in REG.items() for n in ns] + WARP_SHAPES
        i = 0
        for n, m in shapes:
            for mean, cov, H in _sources(n, m):
                sets = OUT_SETS_COV if cov else OUT_SETS_NOCOV
                sh = "".join(k for k in SHARED_SETS[i % len(SHARED_SETS)]
                             if (k == "H" and H) or (k == "R" and cov == "P") or (k == "S" and cov == "S"))
                out.append(Case(dt, n, m, mean, cov, H, shared=sh, K=KS[i % len(KS)],
                                zlay=("own", "scan")[i % 2], zc=("dense", "pad", "zero")[(i // 2) % 3],
                                mask=(i % 5 != 4), outs=sets[i % len(sets)]))
                i += 1
        # every K on each path with every output (the pair walk), and n = m x / P / identity on the tile sizes
        for n, m in ((4, 2), (5, 2), (6, 6)):
            for j, K in enumerate(KS):
                out.append(Case(dt, n, m, "x", "P", True, K=K, zlay=("own", "scan")[j % 2], zc=("dense", "pad")[j % 2],
                                tag="walk"))
        tiles, big, top, refused = warp_shapes(dt)
        for t, m in sorted(tiles.items()):
            out.append(Case(dt, m, m, "x", "P", False, Ns=(5, 37), K=3, tag="tile%d" % t))
        out.append(Case(dt, big, big, "mean", "P", True, Ns=(5, 37), K=2, shared="R", tag="over48k"))
        out.append(Case(dt, top, top, "x", "P", True, Ns=(5, 9), K=2, tag="top"))
        out.append(Case(dt, refused, refused, "x", "P", True, Ns=(3,), K=2, refused=True))
        # one bank per path past the grid-stride cap (sm_count * 16 tiles)
        out.append(Case(dt, 4, 2, "x", "P", True, Ns=(1,), K=3, grid=True))
        out.append(Case(dt, 5, 2, "x", "S", True, Ns=(1,), K=1, shared="S", grid=True))
        out.append(Case(dt, 6, 6, "mean", "P", True, Ns=(1,), K=2, grid=True))
    return out


CASES = _cases()
RUN_CASES = [c for c in CASES if not c.refused]


def _dispatched():
    """{(n, M) register shapes per M} and the instances, parsed from dispatch_m and dispatch."""
    s = src("score.cu")
    dm = body(s, "int dispatch_m(const ScP<T> &p, cudaStream_t s)")
    assert "if (n == M) return launch<T, M, M>(p, s);" in dm
    assert dm.rstrip().endswith("return launch<T, 0, M>(p, s);")
    reg = {}
    parts = re.split(r"if constexpr \(M == (\d+)\)", dm)
    for k in range(1, len(parts), 2):
        M = int(parts[k])
        reg[M] = sorted(int(a) for a, mm in re.findall(r"if \(n == (\d+)\) return launch<T, \1, (\d+)>", parts[k + 1])
                        if int(mm) == M)
    d = body(s, "int dispatch(const bke_score_args &a, cudaStream_t s)")
    ms = [int(a) for a, b_ in re.findall(r"case (\d+): return dispatch_m<T, (\d+)>\(p, s\);", d) if a == b_]
    assert re.search(r"default: return launch<T, 0, 0>\(p, s\);", d)
    shapes = {M: sorted(set([M] + reg.get(M, []))) for M in ms}
    inst = set()
    for dt in (F32, F64):
        for M, ns in shapes.items():
            for n in ns:
                inst.add(k_score(dt, n, M))
            inst.add(k_score(dt, 0, M))
        inst.add(k_score(dt, 0, 0))
    return shapes, inst, s


def test_instance_table_matches_dispatch():
    """CASES reaches exactly the 14 instances per dtype the dispatch can launch, each case routes where the source
    says, and each path sees every source, stride, K, candidate layout, mask and output set; launch()'s shared-memory
    rule is the one warp_smem() restates."""
    shapes, inst, s = _dispatched()
    assert {M: tuple(v) for M, v in shapes.items()} == {M: tuple(sorted(v)) for M, v in REG.items()}
    assert len(inst) == 28
    table = {k for c in CASES for k in c.kernels}
    assert table == inst, (sorted(inst - table), sorted(table - inst))
    # params(): the phase-A width is dim_x with x or P, else dim_z; launch()'s tile and shared-memory rule
    assert "p.n = (a.x || a.P) ? a.dim_x : a.dim_z;" in s
    ln = body(s, "int launch(ScP<T> p, cudaStream_t s)")
    for line in ("p.scratch = (p.m * p.m + p.m + p.n * p.m + 1) & ~1;",
                 "const size_t scr = (size_t)(THREADS / 32) * p.scratch * sizeof(T), budget = 200 * 1024;",
                 "while (p.tile > THREADS / 32 && (size_t)p.tile * per * sizeof(T) + scr > 64 * 1024) p.tile >>= 1;",
                 "smem = (size_t)p.tile * per * sizeof(T) + scr;",
                 "const int64_t tiles = (p.N + p.tile - 1) / p.tile, cap = (int64_t)sm_count() * 16;"):
        assert line in ln, line
    assert "constexpr int THREADS = 128;" in s
    assert "__host__ __device__ __forceinline__ int slot_words(int m) { return m + m * m + 1; }" in src("score_pairs.cuh")
    for dt in (F32, F64):
        tiles, big, top, refused = warp_shapes(dt)
        assert sorted(tiles) == [4, 8, 16, 32, 64, 128]
        cs = [c for c in CASES if c.dt == dt]
        got_tiles = {warp_smem(c.width, c.m, np.dtype(dt).itemsize)[0] for c in cs if c.path == "warp"}
        assert got_tiles >= {4, 8, 16, 32, 64, 128}
        assert any(c.width == big and warp_smem(big, big, np.dtype(dt).itemsize)[1] > 48 * 1024 for c in cs)
        assert any(c.width == top and not c.refused for c in cs) and any(c.refused and c.width == top + 1 for c in cs)
        for path in ("reg", "warp"):
            pc = [c for c in cs if c.path == path and not c.refused]
            assert {c.K for c in pc} >= set(KS), path
            assert {(c.zlay, c.zc) for c in pc} >= {(lz, zc) for lz in ("own", "scan") for zc in ("dense", "pad", "zero")}
            assert {c.mask for c in pc} == {True, False}
            assert any(c.grid for c in pc)
            for k in "HRS":
                assert any(k in c.shared for c in pc) and any(
                    k not in c.shared and (c.H if k == "H" else c.cov == ("P" if k == "R" else "S")) for c in pc), k
            outsets = {c.outs for c in pc}
            assert all((o,) in outsets for o in OUTS) and OUTS in outsets
            assert any(c.width < c.m for c in pc) or path == "reg"
        # every source combination each instance can take
        for n, m in [(n, m) for m, ns in REG.items() for n in ns] + WARP_SHAPES:
            got = {(c.mean, c.cov, c.H) for c in cs if (c.n, c.m) == (n, m) and not c.tag and not c.grid}
            assert got == set(_sources(n, m)), (n, m)


def test_bank_oracle_matches_the_per_track_oracle():
    """stats_oracle.score_bank (vectorised, used here) gives score()'s outputs, including an exactly singular S, an
    indefinite S and missing candidates."""
    rng = np.random.default_rng(0)
    for m in (1, 3, 6):
        N, K = 40, 7
        S = spd(rng, (N,), m, 1.0)
        S[3] = 0.0
        S[5, -1] = 0.0
        S[5, :, -1] = 0.0
        S[7] = -S[7]
        z, zhat, valid = rng.normal(size=(N, K, m)), rng.normal(size=(N, m)), rng.random((N, K)) > 0.2
        a, o = so.score(z, zhat, S, valid), so.score_bank(z, zhat, S, valid)
        for k in ("y", "d2", "mahalanobis", "log_likelihood", "likelihood", "status"):
            assert np.allclose(o[k], a[k], rtol=1e-12, atol=0, equal_nan=True), (m, k)


# ------------------------------------------------------------------------------------------ inputs
def _zlayout(c, N, K, m):
    """(the z array's shape, z_track_stride, z_cand_stride)."""
    w = m + 3 if c.zc == "pad" else m
    kk = 1 if c.zc == "zero" else K
    if c.zlay == "scan":
        return (kk, w), 0, (0 if c.zc == "zero" else w)
    return (N, kk, w), kk * w, (0 if c.zc == "zero" else w)


def _inputs(c, N, seed, edges=False, period=None):
    """The call's arrays rounded to the dtype; a periodic bank repeats the first ``period`` tracks.  Edge tracks at
    30, 91, 152, ... (cov = S)."""
    P0 = period or N
    rng = np.random.default_rng(seed)
    n, m, K, dt = c.n, c.m, c.K, c.dt
    cnt = lambda k: (1,) if k in c.shared else (P0,)
    d = dict(x=rng.normal(size=(P0, n)) * 3, P=spd(rng, (P0,), n, 1.0), H=rng.normal(size=cnt("H") + (m, n)),
             R=spd(rng, cnt("R"), m, 0.5), S=spd(rng, cnt("S"), m, 1.5), mean=rng.normal(size=(P0, m)) * 3)
    zshape, zt, zc = _zlayout(c, P0, K, m)
    d["z"] = rng.normal(size=zshape) * 3
    d = {k: rd(v, dt) for k, v in d.items()}
    valid = (rng.random((P0, K)) >= 0.2) if c.mask else None
    kind = np.zeros(P0, int)
    if edges:
        assert c.cov == "S" and "S" not in c.shared and c.zlay == "own" and c.zc == "dense"
        er = np.random.default_rng(seed + 99)
        for f in range(30, P0, 61):
            k = (SINGULAR, INDEFINITE, ILLCOND, NANCAND)[(f // 61) % 4]
            if m == 1 and k == ILLCOND:
                continue
            kind[f] = k
            U = np.linalg.qr(er.normal(size=(m, m)))[0]
            if k == SINGULAR:                       # a zero last row and column
                d["S"][f, -1] = 0
                d["S"][f, :, -1] = 0
            elif k == INDEFINITE:
                ev = np.linspace(1.0, 2.0, m)
                ev[0] = -1.5
                d["S"][f] = rd((U * ev) @ U.T, dt)
            elif k == ILLCOND:
                d["S"][f] = rd(4 * (U * np.logspace(0, -np.log10(ILLCOND_COND[dt]), m)) @ U.T, dt)
            else:                                   # one NaN candidate
                d["z"][f, K // 2, 0] = np.nan
            if valid is not None:
                valid[f] = True
    if period:
        rep = -(-N // P0)
        for k in ("x", "P", "mean"):
            d[k] = np.tile(d[k], (rep, 1, 1)[:d[k].ndim])[:N]
        for k in ("H", "R", "S"):
            if k not in c.shared:
                d[k] = np.tile(d[k], (rep, 1, 1))[:N]
        if c.zlay == "own":
            d["z"] = np.tile(d["z"], (rep, 1, 1))[:N]
        if valid is not None:
            valid = np.tile(valid, (rep, 1))[:N]
    return d, valid, zt, zc, kind


def _full(a, N):
    return np.broadcast_to(a, (N,) + a.shape[1:]) if a.shape[0] == 1 else a


def _zfull(c, d, N, zt, zc):
    """z as [N, K, m] in the kernel's indexing."""
    m, K = c.m, c.K
    flat = d["z"].reshape(-1)
    i = np.arange(N)[:, None, None] * zt + np.arange(K)[None, :, None] * zc + np.arange(m)[None, None, :]
    return flat[i]


# ------------------------------------------------------------------------------------------ one call
def run(c, N, seed=0, edges=False, period=None, K=None):
    """One call of c on N tracks: (rc, error text, got, inputs, valid, zt, zc, kind)."""
    from filterpy_b200 import _lib
    d, valid, zt, zc, kind = _inputs(c, N, seed, edges, period)
    K = c.K if K is None else K
    m = c.m
    bf = Bufs(c.dt)
    a = _lib.ScoreArgs()
    a.n_tracks, a.n_candidates, a.dim_x, a.dim_z = N, K, c.n, m
    a.dtype = _lib.BKE_F32 if c.dt == F32 else _lib.BKE_F64
    a.x = ptr(bf.put(d["x"])) if c.mean == "x" else None
    a.mean = ptr(bf.put(d["mean"])) if c.mean == "mean" else None
    if c.cov == "P":
        a.P = ptr(bf.put(d["P"]))
        a.R, a.R_stride = ptr(bf.put(d["R"])), 0 if "R" in c.shared else m * m
    elif c.cov == "S":
        a.S, a.S_stride = ptr(bf.put(d["S"])), 0 if "S" in c.shared else m * m
    if c.H:
        a.H, a.H_stride = ptr(bf.put(d["H"])), 0 if "H" in c.shared else m * c.n
    needs_z = any(o in c.outs for o in ("y",) + SCORES)
    if needs_z:
        a.z, a.z_track_stride, a.z_cand_stride = ptr(bf.put(d["z"])), zt, zc
        if valid is not None:
            a.z_valid = ptr(bf.put(valid.astype(np.uint8), dtype=np.uint8))
    shp = dict(zhat=(N, m), y=(N, K, m), d2=(N, K), mahalanobis=(N, K), log_likelihood=(N, K), likelihood=(N, K),
               status=(N,))
    ov = {}
    for k in c.outs:
        ov[k] = bf.out(shp[k], dtype=np.int32, fill=7) if k == "status" else bf.out(shp[k])
        setattr(a, k, ptr(ov[k]))
    rc, err = call("bke_score_measurements", ctypes.byref(a))
    bf.check_guards()
    got = {k: v.cpu().numpy().reshape(shp[k]) for k, v in ov.items()}
    return rc, err, got, d, valid, zt, zc, kind


# ------------------------------------------------------------------------------------------ the oracle and the checks
def oracle(c, d, N, valid, zt, zc):
    m, n = c.m, c.n
    x, P = d["x"][:N], d["P"][:N]
    H = _full(d["H"], N)[:N] if c.H else None
    if c.mean == "mean":
        zhat, zsc = d["mean"][:N], np.abs(d["mean"][:N]).max(axis=1)
    elif H is not None:
        zhat = np.einsum("fmn,fn->fm", H, x)
        zsc = np.einsum("fmn,fn->fm", np.abs(H), np.abs(x)).max(axis=1)
    else:
        zhat, zsc = x, np.abs(x).max(axis=1)
    if c.cov == "S":
        S = _full(d["S"], N)[:N]
    elif c.cov == "P":
        R = _full(d["R"], N)[:N]
        S = (np.einsum("fan,fnk,fbk->fab", H, P, H) if H is not None else P) + R
    else:
        S = np.broadcast_to(np.eye(m), (N, m, m))
    z = _zfull(c, d, N, zt, zc)
    o = so.score_bank(z, zhat, S, None if valid is None else valid[:N])
    o["zhat"], o["zsc"], o["S"], o["z"] = zhat, zsc, S, z
    return o


def _ulps(got, want, dt):
    """|got - want| in ulps of the dtype at want (want in fp64; the ulp of a subnormal is the smallest one)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    sp = np.spacing(np.abs(want).astype(dt)).astype(np.float64)
    return np.abs(got - want) / sp


EXP_ULPS = 2                         # the CUDA math library's bound for exp and expf


def check(c, N, seed, edges=False, period=None):
    """One call against the oracle (on the first period of a periodic bank); returns what the call wrote."""
    rc, err, got, d, valid, zt, zc, kind = run(c, N, seed, edges, period)
    assert rc == 0, err
    dt, m = c.dt, c.m
    Nc = period or N
    what = "%s N=%d seed=%d%s" % (c.id, N, seed, " edges" if edges else "")
    label = "test_gpu_score_instances %s %s" % (c.path, np.dtype(dt).name)
    tol = TOL[c.path][dt]
    if period:
        for k, v in got.items():
            P0 = v[:Nc]
            for s in range(Nc, N, Nc):
                part = v[s:s + Nc]
                assert np.array_equal(part.view(np.uint8), P0[:len(part)].view(np.uint8)), \
                    "%s: %s of period %d differs from the first" % (what, k, s // Nc)
        got = {k: v[:Nc] for k, v in got.items()}
    o = oracle(c, d, Nc, valid, zt, zc)
    v = np.ones((Nc, c.K), bool) if valid is None else valid[:Nc]
    ok = o["status"] == 0 if c.cov else np.ones(Nc, bool)
    if "status" in got:
        assert np.array_equal(got["status"], o["status"]), what + " status"
    exact_zhat = c.mean == "mean" or not c.H
    src_zhat = d["mean"][:Nc] if c.mean == "mean" else d["x"][:Nc]
    if "zhat" in got:
        if exact_zhat:
            assert np.array_equal(got["zhat"], src_zhat.astype(dt)), what + " zhat is not a copy"
        else:
            close(got["zhat"], o["zhat"], o["zsc"], 1.0, tol, what + " zhat", label)
    z = o["z"]
    if "y" in got:
        vy = np.broadcast_to(v[:, :, None], got["y"].shape)
        assert np.all(got["y"][~vy] == 0), what + " y of an invalid pair"
        if exact_zhat:
            want = np.where(vy, z.astype(dt) - src_zhat.astype(dt)[:, None, :], dt(0))
            assert np.array_equal(got["y"], want, equal_nan=True), what + " y is not z - zhat rounded once"
        else:
            ysc = o["zsc"] + np.abs(np.nan_to_num(z)).max(axis=(1, 2))
            fin = np.isfinite(o["y"]).all(axis=(1, 2))
            close(got["y"], o["y"], ysc, 1.0, tol, what + " y", label, rows=fin)
            assert np.array_equal(np.isnan(got["y"]), np.isnan(o["y"])), what + " y NaN pattern"
    if not c.cov:
        return got, kind
    # the per-track scale of d2 and ll: (|y| + the terms of zhat)^2 ||S^-1|| + |log det S| + m, and cond(S)
    SI = np.where(ok[:, None, None], o["SI"], 0.0)
    ysz = np.sqrt(np.nanmax(np.where(v[:, :, None], o["y"], 0.0) ** 2, axis=(1, 2)) * m) + o["zsc"]
    scale = ysz ** 2 * np.linalg.norm(SI, 2, axis=(1, 2)) + np.abs(np.where(ok, o["logdet"], 0.0)) + m
    cond = np.ones(Nc)
    if ok.any():
        cond[ok] = np.linalg.cond(o["S"][ok])
    good = ok[:, None] & v & np.isfinite(o["d2"])
    for k in ("d2", "log_likelihood"):
        if k in got:
            g = got[k]
            inv = np.full(g.shape, LOG_DBL_MIN if k == "log_likelihood" else 0.0).astype(dt)
            assert np.array_equal(g[~v], inv[~v]), what + " %s of an invalid pair" % k
            assert np.all(np.isnan(g[v & ~good])), what + " %s of a singular S or a NaN candidate is not NaN" % k
            close(np.where(good, g, 0.0), np.where(good, o[k], 0.0), scale, cond, tol, what + " " + k, label)
    if "mahalanobis" in got:
        if "d2" in got:
            with np.errstate(invalid="ignore"):
                assert np.array_equal(got["mahalanobis"], np.sqrt(got["d2"]), equal_nan=True), what + " sqrt(d2)"
        else:
            assert np.all(got["mahalanobis"][~v] == 0)
            assert np.all(np.isnan(got["mahalanobis"][v & ~good]))
            mh = got["mahalanobis"].astype(np.float64)
            close(np.where(good, mh * mh, 0.0), np.where(good, o["d2"], 0.0), scale, cond, tol,
                  what + " mahalanobis^2", label)
    if "likelihood" in got:
        lk = got["likelihood"]
        assert np.all(np.isnan(lk[v & ~good])), what + " likelihood of a singular S"
        u = _ulps(lk[~v], np.exp(np.float64(dt(LOG_DBL_MIN))), dt)
        assert np.all(u <= EXP_ULPS), what + " likelihood of an invalid pair: %.1f ulps" % u.max()
        if "log_likelihood" in got:
            u = _ulps(lk[good], np.exp(got["log_likelihood"][good].astype(np.float64)), dt)
            assert u.size == 0 or u.max() <= EXP_ULPS, "%s likelihood is %.1f ulps from exp(log_likelihood) at %r" % (
                what, u.max(), got["log_likelihood"][good][np.argmax(u)])
        else:
            # exp turns an absolute error of ll into a relative one
            rel = np.abs(lk - o["likelihood"]) / np.maximum(o["likelihood"], np.finfo(dt).tiny)
            rel = np.where(good & (o["likelihood"] > 4 * np.finfo(dt).tiny), rel, 0.0)
            err = (rel / (scale * cond)[:, None]).max(initial=0.0)
            assert err <= tol, "%s likelihood: %.3e" % (what, err)
    return got, kind


def _grid_N(c):
    import torch
    tile = THREADS if c.path == "reg" else warp_smem(c.width, c.m, np.dtype(c.dt).itemsize)[0]
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count * tile + 517


PERIOD = 1037


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_instance_vs_oracle(case):
    """Every output of one call against the oracle over the case's bank sizes (and a periodic bank past the
    grid-stride cap); a shape the warp path refuses returns BKE_ERR_UNSUPPORTED with its text and writes nothing."""
    from filterpy_b200 import _lib
    c = case
    if c.refused:
        rc, err, got, *_ = run(c, 3, seed=1)
        smem = warp_smem(c.width, c.m, np.dtype(c.dt).itemsize)[1]
        assert rc == _lib.BKE_ERR_UNSUPPORTED, rc
        assert err == ("bke_score_measurements: dim_x=%d dim_z=%d needs %d B of shared memory per CTA (> %d)"
                       % (c.width, c.m, smem, 200 * 1024)), err
        for k, v in got.items():
            assert np.all(v == (7 if k == "status" else SENT)), k
        return
    for i, N in enumerate(c.Ns):
        check(c, N, seed=N + 7 * i)
    if c.grid:
        check(c, _grid_N(c), seed=5, period=PERIOD)


EDGE_CASES = [Case(dt, n, m, "x", "S", True, K=5, tag="edges") for dt in (F64, F32)
              for n, m in ((4, 2), (3, 3), (5, 2), (8, 6), (1, 1))]


@pytest.mark.gpu
@pytest.mark.parametrize("case", EDGE_CASES, ids=[c.id for c in EDGE_CASES])
def test_edge_tracks_inside_healthy_tiles(case):
    """An exactly singular S (status 1, NaN scores, y still written), an indefinite S (ll uses log|det S|), an
    ill-conditioned S and a NaN candidate (only its pair is NaN) against the oracle; every other track equals a clean
    run bit for bit."""
    c = case
    N = 1037
    clean, _ = check(c, N, seed=3)
    got, kind = check(c, N, seed=3, edges=True)
    okt = kind == EDGE_OK
    for k in clean:
        assert np.array_equal(clean[k][okt], got[k][okt], equal_nan=True), "%s: %s of a healthy track changed" % (c.id, k)
    sing = kind == SINGULAR
    assert np.all(got["status"][sing] == 1) and np.all(got["status"][~sing] == 0)
    assert np.all(np.isfinite(got["y"][sing]))
    nanc = np.nonzero(kind == NANCAND)[0]
    for f in nanc:
        bad = np.isnan(got["d2"][f])
        assert bad.sum() == 1 and bad[c.K // 2], (c.id, f)
    d, *_ = _inputs(c, N, 3, edges=True)
    ind = kind == INDEFINITE
    assert np.all(np.linalg.eigvalsh(d["S"][ind])[:, 0] < 0)


@pytest.mark.gpu
@pytest.mark.parametrize("NK", [(0, 5), (5, 0)], ids=["N0", "K0"])
def test_empty_call_writes_nothing(NK):
    """N = 0 or K = 0 returns BKE_OK and writes nothing, zhat and status included."""
    from filterpy_b200 import _lib
    c = Case(F64, 4, 2, "x", "P", True, K=NK[1])
    N = max(NK[0], 1)
    d, valid, zt, zc, _ = _inputs(c, N, 0)
    bf = Bufs(F64)
    a = _lib.ScoreArgs()
    a.n_tracks, a.n_candidates, a.dim_x, a.dim_z, a.dtype = NK[0], NK[1], 4, 2, _lib.BKE_F64
    a.x, a.P, a.H, a.R = (ptr(bf.put(d[k])) for k in ("x", "P", "H", "R"))
    a.H_stride, a.R_stride = 8, 4
    a.z, a.z_track_stride, a.z_cand_stride = ptr(bf.put(np.zeros(16))), 2, 2
    for k in OUTS:
        setattr(a, k, ptr(bf.out((16,), dtype=np.int32, fill=7) if k == "status" else bf.out((16,))))
    rc, err = call("bke_score_measurements", ctypes.byref(a))
    assert rc == _lib.BKE_OK, err
    bf.check_guards()
    for buf, off, cnt, _ in bf.outs:
        h = buf.cpu().numpy()[off:off + cnt]
        assert np.all(h == (7 if h.dtype.kind == "i" else SENT))


# ------------------------------------------------------------------------------------------ which kernel runs
def _profiled_names():
    def go():
        for c in CASES:
            run(c, c.Ns[0], seed=1)
    return profiled_names(go, r"score_kernel")


@pytest.mark.gpu
def test_dispatch_runs_the_kernels_of_the_table():
    """Each CASES entry, run once, launches the kernel the table names (a refused shape none)."""
    check_launch_order("test_gpu_score_instances", [(c.id, c.kernels) for c in CASES])
