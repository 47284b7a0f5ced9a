"""Every kernel instance behind bke_imm_batch_filter against the fp64 oracle (tests/imm_oracle.imm_batch), through
the C-ABI, with a table that names the kernel each case launches.

bke_imm_batch_filter (csrc/imm.cu) runs imm_batch_kernel<T, N, MZ, G>: one thread per (track, model), the track's
models in an aligned group of G = 2, 4 or 8 lanes (the next power of two >= M), 128 threads per block, the T-epoch
loop inside the kernel.  The instances are 2/1 and 3/1 in fp32 and fp64 and 4/2 in fp32, each at G = 2, 4, 8.
CASES runs every instance at every model count that maps to its G, at 1, 128/G - 1, 128/G + 1 and 1037 tracks (a
partial last block for every G), and names the calls that must be refused before any launch: a shape without an
instance, each state, diagnostic or output array one element off a 16-byte boundary, and the calls with nothing
to do (no tracks, no epochs), which launch nothing and write nothing.

Inputs are rounded to the kernel's dtype before the oracle sees them (mu, cbar and trans are fp64 in both), so only
the kernel's own arithmetic is measured.  Every case has per-model alpha_sq != 1, per-model F / Q / H / R of which
some are shared (stride 0) and some per track, per-track mu and the cbar = mu . trans of a run that continues, non-zero
starting diagnostics (S, SI, K, y, log-likelihood) and zs_valid misses: at epoch 0 on tracks whose starting S is 0
(ll = -inf, L = DBL_MIN, mu = cbar), mid-run, and one track that misses every epoch.  Each error is taken relative to
the track's own scale of that quantity and divided by the largest cond(S) the track's models met; mu, cbar and omega
are compared as absolute errors and log-likelihoods relative to max(|ll|, 1), both divided by the same cond.  Worst
cases measured on an H100 80GB HBM3 (700 W power limit) with BKE_TEST_ERRLOG over every case, output and bank size,
and the bound set from each:

    family                                   T   fp64 worst  bound     fp32 worst  bound
    state  x, P, x_prior, P_prior, means,    1    1.4e-15    6e-15     6.5e-7      3e-6
           covariances, means_p,             2    4.8e-15    2e-14     8.2e-7      3.5e-6
           covariances_p                     8    1.9e-13    8e-13     6.6e-5      3e-4
                                            32    3.6e-13    1.5e-12      -         -
    diag   S, SI, K, y                       1    1.1e-15    5e-15     7.0e-7      3e-6
                                             2    3.6e-15    1.5e-14   1.4e-6      6e-6
                                             8    7.4e-14    3e-13     4.5e-5      2e-4
                                            32    2.5e-13    1e-12        -         -
    ll     log_likelihood                    1    8.9e-16    4e-15     3.7e-7      1.5e-6
                                             2    2.3e-15    1e-14     1.3e-6      5e-6
                                             8    9.0e-14    4e-13     8.6e-5      3.5e-4
                                            32    2.1e-13    8e-13        -         -
    mu     mu, cbar, omega, mus              1    1.3e-15    5e-15     3.5e-7      1.5e-6
                                             2    2.3e-15    1e-14     1.1e-6      4e-6
                                             8    2.6e-14    1e-13     1.2e-5      5e-5
                                            32    2.0e-13    8e-13        -         -

The growth with T is the recursion's own: the models mix every epoch, and m = 1 makes cond(S) = 1, so the
divisor does not absorb it.
"""
import ctypes
import os
import re

import numpy as np
import pytest

from gpu_harness import (F32, F64, ROOT, TNAME, Bufs, body, call, check_launch_order, close, mag, profiled_names, ptr, rd,
                         spd, src, stable_F)

BLOCK = 128                                     # imm.cu kImmBlock
MAX_MODELS = 8                                  # BKE_MM_MAX_MODELS

# bound per family, dtype and T (the recursion's rounding grows with the epochs: see the table above)
TOL = {
    "state": {F64: {1: 6e-15, 2: 2e-14, 8: 8e-13, 32: 1.5e-12}, F32: {1: 3e-6, 2: 3.5e-6, 8: 3e-4}},
    "diag": {F64: {1: 5e-15, 2: 1.5e-14, 8: 3e-13, 32: 1e-12}, F32: {1: 3e-6, 2: 6e-6, 8: 2e-4}},
    "ll": {F64: {1: 4e-15, 2: 1e-14, 8: 4e-13, 32: 8e-13}, F32: {1: 1.5e-6, 2: 5e-6, 8: 3.5e-4}},
    "mu": {F64: {1: 5e-15, 2: 1e-14, 8: 1e-13, 32: 8e-13}, F32: {1: 1.5e-6, 2: 4e-6, 8: 5e-5}},
}


def _bound(c, fam):
    """Family fam's tolerance at case c's dtype and T, and the label of its BKE_TEST_ERRLOG lines."""
    return TOL[fam][c.dt][c.T], "test_gpu_imm_instances %s %s T=%d" % (fam, np.dtype(c.dt).name, c.T)


INSTANCES = {F32: [(2, 1), (3, 1), (4, 2)], F64: [(2, 1), (3, 1)]}
# the arrays validate_imm requires on a 16-byte boundary (per model, then shared)
ALIGNED_MODEL = ("x", "P", "S", "log_likelihood", "K", "y", "SI", "x_prior", "P_prior")
ALIGNED_SHARED = ("means", "covariances", "means_p", "covariances_p")
ERR_SHAPE = "bke_imm_batch_filter: no fused instance for dim_x=%d, dim_z=%d in this dtype"
ERR_ALIGN = "bke_imm_batch_filter: the state, diagnostic and output arrays must be 16-byte aligned"


def group(M):
    """launch_shape: the lanes of a track's group."""
    return 2 if M <= 2 else (4 if M <= 4 else 8)


def k_imm(dt, n, m, G):
    return "imm_batch_kernel<%s, %d, %d, %d>" % (TNAME[dt], n, m, G)


# ------------------------------------------------------------------------------------------ the instance table
class Case:
    """One bke_imm_batch_filter call and the kernel it launches at Np tracks.  kind: "run" (the oracle tests run it
    at every N of Ns), "refused" (BKE_ERR_UNSUPPORTED with the error text err; mis names the array put one element
    off its 16-byte boundary), "empty" (n_tracks = 0 or n_steps = 0: BKE_OK, nothing launched, nothing written)."""

    def __init__(self, kind, dt, n, m, M, T, kernels, Np, Ns=(), mis=None, err=None):
        self.kind, self.dt, self.n, self.m, self.M, self.T = kind, dt, n, m, M, T
        self.kernels, self.Np, self.Ns, self.mis, self.err = list(kernels), Np, tuple(Ns), mis, err

    @property
    def id(self):
        s = "%s-%s-%d_%d-M%d-T%d" % (self.kind, "f32" if self.dt == F32 else "f64", self.n, self.m, self.M, self.T)
        if self.mis:
            s += "-mis_" + self.mis
        return s + "-N%d" % self.Np


# T per model count: 1, 2 and 8 epochs in both dtypes across the model counts
T_OF_M = {2: 8, 3: 1, 4: 2, 5: 8, 6: 1, 7: 2, 8: 8}


def _cases():
    out = []
    for dt in (F64, F32):
        for n, m in INSTANCES[dt]:
            for M in range(2, MAX_MODELS + 1):
                G = group(M)
                tile = BLOCK // G
                out.append(Case("run", dt, n, m, M, T_OF_M[M], [k_imm(dt, n, m, G)], tile + 1,
                                (1, tile - 1, tile + 1, 1037)))
    # long runs in fp64, at G = 4 and G = 8
    for n, m, M in ((2, 1, 3), (3, 1, 6)):
        G = group(M)
        out.append(Case("run", F64, n, m, M, 32, [k_imm(F64, n, m, G)], BLOCK // G + 1, (1, BLOCK // G + 1, 1037)))
    # shapes without an instance
    for dt, n, m in ((F64, 4, 2), (F32, 6, 3), (F64, 6, 3), (F32, 5, 2)):
        out.append(Case("refused", dt, n, m, 3, 2, [], 5, err=ERR_SHAPE % (n, m)))
    # each aligned array one element off its boundary
    for name in ALIGNED_MODEL + ALIGNED_SHARED:
        out.append(Case("refused", F32, 4, 2, 3, 2, [], 5, mis=name, err=ERR_ALIGN))
    out.append(Case("empty", F32, 4, 2, 3, 3, [], 0))
    out.append(Case("empty", F64, 2, 1, 5, 0, [], 9))
    return out


CASES = _cases()
RUN = [c for c in CASES if c.kind == "run"]


# ------------------------------------------------------------------------------------------ the table vs the source
def _dispatched():
    """(the instances launch_imm_batch can launch, {M: G} of launch_shape, the shapes imm_batch_has_instance accepts,
    the arrays validate_imm aligns), parsed from the source."""
    text = src("imm.cu")
    li = body(text, "int launch_imm_batch(const bke_imm_batch_args &a, cudaStream_t s)")
    f32part, f64part = li.split("} else {")
    shapes = {F32: [], F64: []}
    for part, dt in ((f32part, F32), (f64part, F64)):
        for a, b, t, c, e in re.findall(r"if \(n == (\d+) && m == (\d+)\) return launch_shape<(\w+), (\d+), (\d+)>"
                                        r"\(a, s\);", part):
            assert (a, b) == (c, e) and t == TNAME[dt]
            shapes[dt].append((int(a), int(b)))
    assert 'set_error("%s", n, m);' % ERR_SHAPE in li
    ls = body(text, "int launch_shape(const bke_imm_batch_args &a, cudaStream_t s)")
    steps = [(int(k), int(g)) for k, g in re.findall(r"if \(a\.n_models <= (\d+)\) return launch_g<T, N, MZ, (\d+)>", ls)]
    last = re.findall(r"\n\s*return launch_g<T, N, MZ, (\d+)>\(a, s\);", ls)
    assert len(last) == 1
    gmap = {}
    for M in range(2, MAX_MODELS + 1):
        gmap[M] = next((g for k, g in steps if M <= k), int(last[0]))
    lg = body(text, "int launch_g(const bke_imm_batch_args &a, cudaStream_t s)")
    assert "imm_batch_kernel<T, N, MZ, G>" in lg and "grid, kImmBlock, 0, &p, s" in lg
    assert re.search(r"constexpr int kImmBlock = %d;" % BLOCK, text)
    inst = {k_imm(dt, n, m, g) for dt, shp in shapes.items() for n, m in shp for g in set(gmap.values())}
    has = body(text, "bool imm_batch_has_instance(int dim_x, int dim_z, int dtype)")
    accepted = {F32: [], F64: []}
    for a, b, f32 in re.findall(r"\(dim_x == (\d+) && dim_z == (\d+)( && dtype == BKE_F32)?\)", has):
        for dt in ((F32,) if f32 else (F32, F64)):
            accepted[dt].append((int(a), int(b)))
    api = src("api.cu")
    v = body(api, "static int validate_imm(const bke_imm_batch_args *a)")
    al = v[v.index("auto al16"):]
    aligned = (set(re.findall(r"al16\(a->(\w+)\[j\]\)", al)), set(re.findall(r"al16\(a->(\w+)\)", al)))
    assert ERR_ALIGN in al and "return BKE_ERR_UNSUPPORTED;" in al
    with open(os.path.join(ROOT, "include", "bke.h")) as fh:
        assert re.search(r"#define BKE_MM_MAX_MODELS %d\b" % MAX_MODELS, fh.read())
    return inst, gmap, shapes, accepted, aligned


def test_instance_table_matches_dispatch():
    """CASES launches every imm_batch_kernel instance the dispatch can reach and no other, at every model count of
    each G, and names a refused call for every array the alignment check covers: a new shape, lane-group size or
    aligned array in the source, or a removed one, fails here, on a machine without a GPU too."""
    inst, gmap, shapes, accepted, aligned = _dispatched()
    assert shapes == INSTANCES and {dt: sorted(v) for dt, v in accepted.items()} == {dt: sorted(v) for dt, v in
                                                                                    INSTANCES.items()}
    assert all(gmap[M] == group(M) for M in gmap), gmap
    table = {k for c in RUN for k in c.kernels}
    assert table == inst, (sorted(inst - table), sorted(table - inst))
    for dt, shp in INSTANCES.items():
        for n, m in shp:
            got = {c.M for c in RUN if (c.dt, c.n, c.m) == (dt, n, m)}
            assert got == set(range(2, MAX_MODELS + 1)), (dt, n, m, got)
            Ts = {c.T for c in RUN if c.dt == dt}
            assert {1, 2, 8} <= Ts
    assert any(c.T >= 32 for c in RUN if c.dt == F64)
    for c in RUN:                               # 1 track, one group short of and past a block, a partial bank
        tile = BLOCK // group(c.M)
        assert {1, tile + 1, 1037} <= set(c.Ns) and (c.T == 32 or tile - 1 in c.Ns)
        assert all((N * group(c.M)) % BLOCK for N in c.Ns)
    ref = [c for c in CASES if c.kind == "refused"]
    assert {(c.dt, c.n, c.m) for c in ref if not c.mis} == {(F64, 4, 2), (F32, 6, 3), (F64, 6, 3), (F32, 5, 2)}
    for c in ref:
        if not c.mis:
            assert (c.n, c.m) not in INSTANCES[c.dt]
    assert aligned == (set(ALIGNED_MODEL), set(ALIGNED_SHARED)), aligned
    assert {c.mis for c in ref if c.mis} == set(ALIGNED_MODEL + ALIGNED_SHARED)
    assert {(c.Np == 0, c.T == 0) for c in CASES if c.kind == "empty"} == {(True, False), (False, True)}


def test_extended_oracle_reproduces_the_goldens(golden):
    """imm_batch with every starting value it takes given explicitly (zero diagnostics, per-track mu, cbar = mu .
    trans) reproduces each imm_batch_* golden as it does with the defaults, and reports no failure."""
    from imm_oracle import golden_inputs, imm_batch
    for name in ("m2_4_2", "m3_4_2", "m4_4_2", "m3_6_3", "m2_2_1", "m3_3_1", "m2_5_2"):
        g = golden("imm_batch_" + name)
        args = golden_inputs(g)
        N, M, n = g["x0"].shape
        m = g["zs"].shape[2]
        mu = np.broadcast_to(np.asarray(g["mu0"], float), (N, M))
        mu = mu / mu.sum(axis=1, keepdims=True)
        o = imm_batch(*args[:7], mu, *args[8:], S0=np.zeros((N, M, m, m)), ll0=np.zeros((N, M)),
                      K0=np.zeros((N, M, n, m)), y0=np.zeros((N, M, m)), SI0=np.zeros((N, M, m, m)),
                      cbar0=mu @ g["trans"])
        for k in ("x", "P", "xp", "Pp", "mu", "cbar", "omega", "fx", "fP"):
            scale = max(np.abs(g[k]).max(), 1e-300)
            assert np.abs(o[k] - g[k]).max() <= 1e-12 * scale, (name, k)
        np.testing.assert_allclose(o["lik"], g["lik"], rtol=1e-10, atol=0)
        assert not o["status_any"].any()


# ------------------------------------------------------------------------------------------ inputs
def _layout(j):
    """Which of model j's F, Q, H, R are shared by every track (stride 0): a different mix per model, model 0 all per
    track (it is the model the singular-S runs break for one track)."""
    return dict(F=j % 2 == 1, Q=j % 3 == 2, H=j % 2 == 0 and j > 0, R=j % 3 == 1)


def imm_inputs(c, N, seed):
    """The arrays of one call, rounded to the case's dtype, and the tracks whose starting S is 0 / that never measure."""
    rng = np.random.default_rng(seed)
    n, m, M, T, dt = c.n, c.m, c.M, c.T, c.dt
    d = dict(F=[], Q=[], H=[], R=[])
    for j in range(M):
        sh = _layout(j)
        cnt = lambda k: () if sh[k] else (N,)
        d["F"].append(stable_F(rng, cnt("F"), n))
        d["Q"].append(spd(rng, cnt("Q"), n, 0.02 * (j + 1)))
        d["H"].append(rng.normal(size=cnt("H") + (m, n)))
        d["R"].append(spd(rng, cnt("R"), m, 0.3 + 0.2 * j))
    d["alpha_sq"] = np.array([(1.0 + 0.01 * (j + 1)) ** 2 for j in range(M)])
    d["x"] = rng.normal(size=(N, M, n)) * 3
    d["P"] = spd(rng, (N, M), n, 2.0)
    d["S"] = spd(rng, (N, M), m, 1.0)
    d["SI"] = rng.normal(size=(N, M, m, m))
    d["K"] = rng.normal(size=(N, M, n, m))
    d["y"] = rng.normal(size=(N, M, m))
    d["ll"] = -rng.uniform(1.0, 5.0, size=(N, M))
    zero_S = (np.arange(N) % 5) == 2
    d["S"][zero_S] = 0
    trans = 0.6 * np.eye(M) + 0.4 * rng.dirichlet(np.ones(M), size=M)
    d["trans"] = trans / trans.sum(axis=1, keepdims=True)
    d["mu"] = rng.dirichlet(np.ones(M), size=N)
    d["cbar"] = d["mu"] @ d["trans"]
    d["zs"] = rng.normal(size=(T, N, m)) * 3
    valid = rng.random((T, N)) > 0.15
    if T:
        valid[0, zero_S] = False                # ll = -inf for every model: L = DBL_MIN, mu = cbar
    if T > 1 and N:
        valid[T // 2, 0] = False                # a miss mid-run
    never = N // 2 if N > 2 else None
    if never is not None:
        valid[:, never] = False
    d["valid"] = valid
    for k in ("x", "P", "S", "SI", "K", "y", "ll", "zs"):
        d[k] = rd(d[k], dt)
    for k in "FQHR":
        d[k] = [rd(a, dt) for a in d[k]]
    return d


def _per_track(a, N):
    return np.broadcast_to(a, (N,) + a.shape) if a.ndim == 2 else a


def imm_oracle(d, N):
    from imm_oracle import imm_batch
    st = lambda k: np.stack([_per_track(a, N) for a in d[k]], axis=1)
    return imm_batch(d["x"], d["P"], st("F"), st("Q"), st("H"), st("R"), d["alpha_sq"], d["mu"], d["trans"], d["zs"],
                     d["valid"], S0=d["S"], ll0=d["ll"], K0=d["K"], y0=d["y"], SI0=d["SI"], cbar0=d["cbar"])


def run_imm(c, N, d, sticky=False, mis=None):
    """One bke_imm_batch_filter call on the inputs d: (rc, error text, the outputs host-side, Bufs).  Every output
    starts as NaN (status as 5), so an element the kernel never writes shows up."""
    from filterpy_b200 import _lib
    dt, n, m, M, T = c.dt, c.n, c.m, c.M, c.T
    bf = Bufs(dt)
    a = _lib.ImmBatchArgs()
    a.n_tracks, a.dim_x, a.dim_z, a.n_models, a.n_steps = N, n, m, M, T
    a.dtype = _lib.BKE_F32 if dt == F32 else _lib.BKE_F64
    a.flags = _lib.BKE_STATUS_STICKY if sticky else 0
    nan = float("nan")
    views = {}
    shapes = dict(x=(n,), P=(n, n), S=(m, m), SI=(m, m), K=(n, m), y=(m,), log_likelihood=(), x_prior=(n,),
                  P_prior=(n, n))
    src = dict(x="x", P="P", S="S", SI="SI", K="K", y="y", log_likelihood="ll")
    for j in range(M):
        for k, shp in shapes.items():
            off = mis == k and j == 1
            if k in src:
                v = bf.put(d[src[k]][:, j], off, out=True)
            else:
                v = bf.out((N,) + shp, off, fill=nan)
            views[(k, j)] = v
            getattr(a, k)[j] = ptr(v)
        st = bf.out((N,), dtype=np.int32, fill=5)
        views[("status", j)] = st
        a.status[j] = ptr(st)
        for k in "FQHR":
            arr = d[k][j]
            getattr(a, k)[j] = ptr(bf.put(arr))
            getattr(a, k + "_stride")[j] = 0 if arr.ndim == 2 else arr.shape[-1] * arr.shape[-2]
        a.alpha_sq[j] = float(d["alpha_sq"][j])
    for k in ("mu", "cbar"):
        views[k] = bf.put(d[k], out=True, dtype=F64)
        setattr(a, k, ptr(views[k]))
    views["omega"] = bf.out((N, M, M), dtype=F64, fill=nan)
    a.omega = ptr(views["omega"])
    a.trans = ptr(bf.put(d["trans"], dtype=F64))
    a.zs = ptr(bf.put(d["zs"]))
    a.zs_valid = ptr(bf.put(d["valid"].astype(np.uint8), dtype=np.uint8))
    for k, shp in (("means", (n,)), ("covariances", (n, n)), ("means_p", (n,)), ("covariances_p", (n, n))):
        views[k] = bf.out((T, N) + shp, mis == k, fill=nan)
        setattr(a, k, ptr(views[k]))
    views["mus"] = bf.out((T, N, M), dtype=F64, fill=nan)
    a.mus = ptr(views["mus"])
    rc, err = call("bke_imm_batch_filter", ctypes.byref(a))
    got = {}
    for key, v in views.items():
        h = v.cpu().numpy()
        if isinstance(key, tuple):
            k, j = key
            got.setdefault(k, [None] * M)[j] = h.reshape((N,) + shapes.get(k, ()))
        else:
            got[key] = h
    for k in list(shapes) + ["status"]:
        got[k] = np.stack(got[k], axis=1)                           # [N, M, ...]
    got["omega"] = got["omega"].reshape(N, M, M)
    got["mu"], got["cbar"] = got["mu"].reshape(N, M), got["cbar"].reshape(N, M)
    for k, shp in (("means", (n,)), ("covariances", (n, n)), ("means_p", (n,)), ("covariances_p", (n, n)),
                   ("mus", (M,))):
        got[k] = got[k].reshape((T, N) + shp)
    return rc, err, got, bf


def check_imm(c, N, d, got, want, sticky, what):
    sw = lambda a: np.swapaxes(a, 0, 1)                             # [T, N, ...] -> [N, T, ...]
    cond = want["cond"]

    def _cmp(fam, got_, want_, scale, what_):
        """Per track (axis 0), relative to its scale x cond; -inf only where the oracle has it."""
        tol, label = _bound(c, fam)
        close(got_, want_, scale, cond, tol, what_, label, match_inf=True)

    sx = mag(d["x"], sw(want["x"]), sw(want["xp"]), sw(want["fx"]), want["fxp"])
    sP = mag(d["P"], sw(want["P"]), sw(want["Pp"]), sw(want["fP"]), want["fPp"])
    for k, w, s in (("means", "x", sx), ("means_p", "xp", sx), ("covariances", "P", sP), ("covariances_p", "Pp", sP)):
        _cmp("state", sw(got[k]), sw(want[w]), s, what + " " + k)
    _cmp("mu", sw(got["mus"]), sw(want["mu"]), np.ones(N), what + " mus")
    for k, w, s in (("x", "fx", sx), ("P", "fP", sP)):
        _cmp("state", got[k], want[w][-1], s, what + " " + k)
    _cmp("state", got["x_prior"], want["fxp"], sx, what + " x_prior")
    _cmp("state", got["P_prior"], want["fPp"], sP, what + " P_prior")
    Hmax = np.max([np.abs(_per_track(h, N)).reshape(N, -1).max(axis=1) for h in d["H"]], axis=0)
    sy = mag(sw(d["zs"]), d["y"]) + Hmax * np.abs(want["fxp"]).sum(axis=2).max(axis=1)
    _cmp("diag", got["y"], want["fy"], sy, what + " y")
    for k, w, s in (("S", "fS", mag(d["S"], want["fS"])), ("SI", "fSI", mag(d["SI"], want["fSI"])),
                    ("K", "fK", mag(d["K"], want["fK"]))):
        _cmp("diag", got[k], want[w], s, what + " " + k)
    fin = np.where(np.isinf(want["fll"]), 1.0, np.abs(want["fll"]))
    _cmp("ll", got["log_likelihood"] / np.maximum(fin, 1.0), want["fll"] / np.maximum(fin, 1.0), np.ones(N),
         what + " log_likelihood")
    for k, w in (("mu", "mu"), ("cbar", "cbar"), ("omega", "omega")):
        _cmp("mu", got[k], want[w][-1], np.ones(N), what + " " + k)
    st_want = want["status_any"] if sticky else want["status"]
    assert np.array_equal(got["status"], st_want), what + " status"


def _fresh(d):
    return {k: ([a.copy() for a in v] if isinstance(v, list) else np.array(v)) for k, v in d.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("case", RUN, ids=[c.id for c in RUN])
def test_instance_vs_oracle(case):
    """means, covariances, means_p, covariances_p and mus of every epoch, each model's final x, P, x_prior, P_prior,
    S, SI, K, y, log_likelihood and status, and the final mu, cbar and omega against the fp64 oracle, over the case's
    track counts, with and without BKE_STATUS_STICKY."""
    for i, N in enumerate(case.Ns):
        d = imm_inputs(case, N, seed=N + 11 * i + case.M)
        sticky = bool(i % 2)
        rc, err, got, bf = run_imm(case, N, d, sticky=sticky)
        assert rc == 0, err
        bf.check_guards()
        check_imm(case, N, d, got, imm_oracle(d, N), sticky, "%s N=%d%s" % (case.id, N, " sticky" if sticky else ""))


@pytest.mark.gpu
@pytest.mark.parametrize("case", RUN, ids=[c.id for c in RUN])
def test_singular_S_in_one_track(case):
    """H = 0 and R = 0 for model 0 of one track: at every epoch that track measures, that model's S is singular, it
    keeps its prior and its previous log-likelihood, stores S = 0 and reports BKE_STATUS_SINGULAR_S (with
    BKE_STATUS_STICKY the call's first failure; without it the last epoch's, which is OK: the track misses its last
    epoch wherever T > 1).  Every other track is bit-equal to a clean run."""
    N = case.Ns[-1] if case.T < 32 else case.Np
    bad = N // 3
    clean = imm_inputs(case, N, seed=5 + case.M)
    d = _fresh(clean)
    d["H"][0][bad] = 0
    d["R"][0][bad] = 0
    if case.T > 2:
        d["valid"][1, bad] = False               # a miss between two singular epochs: ll = -inf of the kept S = 0
        d["valid"][2, bad] = True
    d["valid"][-1, bad] = False                  # the last epoch misses: its status is OK, the call's worst is not
    d["valid"][0, bad] = True
    for sticky in (False, True):
        rc, err, got, bf = run_imm(case, N, d, sticky=sticky)
        assert rc == 0, err
        bf.check_guards()
        want = imm_oracle(d, N)
        assert want["status_any"][bad, 0] == 1 and not want["status_any"][np.arange(N) != bad].any()
        assert want["status"][bad, 0] == (1 if case.T == 1 else 0)
        check_imm(case, N, d, got, want, sticky, "%s N=%d singular%s" % (case.id, N, " sticky" if sticky else ""))
        rc, err, ref, _ = run_imm(case, N, clean, sticky=sticky)
        assert rc == 0, err
        others = np.arange(N) != bad
        for k, v in got.items():
            ax = 1 if k in ("means", "covariances", "means_p", "covariances_p", "mus") else 0
            a, b = np.compress(others, v, axis=ax), np.compress(others, ref[k], axis=ax)
            assert np.array_equal(a, b, equal_nan=True), "%s: another track changed" % k


# ------------------------------------------------------------------------------------------ refused and empty calls
@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if c.kind != "run"], ids=[c.id for c in CASES if c.kind != "run"])
def test_refused_and_empty_calls(case):
    """A shape without an instance or a misaligned array is BKE_ERR_UNSUPPORTED with its error text; no tracks or no
    epochs is BKE_OK.  Neither writes any output."""
    from filterpy_b200 import _lib
    N = case.Np
    d = imm_inputs(case, N, seed=3)
    rc, err, got, bf = run_imm(case, N, d, mis=case.mis)
    if case.kind == "refused":
        assert rc == _lib.BKE_ERR_UNSUPPORTED and err == case.err, (rc, err)
    else:
        assert rc == _lib.BKE_OK, err
    bf.check_guards()
    for k in ("x", "P", "S", "SI", "K", "y", "mu", "cbar"):
        src = {"mu": d["mu"], "cbar": d["cbar"]}.get(k, d.get(k))
        assert np.array_equal(got[k], np.asarray(src, got[k].dtype).reshape(got[k].shape)), k
    assert np.array_equal(got["log_likelihood"], d["ll"].astype(got["log_likelihood"].dtype))
    for k in ("x_prior", "P_prior", "omega", "means", "covariances", "means_p", "covariances_p", "mus"):
        assert np.all(np.isnan(got[k])), k + " written"
    assert np.all(got["status"] == 5)


# ------------------------------------------------------------------------------------------ which kernel runs
def _run_cases():
    for c in CASES:
        run_imm(c, c.Np, imm_inputs(c, c.Np, seed=1), mis=c.mis)


def _profiled_names():
    """The kernel names of every CASES entry run once at its Np, in launch order."""
    return profiled_names(_run_cases, r"imm_batch_kernel|kf\w*_kernel|fls_\w+_kernel")


@pytest.mark.gpu
def test_dispatch_runs_the_kernels_of_the_table():
    """Each CASES entry, run once at its Np, launches the kernels the table names, in order, template arguments
    included; refused and empty calls launch nothing."""
    check_launch_order("test_gpu_imm_instances", [(c.id, c.kernels) for c in CASES])
