"""Every kernel instance behind bke_poly_filter against the dtype twin of the oracle (tests/poly_oracle.py), bit for
bit in fp64 and fp32, through the C-ABI, with a table that names the kernel each case launches.

launch_typed (csrc/poly.cu) runs 12 poly_kernel<FAM, ORD, BATCH, T> instances per dtype: GH and GHK batch_filter on
<GH, 1, true, T>, the GH and GHK update on their own instance, and one instance per order of GH_ORDER, LSQ and
FADING, which serves both of their modes.  The kernel's arithmetic is explicitly rounded (no contraction), so the
oracle that runs the same operations in the same order and dtype must match every output bit for bit, fp32 included;
a reordered sum, another constant rounding or a fused multiply-add changes a bit.

Every call runs on guarded sentinel buffers (tests/gpu_harness.py).  Each parameter is shared (stride 0) or per
filter by a seeded mask, and a parameter the instance does not read is NULL, or a NaN buffer in some runs (which would
poison the result if it were read).  The state is written back in UPDATE and left alone in BATCH (for LSQ the
counters n[] too).  LSQ counters differ across the bank; the fp32 data holds counters whose gains the double-rounding
detour int64 -> double -> float would change (orders 0 and 1: at order 2 no counter the call accepts gives a product
that rounds differently), and the counter bound is tried at its last accepted and first refused value."""
import ctypes
import os
import re

import numpy as np
import pytest

from gpu_harness import F32, F64, ROOT, TNAME, Bufs, b, body, call, check_launch_order, profiled_names, ptr, src

import poly_oracle as po

GH, GHK, GHO, LSQ, FM = 0, 1, 2, 3, 4                # include/bke.h BKE_POLY_*
UPDATE, BATCH = 0, 1
FNAME = {GH: "GH", GHK: "GHK", GHO: "GH_ORDER", LSQ: "LSQ", FM: "FADING"}
PARAMS = ("g", "h", "k", "dt", "dt2", "hdt2")
NS = (1, 255, 256, 257, 100003)
TS = (1, 2, 64)
INT64_MAX = 2**63 - 1


def k_poly(dt, fam, order, batch):
    return "poly_kernel<%d, %d, %s, %s>" % (fam, order, b(batch), TNAME[dt])


def instance(fam, order, mode):
    """launch_typed's routing: the (FAM, ORD, BATCH) a call runs on."""
    if fam in (GH, GHK):
        return (GH, 1, True) if mode == BATCH else ((GH, 1, False) if fam == GH else (GHK, 2, False))
    return fam, order, False


def reads(fam, order, mode):
    """The parameters the instance reads (api.cu validate_poly's need_*)."""
    batch, gh = mode == BATCH, fam in (GH, GHK)
    ord_ = 1 if fam == GH else 2 if fam == GHK else order
    need = dict(g=fam != LSQ, h=gh or (ord_ >= 1 and fam != LSQ),
                k=(fam == GHK and not batch) or (ord_ == 2 and fam in (GHO, FM)), dt=ord_ >= 1,
                dt2=(fam == GHK and not batch) or (not gh and ord_ == 2), hdt2=fam == LSQ and ord_ == 2)
    return tuple(k for k in PARAMS if need[k])


def outputs(fam, mode):
    """The optional outputs the family and mode have (include/bke.h)."""
    o = ["results"]
    if fam in (GH, GHK):
        o += ["predictions"] if mode == BATCH else ["y", "x_prediction", "dx_prediction"]
        if fam == GHK and mode == UPDATE:
            o.append("ddx_prediction")
    elif fam == GHO and mode == UPDATE:
        o.append("y")
    elif fam == LSQ and mode == UPDATE:
        o.append("K")
    return tuple(o)


def state_width(fam, order):
    return 2 if fam == GH else 3 if fam == GHK else order + 1


# ------------------------------------------------------------------------------------------ the instance table
class Case:
    def __init__(self, dt, fam, order, mode):
        self.dt, self.fam, self.order, self.mode = dt, fam, order, mode
        self.kernels = [k_poly(dt, *instance(fam, order, mode))]

    @property
    def id(self):
        return "%s%s-%s-%s" % (FNAME[self.fam], "" if self.fam in (GH, GHK) else str(self.order),
                               "batch" if self.mode == BATCH else "update", "f32" if self.dt == F32 else "f64")


def _cases():
    out = []
    for dt in (F64, F32):
        for fam in (GH, GHK, GHO, LSQ, FM):
            for order in ((1,) if fam == GH else (2,) if fam == GHK else (0, 1, 2)):
                for mode in (UPDATE, BATCH):
                    out.append(Case(dt, fam, order, mode))
    return out


CASES = _cases()


def test_instance_table_matches_dispatch():
    """CASES reaches every instance launch_typed can launch (24: 12 per dtype) and each case routes where the source
    says it does: GH and GHK batch on <GH, 1, true, T>, one instance per order serving both modes of the others."""
    with open(os.path.join(ROOT, "include", "bke.h")) as fh:
        hdr = fh.read()
    val = {k: int(v) for k, v in re.findall(r"#define BKE_POLY_(\w+) (\d+)", hdr)}
    assert (val["GH"], val["GHK"], val["GH_ORDER"], val["LSQ"], val["FADING"]) == (GH, GHK, GHO, LSQ, FM)
    assert (val["UPDATE"], val["BATCH"]) == (UPDATE, BATCH)
    s = src("poly.cu")
    lt = body(s, "int launch_typed(const bke_poly_args &a, cudaStream_t s)")
    found = {(val[f], int(o), bb == "true") for f, o, bb in re.findall(r"launch_one<BKE_POLY_(\w+), (\d), (true|false), T>", lt)}
    inst = {k_poly(dt, *i) for i in found for dt in (F32, F64)}
    assert len(inst) == 24
    table = {k for c in CASES for k in c.kernels}
    assert table == inst, (sorted(inst - table), sorted(table - inst))
    # the routes
    assert re.search(r"case BKE_POLY_GH:\s*case BKE_POLY_GHK:\s*if \(batch\) return launch_one<BKE_POLY_GH, 1, true, T>\(a, s\);\s*"
                     r"return a.family == BKE_POLY_GH \? launch_one<BKE_POLY_GH, 1, false, T>\(a, s\) : "
                     r"launch_one<BKE_POLY_GHK, 2, false, T>\(a, s\);", lt), lt
    for fam, nxt in (("GH_ORDER", "case BKE_POLY_LSQ:"), ("LSQ", "default:"), ("FADING", "}")):
        seg = lt[lt.index("launch_one<BKE_POLY_%s, 0" % fam) - 40:]
        seg = seg[:seg.index(nxt)] if nxt in seg else seg
        assert re.search(r"a.order == 0 \? launch_one<BKE_POLY_%s, 0, false, T>\(a, s\)\s*: a.order == 1 \? "
                         r"launch_one<BKE_POLY_%s, 1, false, T>\(a, s\) : launch_one<BKE_POLY_%s, 2, false, T>\(a, s\);"
                         % (fam, fam, fam), seg), seg
    assert re.search(r"default:\s*return a.order == 0 \? launch_one<BKE_POLY_FADING", lt)
    assert "return a.dtype == BKE_F64 ? launch_typed<double>(a, s) : launch_typed<float>(a, s);" in s
    # the validator's need_* rules, restated in reads()
    v = body(src("api.cu"), "static int validate_poly(const bke_poly_args &a)")
    for line in ("const bool need_g = fam != BKE_POLY_LSQ;",
                 "const bool need_h = gh || (ord >= 1 && fam != BKE_POLY_LSQ);",
                 "const bool need_k = (fam == BKE_POLY_GHK && !batch) || (ord == 2 && (fam == BKE_POLY_GH_ORDER || "
                 "fam == BKE_POLY_FADING));",
                 "const bool need_dt = ord >= 1;",
                 "const bool need_dt2 = (fam == BKE_POLY_GHK && !batch) || (!gh && ord == 2);",
                 "const bool need_hdt2 = fam == BKE_POLY_LSQ && ord == 2;"):
        assert line in v, line


# ------------------------------------------------------------------------------------------ inputs
# counters whose gains differ through int64 -> double -> float: 1 / n at order 0 (2^60 + 2^36 + 1 rounds to a float
# tie in double), n (n + 1) at order 1 (found by search)
DOUBLE_ROUNDING = {0: (2**60 + 2**36 + 1, 2**61 + 2**37 + 3), 1: (442351154, 806812181)}


def _counters(c, N, T, rng):
    """LSQ counters n[N] on entry: different across the bank, and in fp32 the double-rounding counters (reached at
    the first epoch) in a few filters."""
    n = rng.integers(0, 5000, N).astype(np.int64)
    if c.order == 2:
        big = rng.random(N) < 0.3
        n[big] = rng.integers(2**18, 2**20, big.sum())
    if c.dt == F32 and c.order in DOUBLE_ROUNDING:
        for i, v in enumerate(DOUBLE_ROUNDING[c.order]):
            n[(7 + 61 * i) % N] = v - 1
    return n


def _inputs(c, N, T, seed, shared_mask=None):
    """The call's arrays in the case's dtype: state, zs, parameters (shared ones as one element) and counters."""
    dt = c.dt
    rng = np.random.default_rng(seed)
    S = state_width(c.fam, c.order)
    X = (rng.normal(size=(N, S)) * np.array([10.0, 1.0, 0.1])[:S]).astype(dt)
    v = rng.normal(size=N)
    zs = (X[:, 0].astype(np.float64) + v * np.arange(1, T + 1)[:, None] + rng.normal(size=(T, N))).astype(dt)
    rd = reads(c.fam, c.order, c.mode)
    shared = {k: bool(rng.random() < 0.5) for k in rd} if shared_mask is None else dict(shared_mask)
    raw = dict(g=rng.uniform(0.05, 0.6, N), h=rng.uniform(0.01, 0.2, N), k=rng.uniform(0.001, 0.02, N),
               dt=rng.uniform(0.25, 2.0, N))
    p = {}
    for k in ("g", "h", "k", "dt"):
        p[k] = raw[k].astype(dt)
    p["dt2"] = p["dt"] * p["dt"]
    p["hdt2"] = dt(0.5) * p["dt2"]
    for k in PARAMS:
        if k in rd and shared.get(k):
            p[k] = p[k][:1]                                  # one value for the bank
    n = _counters(c, N, T, rng) if c.fam == LSQ else None
    return X, zs, {k: p[k] for k in rd}, shared, n


def _full(p, N):
    return {k: np.broadcast_to(v, (N,)) for k, v in p.items()}


def oracle(c, X, zs, p, n):
    N = X.shape[0]
    with np.errstate(all="ignore"):
        return po.bank(c.fam, c.order, c.mode == BATCH, X, zs, _full(p, N), n, c.dt)


# ------------------------------------------------------------------------------------------ one call
def _args(c, N, T):
    from filterpy_b200 import _lib
    a = _lib.PolyArgs()
    a.n_filters, a.n_steps, a.family, a.order, a.mode = N, T, c.fam, c.order, c.mode
    a.dtype = _lib.BKE_F32 if c.dt == F32 else _lib.BKE_F64
    return a


def run(c, N, T, seed=0, outs=None, shared_mask=None, unread="null", zs=None, n_max=None, n=None):
    """One call of case c: (rc, error text, got, inputs).  outs: the optional outputs passed (default: all the family
    and mode have); unread: "null" or "nan" for the parameters the instance does not read."""
    X, zs0, p, shared, n0 = _inputs(c, N, T, seed, shared_mask)
    zs = zs0 if zs is None else zs
    n0 = n0 if n is None else n
    outs = outputs(c.fam, c.mode) if outs is None else outs
    bf = Bufs(c.dt)
    a = _args(c, N, T)
    st = {}
    if c.fam in (GH, GHK):
        st["x"], st["dx"] = bf.put(X[:, 0], out=True), bf.put(X[:, 1], out=True)
        a.x, a.dx = ptr(st["x"]), ptr(st["dx"])
        if c.fam == GHK:                                    # GHK batch does not read ddx: NULL, or a buffer it keeps
            if c.mode == UPDATE or unread == "nan":
                st["ddx"] = bf.put(X[:, 2], out=True)
                a.ddx = ptr(st["ddx"])
    else:
        st["x"] = bf.put(X, out=True)
        a.x = ptr(st["x"])
    for k in PARAMS:
        if k in p:
            setattr(a, k, ptr(bf.put(p[k])))
            setattr(a, k + "_stride", 0 if p[k].shape[0] == 1 and shared[k] else 1)
        elif unread == "nan":
            setattr(a, k, ptr(bf.put(np.full(N, np.nan))))
            setattr(a, k + "_stride", 1)
    if c.fam == LSQ:
        st["n"] = bf.put(n0, out=True, dtype=np.int64)
        a.n = ptr(st["n"])
        a.n_max = int(n0.max()) if n_max is None else n_max
    a.z = ptr(bf.put(zs))
    W = 2 if c.fam in (GH, GHK) else c.order + 1
    shp = dict(results=(T + 1, N, W), predictions=(T, N), y=(N,), x_prediction=(N,), dx_prediction=(N,),
               ddx_prediction=(N,), K=(N, c.order + 1))
    ov = {}
    for k in outs:
        ov[k] = bf.out(shp[k])
        setattr(a, k, ptr(ov[k]))
    rc, err = call("bke_poly_filter", ctypes.byref(a))
    bf.check_guards()
    got = {k: v.cpu().numpy().reshape(shp[k]) for k, v in ov.items()}
    for k, v in st.items():
        got["state_" + k] = v.cpu().numpy()
    return rc, err, got, (X, zs, p, n0)


def same(got, want, what):
    """Bit for bit, with NaN wherever the oracle has NaN (any payload)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    nan = np.isnan(want) if want.dtype.kind == "f" else np.zeros(want.shape, bool)
    assert np.array_equal(np.isnan(got) if got.dtype.kind == "f" else nan, nan), what + ": the NaN pattern differs"
    bad = (got != want) | (np.signbit(got) != np.signbit(want)) if want.dtype.kind == "f" else got != want
    bad &= ~nan
    assert not bad.any(), "%s: %d entries differ, first at %s: %r != %r" % (
        what, bad.sum(), np.argwhere(bad)[0], got[tuple(np.argwhere(bad)[0])], want[tuple(np.argwhere(bad)[0])])


def check(c, N, T, seed=0, outs=None, shared_mask=None, unread="null", zs=None):
    rc, err, got, (X, zs, p, n0) = run(c, N, T, seed, outs, shared_mask, unread, zs)
    assert rc == 0, err
    what = "%s N=%d T=%d seed=%d" % (c.id, N, T, seed)
    o = oracle(c, X, zs, p, n0)
    for k in (outs if outs is not None else outputs(c.fam, c.mode)):
        same(got[k], o[k], what + " " + k)
    # the state: written back by UPDATE, untouched by BATCH
    Xw = o["X"] if c.mode == UPDATE else X
    if c.fam in (GH, GHK):
        same(got["state_x"], Xw[:, 0], what + " x")
        same(got["state_dx"], Xw[:, 1], what + " dx")
        if "state_ddx" in got:
            same(got["state_ddx"], Xw[:, 2], what + " ddx")
    else:
        same(got["state_x"].reshape(X.shape), Xw, what + " x")
    if c.fam == LSQ:
        same(got["state_n"], o["n"] if c.mode == UPDATE else n0, what + " n")
        if c.mode == UPDATE:
            assert np.array_equal(o["n"], n0 + T)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_instance_vs_oracle(case):
    """Every output and the state against the oracle, bit for bit, over N x T; each optional output alone and none;
    unread parameters NULL and NaN; every parameter shared and every one per filter."""
    c = case
    i = 0
    for N in NS:
        for T in TS:
            check(c, N, T, seed=1000 * N + T, unread=("null", "nan")[i % 2])
            i += 1
    rd = reads(c.fam, c.order, c.mode)
    for mask in ({k: True for k in rd}, {k: False for k in rd}):
        check(c, 257, 64, seed=5, shared_mask=mask)
    for o in outputs(c.fam, c.mode):
        check(c, 257, 64, seed=6, outs=(o,))
    check(c, 257, 64, seed=7, outs=())


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_nan_and_inf_z_inside_a_healthy_block(case):
    """A NaN and an inf z in single filters follow the oracle entry by entry; every other filter equals a clean run
    bit for bit."""
    c = case
    N, T = 300, 16
    X, zs, p, shared, n0 = _inputs(c, N, T, 11)
    clean = check(c, N, T, seed=11)
    zb = zs.copy()
    zb[3, 100] = np.nan
    zb[5, 200] = np.inf
    zb[0, 201] = -np.inf
    got = check(c, N, T, seed=11, zs=zb)
    ok = np.ones(N, bool)
    ok[[100, 200, 201]] = False
    for k, v in clean.items():
        same(_by_filter(k, got[k], N)[ok], _by_filter(k, v, N)[ok], c.id + " " + k + " of a healthy filter")
    assert np.isnan(got["results"][4, 100]).all() and not np.isnan(got["results"][3, 100]).any()


def _by_filter(k, a, N):
    """An output with the filter axis first."""
    if k == "results":
        return np.moveaxis(a, 1, 0)
    if k == "predictions":
        return a.T
    return a.reshape(N, -1)


# ------------------------------------------------------------------------------------------ the LSQ counter bound
def lsq_top(order):
    """The largest counter whose products (n; n(n+1); n(n+1)(n+2) and 3 n^2 at order 2) fit int64."""
    if order == 0:
        return INT64_MAX
    lo, hi = 1, 2**32 if order == 1 else 2**22
    ok = (lambda t: t * (t + 1) <= INT64_MAX) if order == 1 else \
        (lambda t: t * (t + 1) * (t + 2) <= INT64_MAX and 3 * t * t <= INT64_MAX)
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if ok(mid) else (lo, mid - 1)
    return lo


LSQ_T = 2


@pytest.mark.parametrize("dt", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("order", [0, 1, 2])
def test_lsq_counter_bound_refused(order, dt):
    """n_max one past the last accepted value returns BKE_ERR_BAD_ARG before any device is touched, with every buffer
    as it was (host buffers: the refusal needs no GPU)."""
    from filterpy_b200 import _lib
    N, T = 4, LSQ_T
    top = lsq_top(order)
    bufs = dict(x=np.arange(N * (order + 1), dtype=dt), z=np.ones(T * N, dt), p=np.full(N, 0.5, dt),
                n=np.full(N, 3, np.int64), r=np.full((T + 1) * N * 3, 7, dt), K=np.full(N * 3, 7, dt))
    before = {k: v.copy() for k, v in bufs.items()}
    a = _args(Case(dt, LSQ, order, UPDATE), N, T)
    a.x, a.z, a.n = bufs["x"].ctypes.data, bufs["z"].ctypes.data, bufs["n"].ctypes.data
    a.dt = a.dt2 = a.hdt2 = bufs["p"].ctypes.data
    a.results, a.K = bufs["r"].ctypes.data, bufs["K"].ctypes.data
    a.n_max = top - T + 1
    lib = _lib.load()
    assert lib.bke_poly_filter(ctypes.byref(a), None) == _lib.BKE_ERR_BAD_ARG
    assert "overflows int64" in lib.bke_last_error().decode()
    for k in bufs:
        assert np.array_equal(bufs[k], before[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("dt", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("order", [0, 1, 2])
def test_lsq_counter_bound(order, dt):
    """Counters up to the last accepted n_max run bit for bit; one more is refused with every device buffer
    untouched."""
    from filterpy_b200 import _lib
    top = lsq_top(order)
    for mode in (UPDATE, BATCH):
        c = Case(dt, LSQ, order, mode)
        N, T = 257, LSQ_T
        X, zs, p, shared, n = _inputs(c, N, T, 21)
        n[::3] = top - T
        n[1::7] = top - T - 5
        rc, err, got, _ = run(c, N, T, seed=21, n=n, n_max=top - T)
        assert rc == 0, err
        o = oracle(c, X, zs, p, n)
        for k in outputs(c.fam, c.mode):
            same(got[k], o[k], "%s n_max=top %s" % (c.id, k))
        same(got["state_n"], o["n"] if mode == UPDATE else n, c.id + " n")
        same(got["state_x"].reshape(X.shape), o["X"] if mode == UPDATE else X, c.id + " x")
        rc, err, got, _ = run(c, N, T, seed=21, n=n, n_max=top - T + 1)
        assert rc == _lib.BKE_ERR_BAD_ARG and "overflows int64" in err, (rc, err)
        same(got["state_n"], n, c.id + " n of a refused call")
        same(got["state_x"].reshape(X.shape), X, c.id + " x of a refused call")
        for k in outputs(c.fam, c.mode):
            assert np.all(got[k] == Bufs.SENT), c.id + " %s written by a refused call" % k


# ------------------------------------------------------------------------------------------ the oracle twin (CPU)
def _golden_params(c):
    k = po.consts(c)
    fam = {"gh": GH, "ghk": GHK, "gho": GHO, "lsq": LSQ, "fm": FM}[str(c["family"])]
    if fam == FM:
        p = dict(g=k["G"], h=k.get("H_dt"), k=k.get("K2_dt2"), dt=c["dt"], dt2=k["dt2"])
    else:
        p = dict(g=c["g"], h=c["h"], k=c["k"], dt=c["dt"], dt2=k["dt2"], hdt2=k.get("hdt2"))
    return fam, p, k


def test_twin_reproduces_the_oracle_in_fp64(golden):
    """po.bank at float64 gives run()'s outputs on every golden case: the update and, for GH / GHK, batch_filter."""
    from test_oracle_poly import CASES as GOLDEN
    for name in GOLDEN:
        c = golden(name)
        fam, p, k = _golden_params(c)
        order = int(c["order"])
        N = c["x0"].shape[0]
        n = np.zeros(N, np.int64)
        want = po.run(c)
        o = po.bank(fam, order, False, c["x0"], c["zs"], p, n)
        snap, ep = c["snap"], c["snap"][1:] - 1
        W = o["results"].shape[2]
        assert np.array_equal(o["results"][snap], want["upd_state"][..., :W]), name
        last = c["zs"].shape[0]
        if snap[-1] == last:
            assert np.array_equal(o["X"], want["upd_state"][-1]), name
            for key, out in (("upd_y", "y"), ("upd_xp", "x_prediction"), ("upd_dxp", "dx_prediction"),
                             ("upd_ddxp", "ddx_prediction"), ("upd_K", "K")):
                if key in want:
                    assert np.array_equal(o[out], want[key][-1]), (name, key)
        if fam in (GH, GHK):
            ob = po.bank(fam, order, True, c["x0"], c["zs"], dict(p, h=k["h_dt"]))
            assert np.array_equal(ob["results"][snap], want["bat_res"]), name
            assert np.array_equal(ob["predictions"][ep], want["bat_pred"]), name


class _Probe(np.ndarray):
    """An array that records the dtype of every ufunc result computed from it."""
    seen = []

    def __array_ufunc__(self, ufunc, method, *inputs, **kw):
        args = [np.asarray(v) if isinstance(v, _Probe) else v for v in inputs]
        if "out" in kw:
            kw["out"] = tuple(np.asarray(v) if isinstance(v, _Probe) else v for v in kw["out"])
        r = getattr(ufunc, method)(*args, **kw)
        _Probe.seen.append((ufunc.__name__, np.result_type(r)))
        return r.view(_Probe) if isinstance(r, np.ndarray) else r


@pytest.mark.parametrize("case", [c for c in CASES if c.dt == F32], ids=[c.id for c in CASES if c.dt == F32])
def test_twin_computes_every_intermediate_in_fp32(case):
    """Every floating-point operation the fp32 twin performs yields float32 (no promotion through a Python float, a
    float64 constant or an int64 product converted to double)."""
    c = case
    X, zs, p, shared, n = _inputs(c, 37, 3, 4)
    _Probe.seen = []
    pr = lambda a: a.view(_Probe)
    o = po.bank(c.fam, c.order, c.mode == BATCH, pr(X), pr(zs), {k: pr(np.broadcast_to(v, (37,)).copy())
                                                                  for k, v in p.items()},
                None if n is None else pr(n), F32)
    kinds = {dt for _, dt in _Probe.seen}
    assert _Probe.seen and kinds <= {np.dtype(F32), np.dtype(np.int64)}, kinds
    assert np.dtype(F32) in kinds
    for k, v in o.items():
        assert np.asarray(v).dtype in (np.dtype(F32), np.dtype(np.int64)), k


def _gains_through_double(order, n, dt, dt2):
    """The LSQ gains with every int64 product converted to double and then to float: the detour the kernel must not
    take."""
    f = lambda v: v.astype(F64).astype(F32)
    if order == 0:
        return [F32(1) / f(n)]
    if order == 1:
        return [F32(2) * f(2 * n - 1) / f(n * (n + 1)), F32(6) / (f(n * (n + 1)) * dt)]
    den = f(n * (n + 1) * (n + 2))
    return [F32(3) * f(3 * n**2 - 3 * n + 2) / den, F32(18) * f(2 * n - 1) / (den * dt), F32(60) / (den * dt2)]


@pytest.mark.parametrize("order", [0, 1])
def test_fp32_lsq_data_tells_the_double_rounding_apart(order):
    """The fp32 LSQ cases hold counters whose gains differ between the direct conversion (the kernel's and the
    twin's) and the detour through double, so a kernel that took the detour fails them."""
    c = Case(F32, LSQ, order, UPDATE)
    for N, T in ((257, 64), (100003, 1)):
        X, zs, p, shared, n = _inputs(c, N, T, 1000 * N + T)
        dt = np.broadcast_to(p["dt"], (N,)) if "dt" in p else None
        o = po.bank(LSQ, order, False, X, zs[:1], _full(p, N), n, F32)
        via = _gains_through_double(order, n + 1, dt, None)
        assert any(not np.array_equal(o["K"][:, j], via[j]) for j in range(order + 1)), (N, T)


# ------------------------------------------------------------------------------------------ which kernel runs
def _profiled_names():
    def go():
        for c in CASES:
            run(c, 257, 2, seed=1)
    return profiled_names(go, r"poly_kernel")


@pytest.mark.gpu
def test_dispatch_runs_the_kernels_of_the_table():
    """Each CASES entry, run once, launches the kernel the table names, template arguments included."""
    check_launch_order("test_gpu_poly_instances", [(c.id, c.kernels) for c in CASES])
