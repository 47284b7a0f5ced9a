"""Every kernel instance behind bke_fls_smooth against the fp64 oracle (oracle/fls.fls_bank), through the C-ABI, with
a table that names the kernels each case launches.

bke_fls_smooth (csrc/fls.cu) runs fls_fused_kernel<T, N, M> for the shapes of fused_shape() (1/1, 2/1, 4/2 in fp32 and
fp64, no control input, lag <= BKE_FLS_FUSED_MAX_LAG): one thread per filter, the T-epoch loop and the lag window in
the kernel, the window in dynamic shared memory (above 48 KB for 4/2 fp64 at lag >= 13).  Every other call runs the
per-epoch path: each epoch, the step kernel launch_kf_any (bke_kf_step's dispatch) picks for the shape, then
fls_correct_kernel<T> on the history rows in HBM.  CASES names each fused instance and each per-epoch route the
tests run, and the per-epoch calls refused for their workspace.

Inputs are rounded to the kernel's dtype before the oracle sees them.  Every output starts as NaN (history rows the
call may write, xhat, x_out, P_out, y, S; the workspace as NaN bytes), so a row the kernel never writes shows up.
Each error is taken relative to the filter's own scale of that quantity (the state's for the history, xhat and x_out)
and divided by the largest cond(S) the filter met.  Worst cases measured on an H100 80GB HBM3 (700 W power limit)
with BKE_TEST_ERRLOG over every configuration, output and bank size, and the bound set from each:

    family                                 fp64 worst  bound     fp32 worst  bound
    fused  fls_fused_kernel                  7.6e-15    3e-14     4.2e-6      1.7e-5
    epoch  step kernel + fls_correct_kernel  6.1e-15    2.5e-14   2.0e-6      8e-6
"""
import ctypes
import os
import re

import numpy as np
import pytest

from gpu_harness import (F32, F64, ROOT, TNAME, Bufs, body, call, check_launch_order, close, k_direct, k_fast, k_gen,
                         k_rb, mag, profiled_names, ptr, rb_fpw, rd, spd, src, stable_F)

MAX_LAG = 16                                     # BKE_FLS_FUSED_MAX_LAG
THREADS = 128                                    # fls.cu FLS_THREADS

TOL = {
    "fused": {F64: 3e-14, F32: 1.7e-5},
    "epoch": {F64: 2.5e-14, F32: 8e-6},
}


def _bound(c):
    """Case c's tolerance and the label of its BKE_TEST_ERRLOG lines."""
    return TOL[c.family][c.dt], "test_gpu_fls_instances %s %s" % (c.family, np.dtype(c.dt).name)


FUSED = [(1, 1), (2, 1), (4, 2)]
ERR_WS = ("bke_fls_smooth: this call runs the per-epoch path and needs a workspace of %d bytes "
          "(bke_fls_workspace_bytes), got %d")
ERR_WS_ALIGN = "bke_fls_smooth: workspace must be 16-byte aligned"


def k_fused(dt, n, m):
    return "fls_fused_kernel<%s, %d, %d>" % (TNAME[dt], n, m)


def k_corr(dt):
    return "fls_correct_kernel<%s>" % TNAME[dt]


def smem_bytes(dt, n, lag):
    """launch_fused: the lag window of one block."""
    return lag * n * THREADS * np.dtype(dt).itemsize


def ws_bytes(Nf, n, m, dt):
    """fls.cu WsLayout: x_pre, K, y, SI, v, vn, w (dtype) and the epoch's status (int32), each rounded up to 16 B."""
    es = np.dtype(dt).itemsize
    a16 = lambda b: (b + 15) & ~15
    return sum(a16(Nf * k * es) for k in (n, n * m, m, m * m, n, n, m)) + a16(Nf * 4)


# ------------------------------------------------------------------------------------------ the instance table
class Cfg:
    """One call of a case: N filters, T epochs, lag, count (epochs already taken, with a seeded history), the
    models shared (stride 0) or per filter, and xhat / y / S passed or NULL."""

    def __init__(self, N, T, lag, count=0, shared=False, null=False):
        self.N, self.T, self.lag, self.count, self.shared, self.null = N, T, lag, count, shared, null

    def __repr__(self):
        return "N=%d T=%d lag=%d count=%d%s%s" % (self.N, self.T, self.lag, self.count, " shared" if self.shared else "",
                                                  " null" if self.null else "")


class Case:
    """One fused instance ("fused") or per-epoch route ("epoch"), or a refused per-epoch call ("refused", with ws:
    "null", "short", "mis").  kernels: the launches of the profiled call (cfgs[0]); per epoch on the per-epoch path."""

    def __init__(self, kind, dt, n, m, kernels, cfgs, ctrl=False, ws=None):
        self.kind, self.dt, self.n, self.m, self.kernels, self.cfgs = kind, dt, n, m, list(kernels), list(cfgs)
        self.ctrl, self.ws = ctrl, ws

    @property
    def family(self):
        return "fused" if self.kind == "fused" else "epoch"

    @property
    def id(self):
        s = "%s-%s-%d_%d" % (self.kind, "f32" if self.dt == F32 else "f64", self.n, self.m)
        s += "-ctrl" if self.ctrl else ""
        s += "-" + self.ws if self.ws else ""
        return s + "-lag%d" % self.cfgs[0].lag

    def launches(self):
        c = self.cfgs[0]
        return self.kernels * (c.T if self.kind == "epoch" else 1)


def _fused_cfgs(dt, n):
    out = [Cfg(127, 20, 16, null=True), Cfg(129, 3, 0), Cfg(127, 1, 1, shared=True, null=True), Cfg(129, 5, 2),
           Cfg(1037, 8, 15), Cfg(129, 16, 16, shared=True), Cfg(1, 4, 16),
           Cfg(129, 9, 16, count=10),                                   # count < lag < count + T
           Cfg(1037, 3, 16, count=20, shared=True),                     # count >= lag
           Cfg(127, 2, 15, count=4, null=True)]                         # count + T < lag
    if dt == F64 and n == 4:
        out += [Cfg(129, 14, 13), Cfg(127, 6, 14, count=9, shared=True)]
    return out


def _epoch_cfgs(lag):
    return [Cfg(129, 3, lag), Cfg(1, 2, lag, shared=True, null=True), Cfg(127, lag + 3, lag),
            Cfg(1037, 4, lag, count=lag + 2, shared=True), Cfg(129, 5, lag, count=lag - 2, null=True)]


def _cases():
    out = []
    for dt in (F64, F32):
        for n, m in FUSED:
            out.append(Case("fused", dt, n, m, [k_fused(dt, n, m)], _fused_cfgs(dt, n)))
    L = MAX_LAG + 1
    for dt in (F64, F32):
        f9 = 3 * rb_fpw(dt, 9, 3, 3)
        epoch = [
            (3, 2, True, 3, [k_gen(dt)], 129),
            (4, 2, True, 4, [k_gen(dt)], 129),
            (6, 3, False, 2, [k_direct(dt, 6, 3, True)] if dt == F32 else [k_rb(dt, 6, 3, 3, True, 3, False)],
             129 if dt == F32 else 3 * rb_fpw(dt, 6, 3, 3)),
            (9, 3, False, 5, [k_rb(dt, 9, 3, 3, True, 3, False)], f9),
            (1, 1, False, L, [k_direct(dt, 1, 1, True)], 129),
            (2, 1, False, L, [k_direct(dt, 2, 1, True)], 129),
            # (the TMA kernel takes an epoch only where its slice of zs is 16-byte aligned: N = 128 keeps every one)
            (4, 2, False, L, [k_fast(3, 0, True)] if dt == F32 else [k_direct(dt, 4, 2, True)], 128),
        ]
        for n, m, ctrl, lag, ks, Np in epoch:
            cfgs = _epoch_cfgs(lag)
            cfgs[0] = Cfg(Np, 3, lag)
            out.append(Case("epoch", dt, n, m, ks + [k_corr(dt)], cfgs, ctrl=ctrl))
    # shared models on a row-block route
    out.append(Case("epoch", F64, 9, 3, [k_rb(F64, 9, 3, 3, True, 3, True), k_corr(F64)],
                    [Cfg(3 * rb_fpw(F64, 9, 3, 3), 2, 3, shared=True)]))
    for ws in ("null", "short", "mis"):
        out.append(Case("refused", F32, 6, 3, [], [Cfg(33, 2, 3)], ws=ws))
    return out


CASES = _cases()
RUNS = [c for c in CASES if c.kind != "refused"]


# ------------------------------------------------------------------------------------------ the table vs the source
def _dispatched():
    text = src("fls.cu")
    fs = body(text, "bool fused_shape(int n, int m, int du_used, int dtype, int64_t lag)")
    assert "du_used == 0 && lag <= BKE_FLS_FUSED_MAX_LAG" in fs
    shapes = [(int(a), int(b)) for a, b in re.findall(r"\(n == (\d+) && m == (\d+)\)", fs)]
    lf = body(text, "int launch_fls(const bke_fls_args &a, cudaStream_t s)")
    inst = set()
    for t, n, m in re.findall(r"launch_fused<(\w+), (\d+), (\d+)>\(a, s\)", lf):
        inst.add("fls_fused_kernel<%s, %s, %s>" % (t, n, m))
    assert "launch_per_epoch<float>(a, s) : launch_per_epoch<double>(a, s)" in lf
    assert "fls_correct_kernel<T><<<" in body(text, "int launch_per_epoch(const bke_fls_args &a, cudaStream_t s)")
    assert "int rc = launch_kf_any(k, s);" in text
    assert re.search(r"constexpr int FLS_THREADS = %d;" % THREADS, text)
    assert "const size_t smem = (size_t)a.lag * N * FLS_THREADS * sizeof(T);" in text
    assert ERR_WS.replace("%d", "%zu") in lf.replace('"\n                  "', "") and ERR_WS_ALIGN in lf
    with open(os.path.join(ROOT, "include", "bke.h")) as fh:
        assert re.search(r"#define BKE_FLS_FUSED_MAX_LAG %d\b" % MAX_LAG, fh.read())
    return shapes, inst


def test_instance_table_matches_dispatch():
    """CASES runs every fls_fused_kernel instance launch_fls can launch, at lags 0, 1, 2, 15 and 16 (and 13-16 for the
    4/2 fp64 window above 48 KB), and the per-epoch routes at the first lag past the cap: a new fused shape or a
    changed cap in the source fails here, on a machine without a GPU too."""
    shapes, inst = _dispatched()
    assert shapes == FUSED
    fused = [c for c in CASES if c.kind == "fused"]
    assert {k for c in fused for k in c.kernels} == inst == {k_fused(dt, n, m) for dt in (F32, F64) for n, m in FUSED}
    for c in fused:
        lags = {g.lag for g in c.cfgs}
        assert {0, 1, 2, 15, MAX_LAG} <= lags
        if smem_bytes(c.dt, c.n, MAX_LAG) > 48 * 1024:
            assert {l for l in lags if smem_bytes(c.dt, c.n, l) > 48 * 1024} >= {13, 14, 15, 16}
        assert {1, 127, 129, 1037} <= {g.N for g in c.cfgs}
        assert any(g.T < g.lag for g in c.cfgs) and any(g.T == g.lag for g in c.cfgs) and any(g.T > g.lag for g in c.cfgs)
        assert any(0 < g.count < g.lag < g.count + g.T for g in c.cfgs) and any(g.count >= g.lag > 0 for g in c.cfgs)
        assert any(g.shared for g in c.cfgs) and any(not g.shared for g in c.cfgs)
        assert any(g.null for g in c.cfgs) and any(not g.null for g in c.cfgs)
    assert [c.dt for c in fused if smem_bytes(c.dt, c.n, MAX_LAG) > 48 * 1024] == [F64]
    epoch = {(c.dt, c.n, c.m, c.ctrl, c.cfgs[0].lag > MAX_LAG) for c in CASES if c.kind == "epoch"}
    for dt in (F32, F64):
        assert {(dt, 3, 2, True, False), (dt, 4, 2, True, False), (dt, 6, 3, False, False), (dt, 9, 3, False, False),
                (dt, 1, 1, False, True), (dt, 2, 1, False, True), (dt, 4, 2, False, True)} <= epoch
    assert {c.ws for c in CASES if c.kind == "refused"} == {"null", "short", "mis"}


def test_workspace_bytes_across_the_fused_boundary():
    """bke_fls_workspace_bytes is 0 for the fused calls (up to the cap, without a control input) and the per-epoch
    layout's size past the cap, with a control input, or for any other shape."""
    from filterpy_b200 import _lib
    lib = _lib.load()
    for dt, code in ((F32, _lib.BKE_F32), (F64, _lib.BKE_F64)):
        for Nf in (1, 127, 1037):
            for n, m in FUSED:
                for lag in (0, 1, MAX_LAG):
                    assert lib.bke_fls_workspace_bytes(Nf, n, m, 0, code, lag) == 0
                assert lib.bke_fls_workspace_bytes(Nf, n, m, 0, code, MAX_LAG + 1) == ws_bytes(Nf, n, m, dt)
                assert lib.bke_fls_workspace_bytes(Nf, n, m, 1, code, 2) == ws_bytes(Nf, n, m, dt)
            for n, m in ((3, 1), (2, 2), (6, 3), (9, 3)):
                assert lib.bke_fls_workspace_bytes(Nf, n, m, 0, code, 2) == ws_bytes(Nf, n, m, dt)


# ------------------------------------------------------------------------------------------ inputs
def fls_inputs(c, g, seed):
    rng = np.random.default_rng(seed)
    n, m, N, T, dt = c.n, c.m, g.N, g.T, c.dt
    cnt = () if g.shared else (N,)
    d = dict(x=rng.normal(size=(N, n)) * 3, P=spd(rng, (N,), n, 2.0),
             F=stable_F(rng, cnt, n), Q=spd(rng, cnt, n, 0.05),
             H=rng.normal(size=cnt + (m, n)), R=spd(rng, cnt, m, 0.5), zs=rng.normal(size=(T, N, m)) * 3,
             hist=rng.normal(size=(g.count, N, n)) * 3)
    if c.ctrl:
        d["B"] = rng.normal(size=cnt + (n, 2))
        d["us"] = rng.normal(size=(T, N, 2))
    return {k: rd(v, dt) for k, v in d.items()}


def run_fls(c, g, d, ws=None):
    """One bke_fls_smooth call: (rc, error text, outputs host-side, Bufs)."""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    dt, n, m, N, T = c.dt, c.n, c.m, g.N, g.T
    bf = Bufs(dt)
    nan = float("nan")
    a = _lib.FlsArgs()
    k = a.step
    k.n_filters, k.dim_x, k.dim_z = N, n, m
    k.dtype = _lib.BKE_F32 if dt == F32 else _lib.BKE_F64
    k.x, k.P = ptr(bf.put(d["x"])), ptr(bf.put(d["P"]))
    xo, Po = bf.out((N, n), fill=nan), bf.out((N, n, n), fill=nan)
    k.x_out, k.P_out = ptr(xo), ptr(Po)
    for name in "FQHR":
        arr = d[name]
        setattr(k, name, ptr(bf.put(arr)))
        setattr(k, name + "_stride", 0 if arr.ndim == 2 else arr.shape[-1] * arr.shape[-2])
    if c.ctrl:
        k.dim_u = 2
        k.B = ptr(bf.put(d["B"])); k.B_stride = 0 if d["B"].ndim == 2 else 2 * n
        a.us = ptr(bf.put(d["us"]))
    outs = {}
    if not g.null:
        outs["y"], outs["S"] = bf.out((N, m), fill=nan), bf.out((N, m, m), fill=nan)
        k.y, k.S = ptr(outs["y"]), ptr(outs["S"])
        outs["xhat"] = bf.out((T, N, n), fill=nan)
        a.xhat = ptr(outs["xhat"])
    st = bf.out((N,), dtype=np.int32, fill=5)
    k.status = ptr(st)
    hist = np.concatenate([d["hist"], np.full((T, N, n), nan)])
    xs = bf.put(hist, out=True)
    a.xs_smooth = ptr(xs)
    a.n_steps, a.lag, a.count = T, g.lag, g.count
    a.zs = ptr(bf.put(d["zs"]))
    need = lib.bke_fls_workspace_bytes(N, n, m, 2 if c.ctrl else 0, k.dtype, g.lag)
    wsbuf = torch.full((need + 32,), 255, dtype=torch.uint8, device="cuda")
    base = wsbuf.data_ptr()
    if ws == "null":
        a.workspace, a.workspace_bytes = None, need
    elif ws == "short":
        a.workspace, a.workspace_bytes = base, need - 1
    elif ws == "mis":
        a.workspace, a.workspace_bytes = base + 4, need
    elif need:
        a.workspace, a.workspace_bytes = base, need
    rc, err = call("bke_fls_smooth", ctypes.byref(a))
    got = dict(x=xo.cpu().numpy().reshape(N, n), P=Po.cpu().numpy().reshape(N, n, n), status=st.cpu().numpy(),
               xs=xs.cpu().numpy().reshape(g.count + T, N, n))
    for name, shp in (("y", (N, m)), ("S", (N, m, m)), ("xhat", (T, N, n))):
        if name in outs:
            got[name] = outs[name].cpu().numpy().reshape(shp)
    return rc, err, got, bf, need


def fls_oracle(c, d, g):
    from oracle import fls as ofls
    return ofls.fls_bank(d["x"], d["P"], d["F"], d["H"], d["Q"], d["R"], d["zs"], g.lag, B=d.get("B"), us=d.get("us"),
                         count=g.count, hist=d["hist"] if g.count else None)


def check_fls(c, g, d, got, want, what):
    sw = lambda a: np.swapaxes(a, 0, 1)
    cond = want["cond"]
    tol, label = _bound(c)
    L0 = max(g.count - g.lag + 1, 0) if g.lag else g.count
    # the final rows before the live window are left as they were
    assert np.array_equal(got["xs"][:L0], d["hist"][:L0]), what + " a final history row changed"
    sx = mag(d["x"], sw(want["xs"]), sw(want["xhat"]), want["x"])
    close(sw(got["xs"]), sw(want["xs"]), sx, cond, tol, what + " xs", label)
    close(got["x"], want["x"], sx, cond, tol, what + " x_out", label)
    close(got["P"], want["P"], mag(d["P"], want["P"]), cond, tol, what + " P_out", label)
    assert np.array_equal(got["status"], want["status"]), what + " status"
    if g.null:
        return
    close(sw(got["xhat"]), sw(want["xhat"]), sx, cond, tol, what + " xhat", label)
    H = np.broadcast_to(d["H"], (g.N, c.m, c.n))
    sy = np.abs(d["zs"][-1]).max(axis=1) + np.abs(H).max(axis=(1, 2)) * np.abs(want["xs"][-1]).sum(axis=1) + \
        mag(want["y"])
    close(got["y"], want["y"], sy, cond, tol, what + " y", label)
    close(got["S"], want["S"], mag(want["S"]), cond, tol, what + " S", label)


@pytest.mark.gpu
@pytest.mark.parametrize("case", RUNS, ids=[c.id for c in RUNS])
def test_instance_vs_oracle(case):
    """Every history row, xhat, x_out, P_out, y, S and status against the fp64 oracle, over the case's lags, epoch
    counts, continuations, bank sizes and model layouts, with xhat, y and S passed and NULL."""
    for i, g in enumerate(case.cfgs):
        d = fls_inputs(case, g, seed=17 * i + g.N)
        rc, err, got, bf, _ = run_fls(case, g, d)
        assert rc == 0, err
        bf.check_guards()
        check_fls(case, g, d, got, fls_oracle(case, d, g), "%s %r" % (case.id, g))


@pytest.mark.gpu
@pytest.mark.parametrize("case", RUNS, ids=[c.id for c in RUNS])
def test_singular_S_in_one_filter(case):
    """H = 0 and R = 0 in one filter: its S is singular every epoch, its status is BKE_STATUS_SINGULAR_S, it keeps its
    prior, its rows are the priors, y = z and S = 0 at the last epoch; every other filter is bit-equal to a clean
    run."""
    lag = max(c.lag for c in case.cfgs)
    g = Cfg(129, lag + 3, lag, count=2)
    bad = 70
    clean = fls_inputs(case, g, seed=99)
    d = {k: v.copy() for k, v in clean.items()}
    d["H"][bad] = 0
    d["R"][bad] = 0
    rc, err, got, bf, _ = run_fls(case, g, d)
    assert rc == 0, err
    bf.check_guards()
    want = fls_oracle(case, d, g)
    assert want["status"][bad] == 1 and want["status"].sum() == 1
    check_fls(case, g, d, got, want, "%s %r singular" % (case.id, g))
    assert np.array_equal(got["y"][bad], d["zs"][-1][bad]) and np.all(got["S"][bad] == 0)
    rc, err, ref, _, _ = run_fls(case, g, clean)
    assert rc == 0, err
    others = np.arange(g.N) != bad
    for k, v in got.items():
        ax = 1 if k in ("xs", "xhat") else 0
        assert np.array_equal(np.compress(others, v, axis=ax), np.compress(others, ref[k], axis=ax)), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if c.kind == "refused"],
                         ids=[c.id for c in CASES if c.kind == "refused"])
def test_refused_workspace(case):
    """A per-epoch call with no workspace, one byte short of bke_fls_workspace_bytes, or one off a 16-byte boundary is
    BKE_ERR_BAD_ARG with its error text, and writes nothing."""
    from filterpy_b200 import _lib
    g = case.cfgs[0]
    d = fls_inputs(case, g, seed=1)
    rc, err, got, bf, need = run_fls(case, g, d, ws=case.ws)
    assert rc == _lib.BKE_ERR_BAD_ARG
    want = {"null": ERR_WS % (need, 0), "short": ERR_WS % (need, need - 1), "mis": ERR_WS_ALIGN}[case.ws]
    assert err == want, err
    bf.check_guards()
    for k in ("x", "P", "y", "S", "xhat"):
        assert np.all(np.isnan(got[k])), k
    assert np.all(np.isnan(got["xs"])) and np.all(got["status"] == 5)


# ------------------------------------------------------------------------------------------ which kernel runs
def _run_cases():
    for c in CASES:
        g = c.cfgs[0]
        run_fls(c, g, fls_inputs(c, g, seed=1), ws=c.ws)


def _profiled_names():
    return profiled_names(_run_cases, r"kf\w*_kernel|fls_\w+_kernel")


@pytest.mark.gpu
def test_dispatch_runs_the_kernels_of_the_table():
    """Each CASES entry, run once at its first configuration, launches the kernels the table names, in order: one
    fused kernel, or T x (the step kernel, fls_correct_kernel); a refused call launches nothing.  The profile is
    taken in a process of its own."""
    check_launch_order("test_gpu_fls_instances", [(c.id, c.launches()) for c in CASES])
