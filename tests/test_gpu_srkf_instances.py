"""Every kernel instance behind bke_srkf_step and bke_cholesky_lower against the fp64 oracle, through the C-ABI, with a
table that names the kernel each case launches.

bke_srkf_step (csrc/srkf.cu) runs the register tile srkf_reg_kernel<T, N, M, EX> (one thread per filter) for the shapes
of dispatch() without a control input, when every 16-byte row it loads or stores is aligned; every other call runs
srkf_warp_kernel<T> (one warp per filter, the matrices in the warp's slice of shared memory, 4, 2 or 1 warps per
block, refused above 200 KB per warp).  bke_cholesky_lower runs chol_lower_kernel<T, K> for K = 1 ..
BKE_CHOLESKY_MAX_DIM.  CASES reaches every one of these instances.

Inputs are rounded to the kernel's dtype before the oracle (oracle/srkf.srkf_step_bank, in fp64; scipy's cholesky) sees
them, so only the kernel's own arithmetic is measured.  L has dgeqr2's signs, so every filter's two QR inputs are
checked for a margin from a sign decision (oracle.srkf.dgeqr2_pivot_ratios) before the comparison.  Each error is taken
relative to the filter's own scale of that quantity (the state's for y) and divided by the condition number of what the
filter factors: the larger of its two stacked QR inputs [F L | Lq]' and [[Lr', 0], [(H L)', L']], or the Cholesky input.
Worst cases measured on an H100 80GB HBM3 (700 W power limit) with BKE_TEST_ERRLOG, as error / (scale * cond) over
every case, output and bank size of the family, and the bound set from each:

    family                            fp64 worst  bound     fp32 worst  bound
    reg   srkf_reg_kernel              1.1e-15    4e-15     3.4e-7      1.5e-6
    warp  srkf_warp_kernel             2.3e-16    1e-15     2.2e-7      1e-6
    chol  chol_lower_kernel            2.2e-16    1e-15     1.4e-7      6e-7
"""
import ctypes
import os
import re

import numpy as np
import pytest

from gpu_harness import (BUDGET, F32, F64, ROOT, TNAME, Bufs, b, body, call, check_launch_order, close, mag,
                         profiled_names, ptr, rd, src)

MARGIN = 1e-3                     # the smallest dgeqr2 pivot ratio a compared filter may have

TOL = {
    "reg": {F64: 4e-15, F32: 1.5e-6},
    "warp": {F64: 1e-15, F32: 1e-6},
    "chol": {F64: 1e-15, F32: 6e-7},
}


def _bound(c):
    """Case c's tolerance and the label of its BKE_TEST_ERRLOG lines."""
    return TOL[c.family][c.dt], "test_gpu_srkf_instances %s %s" % (c.family, np.dtype(c.dt).name)


# ------------------------------------------------------------------------------------------ kernel names

def k_reg(dt, n, m, ex):
    return "srkf_reg_kernel<%s, %d, %d, %s>" % (TNAME[dt], n, m, b(ex))


def k_warp(dt):
    return "srkf_warp_kernel<%s>" % TNAME[dt]


def k_chol(dt, k):
    return "chol_lower_kernel<%s, %d>" % (TNAME[dt], k)


# ------------------------------------------------------------------------------------------ the launch shape
def sr_per_warp(n, m):
    """srkf.cu launch_warp: the elements of one warp's slice (x, xp, y, L, T1, H, K, S, SI, W), rounded up to 4."""
    nn, nm, D = n * n, n * m, n + m
    pw = 2 * n + m + nn + max(nn, nm) + 2 * nm + 2 * m * m + max(2 * nn, D * D)
    return (pw + 3) & ~3


def warps_per_block(n, m, dt):
    """api.cu warp_shape: 4 warps per block, halved until the block's slices fit the budget; 0 = refused."""
    b = sr_per_warp(n, m) * np.dtype(dt).itemsize
    for w in (4, 2, 1):
        if b * w <= BUDGET:
            return w
    return 0


def warp_shapes(dt, m=3):
    """(first n with 2 warps per block, first n with 1, the largest accepted n, the first refused n) at dim_z = m."""
    n, out = 1, {}
    while True:
        w = warps_per_block(n, m, dt)
        out.setdefault(w, n)
        if w == 0:
            return out[2], out[1], n - 1, n
        n += 1


# the register shapes of dispatch(), and the arrays launch_reg checks for 16-byte rows (name, elements per filter)
REG = [(4, 2), (1, 1), (2, 2), (3, 1), (4, 1)]


def vec_operands(dt, n, m):
    """kf_rowio.cuh vec_ok: the arrays launch_reg loads or stores as 16-byte vectors (a row of whole vectors)."""
    v = 16 // np.dtype(dt).itemsize
    rows = [("x", n), ("L", n * n), ("F", n * n), ("Lq", n * n), ("H", m * n), ("Lr", m * m), ("z", m),
            ("x_out", n), ("L_out", n * n), ("x_prior", n), ("L_prior", n * n), ("K", n * m), ("y", m),
            ("S1_2", m * m), ("SI1_2", m * m)]
    return [k for k, c in rows if c % v == 0]


# ------------------------------------------------------------------------------------------ the instance table
class Case:
    """One call and the kernels it launches at N = Np.  family "reg" / "warp" (bke_srkf_step) or "chol"
    (bke_cholesky_lower).  models: "per" (stride = the matrix size) or "shared" (stride 0); mis: the array placed one
    element past a 16-byte boundary; inplace: x_out / L_out are x / L; ex: the optional outputs are passed; mode:
    BKE_DO_PREDICT | BKE_DO_UPDATE; ctrl: B u; refused: the call must return BKE_ERR_UNSUPPORTED (no kernel runs);
    grid: one more bank, large enough for the warp kernel's grid-stride loop.  Ns are the bank sizes of the oracle runs."""

    def __init__(self, family, dt, n, m, kernels, Np, Ns, models="per", mis=None, inplace=False, ex=True, mode=3,
                 ctrl=False, refused=False, grid=False):
        self.family, self.dt, self.n, self.m = family, dt, n, m
        self.kernels, self.Np, self.Ns = list(kernels), Np, tuple(Ns)
        self.models, self.mis, self.inplace, self.ex, self.mode = models, mis, inplace, ex, mode
        self.ctrl, self.refused, self.grid = ctrl, refused, grid

    @property
    def id(self):
        s = "%s-%s-%d_%d-%s" % (self.family, "f32" if self.dt == F32 else "f64", self.n, self.m, self.models)
        if self.family != "chol":
            s += "-mode%d" % self.mode + ("" if self.ex else "-noex")
        for flag, name in ((self.mis, "mis_%s" % self.mis), (self.inplace, "inplace"), (self.ctrl, "ctrl"),
                           (self.refused, "refused"), (self.grid, "grid")):
            if flag:
                s += "-" + name
        return s + "-N%d" % self.Np


OUT_SHAPES = lambda n, m: dict(x_prior=(n,), L_prior=(n, n), K=(n, m), y=(m,), S1_2=(m, m), SI1_2=(m, m))  # noqa: E731
TILE_NS = (1, 127, 129, 1037)
WARP_NS = (1, 5, 37)


def _cases():
    out = []
    for dt in (F64, F32):
        # the register tiles: every shape x EX x mode, models shared and per filter, in place
        for n, m in REG:
            for mode in (3, 1, 2):
                for ex in (True, False):
                    out.append(Case("reg", dt, n, m, [k_reg(dt, n, m, ex)], 129, TILE_NS,
                                    models=("per", "shared")[(mode + ex) % 2], ex=ex, mode=mode,
                                    inplace=(mode != 3 and ex) or (mode == 3 and not ex)))
            # one array one element off a 16-byte boundary: the warp kernel, where the tile loads it as vectors
            vec = vec_operands(dt, n, m)
            if vec:
                for i, k in enumerate(vec[::3] if len(vec) > 3 else vec):
                    out.append(Case("reg", dt, n, m, [k_warp(dt)], 33, (1, 33), mis=k,
                                    ex=(i % 2 == 0) or k in OUT_SHAPES(n, m)))
            else:                                   # nothing is loaded as vectors: the tile runs on any address
                out.append(Case("reg", dt, n, m, [k_reg(dt, n, m, True)], 129, (1, 129), mis="x"))
        # a control input: the warp kernel, also at the register shapes
        out.append(Case("warp", dt, 4, 2, [k_warp(dt)], 37, WARP_NS, ctrl=True))
        out.append(Case("warp", dt, 3, 2, [k_warp(dt)], 37, WARP_NS, ctrl=True, models="shared", ex=False))
        out.append(Case("warp", dt, 1, 1, [k_warp(dt)], 37, WARP_NS, ctrl=True, mode=1, inplace=True))
        # the warp kernel's shapes: 4 warps per block, n > 32, n + m > 32, 2 and 1 warps per block, the largest
        # accepted shape and the first refused one
        two, one, top, refused = warp_shapes(dt)
        out += [
            Case("warp", dt, 6, 3, [k_warp(dt)], 37, (1, 5, 37, 1037), grid=True),
            Case("warp", dt, 9, 3, [k_warp(dt)], 37, WARP_NS, models="shared", mode=2, inplace=True),
            Case("warp", dt, 5, 5, [k_warp(dt)], 37, WARP_NS, mode=1, ex=False),
            Case("warp", dt, 2, 3, [k_warp(dt)], 37, WARP_NS, ex=False),
            Case("warp", dt, 33, 2, [k_warp(dt)], 9, (1, 9)),
            Case("warp", dt, 20, 14, [k_warp(dt)], 9, (1, 9), models="shared"),
            Case("warp", dt, two, 3, [k_warp(dt)], 5, (1, 5), mode=2),
            Case("warp", dt, one, 3, [k_warp(dt)], 3, (1, 3), inplace=True),
            Case("warp", dt, top, 3, [k_warp(dt)], 3, (3,), models="shared"),
            Case("warp", dt, refused, 3, [], 3, (3,), refused=True),
        ]
    # the Cholesky factor: every K in both dtypes, models per filter and shared
    for dt in (F64, F32):
        for k in range(1, 17):
            out.append(Case("chol", dt, k, 0, [k_chol(dt, k)], 129, (1, 129, 1037)))
            out.append(Case("chol", dt, k, 0, [k_chol(dt, k)], 129, (129,), models="shared"))
    return out


CASES = _cases()


# ------------------------------------------------------------------------------------------ the table vs the source
def _dispatched():
    """Every kernel instance srkf.cu's dispatch() and launch_chol can launch, parsed from the source."""
    text = src("srkf.cu")
    d = body(text, "int dispatch(const bke_srkf_args &a, cudaStream_t s)")
    shapes = []
    for a, b, c, e in re.findall(r"n == (\d+) && m == (\d+)\) rc = launch_reg<T, (\d+), (\d+)>", d):
        assert (a, b) == (c, e)
        shapes.append((int(a), int(b)))
    assert "return rc == BKE_ERR_UNSUPPORTED ? launch_warp<T>(a, s) : rc;" in d
    assert "if (a.B == nullptr || a.u == nullptr) {" in d
    lr = body(text, "int launch_reg(const bke_srkf_args &a, cudaStream_t s)")
    assert set(re.findall(r"srkf_reg_kernel<T, N, M, (true|false)><<<", lr)) == {"true", "false"}
    inst = {k_reg(dt, n, m, ex) for dt in (F32, F64) for n, m in shapes for ex in (True, False)}
    inst |= {k_warp(dt) for dt in (F32, F64)}
    # launch_chol recurses from K = 1 (launch_cholesky_lower) up to BKE_CHOLESKY_MAX_DIM
    with open(os.path.join(ROOT, "include", "bke.h")) as fh:
        kmax = int(re.search(r"#define BKE_CHOLESKY_MAX_DIM (\d+)", fh.read()).group(1))
    lc = body(text, "int launch_chol(int64_t N, int32_t k, const void *A, int64_t stride, void *L, int32_t *status, "
                    "cudaStream_t s)")
    assert "if constexpr (K < BKE_CHOLESKY_MAX_DIM) return launch_chol<T, K + 1>" in lc
    assert "chol_lower_kernel<T, K><<<" in lc
    assert "launch_chol<float, 1>(" in text and "launch_chol<double, 1>(" in text
    inst |= {k_chol(dt, k) for dt in (F32, F64) for k in range(1, kmax + 1)}
    return inst, shapes, kmax


def test_instance_table_matches_dispatch():
    """CASES launches every instance srkf.cu's dispatch() and launch_chol can reach, and no other: a new register shape
    or Cholesky dimension without a case fails here, on a machine without a GPU too."""
    inst, shapes, kmax = _dispatched()
    assert shapes == REG
    table = {k for c in CASES for k in c.kernels}
    assert table == inst, (sorted(inst - table), sorted(table - inst))
    # every register shape x dtype x EX x mode, and its misaligned call
    got = {(c.dt, c.n, c.m, c.ex, c.mode) for c in CASES if c.family == "reg" and not c.mis}
    assert got == {(dt, n, m, ex, mode) for dt in (F32, F64) for n, m in REG for ex in (True, False) for mode in (1, 2, 3)}
    for dt in (F32, F64):
        for n, m in REG:
            mis = [c for c in CASES if c.family == "reg" and c.mis and (c.dt, c.n, c.m) == (dt, n, m)]
            assert mis and all(c.kernels == ([k_warp(dt)] if vec_operands(dt, n, m) else [k_reg(dt, n, m, True)])
                               for c in mis)
        w = [c for c in CASES if c.family == "warp" and c.dt == dt]
        wpb = {warps_per_block(c.n, c.m, dt) for c in w}
        assert wpb == {0, 1, 2, 4}
        assert any(c.n > 32 for c in w if not c.refused) and any(c.n <= 32 < c.n + c.m for c in w)
        assert any(c.grid for c in w) and any(c.ctrl for c in w)
        # the largest accepted shape and the first refused one
        top = max(c.n for c in w if not c.refused and c.m == 3)
        assert warps_per_block(top + 1, 3, dt) == 0 and any(c.refused and c.n == top + 1 for c in w)
        assert {c.models for c in CASES if c.family == "chol" and c.dt == dt} == {"per", "shared"}
    # the launch formula the warp shapes are chosen from is the launch's own
    lw = body(src("srkf.cu"), "int launch_warp(const bke_srkf_args &a, cudaStream_t s)")
    assert ("int per_warp = 2 * n + m + nn + (nn > nm ? nn : nm) + 2 * nm + 2 * m * m + (2 * nn > D * D ? 2 * nn : D * D);"
            in lw and "per_warp = (per_warp + 3) & ~3;" in lw and "budget = 200 * 1024" in lw)


def test_pivot_ratios_agree_with_the_bank_minimum():
    """dgeqr2_pivot_ratios is dgeqr2_pivot_ratio per matrix."""
    from oracle import srkf as osr
    A = np.random.default_rng(3).normal(size=(7, 9, 4))
    A[2, 5:, 1] = 0
    ra, rs = osr.dgeqr2_pivot_ratios(A)
    assert ra.shape == rs.shape == (7,)
    for i in range(7):
        assert osr.dgeqr2_pivot_ratio(A[i]) == (ra[i], rs[i])
    assert osr.dgeqr2_pivot_ratio(A) == (ra.min(), rs.min())


# ------------------------------------------------------------------------------------------ inputs
def _lower(rng, shape, k, diag, off):
    a = np.tril(off * rng.normal(size=shape + (k, k)), -1)
    return a + np.eye(k) * (diag[0] + diag[1] * rng.random(size=shape + (k,)))[..., None, :]


def _qr_inputs(d, predict):
    """The two stacked matrices a step factors, per filter: [F L | Lq]' (or None) and [[Lr', 0], [(H L)', L']]."""
    from oracle import srkf as osr
    x, L = d["x"], d["L"]
    N, n = x.shape
    T = lambda a: np.swapaxes(a, -1, -2)                                  # noqa: E731
    A = None
    if predict:
        A = np.concatenate([T(d["F"] @ L), np.broadcast_to(T(d["Lq"]), (N, n, n))], axis=-2)
        L = T(osr.dgeqr2(A)[..., :n, :n])
    m = d["H"].shape[-2]
    Mx = np.zeros((N, m + n, m + n))
    Mx[:, :m, :m] = T(np.broadcast_to(d["Lr"], (N, m, m)))
    Mx[:, m:, :m] = T(d["H"] @ L)
    Mx[:, m:, m:] = T(L)
    return A, Mx


def _margin_ok(d, predict):
    from oracle import srkf as osr
    ok = np.ones(d["x"].shape[0], bool)
    for A in _qr_inputs(d, predict):
        if A is not None:
            ra, rs = osr.dgeqr2_pivot_ratios(A)
            ok &= (ra >= MARGIN) & (rs >= MARGIN)
    return ok


def sr_inputs(c, N, seed):
    """The arrays of one bke_srkf_step call, rounded to the case's dtype: L and Lq, Lr lower triangular with a positive
    diagonal, F near I.  A filter whose QR inputs come near a sign decision is drawn again (a shared model: the bank)."""
    rng = np.random.default_rng(seed)
    n, m, dt = c.n, c.m, c.dt
    cnt = () if c.models == "shared" else (N,)
    s = 1 / np.sqrt(n)

    def draw(k):
        d = dict(x=rng.normal(size=(k, n)) * 3, L=_lower(rng, (k,), n, (1.0, 1.0), 0.5 * s), z=rng.normal(size=(k, m)) * 3)
        if c.ctrl:
            d["u"] = rng.normal(size=(k, 2))
        return d

    def models():
        return dict(F=np.eye(n) + 0.2 * s * rng.normal(size=cnt + (n, n)), Lq=_lower(rng, cnt, n, (0.2, 0.3), 0.05 * s),
                    H=rng.normal(size=cnt + (m, n)), Lr=_lower(rng, cnt, m, (0.5, 1.0), 0.2),
                    **({"B": rng.normal(size=cnt + (n, 2))} if c.ctrl else {}))

    d = dict(draw(N), **models())
    d = {k: rd(v, dt) for k, v in d.items()}
    for _ in range(50):
        bad = ~_margin_ok(d, bool(c.mode & 1))
        if not bad.any():
            break
        if c.models == "shared" and bad.all():
            d.update({k: rd(v, dt) for k, v in models().items()})
            continue
        new = {k: rd(v, dt) for k, v in draw(int(bad.sum())).items()}
        if c.models == "per":
            new.update({k: rd(v[:int(bad.sum())], dt) for k, v in models().items()})
        for k, v in new.items():
            d[k] = d[k].copy()
            d[k][bad] = v
    assert _margin_ok(d, bool(c.mode & 1)).all(), "no draw keeps every filter clear of a dgeqr2 sign decision"
    return d


def run_step(c, N, seed=0, sing=None, d=None):
    """One bke_srkf_step of case c on N filters: (rc, error text, got, d, valid).  sing: filters given H = 0 and
    Lr = 0 (S1_2 = 0)."""
    from filterpy_b200 import _lib
    dt, n, m = c.dt, c.n, c.m
    d = dict(sr_inputs(c, N, seed) if d is None else d)
    if sing is not None:
        d["H"], d["Lr"] = d["H"].copy(), d["Lr"].copy()
        d["H"][sing] = 0
        d["Lr"][sing] = 0
    rng = np.random.default_rng(seed + 1)
    valid = (rng.random(N) > 0.2) if c.mode & 2 else None
    if valid is not None and N > 1:
        valid[1] = False
        if sing is not None:
            valid[sing] = True
    bf = Bufs(dt)
    a = _lib.SrkfArgs()
    a.n_filters, a.dim_x, a.dim_z = N, n, m
    a.dtype = _lib.BKE_F32 if dt == F32 else _lib.BKE_F64
    a.flags = c.mode
    xv, Lv = bf.put(d["x"], c.mis == "x", out=c.inplace), bf.put(d["L"], c.mis == "L", out=c.inplace)
    a.x, a.L = ptr(xv), ptr(Lv)
    xo, Lo = (xv, Lv) if c.inplace else (bf.out((N, n), c.mis == "x_out"), bf.out((N, n, n), c.mis == "L_out"))
    a.x_out, a.L_out = ptr(xo), ptr(Lo)
    for k in ("F", "H", "Lq", "Lr"):
        arr = d[k]
        setattr(a, k, ptr(bf.put(arr, c.mis == k)))
        setattr(a, k + "_stride", 0 if arr.ndim == 2 else arr.shape[-1] * arr.shape[-2])
    if c.ctrl:
        a.dim_u = 2
        a.B = ptr(bf.put(d["B"])); a.B_stride = 0 if d["B"].ndim == 2 else 2 * n
        a.u = ptr(bf.put(d["u"])); a.u_stride = 2
    a.z = ptr(bf.put(d["z"], c.mis == "z"))
    if valid is not None:
        a.z_valid = ptr(bf.put(valid.astype(np.uint8), dtype=np.uint8))
    outs = {}
    if c.ex:
        for k, s in OUT_SHAPES(n, m).items():
            outs[k] = bf.out((N,) + s, c.mis == k)
            setattr(a, k, ptr(outs[k]))
    st = bf.out((N,), dtype=np.int32, fill=5)
    a.status = ptr(st)
    rc, err = call("bke_srkf_step", ctypes.byref(a))
    if rc:
        return rc, err, None, d, valid
    bf.check_guards()
    got = dict(x=xo.cpu().numpy().reshape(N, n), L=Lo.cpu().numpy().reshape(N, n, n), status=st.cpu().numpy())
    for k, v in outs.items():
        got[k] = v.cpu().numpy().reshape((N,) + OUT_SHAPES(n, m)[k])
    return rc, err, got, d, valid


def sr_oracle(c, d, valid):
    from oracle import srkf as osr
    o = osr.srkf_step_bank(d["x"], d["L"], d.get("z"), d["F"], d["H"], d["Lq"], d["Lr"], valid=valid,
                           predict=bool(c.mode & 1), update=bool(c.mode & 2), B=d.get("B"), u=d.get("u"))
    A, Mx = _qr_inputs(d, bool(c.mode & 1))
    cond = np.ones(d["x"].shape[0])
    if c.mode & 2:
        cond = np.linalg.cond(Mx)
        cond[~np.isfinite(cond)] = 1             # S1_2 = 0: no reflection, compared exactly
    if A is not None:
        cond = np.maximum(cond, np.linalg.cond(A))
    return o, cond


def check_step(c, N, seed, sing=None):
    rc, err, got, d, valid = run_step(c, N, seed, sing)
    assert rc == 0, err
    want, cond = sr_oracle(c, d, valid)
    what = "%s N=%d seed=%d%s" % (c.id, N, seed, "" if sing is None else " singular")
    tol, label = _bound(c)
    do_p, do_u = bool(c.mode & 1), bool(c.mode & 2)
    prior_x, prior_L = want.get("x_prior", d["x"]), want.get("L_prior", d["L"])
    sx, sL = mag(d["x"], prior_x, want["x"]), mag(d["L"], prior_L, want["L"])
    close(got["x"], want["x"], sx, cond, tol, what + " x", label)
    close(got["L"], want["L"], sL, cond, tol, what + " L", label)
    assert np.array_equal(got["status"], want["status"]), what + " status"
    assert np.all(np.triu(got["L"], 1) == 0), what + " L above its diagonal"
    if not c.ex:
        return got, want
    S = Bufs.SENT
    if do_p:
        close(got["x_prior"], want["x_prior"], sx, cond, tol, what + " x_prior", label)
        close(got["L_prior"], want["L_prior"], sL, cond, tol, what + " L_prior", label)
    else:
        assert np.all(got["x_prior"] == S) and np.all(got["L_prior"] == S), what + " prior written without a predict"
    keys = ("K", "y", "S1_2", "SI1_2")
    if not do_u:
        for k in keys:
            assert np.all(got[k] == S), what + " %s written without an update" % k
        return got, want
    upd = valid
    H = np.broadcast_to(d["H"], (N,) + d["H"].shape[-2:])
    sy = np.abs(H).max(axis=(1, 2)) * np.abs(prior_x).sum(axis=1) + np.abs(d["z"]).max(axis=1)
    close(got["y"], want["y"], sy, cond, tol, what + " y", label, upd)
    for k in ("K", "S1_2", "SI1_2"):
        close(got[k], want[k], mag(np.nan_to_num(want[k])), cond, tol, what + " " + k, label, upd)
    for k in keys:
        assert np.all(got[k][~upd] == S), what + " %s written for a missed measurement" % k
    bad = want["status"] != 0
    if bad.any():                                   # S1_2 = 0: K = SI1_2 = 0 and the prior kept, exactly
        assert np.all(got["K"][bad] == 0) and np.all(got["SI1_2"][bad] == 0), what + " K, SI1_2 of a singular S1_2"
        assert np.array_equal(got["x"][bad], got["x_prior"][bad] if do_p else d["x"][bad]), what + " singular x"
        assert np.array_equal(got["L"][bad], got["L_prior"][bad] if do_p else d["L"][bad]), what + " singular L"
    return got, want


def _tile(c):
    return 128 if c.kernels and c.kernels[0].startswith("srkf_reg") else max(warps_per_block(c.n, c.m, c.dt), 1)


def _grid_N(c):
    """One bank more than the warp kernel's grid (16 blocks per SM) covers in one pass."""
    import torch
    return 16 * torch.cuda.get_device_properties(0).multi_processor_count * warps_per_block(c.n, c.m, c.dt) + 37


STEP_CASES = [c for c in CASES if c.family != "chol"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEP_CASES, ids=[c.id for c in STEP_CASES])
def test_step_instance_vs_oracle(case):
    """bke_srkf_step: x, L, x_prior, L_prior, K, y, S1_2, SI1_2 and status against the fp64 dgeqr2 oracle entrywise,
    over the family's bank sizes, with a z_valid mask, guard elements around every output and outputs a masked filter
    must leave alone; a filter with S1_2 = 0 in every block gets status 1, K = SI1_2 = 0 and keeps its prior, and the
    others are bit-equal to a run without it; a refused shape returns BKE_ERR_UNSUPPORTED and says why."""
    from filterpy_b200 import _lib
    c = case
    if c.refused:
        rc, err, _, _, _ = run_step(c, c.Ns[0], seed=1)
        per = sr_per_warp(c.n, c.m) * np.dtype(c.dt).itemsize
        assert rc == _lib.BKE_ERR_UNSUPPORTED, rc
        assert err == ("bke_srkf_step: dim_x=%d dim_z=%d needs %d B of shared memory per filter (> %d)"
                       % (c.n, c.m, per, BUDGET)), err
        return
    Ns = c.Ns + ((_grid_N(c),) if c.grid else ())
    for i, N in enumerate(Ns):
        check_step(c, N, seed=N + 11 * i)
    if c.mode & 2 and c.models == "per":
        N = Ns[-1]
        t = _tile(c)
        f = np.arange(N)
        sing = f % t == (f // t * 5 + 2) % min(t, N)
        clean, _ = check_step(c, N, seed=21)
        got, _ = check_step(c, N, seed=21, sing=sing)
        for k in clean:
            assert np.array_equal(got[k][~sing], clean[k][~sing]), "%s: %s of a regular filter changed" % (c.id, k)
        assert np.all(got["status"][sing] == 1)


# ------------------------------------------------------------------------------------------ bke_cholesky_lower
def chol_inputs(c, N, seed):
    """SPD matrices (stride 0: one), rounded to the dtype; per filter, also: an indefinite one (a negative diagonal
    entry), a semidefinite one (a [[1, 1], [1, 1]] block or a zero row and column) and one with a NaN diagonal."""
    rng = np.random.default_rng(seed)
    k = c.n
    shape = () if c.models == "shared" else (N,)
    a = rng.normal(size=shape + (k, k))
    A = a @ np.swapaxes(a, -1, -2) / k + 0.5 * np.eye(k)
    A = rd(A, c.dt)
    if c.models == "per" and N >= 8:
        j = rng.integers(0, k, size=N)
        f = np.arange(3, N, 7)
        A[f, j[f], j[f]] *= -1                                  # indefinite
        for f in range(5, N, 11):                               # semidefinite, exactly
            i = j[f]
            b = slice(i, min(i + 2, k))
            A[f, b, :] = 0; A[f, :, b] = 0
            A[f, b, b] = 1 if i + 1 < k else 0
        f = np.arange(6, N, 13)
        A[f, j[f], j[f]] = np.nan
    return A


def chol_oracle(A):
    import scipy.linalg
    L = np.full(A.shape, np.nan)
    st = np.zeros(A.shape[0], np.int32)
    for f in range(A.shape[0]):
        try:
            L[f] = scipy.linalg.cholesky(A[f], lower=True)
        except (np.linalg.LinAlgError, ValueError):
            st[f] = 2
    return L, st


def run_chol(c, N, seed=0):
    dt, k = c.dt, c.n
    A = chol_inputs(c, N, seed)
    Ak = A.copy()
    iu = np.triu_indices(k, 1)
    Ak[..., iu[0], iu[1]] = np.nan                              # the upper triangle is not read
    bf = Bufs(dt)
    Av = bf.put(Ak)
    Lo = bf.out((N, k, k))
    st = bf.out((N,), dtype=np.int32, fill=5)
    rc, err = call("bke_cholesky_lower", ctypes.c_int64(N), ctypes.c_int32(k), ctypes.c_int32(0 if dt == F32 else 1),
                   ctypes.c_void_p(ptr(Av)), ctypes.c_int64(0 if c.models == "shared" else k * k),
                   ctypes.c_void_p(ptr(Lo)), ctypes.c_void_p(ptr(st)))
    assert rc == 0, err
    bf.check_guards()
    return Lo.cpu().numpy().reshape(N, k, k), st.cpu().numpy(), np.broadcast_to(A, (N, k, k))


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if c.family == "chol"],
                         ids=[c.id for c in CASES if c.family == "chol"])
def test_cholesky_instance_vs_scipy(case):
    """bke_cholesky_lower: L against scipy.linalg.cholesky(lower=True), exact zeros above its diagonal, A's upper
    triangle (NaN here) never read, and BKE_STATUS_NOT_PD exactly where scipy raises."""
    from filterpy_b200 import _lib
    assert (_lib.BKE_F32, _lib.BKE_F64) == (0, 1)
    tol, label = _bound(case)
    for i, N in enumerate(case.Ns):
        L, st, A = run_chol(case, N, seed=N + i)
        want, wst = chol_oracle(A)
        what = "%s N=%d" % (case.id, N)
        assert np.array_equal(st, wst), (what, np.nonzero(st != wst))
        if case.models == "per" and N >= 8:
            assert (wst == 2).sum() >= 3
        ok = wst == 0
        assert np.all(np.triu(L[ok], 1) == 0), what + " L above its diagonal"
        close(L, want, mag(np.nan_to_num(want)), np.linalg.cond(np.where(ok[:, None, None], A, np.eye(case.n))), tol,
              what + " L", label, ok)


# ------------------------------------------------------------------------------------------ which kernel runs
def _run_cases():
    for c in CASES:
        if c.family == "chol":
            run_chol(c, c.Np)
        else:
            rc, err, _, _, _ = run_step(c, c.Np)
            assert (rc != 0) == c.refused, (c.id, err)


def _profiled_names():
    """The kernel names of every CASES entry run once at its N, in launch order."""
    return profiled_names(_run_cases, r"srkf_\w+_kernel|chol_lower_kernel")


@pytest.mark.gpu
def test_dispatch_runs_the_kernels_of_the_table():
    """Each CASES entry, run once at its N, launches the kernels the table names, in order, template arguments included
    (a refused shape launches none)."""
    check_launch_order("test_gpu_srkf_instances", [(c.id, c.kernels) for c in CASES])
