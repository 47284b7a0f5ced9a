"""The scaffolding the per-instance GPU tests share: reading the dispatch source, naming kernels, checking which
kernels a table of cases launches, guarded device buffers, the C-ABI call, input helpers and the error-bound
comparisons.  The instance tables, their oracles and their tolerances stay in each test module."""
import json
import os
import re
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "filterpy_b200", "csrc")
F32, F64 = np.float32, np.float64
TNAME = {F32: "float", F64: "double"}
BUDGET = 200 * 1024               # api.cu warp_shape: shared memory per block of a warp-per-filter launch


# ------------------------------------------------------------------------------------------ the source
def src(name):
    """csrc/<name> without its comments (a commented-out dispatch line is not dispatched)."""
    with open(os.path.join(CSRC, name)) as fh:
        return re.sub(r"//[^\n]*|/\*.*?\*/", "", fh.read(), flags=re.S)


def body(text, signature):
    """The body of the function whose definition starts with ``signature`` (up to the closing brace at column 0)."""
    i = text.index(signature)
    return text[i:text.index("\n}\n", i)]


# ------------------------------------------------------------------------------------------ kernel names
def b(v):
    return "true" if v else "false"


def kernel_name(s, prefix):
    """'kf_direct_kernel<double, 4, 2, true, 0>' out of a demangled launch name (namespaces dropped), for a kernel
    whose name matches the regex ``prefix``; None for any other."""
    s = re.sub(r"\(anonymous namespace\)::|\b\w+::", "", s)
    mt = re.search(r"\b(%s)<" % prefix, s)
    if not mt:
        return None
    depth, i = 0, mt.end() - 1
    for j in range(i, len(s)):
        depth += {"<": 1, ">": -1}.get(s[j], 0)
        if depth == 0:
            return re.sub(r"\s+", " ", s[mt.start():j + 1])
    return None


# bke_kf_step's kernels: the KF instance table names them, and so do the FLS per-epoch routes that step on them.
# form: the update form template argument (kf_direct.cu / kf_generic.cu FORM_PLAIN 0, FORM_CORRELATED 1, FORM_ROWS 2)
def k_direct(dt, n, m, ex, form=0):
    return "kf_direct_kernel<%s, %d, %d, %s, %d>" % (TNAME[dt], n, m, b(ex), form)


def k_rb(dt, n, m, rpl, ex, mode, shared):
    return "kf_rowblock_kernel<%s, %d, %d, %d, %s, %d, %s>" % (TNAME[dt], n, m, rpl, b(ex), mode, b(shared))


def k_gen(dt, form=0):
    return "kf_generic_kernel<%s, %d>" % (TNAME[dt], form)


def k_fast(mode, shared, ex):
    return "kf42_f32_kernel<%d, %d, %s, 0, 0, NoPattern>" % (mode, shared, b(ex))


def rb_fpw(dt, n, m, rpl):
    """kf_rowblock.cu's pick_fpw: filters per warp tile, lowered until every tile array is a multiple of 16 bytes."""
    es = np.dtype(dt).itemsize
    for f in range(32 // (n // rpl), 0, -1):
        if all((f * es * k) % 16 == 0 for k in (n, n * n, m * n, m * m, m)):
            return f
    raise AssertionError("no warp tile")


# ------------------------------------------------------------------------------------------ which kernels run
def profiled_names(run_cases, prefix):
    """The names (kernel_name with ``prefix``) of the kernels run_cases() launches, in launch order (torch.profiler,
    CUDA activity)."""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run_cases()
    names = [kernel_name(e.name, prefix) for e in sorted(prof.events(), key=lambda e: e.time_range.start)]
    return [k for k in names if k]


def check_launch_order(module, expected):
    """``expected``: (case id, the kernel names the case launches) per case, in the order ``module``'s
    _profiled_names() runs them.  The names are profiled in a process of their own: after a session of this size the
    profiler of the same process reports no kernels to the sessions that follow it (other tests')."""
    code = ("import json, sys; sys.path[:0] = %r; import %s as t; print(json.dumps(t._profiled_names()))"
            % ([HERE, ROOT], module))
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    pos, bad = 0, []
    for cid, want in expected:
        got = names[pos:pos + len(want)]
        if got != want:
            bad.append((cid, want, got))
            break                                       # everything after a wrong count is shifted
        pos += len(want)
    assert not bad and pos == len(names), (bad, names[pos:pos + 5])


# ------------------------------------------------------------------------------------------ buffers and calls
class Bufs:
    """Device buffers, each with a 16-byte NaN guard before it (plus one element when it is misaligned) and five NaN
    elements after it; outputs start as a finite sentinel, so an element a kernel must leave alone can be checked."""
    SENT = 12345.0

    def __init__(self, dt):
        self.dt, self.keep, self.outs = dt, [], []

    def put(self, a, mis=False, out=False, dtype=None):
        import torch
        dtype = dtype or self.dt
        a = np.ascontiguousarray(a, dtype=dtype)
        es = a.itemsize
        off = 16 // es + (1 if mis else 0)
        tdt = {np.dtype(F32): torch.float32, np.dtype(F64): torch.float64, np.dtype(np.int32): torch.int32,
               np.dtype(np.int64): torch.int64, np.dtype(np.uint8): torch.uint8}[a.dtype]
        fill = float("nan") if tdt in (torch.float32, torch.float64) else -7
        buf = torch.full((off + a.size + 5,), fill, dtype=tdt, device="cuda")
        buf[off:off + a.size] = torch.from_numpy(a.reshape(-1)).cuda()
        view = buf[off:off + a.size]
        self.keep.append(buf)
        if out:
            self.outs.append((buf, off, a.size, a.shape))
        return view

    def out(self, shape, mis=False, dtype=None, fill=None):
        return self.put(np.full(shape, self.SENT if fill is None else fill), mis, True, dtype)

    def check_guards(self):
        for buf, off, cnt, _ in self.outs:
            h = buf.cpu().numpy()
            pre, post = h[:off], h[off + cnt:]
            if h.dtype.kind == "f":
                assert np.all(np.isnan(pre)) and np.all(np.isnan(post)), "write outside an output array"
            else:
                assert np.all(pre == -7) and np.all(post == -7), "write outside an output array"


def ptr(t):
    return None if t is None else t.data_ptr()


def call(fn, *args):
    """The C-ABI function ``fn`` on ``args`` and the current stream, then a device synchronize: (rc, error text)."""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    rc = getattr(lib, fn)(*args, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc, lib.bke_last_error().decode() if rc else ""


def call_ok(fn, *args):
    from filterpy_b200 import _lib
    rc, err = call(fn, *args)
    assert rc == _lib.BKE_OK, err


# ------------------------------------------------------------------------------------------ inputs
def rd(a, dt):
    """``a`` rounded to dtype dt, as fp64."""
    return np.asarray(a, np.float64).astype(dt).astype(np.float64)


def spd(rng, shape, k, scale):
    a = rng.normal(size=shape + (k, k))
    return scale * (a @ np.swapaxes(a, -1, -2) / k + np.eye(k))


def stable_F(rng, shape, n):
    """I + 0.15 G, scaled to a spectral radius of at most 0.98: a recursion of 32 epochs neither grows nor decays so
    far that its rounding says more about the model than about the kernel."""
    F = np.eye(n) + 0.15 * rng.normal(size=shape + (n, n))
    rho = np.abs(np.linalg.eigvals(F)).max(axis=-1)
    return F * np.minimum(1.0, 0.98 / rho)[..., None, None]


def corr_spd(rng, N, d, sd):
    """N random SPD matrices with correlated entries: sd_i sd_j (A A'/d + I/2)_ij, A standard normal."""
    A = rng.standard_normal((N, d, d))
    return (A @ np.swapaxes(A, 1, 2) / d + 0.5 * np.eye(d)) * np.outer(sd, sd)


SIGMA_DT = 0.1
SIGMA_FX = {"LINEAR": 0, "CONST_VEL": 1}                        # include/bke.h (and oracle/ukf.py)
SIGMA_HX = {"LINEAR": 0, "RANGE_AZ_EL": 1, "RANGE_BEARING": 2}


def sigma_problem(n, m, fx, hx, N=1037, T=3, seed=0):
    """A bank for the sigma-point families (UKF, CKF, EnKF) on the device models fx / hx (SIGMA_FX / SIGMA_HX names):
    x, correlated P, the model matrices in both layouts (shared by the bank / one per filter), T epochs of z and a
    ~20 % mask of missing measurements, with dt = SIGMA_DT.  The range models see targets 100-500 m from a sensor at
    the origin, well inside (-pi, pi) in azimuth, with R of sd 1 m in range and 0.005 rad in the angles."""
    from oracle import ukf as oukf
    rng = np.random.default_rng(seed)
    ranged = hx != "LINEAR"
    if ranged:
        x = np.zeros((N, n))
        x[:, 1::2] = rng.uniform(-10, 10, (N, n // 2))
        x[:, 0] = rng.uniform(100, 500, N); x[:, 2] = rng.uniform(-300, 300, N)
        if n == 6:
            x[:, 4] = rng.uniform(20, 200, N)
        sd = np.tile([2.0, 0.5], n // 2)
        rsd = np.array([1.0, 0.005, 0.005])[:m]
    else:
        x = rng.normal(0.0, 5.0, (N, n))
        sd = rng.uniform(0.5, 2.0, n)
        rsd = rng.uniform(0.5, 2.0, m)
    P = corr_spd(rng, N, n, sd)
    Q = corr_spd(rng, N, n, 0.1 * sd)
    R = corr_spd(rng, N, m, rsd)
    F = Fpf = H = Hpf = None
    if fx == "LINEAR":
        F = np.eye(n)
        if n % 2 == 0:
            F[np.arange(0, n, 2), np.arange(1, n, 2)] = SIGMA_DT
        eps = 0.002 if ranged else 0.1
        F = F + eps * rng.standard_normal((n, n))
        Fpf = F + eps * rng.standard_normal((N, n, n))
    if hx == "LINEAR":
        H = rng.standard_normal((m, n))
        Hpf = H + 0.1 * rng.standard_normal((N, m, n))
    truth = x + sd * rng.standard_normal((N, n))
    zs = np.empty((T, N, m))
    for t in range(T):
        truth = oukf.fx_apply(SIGMA_FX[fx], truth, SIGMA_DT, Fpf)
        zs[t] = oukf.hx_apply(SIGMA_HX[hx], truth, Hpf) + rsd * rng.standard_normal((N, m))
    valid = rng.random((T, N)) >= 0.2
    return dict(x=x, P=P, zs=zs, valid=valid, shared=dict(F=F, H=H, Q=Q[0], R=R[0]), per=dict(F=Fpf, H=Hpf, Q=Q, R=R))


def mag(*arrs):
    """Per filter (axis 0): the largest |entry| over the given arrays."""
    return np.max([np.abs(a).reshape(a.shape[0], -1).max(axis=1) for a in arrs], axis=0)


# ------------------------------------------------------------------------------------------ comparisons
def errlog(label, what, err, tol):
    """One BKE_TEST_ERRLOG line: label (module, family, dtype, ...), what, the worst error and the bound."""
    log = os.environ.get("BKE_TEST_ERRLOG")
    if log:
        with open(log, "a") as fh:
            fh.write("%s %s max_err=%.3e tol=%.1e\n" % (label, what, err, tol))


def close(got, want, scale, cond, tol, what, label, rows=None, match_inf=False):
    """|got - want| <= tol * scale * cond per filter: axis 0 of got and want indexes the filters, scale and cond (or a
    scalar cond) hold one value each; rows, if given, selects the filters compared.  Every compared entry of got is
    finite, except with match_inf, where got has exactly the infinities of want and the rest is compared."""
    got = np.asarray(got, np.float64); want = np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    scale = np.maximum(scale, 1e-300)
    cond = np.broadcast_to(np.asarray(cond, np.float64), scale.shape)
    if rows is not None:
        got, want, scale, cond = got[rows], want[rows], scale[rows], cond[rows]
    inf = np.isinf(want) if match_inf else np.zeros(want.shape, bool)
    assert np.array_equal(got[inf], want[inf]), "%s: an infinity differs" % what
    assert np.all(np.isfinite(got[~inf])), "%s: not finite" % what
    if inf.all():
        return
    sh = (-1,) + (1,) * (want.ndim - 1)
    e = np.where(inf, 0.0, np.abs(got - np.where(inf, 0.0, want)))
    err = e / (scale.reshape(sh) * cond.reshape(sh))
    errlog(label, what, err.max(), tol)
    assert err.max() <= tol, "%s: max err %.3e of the filter's scale x cond > %.1e" % (what, err.max(), tol)


RTOL = {np.float64: 1e-6, np.float32: 1e-3}


def rel_close(got, want, rtol, what=""):
    """|got - want| <= rtol * max(|want|, 1e-2 * max|want| of the same filter): element-wise
    relative error, with entries that are (near) zero by cancellation measured against the
    filter's own scale."""
    got = np.asarray(got, dtype=np.float64); want = np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.all(np.isfinite(got)), what
    if want.ndim > 1:
        floor = 1e-2 * np.abs(want).max(axis=tuple(range(1, want.ndim)), keepdims=True)
    else:
        floor = 1e-2 * np.abs(want)
    err = np.abs(got - want) / np.maximum(np.maximum(np.abs(want), floor), 1e-300)
    log = os.environ.get("BKE_TEST_ERRLOG")
    if log and err.size:
        import inspect
        caller = inspect.stack()[1]
        with open(log, "a") as fh:
            fh.write("%s:%d %s max_rel_err=%.3e rtol=%.1e\n" % (os.path.basename(caller.filename), caller.lineno, what, err.max(), rtol))
    assert err.size == 0 or err.max() <= rtol, "%s: max rel err %.3e > %.1e" % (what, err.max(), rtol)
