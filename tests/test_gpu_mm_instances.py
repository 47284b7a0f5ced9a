"""Every kernel instance of csrc/mix.cu (the IMM / MMAE mixing launches) against the fp64 bank oracle
(oracle/imm.py), through the C-ABI.

The goldens reach these kernels only at dim_x = 4 with 2 or 3 models on aligned buffers.  Here every
instance that mix.cu dispatches runs: the row-parallel k_mm_rows<T, NX, MM, MIX> at NX = 2, 4, 6 and MM = 2, 3,
4; the element-parallel k_mm_mix / k_mm_estimate with a compile-time model count and with the run-time one
(M = 1 and 5..8), reached through other dim_x or buffers one element past a 16-byte boundary; the MMAE
covariance (the reference's zip over the components of x) with M below, equal to and above dim_x; and the
probabilities kernel at its DBL_MIN floor.  Inputs are rounded to the kernel's dtype before the oracle sees
them, so only the kernel's own rounding is measured."""
import ctypes
import os
import re

import numpy as np
import pytest

from gpu_harness import CSRC, F32, F64, TNAME, call_ok, check_launch_order, close, mag, profiled_names

# Relative to the track's scale: the largest |x_j| of its inputs for x (a combined mean can cancel to ~0), the
# largest |entry| of the output for P.  Worst cases measured on an H100 with BKE_TEST_ERRLOG: x 2.7e-16 and
# P 7.7e-16 (fp64), x 1.4e-7 and P 3.3e-7 (fp32); the probabilities 3.9 ulp.
TOL = {F64: 1e-14, F32: 2e-6}
LABEL = "test_gpu_mm_instances"
PROB_ULPS = 6


def _instances():
    """(op, dtype, dim_x, M, misaligned, expected kernel).  The kernel is named as mix.cu instantiates it
    ("rows<NX,MM>", "mix<MM>", "estimate<MM>", MM = 0 for the run-time model count)."""
    out = []
    for dt in (F32, F64):
        for op in ("mix", "estimate"):
            for nx in (2, 4, 6):
                for mm in (2, 3, 4):
                    out.append((op, dt, nx, mm, False, "rows<%d,%d>" % (nx, mm)))
            # element kernels, compile-time model count: a dim_x without a row instance, and a row shape whose
            # buffers start one element past a 16-byte boundary
            for mm, nx in ((2, 3), (3, 5), (4, 1)):
                out.append((op, dt, nx, mm, False, "%s<%d>" % (op, mm)))
            for mm, nx in ((2, 2), (3, 4), (4, 6)):
                out.append((op, dt, nx, mm, True, "%s<%d>" % (op, mm)))
            # run-time model count: M = 1 and 5..8, aligned row shapes included (they have no row instance)
            for M, nx, mis in ((1, 4, False), (5, 4, False), (6, 2, True), (7, 3, False), (8, 6, False), (8, 64, False)):
                out.append((op, dt, nx, M, mis, "%s<0>" % op))
        # MMAE covariance (estimate only): M < dim_x, M = dim_x and M > dim_x, aligned row shapes included
        for M, nx, mis in ((2, 4, False), (3, 3, False), (4, 2, False), (1, 6, False), (5, 5, True), (8, 3, False),
                           (6, 6, False)):
            out.append(("mmae", dt, nx, M, mis, "estimate<%d>" % (M if M <= 4 and M > 1 else 0)))
    return out


INSTANCES = _instances()
INSTANCE_IDS = ["%s-%s-n%d-M%d%s" % (op, "f32" if dt == F32 else "f64", n, M, "-mis" if mis else "")
                for op, dt, n, M, mis, _ in INSTANCES]


def test_instance_list_matches_dispatch_table():
    """INSTANCES covers every kernel mix.cu instantiates: a new row shape or model count in the dispatch
    fails here, on a machine without a GPU too."""
    with open(os.path.join(CSRC, "mix.cu")) as fh:
        text = fh.read()
    nx = sorted(int(v) for v in re.findall(r"launch_rows_m<T,\s*(\d+)>\(p, op, s\)", text))
    mm = sorted(int(c) for c, v in re.findall(r"case (\d+): return launch_rows<T, NX, (\d+)>", text) if c == v)
    assert nx == [2, 4, 6] and mm == [2, 3, 4]
    dispatched = {"rows<%d,%d>" % (a, b) for a in nx for b in mm}
    for kern in ("mix", "estimate"):
        cases = re.findall(r"case (\d+): k_mm_%s<T, (\d+)>" % kern, text)
        assert all(c == v for c, v in cases)
        dispatched |= {"%s<%s>" % (kern, v) for _, v in cases}
        assert re.search(r"default: k_mm_%s<T, 0>" % kern, text)
        dispatched.add("%s<0>" % kern)
    for dt in (F32, F64):
        for op in ("mix", "estimate"):
            got = {k for o, d, _, _, _, k in INSTANCES if o == op and d == dt}
            assert got == {k for k in dispatched if k.startswith("rows") or k.startswith(op)}, (op, dt)
        got = {k for o, d, _, _, _, k in INSTANCES if o == "mmae" and d == dt}
        assert got == {k for k in dispatched if k.startswith("estimate")}
    # the row instances are only reached for MIX / IMM estimate on aligned buffers
    assert "launch_rows_m<T, 4>" in text and "!(a.flags & BKE_MM_MMAE)" in text


# ------------------------------------------------------------------------------------------ C-ABI helpers
def _dev(a, dtype, offset=0, guard=0):
    """A device copy of ``a`` in ``dtype`` that starts ``offset`` elements into its allocation (the caching
    allocator's blocks are 512-byte aligned, so offset 1 is one element past a 16-byte boundary) and is followed
    by ``guard`` NaN elements.  Returns (view, backing tensor)."""
    import torch
    a = np.ascontiguousarray(a, dtype=dtype)
    buf = torch.full((offset + a.size + guard,), float("nan"), dtype=torch.float32 if dtype == F32 else torch.float64,
                     device="cuda")
    buf[offset:offset + a.size] = torch.from_numpy(a.reshape(-1)).cuda()
    return buf[offset:offset + a.size].view(a.shape), buf


def _args(n_tracks, dim_x, M, dtype, flags=0):
    from filterpy_b200 import _lib
    a = _lib.MmArgs()
    a.n_tracks, a.dim_x, a.n_models = n_tracks, dim_x, M
    a.dtype, a.flags = (_lib.BKE_F32 if dtype == F32 else _lib.BKE_F64), flags
    return a


def _inputs(N, n, M, dtype, seed):
    """Per-model states (M, N, n) / (M, N, n, n) with spread means and SPD covariances, rounded to ``dtype``;
    mixing weights omega (N, M, M) whose columns sum to 1, and mode probabilities mu (N, M)."""
    rng = np.random.default_rng(seed)
    xs = rng.normal(size=(M, N, n)) * 3 + np.arange(M)[:, None, None]
    A = rng.normal(size=(M, N, n, n))
    Ps = A @ np.swapaxes(A, -1, -2) / n + np.eye(n)
    om = rng.uniform(0.05, 1.0, (N, M, M))
    om /= om.sum(axis=1, keepdims=True)
    mu = rng.uniform(0.05, 1.0, (N, M))
    mu /= mu.sum(axis=1, keepdims=True)
    return xs.astype(dtype).astype(F64), Ps.astype(dtype).astype(F64), om, mu


def run_instance(op, dtype, n, M, misaligned, N, shared, seed=0):
    """One bke_mm_mix / bke_mm_estimate call; returns (x_out, P_out) as (outs, N, n) / (outs, N, n, n), the
    oracle's, and each track's largest |x_j|."""
    import torch
    from filterpy_b200 import _lib
    from oracle import imm as oimm
    xs, Ps, om, mu = _inputs(N, n, M, dtype, seed)
    off, G = (1 if misaligned else 0), 5
    keep = []
    a = _args(N, n, M, dtype, _lib.BKE_MM_MMAE if op == "mmae" else 0)
    for j in range(M):
        xv, xb = _dev(xs[j], dtype, off); Pv, Pb = _dev(Ps[j], dtype, off)
        a.x[j], a.P[j] = xv.data_ptr(), Pv.data_ptr()
        keep += [xb, Pb]
    outs = M if op == "mix" else 1
    xo, Po = [], []
    for i in range(outs):
        xv, xb = _dev(np.zeros((N, n)), dtype, off, G); Pv, Pb = _dev(np.zeros((N, n, n)), dtype, off, G)
        a.x_out[i], a.P_out[i] = xv.data_ptr(), Pv.data_ptr()
        xo.append((xv, xb)); Po.append((Pv, Pb))
    w = (om if op == "mix" else mu)
    w = w[0] if shared else w
    wd = torch.from_numpy(np.ascontiguousarray(w)).cuda()
    keep.append(wd)
    if op == "mix":
        a.omega, a.weights_stride = wd.data_ptr(), (0 if shared else M * M)
        call_ok("bke_mm_mix", ctypes.byref(a))
        want = oimm.mm_mix_bank(xs, Ps, w)
    else:
        a.mu, a.weights_stride = wd.data_ptr(), (0 if shared else M)
        call_ok("bke_mm_estimate", ctypes.byref(a))
        wx, wP = oimm.mm_estimate_bank(xs, Ps, w, mmae=(op == "mmae"))
        want = (wx[None], wP[None])
    for (v, b), cnt in [(t, N * n) for t in xo] + [(t, N * n * n) for t in Po]:
        bh = b.cpu().numpy()
        assert np.all(np.isnan(bh[:off])) and np.all(np.isnan(bh[off + cnt:])), "write outside the output array"
    got = (np.array([v.cpu().numpy() for v, _ in xo], F64), np.array([v.cpu().numpy() for v, _ in Po], F64))
    return got, want, np.abs(xs).max(axis=(0, 2))


@pytest.mark.gpu
@pytest.mark.parametrize("inst", INSTANCES, ids=INSTANCE_IDS)
def test_instance_vs_bank_oracle(inst):
    op, dtype, n, M, mis, _ = inst
    for N in ((1, 255, 1037) if n < 32 else (1, 255)):          # dim_x = 64: 32 KB of P per track and model
        for shared in (False, True):
            (gx, gP), (wx, wP), xs = run_instance(op, dtype, n, M, mis, N, shared, seed=N + M)
            what = "%s %s n=%d M=%d N=%d shared=%d" % (op, np.dtype(dtype).name, n, M, N, shared)
            for i in range(gx.shape[0]):
                close(gx[i], wx[i], xs, 1, TOL[dtype], what + " x[%d]" % i, LABEL)
                close(gP[i], wP[i], mag(wP[i]), 1, TOL[dtype], what + " P[%d]" % i, LABEL)


def _kernel(op, dtype, kern):
    """The launch name of INSTANCES' kernel ``kern`` of op in dtype."""
    k, args = re.match(r"(\w+)<([\d,]+)>", kern).groups()
    if k == "rows":
        return "k_mm_rows<%s, %s, %s>" % (TNAME[dtype], ", ".join(args.split(",")), "true" if op == "mix" else "false")
    return "k_mm_%s<%s, %s>" % (k, TNAME[dtype], args)


def _run_cases():
    for op, dtype, n, M, mis, _ in INSTANCES:
        run_instance(op, dtype, n, M, mis, 1, False)


def _profiled_names():
    return profiled_names(_run_cases, r"k_mm_\w+")


@pytest.mark.gpu
def test_dispatch_runs_the_kernel_of_the_table():
    """Each INSTANCES entry launches the kernel the table names (kernel names from torch.profiler)."""
    check_launch_order("test_gpu_mm_instances",
                       [(i, [_kernel(op, dt, kern)]) for i, (op, dt, _, _, _, kern) in zip(INSTANCE_IDS, INSTANCES)])


@pytest.mark.gpu
def test_mix_and_estimate_grid_stride_2e20_tracks():
    """2^20 tracks, dim_x = 4, M = 3, fp32: more threads than one grid holds, so every thread loops."""
    for op in ("mix", "estimate"):
        for mis in (False, True):
            (gx, gP), (wx, wP), xs = run_instance(op, F32, 4, 3, mis, 1 << 20, False, seed=7)
            for i in range(gx.shape[0]):
                close(gx[i], wx[i], xs, 1, TOL[F32], "%s 2^20 mis=%d x[%d]" % (op, mis, i), LABEL)
                close(gP[i], wP[i], mag(wP[i]), 1, TOL[F32], "%s 2^20 mis=%d P[%d]" % (op, mis, i), LABEL)


# ------------------------------------------------------------------------------------------ probabilities
PROB_CASES = {
    # name: (M, ll generator)
    "normal": (3, lambda rng, N, M: rng.uniform(-12, -1, (N, M))),
    "all_floored": (3, lambda rng, N, M: np.full((N, M), -800.0)),           # exp underflows: every L is DBL_MIN
    "one_floored": (4, lambda rng, N, M: np.concatenate([np.full((N, 1), -800.0), rng.uniform(-12, -1, (N, M - 1))], 1)),
    "minus_inf": (2, lambda rng, N, M: np.where(rng.random((N, M)) < 0.3, -np.inf, rng.uniform(-9, -1, (N, M)))),
    "one_model": (1, lambda rng, N, M: rng.uniform(-12, -1, (N, M))),
    "eight_models": (8, lambda rng, N, M: rng.uniform(-40, -1, (N, M))),
}


def _ulp_close(got, want, ulps, what):
    got = np.asarray(got, F64); want = np.asarray(want, F64)
    err = np.abs(got - want) / np.maximum(np.abs(want), np.finfo(F64).tiny) / np.finfo(F64).eps
    log = os.environ.get("BKE_TEST_ERRLOG")
    if log:
        with open(log, "a") as fh:
            fh.write("test_gpu_mm_instances %s max_ulps=%.2f tol=%d\n" % (what, err.max(), ulps))
    assert err.max() <= ulps, "%s: %.2f ulp > %d" % (what, err.max(), ulps)


PROB_PARAMS = [(mode, case) for mode in ("imm", "mmae") for case in PROB_CASES] + \
    [("from_mu", "normal"), ("from_mu", "one_model"), ("from_mu", "eight_models")]


@pytest.mark.gpu
@pytest.mark.parametrize("mode,case", PROB_PARAMS, ids=["%s-%s" % p for p in PROB_PARAMS])
@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_probabilities_vs_bank_oracle(mode, case, dtype):
    """bke_mm_probabilities: L = exp(ll) floored at DBL_MIN, mu = prior L / sum (IMM: prior cbar; MMAE: mu),
    then cbar = mu . trans and omega (IMM, from_mu).  The log-likelihoods are the dtype's (what the KF bank
    writes); everything after is fp64 and agrees to a few ulp."""
    import torch
    from filterpy_b200 import _lib
    from oracle import imm as oimm
    M, gen = PROB_CASES[case]
    for N in (1, 1037):
        rng = np.random.default_rng(N + M)
        ll = gen(rng, N, M).astype(dtype)
        mu = rng.uniform(0.05, 1.0, (N, M)); mu /= mu.sum(1, keepdims=True)
        trans = rng.uniform(0.05, 1.0, (M, M)); trans /= trans.sum(1, keepdims=True)
        cbar = mu @ trans
        flags = {"imm": 0, "mmae": _lib.BKE_MM_MMAE, "from_mu": _lib.BKE_MM_FROM_MU}[mode]
        a = _args(N, 0, M, dtype, flags)
        lld = [torch.from_numpy(np.ascontiguousarray(ll[:, j])).cuda() for j in range(M)]
        for j in range(M):
            a.log_likelihood[j] = lld[j].data_ptr()
        t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in
             dict(mu=mu, cbar=cbar, trans=trans, omega=np.zeros((N, M, M))).items()}
        a.mu, a.cbar, a.omega, a.trans = (t[k].data_ptr() for k in ("mu", "cbar", "omega", "trans"))
        call_ok("bke_mm_probabilities", ctypes.byref(a))
        what = "%s %s %s N=%d" % (mode, case, np.dtype(dtype).name, N)
        llf = ll.astype(F64)
        if mode == "mmae":
            _ulp_close(t["mu"].cpu().numpy(), oimm.mm_probabilities_bank(mu, llf, mmae=True), PROB_ULPS, what + " mu")
            assert np.array_equal(t["cbar"].cpu().numpy(), cbar)          # MMAE has no cbar / omega
            continue
        wmu, wcb, wom = oimm.mm_probabilities_bank(mu, None if mode == "from_mu" else llf, cbar, trans)
        got_mu = t["mu"].cpu().numpy()
        if mode == "from_mu":
            assert np.array_equal(got_mu, mu)
        _ulp_close(got_mu, wmu, PROB_ULPS, what + " mu")
        _ulp_close(t["cbar"].cpu().numpy(), wcb, PROB_ULPS, what + " cbar")
        _ulp_close(t["omega"].cpu().numpy(), wom, PROB_ULPS, what + " omega")


# ------------------------------------------------------------------------------------------ argument checks
def _valid_args(op, dtype=F64):
    """Arguments that pass validation for op 0 (probabilities), 1 (mix), 2 (estimate): N = 1, dim_x = 2, M = 2,
    every pointer into one host buffer large enough for all of them (validation runs before the device check,
    so nothing is read from them on a machine without a GPU)."""
    from filterpy_b200 import _lib
    buf = np.zeros(4096)
    base = buf.ctypes.data
    a = _args(1, 2, 2, dtype)
    for j in range(2):
        a.x[j], a.P[j], a.log_likelihood[j] = base + 64 * j, base + 256 + 64 * j, base + 512 + 64 * j
        a.x_out[j], a.P_out[j] = base + 1024 + 64 * j, base + 1280 + 64 * j
    a.mu, a.cbar, a.omega, a.trans = base + 2048, base + 2112, base + 2176, base + 2304
    a.weights_stride = 4 if op == 1 else 2
    return a, buf


def _call(op, a):
    from filterpy_b200 import _lib
    lib = _lib.load()
    fn = (lib.bke_mm_probabilities, lib.bke_mm_mix, lib.bke_mm_estimate)[op]
    return fn(ctypes.byref(a), None)


BAD = [
    # (name, ops, edit, expected return code name)
    ("n_models_0", (0, 1, 2), lambda a: setattr(a, "n_models", 0), "BKE_ERR_UNSUPPORTED"),
    ("n_models_9", (0, 1, 2), lambda a: setattr(a, "n_models", 9), "BKE_ERR_UNSUPPORTED"),
    ("dim_x_0", (1, 2), lambda a: setattr(a, "dim_x", 0), "BKE_ERR_BAD_ARG"),
    ("dim_x_65", (1, 2), lambda a: setattr(a, "dim_x", 65), "BKE_ERR_BAD_ARG"),
    ("bad_dtype", (0, 1, 2), lambda a: setattr(a, "dtype", 7), "BKE_ERR_BAD_ARG"),
    ("negative_tracks", (0, 1, 2), lambda a: setattr(a, "n_tracks", -1), "BKE_ERR_BAD_ARG"),
    ("x_out_aliases_x", (1, 2), lambda a: a.x_out.__setitem__(0, a.x[1]), "BKE_ERR_BAD_ARG"),
    ("P_out_aliases_P", (1, 2), lambda a: a.P_out.__setitem__(0, a.P[0]), "BKE_ERR_BAD_ARG"),
    ("x_out_1_aliases_x", (1,), lambda a: a.x_out.__setitem__(1, a.x[0]), "BKE_ERR_BAD_ARG"),
    ("null_x", (1, 2), lambda a: a.x.__setitem__(1, None), "BKE_ERR_BAD_ARG"),
    ("null_P_out", (1, 2), lambda a: a.P_out.__setitem__(0, None), "BKE_ERR_BAD_ARG"),
    ("null_mu", (0, 2), lambda a: setattr(a, "mu", None), "BKE_ERR_BAD_ARG"),
    ("null_omega", (0, 1), lambda a: setattr(a, "omega", None), "BKE_ERR_BAD_ARG"),
    ("null_cbar", (0,), lambda a: setattr(a, "cbar", None), "BKE_ERR_BAD_ARG"),
    ("null_trans", (0,), lambda a: setattr(a, "trans", None), "BKE_ERR_BAD_ARG"),
    ("null_log_likelihood", (0,), lambda a: a.log_likelihood.__setitem__(1, None), "BKE_ERR_BAD_ARG"),
    ("negative_stride", (1, 2), lambda a: setattr(a, "weights_stride", -1), "BKE_ERR_BAD_ARG"),
]


@pytest.mark.parametrize("name,ops,edit,rc", BAD, ids=[b[0] for b in BAD])
def test_argument_checks(name, ops, edit, rc):
    """Every rejected argument returns its code before anything touches a device (these run without a GPU)."""
    from filterpy_b200 import _lib
    for op in ops:
        a, buf = _valid_args(op)
        edit(a)
        assert _call(op, a) == getattr(_lib, rc), (name, op, _lib.load().bke_last_error())


def test_argument_checks_accept_what_they_should():
    """n_tracks = 0 returns BKE_OK without a device; MMAE probabilities need no cbar / omega / trans and
    from_mu probabilities no log-likelihoods — without a GPU those get as far as the device check."""
    import torch
    from filterpy_b200 import _lib
    for op in (0, 1, 2):
        a, buf = _valid_args(op)
        a.n_tracks = 0
        assert _call(op, a) == _lib.BKE_OK
        a.x[0] = None; a.mu = None
        assert _call(op, a) == _lib.BKE_OK          # nothing to do: the pointers are not looked at
    if torch.cuda.is_available():
        return                                      # the remaining cases would launch on host pointers
    a, buf = _valid_args(0)
    a.flags = _lib.BKE_MM_MMAE; a.cbar = a.omega = a.trans = None
    assert _call(0, a) == _lib.BKE_ERR_CUDA
    a, buf = _valid_args(0)
    a.flags = _lib.BKE_MM_FROM_MU
    for j in range(2):
        a.log_likelihood[j] = None
    assert _call(0, a) == _lib.BKE_ERR_CUDA
