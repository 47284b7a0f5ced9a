"""GPU parity of every pre-built UKF / CKF kernel instance, the UKF RTS smoother and the stand-alone sigma
points / unscented transform against the fp64 oracle (oracle/ukf.py, oracle/ckf.py).

The golden vectors pin the oracle to the reference at 6/3 and 4/2.  These tests carry the comparison to every
(dim_x, dim_z, fx, hx) instance that ukf.cu and ckf.cu dispatch, to both layouts of each model matrix (shared by
the bank or one per filter), to banks that leave the last CTA part-empty, and to the edges of the kernels with
a run-time size: the smoother's n <= 8, the grid-stride loops and the > 48 KB shared-memory path of ut.cu."""
import ctypes
import os
import re

import numpy as np
import pytest

from gpu_harness import corr_spd as _corr_spd, sigma_problem as _problem, rel_close, RTOL

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "filterpy_b200", "csrc")
DT = 0.1
FX = {"LINEAR": 0, "CONST_VEL": 1}                              # include/bke.h (and oracle/ukf.py)
HX = {"LINEAR": 0, "RANGE_AZ_EL": 1, "RANGE_BEARING": 2}
DTYPES = pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])

# the pre-built (dim_x, dim_z, fx, hx) instances, in the order ukf.cu and ckf.cu dispatch them
INSTANCES = [
    (6, 3, "CONST_VEL", "RANGE_AZ_EL"),
    (6, 3, "CONST_VEL", "LINEAR"),
    (6, 3, "LINEAR", "LINEAR"),
    (6, 3, "LINEAR", "RANGE_AZ_EL"),
    (4, 2, "CONST_VEL", "RANGE_BEARING"),
    (4, 2, "LINEAR", "RANGE_BEARING"),
    (4, 2, "CONST_VEL", "LINEAR"),
    (4, 2, "LINEAR", "LINEAR"),
    (1, 1, "LINEAR", "LINEAR"),
    (2, 1, "LINEAR", "LINEAR"),
    (2, 1, "CONST_VEL", "LINEAR"),
    (2, 2, "LINEAR", "LINEAR"),
    (3, 1, "LINEAR", "LINEAR"),
    (3, 3, "LINEAR", "LINEAR"),
    (4, 4, "LINEAR", "LINEAR"),
]
INSTANCE_IDS = ["%d_%d_%s_%s" % (n, m, fx.lower(), hx.lower()) for n, m, fx, hx in INSTANCES]


@pytest.mark.parametrize("src", ["ukf.cu", "ukf_simplex.cu", "ckf.cu", "enkf.cu"])
def test_instance_table_is_the_dispatch_table(src):
    """INSTANCES is BKE_SIGMA_INSTANCES (sigma_launch.cuh), the one table from which ukf.cu, ckf.cu and enkf.cu
    dispatch and ukf_simplex.cu instantiates: an instance added there without being added to the tests below
    fails here, on a machine without a GPU too, and so does a row written into one of the four files by hand."""
    with open(os.path.join(CSRC, "sigma_launch.cuh")) as fh:
        table = re.search(r"#define BKE_SIGMA_INSTANCES\(X\)((?:.*\\\n)*.*)", fh.read()).group(1)
    row = r"\w+\(\s*(\d+)\s*,\s*(\d+)\s*,\s*BKE_FX_(\w+)\s*,\s*BKE_HX_(\w+)\s*\)"
    got = [(int(n), int(m), fx, hx) for n, m, fx, hx in re.findall(row, table)]
    assert got == INSTANCES
    with open(os.path.join(CSRC, src)) as fh:
        text = fh.read()
    assert re.search(r"^\s*BKE_SIGMA_INSTANCES\(\w+\)", text, re.M)
    assert not re.findall(row, text)                 # no hand-written row next to the table


# ----------------------------------------------------------------------------------------------- problems
def _take(mats, N):
    return {k: (v[:N] if v is not None and v.ndim == 3 else v) for k, v in mats.items()}


def _filter(kind, inst, mats, N, dtype, pts, diagnostics=True):
    from filterpy_b200.kalman import (UnscentedKalmanFilter, CubatureKalmanFilter, MerweScaledSigmaPoints,
                                      LinearFx, ConstVelFx, LinearHx, RangeAzElHx, RangeBearingHx)
    n, m, fx, hx = inst
    f = LinearFx(mats["F"]) if fx == "LINEAR" else ConstVelFx()
    h = LinearHx(mats["H"]) if hx == "LINEAR" else (RangeAzElHx() if hx == "RANGE_AZ_EL" else RangeBearingHx())
    if kind == "ukf":
        u = UnscentedKalmanFilter(n, m, DT, h, f, MerweScaledSigmaPoints(n, *pts), n_filters=N, dtype=dtype,
                                  diagnostics=diagnostics)
    else:
        u = CubatureKalmanFilter(n, m, DT, h, f, n_filters=N, dtype=dtype, diagnostics=diagnostics)
    u.Q = mats["Q"]; u.R = mats["R"]
    return u


def _oracle_step(kind, inst, x, P, z, mats, valid, pts):
    from oracle import ukf as oukf, ckf as ockf
    _, _, fx, hx = inst
    if kind == "ukf":
        return oukf.ukf_step_bank(x, P, z, mats["Q"], mats["R"], DT, *pts, FX[fx], HX[hx], F=mats["F"], H=mats["H"], valid=valid)
    return ockf.ckf_step_bank(x, P, z, mats["Q"], mats["R"], DT, FX[fx], HX[hx], F=mats["F"], H=mats["H"], valid=valid)


def _loglik(S, y):
    """log N(y; 0, S) per filter."""
    q = np.einsum("na,nab,nb->n", y, np.linalg.inv(S), y)
    return -0.5 * (q + np.linalg.slogdet(S)[1] + y.shape[-1] * np.log(2 * np.pi))


# fp32 against the fp64 oracle, 3 epochs from random correlated P through random F and H: measured worst cases
# on the H100 5.3e-3 (S of the 6/3 linear UKF; x, P and the priors 2.5e-3) and 6.0e-3 (K).  fp64: 1e-6 / 1e-5,
# measured worst case 4e-11
STEP_TOL = {np.float64: (RTOL[np.float64], 1e-5), np.float32: (1e-2, 2e-2)}


def _compare(f, o, z, v, dtype, what):
    """Posterior and prior everywhere; K, S, the predicted measurement z - y and the log-likelihood where the
    filter had a measurement (elsewhere the kernel leaves them as they were)."""
    tol, ktol = STEP_TOL[dtype]
    rel_close(f.x.cpu().numpy(), o["x"], tol, "x " + what)
    rel_close(f.P.cpu().numpy(), o["P"], tol, "P " + what)
    rel_close(f.x_prior.cpu().numpy(), o["x_prior"], tol, "x_prior " + what)
    rel_close(f.P_prior.cpu().numpy(), o["P_prior"], tol, "P_prior " + what)
    if v.any():
        rel_close(f.K.cpu().numpy()[v], o["K"][v], ktol, "K " + what)
        rel_close(f.S.cpu().numpy()[v], o["S"][v], max(tol, 1e-5), "S " + what)
        # y = z - z^ cancels most digits of z: compare the predicted measurement z^ = z - y instead, each
        # component against the larger of its own size and its standard deviation sqrt(S_aa) (with dim_z = 1
        # a z^ near 0 has no other component to measure it against)
        zf = z.astype(dtype).astype(np.float64)                      # the z the filter was given
        got, want = (zf - f.y.cpu().numpy())[v], (z - o["y"])[v]
        scale = np.maximum(np.abs(want), np.sqrt(np.diagonal(o["S"][v], axis1=1, axis2=2)))
        err = np.abs(got - want) / scale
        assert err.max() <= max(tol, 1e-5), "z - y %s: %.3e" % (what, err.max())
        ll = _loglik(o["S"][v], o["y"][v])
        err = np.abs(f.log_likelihood.cpu().numpy()[v] - ll) / np.maximum(np.abs(ll), 1.0)
        assert err.max() <= max(10 * RTOL[dtype], 1e-5), "loglik %s: %.3e" % (what, err.max())


def _merwe(n, pts):
    return (pts[0], pts[1], 3.0 - n if pts[2] == "3-n" else pts[2])


# alpha = 0.5, kappa = 0: centre weight -3 at every n; alpha = 1, kappa = 3 - n: (3 - n) / 3, positive for n < 3
STEP_CASES = [("ukf", (0.5, 2.0, 0.0)), ("ukf", (1.0, 2.0, "3-n")), ("ckf", None)]
STEP_IDS = ["ukf_a0.5_k0", "ukf_a1_k3-n", "ckf"]


# ----------------------------------------------------------------------------------------- instance matrix
@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("inst", INSTANCES, ids=INSTANCE_IDS)
@pytest.mark.parametrize("kind,pts", STEP_CASES, ids=STEP_IDS)
def test_instance_vs_oracle(kind, pts, inst, dtype):
    """Every pre-built instance: banks of 1 and 1037 filters (the last of 9 CTAs holds 13), F / H / Q / R
    shared and per filter, 3 predict + update epochs with ~20 % of the measurements missing."""
    n = inst[0]
    pts = None if pts is None else _merwe(n, pts)
    pr = _problem(*inst, seed=INSTANCES.index(inst))
    for N in (1, 1037):
        for layout in ("shared", "per"):
            mats = _take(pr[layout], N)
            f = _filter(kind, inst, mats, N, dtype, pts)
            x, P = pr["x"][:N], pr["P"][:N]
            f.x = x; f.P = P
            for t in range(pr["zs"].shape[0]):
                z, v = pr["zs"][t, :N], pr["valid"][t, :N]
                f.predict(); f.update(z, valid=v)
                o = _oracle_step(kind, inst, x, P, z, mats, v, pts)
                x, P = o["x"], o["P"]
                _compare(f, o, z, v, dtype, "%s N=%d t=%d" % (layout, N, t))
                assert int(f.status.sum().item()) == 0


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("inst", INSTANCES, ids=INSTANCE_IDS)
@pytest.mark.parametrize("kind", ["ukf", "ckf"])
def test_instance_diagnostics_off_split_and_not_pd(kind, inst, dtype):
    """Every pre-built instance, 1037 filters: without the optional outputs against the oracle; a predict
    launched on its own (flushed by reading x) and then the update give bit for bit the fused step; and
    P = -I in one filter of each CTA flags that filter (status 2) and changes no other filter by a bit."""
    pts = (0.5, 2.0, 0.0)
    pr = _problem(*inst, seed=100 + INSTANCES.index(inst))
    N, T = pr["x"].shape[0], pr["zs"].shape[0]

    mats = pr["shared"]
    c = _filter(kind, inst, mats, N, dtype, pts, diagnostics=False)
    c.x = pr["x"]; c.P = pr["P"]
    x, P = pr["x"], pr["P"]
    for t in range(T):
        c.predict(); c.update(pr["zs"][t], valid=pr["valid"][t])
        o = _oracle_step(kind, inst, x, P, pr["zs"][t], mats, pr["valid"][t], pts)
        x, P = o["x"], o["P"]
    rel_close(c.x.cpu().numpy(), x, STEP_TOL[dtype][0], "x, diagnostics off")
    rel_close(c.P.cpu().numpy(), P, STEP_TOL[dtype][0], "P, diagnostics off")

    bad = [c0 + (37 * i + 5) % min(128, N - c0) for i, c0 in enumerate(range(0, N, 128))]
    good = np.ones(N, bool); good[bad] = False
    Pbad = pr["P"].copy(); Pbad[bad] = -np.eye(inst[0])
    fused, split, flagged = (_filter(kind, inst, pr["per"], N, dtype, pts) for _ in range(3))
    for f, P0 in ((fused, pr["P"]), (split, pr["P"]), (flagged, Pbad)):
        f.x = pr["x"]; f.P = P0
    for t in range(T):
        z, v = pr["zs"][t], pr["valid"][t]
        fused.predict(); fused.update(z, valid=v)
        split.predict(); split.x; split.update(z, valid=v)
        flagged.predict(); flagged.update(z, valid=v)
        xa, Pa = fused.x.cpu().numpy(), fused.P.cpu().numpy()
        assert np.array_equal(split.x.cpu().numpy(), xa) and np.array_equal(split.P.cpu().numpy(), Pa), t
        st = flagged.status.cpu().numpy()
        assert (st[bad] == 2).all() and (st[good] == 0).all(), (t, st[bad], np.flatnonzero(st[good]))
        assert np.array_equal(flagged.x.cpu().numpy()[good], xa[good]), t
        assert np.array_equal(flagged.P.cpu().numpy()[good], Pa[good]), t


# ------------------------------------------------------------------------------------------- angle paths
@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("case", ["azimuth_cut", "close_range"])
@pytest.mark.parametrize("fx", ["CONST_VEL", "LINEAR"])
@pytest.mark.parametrize("hx", ["RANGE_AZ_EL", "RANGE_BEARING"])
@pytest.mark.parametrize("kind", ["ukf", "ckf"])
def test_angle_paths_vs_oracle(kind, hx, fx, case, dtype):
    """The UKF kernel evaluates the angles of the sigma points relative to the mean point (a short series for
    small angular offsets, the library atan2 otherwise) and wraps into (-pi, pi]; the CKF's run-time loop calls
    atan2 directly.  Both against the oracle's plain np.arctan2: targets straddling the +-pi azimuth cut, and
    targets so close that the sigma points span wide angles.

    In fp32, filters with an fp64 oracle sigma point within 1e-5 rad of +-pi are left out: that close, rounding
    decides on which side of the cut the point lies.  (An fp32 position 300-900 m out carries ~1e-7 rad of
    rounding, so 1e-5 rad leaves a factor 100; at 1e-4 rad the CKF's wider points left out 11 % of the bank.)
    The filters whose points straddle the cut average angles near +pi and -pi: their S and P come out of sums
    that cancel, measured to amplify rounding ~3e5-fold in fp64 (3.7e-11).  fp32 there is held to 5e-2
    (measured worst case 1.4e-2, P); the close-range case to RTOL."""
    from filterpy_b200.common import workloads as wl
    from oracle import ukf as oukf
    N = 3000
    n, m = (6, 3) if hx == "RANGE_AZ_EL" else (4, 2)
    w = wl.ukf_bank_cv3d(N, seed=77, steps=1)
    rng = np.random.default_rng(5)
    x = w["x"].copy()
    if case == "azimuth_cut":
        x[:, 0] = -rng.uniform(300, 900, N); x[:, 2] = rng.uniform(-1.5, 1.5, N); x[:, 4] = rng.uniform(-50, 50, N)
    else:
        x[:, 0] = rng.uniform(2, 6, N) * rng.choice([-1, 1], N); x[:, 2] = rng.uniform(2, 6, N) * rng.choice([-1, 1], N)
        x[:, 4] = rng.uniform(-4, 4, N)
    px, py, pz = x[:, 0], x[:, 2], x[:, 4]
    if n == 6:
        z = np.stack([np.sqrt(px * px + py * py + pz * pz), np.arctan2(py, px), np.arctan2(pz, np.sqrt(px * px + py * py))], 1)
        z = z + rng.normal(size=z.shape) * np.array([0.5, 0.002, 0.002])
    else:
        z = np.stack([np.sqrt(px * px + py * py), np.arctan2(py, px)], 1) + rng.normal(size=(N, 2)) * np.array([0.5, 0.002])
    x, P, Q, F = x[:, :n], w["P"][:, :n, :n], w["Q"][:, :n, :n], w["F"][:n, :n]
    mats = dict(F=F if fx == "LINEAR" else None, H=None, Q=Q, R=w["R"][:, :m, :m])
    inst, pts = (n, m, fx, hx), (0.5, 2.0, 0.0)
    f = _filter(kind, inst, mats, N, dtype, pts)
    f.x = x; f.P = P
    f.predict(); f.update(z)
    o = _oracle_step(kind, inst, x, P, z, mats, None, pts)
    ok = np.isfinite(o["x"]).all(axis=1) & (f.status.cpu().numpy() == 0)
    assert ok.mean() > 0.95
    if dtype == np.float32:
        sig = oukf.merwe_sigma_points(o["x_prior"], o["P_prior"], *pts) if kind == "ukf" else o["sigmas_f"]
        near_cut = (np.pi - np.abs(np.arctan2(sig[..., 2], sig[..., 0]))).min(axis=1) < 1e-5
        print("%s %s %s %s fp32: %d of %d filters near the cut left out" % (kind, hx, fx, case, near_cut.sum(), N))
        assert near_cut.mean() < 0.05
        ok &= ~near_cut
    rtol = 5e-2 if (dtype == np.float32 and case == "azimuth_cut") else RTOL[dtype]
    rel_close(f.x.cpu().numpy()[ok], o["x"][ok], rtol, "x " + case)
    rel_close(f.P.cpu().numpy()[ok], o["P"][ok], rtol, "P " + case)
    rel_close(f.S.cpu().numpy()[ok], o["S"][ok], rtol, "S " + case)


# -------------------------------------------------------------------------------------- UKF RTS smoother
RTS_SHAPES = [(n, "LINEAR", lay) for n in range(1, 9) for lay in ("shared", "per")] + [(n, "CONST_VEL", None) for n in (2, 4, 6, 8)]


def _rts_problem(n, fx, F_layout, T, Q_layout, dts_kind, N=65, seed=0):
    """Xs, Ps of an oracle UKF forward pass (linear measurement of half the state), with the Q, F and dts the
    smoother is then given."""
    from oracle import ukf as oukf
    rng = np.random.default_rng(seed)
    pts = (0.5, 2.0, 0.0) if n % 2 == 0 else (1.0, 2.0, 3.0 - n)
    m = max(1, n // 2)
    sd = rng.uniform(0.5, 2.0, n)
    x = rng.normal(0.0, 3.0, (N, n))
    P = _corr_spd(rng, N, n, sd)
    Q = _corr_spd(rng, N, n, 0.2 * sd)
    Q = Q[0] if Q_layout == "shared" else Q
    F = None
    if fx == "LINEAR":
        F = np.eye(n) + 0.1 * rng.standard_normal((n, n))
        if F_layout == "per":
            F = F + 0.05 * rng.standard_normal((N, n, n))
    H = rng.standard_normal((m, n)); R = np.eye(m) * 0.5
    dts = {"none": None, "scalar": 0.25, "epochs": rng.uniform(0.05, 0.3, T)}[dts_kind]
    dt_k = [DT] * T if dts is None else ([dts] * T if np.isscalar(dts) else list(dts))
    Xs, Ps = np.empty((T, N, n)), np.empty((T, N, n, n))
    for k in range(T):
        z = x @ H.T + rng.normal(0.0, 1.0, (N, m))
        o = oukf.ukf_step_bank(x, P, z, Q, R, dt_k[k], *pts, FX[fx], HX["LINEAR"], F=F, H=H)
        x, P = o["x"], o["P"]
        Xs[k], Ps[k] = x, P
    return dict(Xs=Xs, Ps=Ps, Q=Q, F=F, H=H, dts=dts, dt_k=dt_k, pts=pts)


def _rts_filter(n, fx, pr, N, dtype):
    from filterpy_b200.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, LinearFx, ConstVelFx, LinearHx
    f = LinearFx(pr["F"]) if fx == "LINEAR" else ConstVelFx()
    u = UnscentedKalmanFilter(n, pr["H"].shape[0], DT, LinearHx(pr["H"]), f, MerweScaledSigmaPoints(n, *pr["pts"]),
                              n_filters=N, dtype=dtype)
    u.Q = pr["Q"]
    return u


def _rts_oracle(n, fx, pr, dtype):
    """oracle.ukf.ukf_rts_smoother filter by filter, on the inputs as the kernel sees them (rounded to dtype)."""
    from oracle import ukf as oukf
    r = lambda a: None if a is None else np.asarray(a).astype(dtype).astype(np.float64)      # noqa: E731
    Xs, Ps, Q, F = r(pr["Xs"]), r(pr["Ps"]), r(pr["Q"]), r(pr["F"])
    dts = list(r(pr["dt_k"]))
    T, N = Xs.shape[:2]
    xs, Pso, Ks = np.empty_like(Xs), np.empty_like(Ps), np.empty_like(Ps)
    for i in range(N):
        if fx == "LINEAR":
            Fi = F if F.ndim == 2 else F[i]
            fxi = lambda s, dt, Fi=Fi: Fi @ s                                                 # noqa: E731
        else:
            fxi = lambda s, dt: oukf.fx_apply(FX["CONST_VEL"], s, dt)                         # noqa: E731
        xs[:, i], Pso[:, i], Ks[:, i] = oukf.ukf_rts_smoother(Xs[:, i], Ps[:, i], Q if Q.ndim == 2 else Q[i], fxi, dts, *pr["pts"])
    return xs, Pso, Ks


def _per_filter(a):
    """[T, N, ...] -> [N, T, ...]: rel_close measures near-zero entries against their own filter's scale."""
    return np.swapaxes(np.asarray(a), 0, 1)


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("n,fx,F_layout", RTS_SHAPES, ids=["%d_%s_%s" % (n, fx.lower(), lay) for n, fx, lay in RTS_SHAPES])
def test_ukf_rts_smoother_vs_oracle(n, fx, F_layout, dtype):
    """The smoother kernel (run-time n <= 8) at every n with a linear fx, F shared and per filter, and with
    constant velocity at every even n; Q shared and per filter; dts None (the filter's dt), a scalar and one
    per epoch (every pairing at T = 2, two at T = 17); T = 1, 2, 17 epochs of 65 filters (the last of the
    64-thread blocks holds one).  fp32 after 16 backward steps, each with a Gauss-Jordan inverse: measured
    worst case 1.2e-2 (K at n = 7; x 4.5e-3, P 3.4e-3) on the H100, held to 3e-2."""
    import torch
    N = 65
    combos = [(T, q, d) for T in (1, 2) for q in ("shared", "per") for d in ("none", "scalar", "epochs")]
    for T, Q_layout, dts_kind in combos + [(17, "shared", "scalar"), (17, "per", "epochs")]:
        what = "T=%d Q %s dts %s" % (T, Q_layout, dts_kind)
        pr = _rts_problem(n, fx, F_layout, T, Q_layout, dts_kind, N, seed=T * 10 + n)
        u = _rts_filter(n, fx, pr, N, dtype)
        xs, Ps, Ks = (a.cpu().numpy() for a in u.rts_smoother(torch.from_numpy(pr["Xs"]), torch.from_numpy(pr["Ps"]), dts=pr["dts"]))
        if T == 1:                                               # nothing to smooth: the inputs come back, K = 0
            assert np.array_equal(xs, pr["Xs"].astype(dtype)) and np.array_equal(Ps, pr["Ps"].astype(dtype)), what
            assert not Ks.any(), what
            continue
        wx, wP, wK = _rts_oracle(n, fx, pr, dtype)
        rtol = RTOL[dtype] if dtype == np.float64 else 3e-2
        rel_close(_per_filter(xs), _per_filter(wx), rtol, "xs " + what)
        rel_close(_per_filter(Ps), _per_filter(wP), rtol, "Ps " + what)
        rel_close(_per_filter(Ks[:-1]), _per_filter(wK[:-1]), rtol, "Ks " + what)
        assert not Ks[-1].any(), what


def _rts_raw(u, Xs, Ps):
    """bke_ukf_rts_smoother through the C-ABI, for the per-filter status the bank-mode method does not return."""
    import torch
    from filterpy_b200 import _lib
    from filterpy_b200._dev import bke_dtype
    T, N, n = Xs.shape
    Xt, Pt = (torch.from_numpy(np.ascontiguousarray(a)).cuda().to(u._dtype) for a in (Xs, Ps))
    xs, Pso, Ks = torch.empty_like(Xt), torch.empty_like(Pt), torch.empty_like(Pt)
    status = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    a = _lib.UkfRtsArgs()
    a.n_filters, a.n_steps, a.dim_x, a.dtype, a.fx_model = N, T, n, bke_dtype(u._dtype), u.fx.model
    a.alpha, a.beta, a.kappa, a.dt = u.points_fn.alpha, u.points_fn.beta, u.points_fn.kappa, float(u._dt)
    a.Xs, a.Ps, a.x_out, a.P_out, a.K, a.status = Xt.data_ptr(), Pt.data_ptr(), xs.data_ptr(), Pso.data_ptr(), Ks.data_ptr(), status.data_ptr()
    a.Q, a.Q_stride = u._Q.data_ptr(), u._stride(u._Q)
    if u._F is not None:
        a.F, a.F_stride = u._F.data_ptr(), u._stride(u._F)
    _lib.check(_lib.load().bke_ukf_rts_smoother(ctypes.byref(a), None))
    torch.cuda.synchronize()
    return xs.cpu().numpy(), Pso.cpu().numpy(), Ks.cpu().numpy(), status.cpu().numpy()


@pytest.mark.gpu
@DTYPES
def test_ukf_rts_smoother_not_pd_flags_one_filter(dtype):
    """A non-PD Ps[k] in one filter: that filter's status is 2, epochs after k are smoothed as before, k and
    the epochs before it come back as given with K = 0; every other filter is bit-equal to the clean run."""
    N, T, k, j = 65, 17, 8, 33
    pr = _rts_problem(4, "LINEAR", "per", T, "per", "none", N, seed=5)
    u = _rts_filter(4, "LINEAR", pr, N, dtype)
    Pbad = pr["Ps"].copy(); Pbad[k, j] = -np.eye(4)
    x0, P0, K0, s0 = _rts_raw(u, pr["Xs"], pr["Ps"])
    x1, P1, K1, s1 = _rts_raw(u, pr["Xs"], Pbad)
    assert not s0.any()
    assert s1[j] == 2 and not np.delete(s1, j).any()
    others = np.arange(N) != j
    for a, b in ((x1, x0), (P1, P0), (K1, K0)):
        assert np.array_equal(a[:, others], b[:, others])
        assert np.array_equal(a[k + 1:, j], b[k + 1:, j])
    assert np.array_equal(x1[:k + 1, j], pr["Xs"][:k + 1, j].astype(dtype))
    assert np.array_equal(P1[:k + 1, j], Pbad[:k + 1, j].astype(dtype))
    assert not K1[:k + 1, j].any()


# ------------------------------------------------------------------------ stand-alone sigma points and UT
def _sigma_raw(x, P, alpha, beta, kappa):
    """bke_merwe_sigma_points through the C-ABI, with its per-filter status."""
    import torch
    from filterpy_b200 import _lib
    from filterpy_b200._dev import bke_dtype
    N, n = x.shape
    sig = torch.empty(N, 2 * n + 1, n, dtype=x.dtype, device=x.device)
    status = torch.full((N,), -1, dtype=torch.int32, device=x.device)
    _lib.check(_lib.load().bke_merwe_sigma_points(N, n, bke_dtype(x.dtype), alpha, beta, kappa, x.data_ptr(), P.data_ptr(),
                                                  sig.data_ptr(), status.data_ptr(), None))
    torch.cuda.synchronize()
    return sig, status.cpu().numpy()


def _subset(N, seed):
    """All filters of a small bank; of a large one a random 300 and the last 64 (the grid-stride loop's tail)."""
    if N <= 64:
        return np.arange(N)
    return np.unique(np.concatenate([np.random.default_rng(seed).choice(N, 300, replace=False), np.arange(N - 64, N)]))


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("n", range(1, 33))
def test_sigma_points_vs_oracle(n, dtype):
    """k_sigma_points at every n it accepts, for 1, 5 and 20011 filters (the grid holds 16 x SMs blocks of 4
    warps, one filter per warp: 20011 runs the grid-stride loop), with asymmetric garbage in P's lower
    triangle (only the upper one is read, like scipy.linalg.cholesky); non-PD filters are flagged, alone."""
    import torch
    from oracle import ukf as oukf
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    alpha, beta, kappa = (0.5, 2.0, 0.0) if n % 2 else (1.0, 2.0, 3.0 - n)
    g = torch.Generator(device="cuda").manual_seed(1000 + n)
    kw = dict(generator=g, device="cuda", dtype=torch.float64)
    tol = 1e-10 if dtype == np.float64 else RTOL[dtype]
    lower = torch.tril(torch.ones(n, n, dtype=torch.bool, device="cuda"), -1)
    for N in (1, 5, 20011):
        x = torch.randn(N, n, **kw)
        A = torch.randn(N, n, n, **kw)
        P = A @ A.transpose(1, 2) / n + torch.eye(n, dtype=torch.float64, device="cuda")
        P = torch.where(lower, 100 * torch.randn(N, n, n, **kw), P).to(tdt).contiguous()
        x = x.to(tdt).contiguous()
        sig, st = _sigma_raw(x, P, alpha, beta, kappa)
        assert not st.any(), N
        sel = torch.from_numpy(_subset(N, n)).cuda()
        want = oukf.merwe_sigma_points(x[sel].double().cpu().numpy(), P[sel].double().cpu().numpy(), alpha, beta, kappa)
        rel_close(sig[sel].cpu().numpy(), want, tol, "sigmas N=%d" % N)
        if N == 5:
            Pb = P.clone()
            Pb[1] = -torch.eye(n, dtype=tdt, device="cuda")
            Pb[3, n - 1, n - 1] = -1.0                           # fails at the last pivot only
            sb, sst = _sigma_raw(x, Pb, alpha, beta, kappa)
            assert sst.tolist() == [0, 2, 0, 2, 0]
            assert torch.equal(sb[[0, 2, 4]], sig[[0, 2, 4]])


UT_SHAPES = [(2 * n + 1, n) for n in (1, 3, 9, 16, 32, 64)] + [(1, 5), (256, 64)]


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("k,n", UT_SHAPES, ids=["k%d_n%d" % s for s in UT_SHAPES])
def test_unscented_transform_vs_oracle(k, n, dtype):
    """k_unscented_transform from 1 point to the 256 x 64 the C-ABI accepts, for 1 and 20011 filters, noise
    none, shared and per filter.  A warp holds k * n + n words of shared memory: from fp64 n = 28 a block of 4
    warps needs > 48 KB, and at (129, 64) fp64 and (256, 64) more than a block can have, where the launch uses
    fewer warps per block."""
    import torch
    from filterpy_b200.kalman import unscented_transform
    from oracle import ukf as oukf
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    rng = np.random.default_rng(k * 100 + n)
    if k == 2 * n + 1:
        Wm, Wc = oukf.merwe_weights(n, 0.5, 2.0, 0.0)
    else:
        Wm = rng.uniform(0.5, 1.5, k); Wm /= Wm.sum()
        Wc = rng.uniform(0.5, 1.5, k) * (2.0 / k)
    r = lambda a: np.asarray(a).astype(dtype).astype(np.float64)                               # noqa: E731
    g = torch.Generator(device="cuda").manual_seed(k * 100 + n)
    kw = dict(generator=g, device="cuda", dtype=torch.float64)
    tol = 1e-10 if dtype == np.float64 else RTOL[dtype]
    for N in (1, 20011):
        L = torch.randn(N, n, n, **kw) / np.sqrt(n)
        sig = (10 * torch.randn(N, 1, n, **kw) + torch.randn(N, k, n, **kw) @ L.transpose(1, 2)).to(tdt).contiguous()
        B = torch.randn(N, n, n, **kw)
        noise_pf = (B @ B.transpose(1, 2) / n).to(tdt).contiguous()
        sel = _subset(N, k + n)
        for noise in ("none", "shared", "per"):
            nz = {"none": None, "shared": noise_pf[0], "per": noise_pf}[noise]
            x, P = unscented_transform(sig, Wm, Wc, noise_cov=nz)
            s = sig[torch.from_numpy(sel).cuda()].double().cpu().numpy()
            nzw = None if nz is None else (nz.double().cpu().numpy() if noise == "shared" else nz[torch.from_numpy(sel).cuda()].double().cpu().numpy())
            wx, wP = oukf.unscented_transform(s, r(Wm), r(Wc), nzw)
            rel_close(x.cpu().numpy()[sel], wx, tol, "x N=%d noise %s" % (N, noise))
            rel_close(P.cpu().numpy()[sel], wP, tol, "P N=%d noise %s" % (N, noise))
