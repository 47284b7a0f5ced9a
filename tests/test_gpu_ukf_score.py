"""GPU parity of bke_ukf_score / UnscentedKalmanFilter.score_measurements: every pre-built instance (both dtypes, both
point sets) against the fp64 oracle (tests/ukf_score_oracle.py), the reference goldens through the public method in
bank and single mode, the status rules, that scoring leaves the filter untouched, and the torch op."""
import numpy as np
import pytest
import torch

import ukf_score_oracle as uso
from gpu_harness import RTOL
from test_gpu_sigma_instances import INSTANCES, INSTANCE_IDS, FX, HX, _corr_spd
from test_oracle_ukf_score import CASES, load
from oracle import ukf as oukf

DTYPES = pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
# the distinct (dim_x, dim_z, hx) of the instance table: the score does not run fx
SCORE_INSTANCES = list(dict.fromkeys((n, m, hx) for n, m, _, hx in INSTANCES))
SCORE_IDS = ["%d_%d_%s" % (n, m, hx.lower()) for n, m, hx in SCORE_INSTANCES]
POINTS = {"merwe": ("merwe", 0.5, 2.0, 0.0), "simplex": ("simplex",)}
# against the fp64 oracle, the log-likelihood tolerance of the UKF instance tests (test_gpu_sigma_instances.py):
# max(10 RTOL, 1e-5) relative to max(|ll|, 1), 1e-2 in fp32 and 1e-5 in fp64; d2 to the same, relative to max(d2, m)
LL_TOL = {dt: max(10 * RTOL[dt], 1e-5) for dt in (np.float64, np.float32)}


def _problem(n, m, hx, N, K, seed, shared_scan):
    rng = np.random.default_rng(seed)
    if hx != "LINEAR":
        x = np.zeros((N, n))
        x[:, 1::2] = rng.uniform(-10, 10, (N, n // 2))
        x[:, 0] = rng.uniform(100, 500, N); x[:, 2] = rng.uniform(-300, 300, N)
        if n == 6:
            x[:, 4] = rng.uniform(20, 200, N)
        sd = np.tile([2.0, 0.5], n // 2)
        rsd = np.array([1.0, 0.005, 0.005])[:m]
        H = None
    else:
        x = rng.normal(0.0, 5.0, (N, n))
        sd = rng.uniform(0.5, 2.0, n)
        rsd = rng.uniform(0.5, 2.0, m)
        H = rng.standard_normal((N, m, n))
    P = _corr_spd(rng, N, n, sd)
    R = _corr_spd(rng, N, m, rsd)
    z0 = oukf.hx_apply(HX[hx], x + sd * rng.standard_normal((N, n)), H)
    z = z0[:, None, :] + 2 * rsd * rng.standard_normal((N, K, m))
    if shared_scan:
        z = z[:1]
    valid = rng.random((N, K)) >= 0.2
    return x, P, R, H, z, valid


def _ukf(n, m, hx, pts, N, dtype, H=None, **kw):
    from filterpy_b200.kalman import (UnscentedKalmanFilter, MerweScaledSigmaPoints, SimplexSigmaPoints, ConstVelFx,
                                      LinearFx, LinearHx, RangeAzElHx, RangeBearingHx)
    h = LinearHx(H) if hx == "LINEAR" else (RangeAzElHx() if hx == "RANGE_AZ_EL" else RangeBearingHx())
    p = SimplexSigmaPoints(n) if pts[0] == "simplex" else MerweScaledSigmaPoints(n, *pts[1:])
    f = ConstVelFx() if n % 2 == 0 else LinearFx(np.eye(n))
    return UnscentedKalmanFilter(n, m, 0.1, h, f, p, n_filters=N, dtype=dtype, **kw)


def _close(got, want, tol, what, scale=None):
    got = np.asarray(got, np.float64)
    scale = np.maximum(np.abs(want), 1.0) if scale is None else scale
    err = np.abs(got - want) / scale
    assert err.max() <= tol, "%s: %.3e" % (what, err.max())


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("points", sorted(POINTS))
@pytest.mark.parametrize("inst", SCORE_INSTANCES, ids=SCORE_IDS)
def test_instance_vs_oracle(inst, points, dtype):
    """Every pre-built instance: N = 1037 (the last CTA holds 13 tracks), K in {1, 7, 33, 300}, per-track and
    shared scans, ~20 % missing candidates."""
    n, m, hx = inst
    pts = POINTS[points]
    N = 1037
    for K in (1, 7, 33, 300):
        for shared in (False, True):
            x, P, R, H, z, valid = _problem(n, m, hx, N, K, seed=K + 1000 * shared, shared_scan=shared)
            u = _ukf(n, m, hx, pts, N, dtype, H=H)
            u.x = x; u.P = P; u.R = R
            ll, maha = u.score_measurements(z, valid=valid)
            torch.cuda.synchronize()
            o = uso.ukf_score_bank(x, P, z, R, pts, hx_model=HX[hx], H=H, valid=valid)
            assert (o["status"] == 0).all()
            what = "K=%d shared=%s" % (K, shared)
            ll, maha = ll.cpu().numpy(), maha.cpu().numpy()
            _close(ll, o["log_likelihood"], LL_TOL[dtype], "ll " + what)
            d2 = o["d2"]
            _close(maha ** 2, d2, LL_TOL[dtype], "d2 " + what, scale=np.maximum(d2, m))
            assert (maha[~valid] == 0).all() and (ll[~valid] == dtype(uso.so.LOG_DBL_MIN)).all()


def _golden_filter(name, dtype, n_filters, f=None):
    """The golden's bank (n_filters) or its filter f in single mode (n_filters None)."""
    from filterpy_b200.kalman import (UnscentedKalmanFilter, MerweScaledSigmaPoints, SimplexSigmaPoints,
                                      JulierSigmaPoints, ConstVelFx, LinearHx, RangeAzElHx, RangeBearingHx,
                                      DeviceHx, DeviceFn)
    from filterpy_b200.common import workloads as wl
    g = load(name)
    n, m = g["x"].shape[1], g["z"].shape[2]
    pts = {"julier": lambda: JulierSigmaPoints(n, kappa=1.5), "simplex_rb": lambda: SimplexSigmaPoints(n),
           "hooks_rb": lambda: MerweScaledSigmaPoints(n, .8, 2., 0.)}.get(name, lambda: MerweScaledSigmaPoints(n, .5, 2., 0.))()
    kw = {}
    if name in ("cv_rae", "julier"):
        hx = RangeAzElHx()
    elif name == "lin":
        hx = LinearHx(np.array([[1., 0, 0, 0], [0, 0, 1, 0]]))
    elif name == "user_rb":
        # the defaults serve the predict a score flushes; the score passes the same values as hx_args
        sel = (lambda v: v) if f is None else (lambda v: float(v[f]))
        hx = DeviceHx(wl.OFFSET_RB_HX_SOURCE, ("sx", "sy"), sx=sel(g["sx"]), sy=sel(g["sy"]))
    else:
        hx = RangeBearingHx()
    if name == "hooks_rb":
        hk = DeviceFn(wl.RB_HOOKS_SOURCE)
        kw = dict(residual_z=hk, z_mean_fn=hk)
    return g, UnscentedKalmanFilter(n, m, float(g["dt"]), hx, ConstVelFx(), pts, n_filters=n_filters, dtype=dtype, **kw)


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("name", sorted(CASES))
def test_goldens_bank_and_single(name, dtype):
    """The reference's log_likelihood / mahalanobis of update(z_ik) after predict(): the whole bank in one call
    (predict pending), then each filter in single mode."""
    g, u = _golden_filter(name, dtype, g_N := load(name)["x"].shape[0])
    u.x = g["x"]; u.P = g["P"]; u.Q = g["Q"]; u.R = g["R"]
    hx_args = dict(sx=g["sx"], sy=g["sy"]) if name == "user_rb" else {}
    u.predict()
    ll, maha = u.score_measurements(g["z"], **hx_args)
    tol = 1e-8 if dtype == np.float64 else LL_TOL[dtype]
    _close(ll.cpu().numpy(), g["ref_ll"], tol, "bank ll")
    _close(maha.cpu().numpy(), g["ref_maha"], tol, "bank maha")
    for f in range(g_N):
        g, s = _golden_filter(name, dtype, None, f)
        s.x = g["x"][f]; s.P = g["P"][f]; s.Q = g["Q"][f]; s.R = g["R"][f]
        s.predict()
        for k in range(g["z"].shape[1]):
            kw = {a: float(v[f]) for a, v in hx_args.items()}
            l1, d1 = s.score_measurements(g["z"][f, k], **kw)
            assert isinstance(l1, float)
            _close(l1, g["ref_ll"][f, k], tol, "single ll")
            _close(d1, g["ref_maha"][f, k], tol, "single maha")


@pytest.mark.gpu
@DTYPES
def test_status_rules(dtype):
    """One track with an indefinite P and one with a singular S get NaN and their status; their neighbours are
    unaffected; single mode raises LinAlgError."""
    n, m, N, K = 4, 2, 300, 9
    x, P, R, H, z, valid = _problem(n, m, "LINEAR", N, K, seed=5, shared_scan=False)
    H[:] = np.array([[1., 0, 0, 0], [0, 0, 1, 0]])
    P[17] = -np.eye(n)
    R[130] = 0.0
    H[130] = 0.0                                                      # S = 0 + R = 0: singular
    u = _ukf(n, m, "LINEAR", POINTS["merwe"], N, dtype, H=H)
    u.x = x; u.P = P; u.R = R
    ll, maha = u.score_measurements(z)
    ll, maha = ll.cpu().numpy(), maha.cpu().numpy()
    o = uso.ukf_score_bank(x, P, z, R, POINTS["merwe"], H=H)
    assert o["status"][17] == 2 and o["status"][130] == 1
    # the status the device writes (the method keeps it to itself; the torch op returns it)
    from filterpy_b200 import _lib, torch_ops
    torch_ops.load()
    tdt = {np.float64: torch.float64, np.float32: torch.float32}[dtype]
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to("cuda", tdt)  # noqa: E731
    _, _, st = torch.ops.bke.ukf_score_measurements(t(x), t(P), t(R), t(z), 0.5, 2.0, 0.0, _lib.BKE_HX_LINEAR, t(H))
    st = st.cpu().numpy()
    assert st[17] == _lib.BKE_STATUS_NOT_PD and st[130] == _lib.BKE_STATUS_SINGULAR_S
    assert (st[ok_tracks := np.setdiff1d(np.arange(N), [17, 130])] == 0).all(), ok_tracks
    assert np.isnan(ll[17]).all() and np.isnan(ll[130]).all() and np.isnan(maha[17]).all()
    ok = np.ones(N, bool); ok[[17, 130]] = False
    _close(ll[ok], o["log_likelihood"][ok], LL_TOL[dtype], "neighbours")
    from filterpy_b200.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, ConstVelFx, LinearHx
    for bad in (17, 130):
        s = UnscentedKalmanFilter(n, m, 0.1, LinearHx(H[bad]), ConstVelFx(), MerweScaledSigmaPoints(n, .5, 2., 0.), dtype=dtype)
        s.x = x[bad]; s.P = P[bad]; s.R = R[bad]
        with pytest.raises(np.linalg.LinAlgError):
            s.score_measurements(z[bad, 0])


def _snapshot(u):
    names = ["x", "P", "S", "SI", "K", "y", "log_likelihood", "x_prior", "P_prior", "z"]
    out = {}
    for k in names:
        v = getattr(u, "_" + k, None) if k != "z" else u._z
        out[k] = None if v is None else v.clone()
    for k in ("_S", "_SI", "_K", "_y", "_ll", "_x_prior", "_P_prior", "_x_post", "_P_post"):
        v = getattr(u, k, None)
        out[k] = None if v is None else v.clone()
    return out


def _same(a, b):
    for k in a:
        if a[k] is None:
            assert b[k] is None, k
        else:
            assert torch.equal(a[k], b[k]), k


@pytest.mark.gpu
@DTYPES
def test_no_mutation_and_pending_predict(dtype):
    """Scoring changes nothing: with no predict pending, x, P and every diagnostic are bit for bit as before and
    the next update equals a run without the score call; with a predict pending, the predict is committed (x_prior /
    P_prior hold it) and score + update matches the oracle's predict + update."""
    from filterpy_b200.common import workloads as wl
    N, K = 1037, 7
    w = wl.ukf_bank_cv3d(N, seed=11, steps=2)

    def make():
        u = _ukf(6, 3, "RANGE_AZ_EL", POINTS["merwe"], N, dtype)
        u.x = w["x"]; u.P = w["P"]; u.Q = w["Q"]; u.R = w["R"]
        u.predict(); u.update(w["zs"][0])
        return u
    cand = np.repeat(w["zs"][1][:, None, :], K, 1)
    a, b = make(), make()
    before = _snapshot(a)
    a.score_measurements(cand)
    torch.cuda.synchronize()
    _same(before, _snapshot(a))
    a.update(w["zs"][1]); b.update(w["zs"][1])
    assert torch.equal(a._x, b._x) and torch.equal(a._P, b._P)

    u = make()
    x0, P0 = u._x.cpu().numpy().astype(np.float64), u._P.cpu().numpy().astype(np.float64)
    u.predict()
    ll, _ = u.score_measurements(cand)
    o = oukf.ukf_step_bank(x0, P0, w["zs"][1], w["Q"], w["R"], 0.1, .5, 2., 0., oukf.FX_CONST_VEL, oukf.HX_RANGE_AZ_EL)
    tol = 1e-6 if dtype == np.float64 else 1e-2
    _close(u.x_prior.cpu().numpy(), o["x_prior"], tol, "x_prior")
    _close(u.P_prior.cpu().numpy(), o["P_prior"], tol, "P_prior")
    u.update(w["zs"][1])
    _close(u.x.cpu().numpy(), o["x"], tol, "x")
    _close(u.P.cpu().numpy(), o["P"], tol, "P", scale=np.maximum(np.abs(o["P"]), 1.0))
    so = uso.ukf_score_bank(o["x_prior"], o["P_prior"], cand, w["R"], POINTS["merwe"], hx_model=oukf.HX_RANGE_AZ_EL)
    _close(ll.cpu().numpy(), so["log_likelihood"], LL_TOL[dtype], "ll after pending predict")


@pytest.mark.gpu
@DTYPES
@pytest.mark.parametrize("points", sorted(POINTS))
def test_torch_op_equals_method(points, dtype):
    from filterpy_b200 import _lib, torch_ops
    torch_ops.load()
    n, m, N, K = 4, 2, 500, 11
    x, P, R, H, z, valid = _problem(n, m, "RANGE_BEARING", N, K, seed=3, shared_scan=False)
    pts = POINTS[points]
    u = _ukf(n, m, "RANGE_BEARING", pts, N, dtype)
    u.x = x; u.P = P; u.R = R
    ll, maha = u.score_measurements(z, valid=valid)
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to("cuda", {np.float64: torch.float64, np.float32: torch.float32}[dtype])  # noqa: E731
    al, be, ka = (0.5, 2.0, 0.0) if points == "merwe" else (1.0, 0.0, 0.0)
    l2, d2, st = torch.ops.bke.ukf_score_measurements(t(x), t(P), t(R), t(z), al, be, ka, _lib.BKE_HX_RANGE_BEARING, None,
                                                      torch.as_tensor(valid, device="cuda").to(torch.uint8).contiguous(),
                                                      points == "simplex")
    assert torch.equal(l2, ll) and torch.equal(d2, maha) and int(st.sum()) == 0


@pytest.mark.gpu
def test_score_shared_memory_limit_of_runtime_models():
    """A run-time model whose score slots (m + m^2 + 1 words per track) exceed a CTA's shared memory steps, and its
    score is refused with a clear error instead of a failed launch."""
    from filterpy_b200.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, ConstVelFx, DeviceHx
    src = """
__device__ void hx(const real *x, real *z, const real *args) { for (int a = 0; a < BKE_DIM_Z; a++) z[a] = x[a % 4] * (a + 1); }
"""
    N, m = 200, 12
    u = UnscentedKalmanFilter(4, m, 0.1, DeviceHx(src), ConstVelFx(), MerweScaledSigmaPoints(4, .5, 2., 0.), n_filters=N)
    u.R = np.eye(m) * 0.5
    u.predict(); u.update(np.zeros((N, m)))
    assert int(u.status.sum().item()) == 0
    with pytest.raises(NotImplementedError, match="shared memory"):
        u.score_measurements(np.zeros((N, 3, m)))
