"""GPU parity: UKF bank (CUDA through the C-ABI) vs the reference's golden vectors and the oracle."""
import numpy as np
import pytest

from gpu_harness import rel_close, RTOL

pytestmark = pytest.mark.gpu


def build(g, dtype, kind, N=None, diagnostics=True):
    from filterpy_b200.kalman import (UnscentedKalmanFilter, MerweScaledSigmaPoints, LinearFx, ConstVelFx,
                                      LinearHx, RangeAzElHx)
    pts = MerweScaledSigmaPoints(6, float(g["alpha"]), float(g["beta"]), float(g["kappa"]))
    fx = LinearFx(g["F"]) if kind == "lin" else ConstVelFx()
    hx = LinearHx(g["H"]) if kind == "lin" else RangeAzElHx()
    N = g["x"].shape[0] if N is None else N
    u = UnscentedKalmanFilter(6, 3, float(g["dt"]), hx, fx, pts, n_filters=N, dtype=dtype, diagnostics=diagnostics)
    u.x = g["x"]; u.P = g["P"]; u.Q = g["Q"]; u.R = g["R"]
    return u


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name,kind", [("ukf_bank_rae", "rae"), ("ukf_bank_lin", "lin")])
def test_ukf_bank_vs_reference_golden(golden, name, kind, dtype):
    g = golden(name)
    u = build(g, dtype, kind)
    rtol = RTOL[dtype]       # fp32: 1e-3 (north_star); measured worst case 9.2e-4 (P_prior of the range/az/el bank)
    for t in range(g["zs"].shape[0]):
        v = g["valid"][t]
        u.predict(); u.update(g["zs"][t], valid=v)
        rel_close(u.x.cpu().numpy(), g["ref_x"][t], rtol, "x t=%d" % t)
        rel_close(u.P.cpu().numpy(), g["ref_P"][t], rtol, "P t=%d" % t)
        rel_close(u.x_prior.cpu().numpy(), g["ref_x_prior"][t], rtol, "x_prior")
        rel_close(u.P_prior.cpu().numpy(), g["ref_P_prior"][t], rtol, "P_prior")
        rel_close(u.K.cpu().numpy()[v], g["ref_K"][t][v], max(rtol, 1e-5), "K")
        rel_close(u.S.cpu().numpy()[v], g["ref_S"][t][v], max(rtol, 1e-5), "S")
        assert int(u.status.sum().item()) == 0


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name,kind", [("ukf_julier_rae", "rae"), ("ukf_julier_lin", "lin")])
def test_ukf_julier_bank_vs_reference_golden(golden, name, kind, dtype):
    """UKF bank on JulierSigmaPoints (sigma_points.py:211-383) against vectors from the reference;
    the linear case has kappa < 0, i.e. a negative centre weight."""
    from filterpy_b200.kalman import UnscentedKalmanFilter, JulierSigmaPoints, LinearFx, ConstVelFx, LinearHx, RangeAzElHx
    g = golden(name)
    pts = JulierSigmaPoints(6, float(g["kappa"]))
    fx = LinearFx(g["F"]) if kind == "lin" else ConstVelFx()
    hx = LinearHx(g["H"]) if kind == "lin" else RangeAzElHx()
    u = UnscentedKalmanFilter(6, 3, float(g["dt"]), hx, fx, pts, n_filters=g["x"].shape[0], dtype=dtype)
    u.x = g["x"]; u.P = g["P"]; u.Q = g["Q"]; u.R = g["R"]
    rtol = RTOL[dtype]
    for t in range(g["zs"].shape[0]):
        v = g["valid"][t]
        u.predict(); u.update(g["zs"][t], valid=v)
        rel_close(u.x.cpu().numpy(), g["ref_x"][t], rtol, "x t=%d" % t)
        rel_close(u.P.cpu().numpy(), g["ref_P"][t], rtol, "P t=%d" % t)
        rel_close(u.x_prior.cpu().numpy(), g["ref_x_prior"][t], rtol, "x_prior")
        rel_close(u.P_prior.cpu().numpy(), g["ref_P_prior"][t], rtol, "P_prior")
        rel_close(u.K.cpu().numpy()[v], g["ref_K"][t][v], max(rtol, 1e-5), "K")
        rel_close(u.S.cpu().numpy()[v], g["ref_S"][t][v], max(rtol, 1e-5), "S")
        assert int(u.status.sum().item()) == 0


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name,linear", [("ukf_user_ct_rb", False), ("ukf_user_ct_lin", True)])
def test_ukf_user_models_vs_reference_golden(golden, name, linear, dtype):
    """fx / hx OUTSIDE the built-in set, compiled at run time from CUDA text (NVRTC): coordinated turn with a
    per-filter turn rate (fx_args of UKF.predict, UKF.py:364) and range / bearing from an offset sensor
    (hx_args of UKF.update, UKF.py:413) — against the reference run with the same functions as Python
    callables; the second case pairs the user fx with the built-in linear hx."""
    from filterpy_b200.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, DeviceFx, DeviceHx, LinearHx
    from filterpy_b200.common import workloads as wl
    g = golden(name)
    N = g["x"].shape[0]
    fx = DeviceFx(wl.CT_FX_SOURCE, arg_names=("omega",))
    hx = LinearHx(g["H"]) if linear else DeviceHx(wl.OFFSET_RB_HX_SOURCE, arg_names=("sx", "sy"))
    pts = MerweScaledSigmaPoints(4, float(g["alpha"]), float(g["beta"]), float(g["kappa"]))
    u = UnscentedKalmanFilter(4, 2, float(g["dt"]), hx, fx, pts, n_filters=N, dtype=dtype)
    u.x = g["x"]; u.P = g["P"]; u.Q = g["Q"]; u.R = g["R"]
    rtol = RTOL[dtype]
    for t in range(g["zs"].shape[0]):
        v = g["valid"][t]
        u.predict(omega=g["omega"])
        if linear:
            u.update(g["zs"][t], valid=v)
        else:
            u.update(g["zs"][t], valid=v, sx=float(g["sensor"][0]), sy=float(g["sensor"][1]))
        rel_close(u.x.cpu().numpy(), g["ref_x"][t], rtol, "x t=%d" % t)
        rel_close(u.P.cpu().numpy(), g["ref_P"][t], rtol, "P t=%d" % t)
        rel_close(u.x_prior.cpu().numpy(), g["ref_x_prior"][t], rtol, "x_prior")
        rel_close(u.P_prior.cpu().numpy(), g["ref_P_prior"][t], rtol, "P_prior")
        rel_close(u.K.cpu().numpy()[v], g["ref_K"][t][v], max(rtol, 1e-5), "K")
        rel_close(u.S.cpu().numpy()[v], g["ref_S"][t][v], max(rtol, 1e-5), "S")
        assert int(u.status.sum().item()) == 0


def test_ukf_user_model_errors():
    from filterpy_b200 import _lib
    from filterpy_b200.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, DeviceFx, LinearHx
    from filterpy_b200.common import workloads as wl
    pts = MerweScaledSigmaPoints(4, .5, 2., 0.)
    H = np.eye(2, 4)
    with pytest.raises(ValueError, match="no_such_thing"):      # the compiler's message reaches the caller
        UnscentedKalmanFilter(4, 2, .1, LinearHx(H), DeviceFx("__device__ void fx(const real *x, real *o, real dt, const real *a) { o[0] = no_such_thing; }"),
                              pts, n_filters=4)
    u = UnscentedKalmanFilter(4, 2, .1, LinearHx(H), DeviceFx(wl.CT_FX_SOURCE, arg_names=("omega",)), pts, n_filters=4)
    u.predict()
    with pytest.raises(TypeError, match="omega"):                 # the model's argument has no value
        u.update(np.zeros((4, 2)))


@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-6), (np.float32, 2e-3)])
def test_ukf_user_fx_rts_smoother_vs_reference_golden(golden, dtype, tol):
    """UKF.rts_smoother (UKF.py:634-739) around a user-supplied fx: the smoother kernel is compiled at run
    time with the same text; the reference ran the Python callable with its default turn rate (:712)."""
    import torch
    from filterpy_b200.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, DeviceFx, LinearHx
    from filterpy_b200.common import workloads as wl
    g = golden("ukf_user_rts")
    T, N, n = g["Xs"].shape
    u = UnscentedKalmanFilter(4, 2, float(g["dt"]), LinearHx(g["H"]), DeviceFx(wl.CT_FX_SOURCE, arg_names=("omega",), omega=float(g["omega"])),
                              MerweScaledSigmaPoints(4, float(g["alpha"]), float(g["beta"]), float(g["kappa"])), n_filters=N, dtype=dtype)
    u.Q = g["Q"]
    x, P, K = u.rts_smoother(torch.from_numpy(g["Xs"]), torch.from_numpy(g["Ps"]))
    from test_gpu_next_rows import rel_close as close_abs          # the built-in models' RTS tests use the same measure
    close_abs(x.cpu().numpy(), g["x"], tol)
    close_abs(P.cpu().numpy(), g["P"], tol, atol_scale=4.0 if dtype == np.float32 else 1.0)
    close_abs(K.cpu().numpy(), g["K"], tol * 10, atol_scale=4.0)


def test_julier_sigma_points_standalone(golden):
    from filterpy_b200.kalman import JulierSigmaPoints
    g = golden("julier_sigma")
    for i in range(4):
        pts = JulierSigmaPoints(4, float(g["kappa%d" % i]))
        rel_close(pts.sigma_points(g["x"], g["P"]), g["sigmas%d" % i], 1e-12, "julier sigmas kappa=%g" % pts.kappa)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_ukf_256k_vs_oracle_subset(dtype):
    """BASELINE config 4 size (2^18 filters, n=6, m=3, range/azimuth/elevation): full bank on the
    GPU, a 4096-filter random subset checked against the oracle, 3 epochs."""
    from filterpy_b200.common import workloads as wl
    from oracle import ukf as oukf
    N, T = 1 << 18, 3
    w = wl.ukf_bank_cv3d(N, seed=2468, steps=T)
    g = dict(w, alpha=0.5, beta=2.0, kappa=0.0, dt=0.1)
    u = build(g, dtype, "rae", diagnostics=False)
    sel = np.random.default_rng(0).choice(N, 4096, replace=False)
    x, P = w["x"][sel], w["P"][sel]
    for t in range(T):
        u.predict(); u.update(w["zs"][t])
        o = oukf.ukf_step_bank(x, P, w["zs"][t][sel], w["Q"][sel], w["R"][sel], 0.1, 0.5, 2.0, 0.0,
                               oukf.FX_CONST_VEL, oukf.HX_RANGE_AZ_EL)
        x, P = o["x"], o["P"]
    rtol = RTOL[dtype]       # fp32: 1e-3 (north_star); measured worst case 8.8e-4 after 3 steps of the 2^18 bank
    rel_close(u.x.cpu().numpy()[sel], x, rtol, "x"); rel_close(u.P.cpu().numpy()[sel], P, rtol, "P")


def test_ukf_matches_linear_kf_on_linear_model():
    """test_ukf.py:893-979: on a linear model the UKF equals the linear KF (atol 1e-7 there)."""
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.common import workloads as wl
    N, T = 512, 10
    w = wl.ukf_bank_cv3d(N, seed=1, steps=T, linear_hx=True)
    g = dict(w, alpha=0.5, beta=2.0, kappa=0.0, dt=0.1)
    u = build(g, np.float64, "lin", diagnostics=False)
    kf = KalmanFilter(6, 3, n_filters=N, diagnostics=False)
    kf.x = w["x"]; kf.P = w["P"]; kf.F = w["F"]; kf.H = w["H"]; kf.Q = w["Q"]; kf.R = w["R"]
    for t in range(T):
        u.predict(); u.update(w["zs"][t])
        kf.predict(); kf.update(w["zs"][t])
    np.testing.assert_allclose(u.x.cpu().numpy(), kf.x.cpu().numpy(), rtol=1e-7, atol=1e-7)
    np.testing.assert_allclose(u.P.cpu().numpy(), kf.P.cpu().numpy(), rtol=1e-6, atol=1e-7)


def test_ukf_single_mode_batch_filter_equals_loop(golden):
    """test_ukf.py:506: batch_filter == the predict/update loop (bit-equal there)."""
    from filterpy_b200.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, ConstVelFx, RangeAzElHx
    g = golden("ukf_bank_rae")

    def mk():
        u = UnscentedKalmanFilter(6, 3, 0.1, RangeAzElHx(), ConstVelFx(), MerweScaledSigmaPoints(6, .5, 2., 0.))
        u.x = g["x"][0]; u.P = g["P"][0]; u.Q = g["Q"][0]; u.R = g["R"][0]
        return u
    a, b = mk(), mk()
    zs = [g["zs"][t, 0] for t in range(5)]
    M, C = a.batch_filter(zs)
    xs = []
    for z in zs:
        b.predict(); b.update(z); xs.append(b.x.copy())
    assert M.shape == (5, 6) and C.shape == (5, 6, 6)
    assert np.array_equal(M, np.array(xs))
    with pytest.raises(NotImplementedError):
        UnscentedKalmanFilter(6, 3, 0.1, lambda x: x[:3], lambda x, dt: x, MerweScaledSigmaPoints(6, .5, 2., 0.))
    with pytest.raises(TypeError):
        a.batch_filter(3.0)


def test_ukf_not_pd_status():
    from filterpy_b200.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, ConstVelFx, LinearHx
    H = np.zeros((1, 2)); H[0, 0] = 1
    u = UnscentedKalmanFilter(2, 1, 1.0, LinearHx(H), ConstVelFx(), MerweScaledSigmaPoints(2, .5, 2., 1.), n_filters=3)
    P = np.array([np.eye(2), -np.eye(2), np.eye(2)])
    u.P = P
    u.predict(); u.update(np.zeros((3, 1)))
    assert u.status.cpu().numpy().tolist() == [0, 2, 0]


def test_sigma_points_and_unscented_transform_standalone(golden):
    """sigma_points.py:124-177 / unscented_transform.py:99-128 as stand-alone calls (test_ukf.py:112-189)."""
    import torch
    from filterpy_b200.kalman import MerweScaledSigmaPoints, unscented_transform
    from oracle import ukf as oukf
    g = golden("ukf_sigma")
    pts = MerweScaledSigmaPoints(6, float(g["alpha"]), float(g["beta"]), float(g["kappa"]))
    sig = pts.sigma_points(g["x"], g["P"])
    assert sig.shape == (13, 6)
    np.testing.assert_allclose(sig, g["sigmas"], rtol=1e-12, atol=1e-13)
    # sigma points + UT recover the mean and covariance (test_ukf.py:132-134)
    x, P = unscented_transform(sig, pts.Wm, pts.Wc)
    np.testing.assert_allclose(x, g["x"], atol=1e-12); np.testing.assert_allclose(P, g["P"], atol=1e-11)
    # bank, both dtypes, against the oracle
    rng = np.random.default_rng(0)
    N = 1000
    A = rng.standard_normal((N, 6, 6)); Pb = np.einsum("nij,nkj->nik", A, A) + np.eye(6); xb = rng.standard_normal((N, 6))
    for dt, tol in ((torch.float64, 1e-10), (torch.float32, 2e-4)):
        sb = pts.sigma_points(torch.from_numpy(xb).cuda().to(dt), torch.from_numpy(Pb).cuda().to(dt))
        want = oukf.merwe_sigma_points(xb, Pb, pts.alpha, pts.beta, pts.kappa)
        np.testing.assert_allclose(sb.cpu().numpy(), want, rtol=tol, atol=tol * 10)
        Q = np.eye(6) * 0.1
        xm, Pm = unscented_transform(sb, pts.Wm, pts.Wc, noise_cov=Q)
        wx, wP = oukf.unscented_transform(want, pts.Wm, pts.Wc, Q)
        np.testing.assert_allclose(xm.cpu().numpy(), wx, rtol=tol * 10, atol=tol * 100)
        np.testing.assert_allclose(Pm.cpu().numpy(), wP, rtol=tol * 100, atol=tol * 1000)
    with pytest.raises(np.linalg.LinAlgError):
        pts.sigma_points(np.zeros(6), -np.eye(6))
    with pytest.raises(NotImplementedError):
        unscented_transform(sig, pts.Wm, pts.Wc, mean_fn=lambda s, w: s[0])
