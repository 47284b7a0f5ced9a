"""GPU parity: CKF bank (CUDA through the mirror and the C-ABI) vs the reference's golden vectors and the oracle."""
import numpy as np
import pytest

from gpu_harness import rel_close, RTOL

pytestmark = pytest.mark.gpu


def _ops(g):
    return [str(o) for o in g["ops"]] if "ops" in g else ["predict+update"] * g["zs"].shape[0]


def make(name, g, dtype, N=None, diagnostics=True):
    from filterpy_b200.kalman import CubatureKalmanFilter, LinearFx, ConstVelFx, LinearHx, RangeAzElHx, DeviceFx, DeviceHx
    from filterpy_b200.common import workloads as wl
    if name == "ckf_user_ct_rb":
        fx, hx, n, m = DeviceFx(wl.CT_FX_SOURCE, arg_names=("omega",)), DeviceHx(wl.OFFSET_RB_HX_SOURCE, arg_names=("sx", "sy")), 4, 2
    elif name == "ckf_bank_rae":
        fx, hx, n, m = ConstVelFx(), RangeAzElHx(), 6, 3
    else:
        fx, hx, n, m = LinearFx(g["F"]), LinearHx(g["H"]), 6, 3
    N = g["x"].shape[0] if N is None else N
    c = CubatureKalmanFilter(n, m, float(g["dt"]), hx, fx, n_filters=N, dtype=dtype, diagnostics=diagnostics)
    c.x = g["x"]; c.P = g["P"]; c.Q = g["Q"]; c.R = g["R"]
    return c


def run_ops(c, name, g, t, op):
    fa = (g["omega"],) if name == "ckf_user_ct_rb" else ()
    ha = (float(g["sensor"][0]), float(g["sensor"][1])) if name == "ckf_user_ct_rb" else ()
    if op.startswith("predict"):
        c.predict(fx_args=fa)
    if op == "predict+read+update":
        c.x                                               # flushes the predict on its own
    if op == "predict+none":
        c.update(None)
    else:
        c.update(g["zs"][t], R=0.5 if op == "predict+update_R" else None, hx_args=ha, valid=g["valid"][t])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["ckf_bank_rae", "ckf_bank_lin", "ckf_user_ct_rb", "ckf_call_order"])
def test_ckf_vs_reference_golden(golden, name, dtype):
    """Every recorded output after every call, including updates without a predict (stale points) and
    an update on a new filter (zero points), the user models through NVRTC and a scalar R."""
    g = golden(name)
    c = make(name, g, dtype)
    rtol = RTOL[dtype]
    for t, op in enumerate(_ops(g)):
        run_ops(c, name, g, t, op)
        v = g["valid"][t] & (op != "predict+none")
        rel_close(c.x.cpu().numpy(), g["ref_x"][t], rtol, "x t=%d" % t)
        rel_close(c.P.cpu().numpy(), g["ref_P"][t], rtol, "P t=%d" % t)
        rel_close(c.x_prior.cpu().numpy(), g["ref_x_prior"][t], rtol, "x_prior")
        rel_close(c.P_prior.cpu().numpy(), g["ref_P_prior"][t], rtol, "P_prior")
        rel_close(c.sigmas_f.cpu().numpy(), g["ref_sigmas_f"][t], rtol, "sigmas_f")
        if v.any():
            # the call-order case ends with an update that reuses the last predict's points and applies the
            # gain a second time; fp32 K is then within 1.7e-3 of the reference (measured on the H100)
            ktol = 2e-3 if (name == "ckf_call_order" and dtype == np.float32) else max(rtol, 1e-5)
            rel_close(c.K.cpu().numpy()[v], g["ref_K"][t][v], ktol, "K")
            rel_close(c.S.cpu().numpy()[v], g["ref_S"][t][v], max(rtol, 1e-5), "S")
            # y = z - z^ cancels most digits of z: compare the predicted measurement z^ = z - y instead
            zf = g["zs"][t].astype(dtype).astype(np.float64)          # the z the filter was given
            rel_close((zf - c.y.cpu().numpy())[v], (g["zs"][t] - g["ref_y"][t])[v], max(rtol, 1e-5), "z - y")
            rel_close(c.log_likelihood.cpu().numpy()[v], g["ref_loglik"][t][v], max(10 * rtol, 1e-5), "loglik")
        assert int(c.status.sum().item()) == 0


def test_split_equals_fused_and_diagnostics_off(golden):
    g = golden("ckf_bank_rae")
    a, b = make("ckf_bank_rae", g, np.float64), make("ckf_bank_rae", g, np.float64)
    for t in range(3):
        a.predict(); a.update(g["zs"][t])
        b.predict(); b.x; b.update(g["zs"][t])               # predict-only launch, then update-only launch
        assert np.array_equal(a.x.cpu().numpy(), b.x.cpu().numpy())
        assert np.array_equal(a.P.cpu().numpy(), b.P.cpu().numpy())
    c = make("ckf_bank_rae", g, np.float64, diagnostics=False)
    c.predict(); c.update(g["zs"][0])
    with pytest.raises(NotImplementedError, match="diagnostics"):
        c.update(g["zs"][1])
    c.predict(); c.x; c.update(g["zs"][1])                     # a predict on its own keeps its points
    d = make("ckf_bank_rae", g, np.float64, diagnostics=False)
    d.update(g["zs"][0])                                      # a new filter's zero points, as in the reference


def test_missing_measurements_not_pd_and_single_mode():
    from filterpy_b200.kalman import CubatureKalmanFilter, ConstVelFx, LinearHx
    H = np.zeros((1, 2)); H[0, 0] = 1
    c = CubatureKalmanFilter(2, 1, 1.0, LinearHx(H), ConstVelFx(), n_filters=3)
    c.P = np.array([np.eye(2), -np.eye(2), np.eye(2)])
    c.predict(); c.update(np.zeros((3, 1)), valid=[1, 1, 0])
    assert c.status.cpu().numpy().tolist() == [0, 2, 0]
    rel_close(c.x.cpu().numpy()[2], c.x_prior.cpu().numpy()[2], 0, "valid=0 keeps the prior")
    rel_close(c.P.cpu().numpy()[2], c.P_prior.cpu().numpy()[2], 0, "valid=0 keeps the prior")
    c.predict(); xp = c.x.clone(); c.update(None)
    assert np.array_equal(c.x.cpu().numpy(), xp.cpu().numpy(), equal_nan=True)     # filter 1 is NaN (not PD)
    s = CubatureKalmanFilter(2, 1, 1.0, LinearHx(H), ConstVelFx())
    s.P = -np.eye(2)
    s.predict()
    with pytest.raises(np.linalg.LinAlgError):
        s.update(np.array([1.0]))
    with pytest.raises(NotImplementedError):
        CubatureKalmanFilter(2, 1, 1.0, lambda x: x[:1], lambda x, dt: x)


@pytest.mark.parametrize("shared", [True, False])
def test_ragged_bank_and_model_strides(shared):
    """N not a multiple of the 128-filter CTA; F, H, Q, R shared by the bank or per filter."""
    from filterpy_b200.kalman import CubatureKalmanFilter, LinearFx, LinearHx
    from filterpy_b200.common import workloads as wl
    from oracle import ckf as ockf
    N = 1000 + 37
    w = wl.ukf_bank_cv3d(N, seed=4, steps=2, linear_hx=True)
    F, H, Q, R = w["F"], w["H"], w["Q"], w["R"]
    if not shared:
        F = np.broadcast_to(F, (N, 6, 6)).copy() * (1 + 1e-3 * np.arange(N))[:, None, None]
        H = np.broadcast_to(H, (N, 3, 6)).copy()
    else:
        Q, R = Q[0], R[0]
    c = CubatureKalmanFilter(6, 3, 0.1, LinearHx(H), LinearFx(F), n_filters=N, diagnostics=False)
    c.x = w["x"]; c.P = w["P"]; c.Q = Q; c.R = R
    x, P = w["x"], w["P"]
    for t in range(2):
        c.predict(); c.update(w["zs"][t])
        o = ockf.ckf_step_bank(x, P, w["zs"][t], Q, R, 0.1, ockf.FX_LINEAR, ockf.HX_LINEAR, F=F, H=H)
        x, P = o["x"], o["P"]
    rel_close(c.x.cpu().numpy(), x, 1e-9, "x"); rel_close(c.P.cpu().numpy(), P, 1e-9, "P")


def _raw_moment_cov(X, noise):
    """ckf_transform's raw second moments in the points' own precision (CubatureKalmanFilter.py:89-96)."""
    m = X.shape[-2]
    x = X.sum(axis=-2) / X.dtype.type(m)
    P = np.einsum("nka,nkb->nab", X, X) - X.dtype.type(m) * np.einsum("na,nb->nab", x, x)
    return P * X.dtype.type(1.0 / m) + noise


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_ckf_256k_vs_oracle_subset(dtype):
    """2^18 filters, n=6, m=3, CV + range/azimuth/elevation (the UKF's C4 geometry): the whole bank on
    the GPU, a 4096-filter subset checked against the fp64 centred oracle.  In fp32 the raw-moment form of
    the reference would miss the 1e-3 tolerance on this geometry; the test shows that it does."""
    from filterpy_b200.common import workloads as wl
    from oracle import ckf as ockf
    N, T = 1 << 18, 3
    w = wl.ukf_bank_cv3d(N, seed=2468, steps=T)
    g = dict(w, dt=0.1)
    c = make("ckf_bank_rae", g, dtype, diagnostics=False)
    sel = np.random.default_rng(0).choice(N, 4096, replace=False)
    x, P = w["x"][sel], w["P"][sel]
    raw_err = 0.0
    for t in range(T):
        c.predict(); c.update(w["zs"][t])
        o = ockf.ckf_step_bank(x, P, w["zs"][t][sel], w["Q"][sel], w["R"][sel], 0.1, ockf.FX_CONST_VEL, ockf.HX_RANGE_AZ_EL)
        if t == 0:
            raw = _raw_moment_cov(o["sigmas_f"].astype(np.float32), w["Q"][sel].astype(np.float32))
            raw_err = np.abs(raw - o["P_prior"]).max() / np.abs(o["P_prior"]).max()
        x, P = o["x"], o["P"]
    rtol = RTOL[dtype]
    rel_close(c.x.cpu().numpy()[sel], x, rtol, "x"); rel_close(c.P.cpu().numpy()[sel], P, rtol, "P")
    assert raw_err > 1e-3, raw_err                    # what the centred sums avoid


def test_torch_op_equals_mirror(golden):
    import torch
    from filterpy_b200 import torch_ops, _lib
    ops = torch_ops.load()
    g = golden("ckf_bank_rae")
    c = make("ckf_bank_rae", g, np.float64, diagnostics=False)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()      # noqa: E731
    x, P = ops.ckf_step(dev(g["x"]), dev(g["P"]), dev(g["Q"]), dev(g["R"]), dev(g["zs"][0]), 0.1,
                        _lib.BKE_FX_CONST_VEL, _lib.BKE_HX_RANGE_AZ_EL)
    c.predict(); c.update(g["zs"][0])
    assert torch.equal(x, c.x) and torch.equal(P, c.P)


def test_ukf_and_ckf_handles_do_not_mix():
    import ctypes
    import torch
    from filterpy_b200 import _lib
    from filterpy_b200.common import workloads as wl
    lib = _lib.load()
    inc = _lib.kernel_include_dirs().encode()
    hu, hc, he = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    _lib.check(lib.bke_ukf_model_compile(4, 2, 1, _lib.BKE_FX_USER, _lib.BKE_HX_LINEAR, wl.CT_FX_SOURCE.encode(), inc, ctypes.byref(hu)))
    _lib.check(lib.bke_ckf_model_compile(4, 2, 1, _lib.BKE_FX_USER, _lib.BKE_HX_LINEAR, wl.CT_FX_SOURCE.encode(), inc, ctypes.byref(hc)))
    _lib.check(lib.bke_enkf_model_compile(4, 2, 1, _lib.BKE_FX_USER, _lib.BKE_HX_LINEAR, wl.CT_FX_SOURCE.encode(), inc, ctypes.byref(he)))
    N = 4
    t = {k: torch.zeros(s, dtype=torch.float64, device="cuda") for k, s in
         dict(x=(N, 4), P=(N, 4, 4), Q=(4, 4), R=(2, 2), H=(2, 4), z=(N, 2), sf=(N, 8, 4), args=(1,)).items()}
    for cls in (_lib.UkfArgs, _lib.CkfArgs):
        a = cls()
        a.n_filters, a.dim_x, a.dim_z, a.dtype = N, 4, 2, 1
        a.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
        a.fx_model, a.hx_model = _lib.BKE_FX_USER, _lib.BKE_HX_LINEAR
        a.x = a.x_out = t["x"].data_ptr(); a.P = a.P_out = t["P"].data_ptr()
        a.Q, a.R, a.H, a.z = t["Q"].data_ptr(), t["R"].data_ptr(), t["H"].data_ptr(), t["z"].data_ptr()
        if cls is _lib.UkfArgs:
            a.alpha, a.beta, a.kappa = 0.5, 2.0, 0.0
            rc = lib.bke_ukf_step_model(a, hc, t["args"].data_ptr(), 0, None, 0, None)
            assert rc == _lib.BKE_ERR_BAD_ARG and b"compiled for the CKF" in lib.bke_last_error(), rc
            rc = lib.bke_ukf_step_model(a, he, t["args"].data_ptr(), 0, None, 0, None)
            assert b"compiled for the EnKF" in lib.bke_last_error()        # the family the handle was compiled for
        else:
            a.sigmas_f = t["sf"].data_ptr()
            rc = lib.bke_ckf_step_model(a, hu, t["args"].data_ptr(), 0, None, 0, None)
            assert b"compiled for the UKF" in lib.bke_last_error()
        assert rc == _lib.BKE_ERR_BAD_ARG, rc
    a = _lib.CkfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags = N, 4, 2, 1, _lib.BKE_DO_UPDATE
    a.fx_model, a.hx_model = _lib.BKE_FX_CONST_VEL, _lib.BKE_HX_LINEAR
    a.x = a.x_out = t["x"].data_ptr(); a.P = a.P_out = t["P"].data_ptr()
    a.R, a.H, a.z = t["R"].data_ptr(), t["H"].data_ptr(), t["z"].data_ptr()
    assert lib.bke_ckf_step(a, None) == _lib.BKE_ERR_BAD_ARG             # update-only without sigmas_f
    lib.bke_ukf_model_free(hu); lib.bke_ukf_model_free(hc); lib.bke_ukf_model_free(he)
