"""CPU: the simplex point set (SimplexSigmaPoints) — the oracle against the reference's golden vectors, the
kernels' closed form of the offsets against the oracle, the mirror object, and the simplex programs through
NVRTC (no GPU needed)."""
import ctypes

import numpy as np
import pytest

import ukf_hooks_oracle as oh
import ukf_simplex_oracle as osx
from oracle import ukf as oukf
from filterpy_b200.common import workloads as wl

SIGMA_NS = (1, 2, 3, 4, 6, 9)
BANKS = {"ukf_simplex_bank_rae": (oukf.FX_CONST_VEL, oukf.HX_RANGE_AZ_EL),
         "ukf_simplex_bank_rb": (oukf.FX_CONST_VEL, oukf.HX_RANGE_BEARING),
         "ukf_simplex_bank_lin": (oukf.FX_LINEAR, oukf.HX_LINEAR)}


def _err(a, b):
    return np.abs(np.asarray(a, float) - b).max() / max(np.abs(b).max(), 1e-300)


def hx_rb(x):
    return np.array([np.sqrt(x[0] * x[0] + x[2] * x[2]), np.arctan2(x[2], x[0])])


def fx_cv(x, dt):
    return oukf.fx_apply(oukf.FX_CONST_VEL, x, dt)


# ------------------------------------------------------------------------------------------- oracle
def test_sigma_points_oracle_matches_golden(golden):
    g = golden("ukf_simplex_sigma")
    for n in SIGMA_NS:
        x, P = g["x%d" % n], g["P%d" % n]
        assert np.array_equal(osx.simplex_sigma_points(x, P), g["sigmas%d" % n]), n
        Wm, Wc = osx.simplex_weights(n)
        assert Wm is Wc and np.array_equal(Wm, g["Wm%d" % n])
    x = g["x_scalar"]
    assert np.array_equal(osx.simplex_sigma_points(x, np.eye(3) * float(g["P_scalar"])), g["sigmas_scalar"])


@pytest.mark.parametrize("n", range(1, 17))
def test_closed_form_matches_oracle(n):
    """The offsets the kernels form (suffix sums of scaled rows of U) against the reference's Istar product."""
    rng = np.random.default_rng(n)
    A = rng.standard_normal((8, n, n))
    P = A @ np.swapaxes(A, 1, 2) + 0.1 * np.eye(n)
    x = rng.standard_normal((8, n))
    want = osx.simplex_sigma_points(x, P) - x[:, None, :]
    got = osx.simplex_offsets_closed_form(P)
    assert _err(got, want) < 1e-14
    # the sparsity the register plan relies on: D_j (j >= 2) is zero left of column j-1, D_n is e_{n-1} * c
    for j in range(2, n + 1):
        assert not got[:, j, :j - 1].any()


@pytest.mark.parametrize("name", sorted(BANKS))
def test_bank_oracle_matches_golden(golden, name):
    g = golden(name)
    fxm, hxm = BANKS[name]
    F = g["F"] if fxm == oukf.FX_LINEAR else None
    H = g["H"] if hxm == oukf.HX_LINEAR else None
    x, P = g["x"], g["P"]
    for t in range(g["zs"].shape[0]):
        R = g["R_override"] if ("R_override" in g and t % 2) else g["R"]
        v = g["valid"][t]
        o = osx.ukf_step_bank(x, P, g["zs"][t], g["Q"], R, float(g["dt"]), fxm, hxm, F=F, H=H, valid=v)
        x, P = o["x"], o["P"]
        for k in ("x", "P", "x_prior", "P_prior"):
            assert _err(o[k], g["ref_" + k][t]) < 1e-9, (k, t)
        for k in ("K", "S", "y"):
            assert _err(o[k][v], g["ref_" + k][t][v]) < 1e-9, (k, t)


def test_user_model_oracle_matches_golden(golden):
    g = golden("ukf_simplex_user_ct_rb")
    sx, sy = g["sensor"]
    for f in range(g["x"].shape[0]):
        x, P = g["x"][f], g["P"][f]
        for t in range(g["zs"].shape[0]):
            x, P, sf = osx.ukf_predict_single(x, P, g["Q"][f], lambda s, dt: wl.ct_fx(s, dt, g["omega"][f]), float(g["dt"]))
            if g["valid"][t, f]:
                x, P, y, K, S, SI = osx.ukf_update_single(x, P, sf, g["zs"][t, f], g["R"][f], lambda s: wl.offset_rb_hx(s, sx, sy))
                assert _err(K, g["ref_K"][t, f]) < 1e-9 and _err(S, g["ref_S"][t, f]) < 1e-9
            assert _err(x, g["ref_x"][t, f]) < 1e-9 and _err(P, g["ref_P"][t, f]) < 1e-9


@pytest.mark.parametrize("case", ["cv", "ct"])
def test_rts_oracle_matches_golden(golden, case):
    g = golden("ukf_simplex_rts")
    om, dt = float(g["omega"]), float(g["dt"])
    fx = fx_cv if case == "cv" else (lambda s, dt: wl.ct_fx(s, dt, om))
    Xs, Ps = g[case + "_Xs"], g[case + "_Ps"]
    T, N, _ = Xs.shape
    for f in range(N):
        xs, ps, ks = osx.ukf_rts_smoother(Xs[:, f], Ps[:, f], g[case + "_Q"][f], fx, [dt] * T)
        assert _err(xs, g[case + "_ref_x"][:, f]) < 1e-9 and _err(ps, g[case + "_ref_P"][:, f]) < 1e-9
        assert _err(ks, g[case + "_ref_K"][:, f]) < 1e-9


def test_hooks_oracle_matches_golden(golden):
    """residual_z / z_mean_fn on the simplex points, one filter at a time (UKF.py:393-481); without them the
    same filters cross the +-pi cut into a different answer."""
    g = golden("ukf_simplex_hooks_rb")
    Wm, Wc = osx.simplex_weights(4)

    def run(hooked):
        xs = np.zeros_like(g["ref_x"])
        for f in range(g["x"].shape[0]):
            x, P = g["x"][f], g["P"][f]
            for t in range(g["zs"].shape[0]):
                sf = np.array([fx_cv(s, float(g["dt"])) for s in osx.simplex_sigma_points(x, P)])
                x, P = oh.unscented_transform(sf, Wm, Wc, g["Q"][f])
                if g["valid"][t, f]:
                    sig = osx.simplex_sigma_points(x, P)
                    sh = np.array([hx_rb(s) for s in sig])
                    rz = wl.rb_residual_z if hooked else np.subtract
                    zp, S = oh.unscented_transform(sh, Wm, Wc, g["R"][f], wl.rb_z_mean if hooked else None, rz)
                    Pxz = sum(Wc[k] * np.outer(sig[k] - x, rz(sh[k], zp)) for k in range(5))
                    K = Pxz @ np.linalg.inv(S)
                    x = x + K @ rz(g["zs"][t, f], zp)
                    P = P - K @ S @ K.T
                xs[t, f] = x
        return xs
    xs = run(True)
    assert _err(xs, g["ref_x"]) < 1e-9
    assert np.abs(run(False) - g["ref_x"]).max() > 1.0


# ------------------------------------------------------------------------------------------- mirror
def test_mirror_object():
    from filterpy_b200.kalman import SimplexSigmaPoints
    for n in SIGMA_NS:
        p = SimplexSigmaPoints(n)
        assert p.num_sigmas() == n + 1 and p.n == n and p.alpha == 1
        assert p.Wm is p.Wc and np.array_equal(p.Wm, np.full(n + 1, 1. / (n + 1)))
    p = SimplexSigmaPoints(4, alpha=0.3)
    assert p.alpha == 0.3 and "alpha=0.3" in repr(p) and "n=4" in repr(p)
    with pytest.raises(NotImplementedError):
        SimplexSigmaPoints(4, sqrt_method=np.linalg.cholesky)
    with pytest.raises(NotImplementedError):
        SimplexSigmaPoints(4, subtract=np.subtract)


def test_compute_without_a_device_raises():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from filterpy_b200 import _lib
    from filterpy_b200.kalman import SimplexSigmaPoints, UnscentedKalmanFilter, ConstVelFx, RangeBearingHx
    with pytest.raises(_lib.BkeError):
        SimplexSigmaPoints(2).sigma_points(np.zeros(2), np.eye(2))
    with pytest.raises(_lib.BkeError):
        UnscentedKalmanFilter(4, 2, 1.0, RangeBearingHx(), ConstVelFx(), SimplexSigmaPoints(4), n_filters=8)
    lib = _lib.load()
    x, P, sig = np.zeros((1, 2)), np.eye(2)[None].copy(), np.zeros((1, 3, 2))
    assert lib.bke_simplex_sigma_points(1, 2, _lib.BKE_F64, x.ctypes.data, P.ctypes.data, sig.ctypes.data, None, None) == _lib.BKE_ERR_CUDA
    assert lib.bke_simplex_sigma_points(1, 33, _lib.BKE_F64, x.ctypes.data, P.ctypes.data, sig.ctypes.data, None, None) == _lib.BKE_ERR_BAD_ARG


# ------------------------------------------------------------------------------------------- NVRTC
def _lib():
    from filterpy_b200 import _lib
    return _lib, _lib.load(), _lib.kernel_include_dirs().encode()


@pytest.mark.parametrize("dtype", [0, 1])
def test_simplex_programs_compile_with_nvrtc(dtype):
    L, lib, inc = _lib()
    S = L.BKE_UKF_SIMPLEX
    user = (wl.CT_FX_SOURCE + "\n" + wl.OFFSET_RB_HX_SOURCE).encode()
    assert lib.bke_debug_ukf_model_points_cubin_bytes(4, 2, dtype, L.BKE_FX_USER, L.BKE_HX_USER, 0, S, user, inc) > 0
    assert lib.bke_debug_ukf_model_points_cubin_bytes(4, 2, dtype, L.BKE_FX_USER, L.BKE_HX_LINEAR, 0, S, wl.CT_FX_SOURCE.encode(), inc) > 0
    rb = wl.RB_HOOKS_SOURCE.encode()
    mask = L.BKE_HOOK_RESIDUAL_Z | L.BKE_HOOK_Z_MEAN
    assert lib.bke_debug_ukf_model_points_cubin_bytes(4, 2, dtype, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING, mask, S, rb, inc) > 0
    ctrv = "\n".join([wl.CTRV_FX_SOURCE, wl.CTRV_RB_HX_SOURCE, wl.RB_HOOKS_SOURCE, wl.CTRV_X_HOOKS_SOURCE]).encode()
    allm = mask | L.BKE_HOOK_X_MEAN | L.BKE_HOOK_RESIDUAL_X | L.BKE_HOOK_STATE_ADD
    assert lib.bke_debug_ukf_model_points_cubin_bytes(5, 2, dtype, L.BKE_FX_USER, L.BKE_HX_USER, allm, S, ctrv, inc) > 0


def test_points_zero_is_the_merwe_compile():
    L, lib, inc = _lib()
    src = (wl.CT_FX_SOURCE + "\n" + wl.OFFSET_RB_HX_SOURCE).encode()
    a = lib.bke_debug_ukf_model_cubin_bytes(4, 2, 1, L.BKE_FX_USER, L.BKE_HX_USER, src, inc)
    assert a > 0 and lib.bke_debug_ukf_model_points_cubin_bytes(4, 2, 1, L.BKE_FX_USER, L.BKE_HX_USER, 0, 0, src, inc) == a
    rb = wl.RB_HOOKS_SOURCE.encode()
    mask = L.BKE_HOOK_RESIDUAL_Z | L.BKE_HOOK_Z_MEAN
    h = lib.bke_debug_ukf_model_hooks_cubin_bytes(4, 2, 1, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING, mask, rb, inc)
    assert h > 0 and lib.bke_debug_ukf_model_points_cubin_bytes(4, 2, 1, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING, mask, 0, rb, inc) == h


def test_simplex_compile_refusals():
    L, lib, inc = _lib()
    src = wl.CT_FX_SOURCE.encode()
    # an unknown point set
    assert lib.bke_debug_ukf_model_points_cubin_bytes(4, 2, 1, L.BKE_FX_USER, L.BKE_HX_LINEAR, 0, 64, src, inc) == 0
    assert "BKE_UKF_SIMPLEX" in lib.bke_last_error().decode()
    out = ctypes.c_void_p()
    assert lib.bke_ukf_model_compile_points(4, 2, 1, L.BKE_FX_USER, L.BKE_HX_LINEAR, 0, 1, src, inc, ctypes.byref(out)) == L.BKE_ERR_BAD_ARG
    # neither a user function nor a hook: the pre-built simplex instances serve that
    assert lib.bke_debug_ukf_model_points_cubin_bytes(4, 2, 1, L.BKE_FX_CONST_VEL, L.BKE_HX_LINEAR, 0, L.BKE_UKF_SIMPLEX, b"", inc) == 0
    # the simplex text sees BKE_N_SIGMAS = n + 1
    probe = (wl.CT_FX_SOURCE + "\nstatic_assert(BKE_N_SIGMAS == BKE_DIM_X + 1, \"n + 1 points\");\n").encode()
    assert lib.bke_debug_ukf_model_points_cubin_bytes(4, 2, 1, L.BKE_FX_USER, L.BKE_HX_LINEAR, 0, L.BKE_UKF_SIMPLEX, probe, inc) > 0
