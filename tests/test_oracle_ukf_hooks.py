"""CPU: the hooked UKF / CKF oracle against the reference's golden vectors (and the hook-free oracle against
them, which must NOT match), hooked programs through NVRTC, and the refusals."""
import numpy as np
import pytest

import ukf_hooks_oracle as oh
from oracle import ckf as ockf
from oracle import ukf as oukf
from filterpy_b200.common import workloads as wl

RB_HOOKS = dict(residual_z=wl.rb_residual_z, z_mean_fn=wl.rb_z_mean)
CTRV_HOOKS = dict(residual_z=wl.rb_residual_z, z_mean_fn=wl.rb_z_mean, residual_x=wl.ctrv_residual_x,
                  state_add=wl.ctrv_state_add, x_mean_fn=wl.ctrv_x_mean)


def _err(a, b):
    return np.abs(np.asarray(a, float) - b).max() / max(np.abs(b).max(), 1e-300)


def hx_rb(x):
    return np.array([np.sqrt(x[0] * x[0] + x[2] * x[2]), np.arctan2(x[2], x[0])])


def fx_cv(x, dt):
    return oukf.fx_apply(oukf.FX_CONST_VEL, x, dt)


def _single(g, name, hooks):
    N = g["x"].shape[0]
    ab = (float(g["alpha"]), float(g["beta"]), float(g["kappa"]))
    xs = np.zeros_like(g["ref_x"])
    worst = 0.0
    for f in range(N):
        x, P = g["x"][f], g["P"][f]
        for t in range(g["zs"].shape[0]):
            z = g["zs"][t, f] if g["valid"][t, f] else None
            if name == "ukf_hooks_rb":
                o = oh.ukf_step_single(x, P, z, g["Q"][f], g["R"][f], fx_cv, hx_rb, float(g["dt"]), *ab, hooks)
            else:
                o = oh.ukf_step_single(x, P, z, g["Q"][f], g["R"][f], wl.ctrv_fx, wl.ctrv_rb_hx, float(g["dt"]), *ab, hooks,
                                       hx_args=dict(sx=g["sensor"][0], sy=g["sensor"][1]))
            x, P = o["x"], o["P"]
            xs[t, f] = x
            worst = max(worst, _err(P, g["ref_P"][t, f]), _err(o["x_prior"], g["ref_x_prior"][t, f]))
            if z is not None:
                worst = max(worst, _err(o["K"], g["ref_K"][t, f]), _err(o["S"], g["ref_S"][t, f]),
                            _err(o["y"], g["ref_y"][t, f]), _err(o["loglik"], g["ref_loglik"][t, f]))
    return xs, worst


@pytest.mark.parametrize("name,hooks", [("ukf_hooks_rb", RB_HOOKS), ("ukf_hooks_ctrv", CTRV_HOOKS)])
def test_single_oracle_with_hooks_matches_golden(golden, name, hooks):
    g = golden(name)
    xs, worst = _single(g, name, hooks)
    assert max(worst, _err(xs, g["ref_x"])) < 1e-9
    # without the hooks the same filters cross the +-pi cut into a different answer
    xs_plain, _ = _single(g, name, {})
    assert np.abs(xs_plain - g["ref_x"]).max() > 1.0


def test_bank_oracle_with_hooks_matches_golden(golden):
    g = golden("ukf_hooks_rb")
    ab = (float(g["alpha"]), float(g["beta"]), float(g["kappa"]))
    x, P = g["x"], g["P"]
    xp, Pp = g["x"], g["P"]
    for t in range(g["zs"].shape[0]):
        o = oh.ukf_step_bank_hooks(x, P, g["zs"][t], g["Q"], g["R"], float(g["dt"]), *ab, oukf.FX_CONST_VEL,
                                   oukf.HX_RANGE_BEARING, angle_z=(1,), z_mean=True, valid=g["valid"][t])
        x, P = o["x"], o["P"]
        assert _err(x, g["ref_x"][t]) < 1e-9 and _err(P, g["ref_P"][t]) < 1e-9
        v = g["valid"][t]
        assert _err(o["K"][v], g["ref_K"][t][v]) < 1e-9 and _err(o["y"][v], g["ref_y"][t][v]) < 1e-9
        p = oukf.ukf_step_bank(xp, Pp, g["zs"][t], g["Q"], g["R"], float(g["dt"]), *ab, oukf.FX_CONST_VEL,
                               oukf.HX_RANGE_BEARING, valid=v)
        xp, Pp = p["x"], p["P"]
    assert np.abs(xp - g["ref_x"][-1]).max() > 1.0           # the hook-free oracle does not match


def test_rts_oracle_with_hooks_matches_golden(golden):
    g = golden("ukf_hooks_ctrv_rts")
    ab = (float(g["alpha"]), float(g["beta"]), float(g["kappa"]))
    T, N, n = g["Xs"].shape
    for f in range(N):
        xs, ps, ks = oh.ukf_rts_smoother_hooks(g["Xs"][:, f], g["Ps"][:, f], g["Q"][f], wl.ctrv_fx, [float(g["dt"])] * T, *ab,
                                              x_mean_fn=wl.ctrv_x_mean, residual_x=wl.ctrv_residual_x)
        assert _err(xs, g["ref_x"][:, f]) < 1e-9 and _err(ps, g["ref_P"][:, f]) < 1e-9 and _err(ks, g["ref_K"][:, f]) < 1e-9


def test_ckf_oracle_with_residual_z_matches_golden(golden):
    g = golden("ckf_hooks_rb")
    N = g["x"].shape[0]
    for f in range(N):
        x, P = g["x"][f][:, None], g["P"][f]
        for t in range(g["zs"].shape[0]):
            x, P, sf = ockf.ckf_predict_single(x, P, g["Q"][f], fx_cv, float(g["dt"]))
            if g["valid"][t, f]:
                x, P, y, K, S, SI = oh.ckf_update_single_hooks(x, P, sf, g["zs"][t, f][:, None], g["R"][f], hx_rb,
                                                               wl.rb_residual_z)
                z = g["zs"][t, f]                      # y = z - z^ cancels most digits: compare z^ = z - y
                assert _err(z - y.ravel(), z - g["ref_y"][t, f]) < 1e-9
            assert _err(x.ravel(), g["ref_x"][t, f]) < 1e-9 and _err(P, g["ref_P"][t, f]) < 1e-9
    x, P = g["x"], g["P"]
    for t in range(g["zs"].shape[0]):
        o = oh.ckf_step_bank_hooks(x, P, g["zs"][t], g["Q"], g["R"], float(g["dt"]), ockf.FX_CONST_VEL, ockf.HX_RANGE_BEARING,
                                   angle_z=(1,), valid=g["valid"][t])
        x, P = o["x"], o["P"]
        assert _err(x, g["ref_x"][t]) < 1e-9 and _err(P, g["ref_P"][t]) < 1e-9


# --------------------------------------------------------------------------- NVRTC and refusals
def _lib():
    from filterpy_b200 import _lib
    return _lib, _lib.load(), _lib.kernel_include_dirs().encode()


def _rb_mask(L):
    return L.BKE_HOOK_RESIDUAL_Z | L.BKE_HOOK_Z_MEAN


def _all_mask(L):
    return L.BKE_HOOK_X_MEAN | L.BKE_HOOK_Z_MEAN | L.BKE_HOOK_RESIDUAL_X | L.BKE_HOOK_RESIDUAL_Z | L.BKE_HOOK_STATE_ADD


@pytest.mark.parametrize("dtype", [0, 1])
def test_hooked_programs_compile_with_nvrtc(dtype):
    L, lib, inc = _lib()
    rb = wl.RB_HOOKS_SOURCE.encode()
    assert lib.bke_debug_ukf_model_hooks_cubin_bytes(4, 2, dtype, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING, _rb_mask(L), rb, inc) > 0
    ctrv = "\n".join([wl.CTRV_FX_SOURCE, wl.CTRV_RB_HX_SOURCE, wl.RB_HOOKS_SOURCE, wl.CTRV_X_HOOKS_SOURCE]).encode()
    assert lib.bke_debug_ukf_model_hooks_cubin_bytes(5, 2, dtype, L.BKE_FX_USER, L.BKE_HX_USER, _all_mask(L), ctrv, inc) > 0
    assert lib.bke_debug_ckf_model_hooks_cubin_bytes(4, 2, dtype, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING,
                                                     L.BKE_HOOK_RESIDUAL_Z, rb, inc) > 0


def test_hooks_zero_is_the_plain_compile():
    L, lib, inc = _lib()
    src = (wl.CT_FX_SOURCE + "\n" + wl.OFFSET_RB_HX_SOURCE).encode()
    for plain, hooked in ((lib.bke_debug_ukf_model_cubin_bytes, lib.bke_debug_ukf_model_hooks_cubin_bytes),
                          (lib.bke_debug_ckf_model_cubin_bytes, lib.bke_debug_ckf_model_hooks_cubin_bytes)):
        a = plain(4, 2, 1, L.BKE_FX_USER, L.BKE_HX_USER, src, inc)
        assert a > 0 and hooked(4, 2, 1, L.BKE_FX_USER, L.BKE_HX_USER, 0, src, inc) == a
        # hooks == 0 keeps the plain call's checks: no user function is refused
        assert hooked(4, 2, 1, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING, 0, b"", inc) == 0


def test_hook_refusals():
    L, lib, inc = _lib()
    rb = wl.RB_HOOKS_SOURCE.encode()
    # a hook named in the mask that the text does not define: NVRTC's log names it
    assert lib.bke_debug_ukf_model_hooks_cubin_bytes(4, 2, 1, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING,
                                                     _rb_mask(L) | L.BKE_HOOK_STATE_ADD, rb, inc) == 0
    msg = lib.bke_last_error().decode()
    assert "state_add" in msg and "UKF" in msg
    # dim_x > 8
    assert lib.bke_debug_ukf_model_hooks_cubin_bytes(10, 2, 1, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING, _rb_mask(L), rb, inc) == 0
    assert "dim_x = 8" in lib.bke_last_error().decode()
    out = __import__("ctypes").c_void_p()
    assert lib.bke_ukf_model_compile_hooks(10, 2, 1, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING, _rb_mask(L), rb, inc,
                                           __import__("ctypes").byref(out)) == L.BKE_ERR_UNSUPPORTED
    # the CKF calls residual_z only; unknown bits
    assert lib.bke_debug_ckf_model_hooks_cubin_bytes(4, 2, 1, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING, _rb_mask(L), rb, inc) == 0
    assert "residual_z" in lib.bke_last_error().decode()
    assert lib.bke_debug_ukf_model_hooks_cubin_bytes(4, 2, 1, L.BKE_FX_CONST_VEL, L.BKE_HX_RANGE_BEARING, 64, rb, inc) == 0


def test_python_callable_hooks_still_raise():
    from filterpy_b200.kalman import (UnscentedKalmanFilter, CubatureKalmanFilter, MerweScaledSigmaPoints,
                                      ConstVelFx, RangeBearingHx, DeviceFn)
    pts = MerweScaledSigmaPoints(4, .8, 2., 0.)
    for kw in RB_HOOKS.items():
        with pytest.raises(NotImplementedError):
            UnscentedKalmanFilter(4, 2, 1.0, RangeBearingHx(), ConstVelFx(), pts, **dict([kw]))
    with pytest.raises(NotImplementedError):
        UnscentedKalmanFilter(4, 2, 1.0, RangeBearingHx(), ConstVelFx(), pts, sqrt_fn=np.linalg.cholesky)
    with pytest.raises(NotImplementedError):
        CubatureKalmanFilter(4, 2, 1.0, RangeBearingHx(), ConstVelFx(), residual_z=wl.rb_residual_z)
    with pytest.raises(NotImplementedError):              # stored but never called by the reference's CKF
        CubatureKalmanFilter(4, 2, 1.0, RangeBearingHx(), ConstVelFx(), residual_x=DeviceFn(""))


def test_device_hooks_mask_and_dedup():
    from filterpy_b200 import _lib as L
    from filterpy_b200.kalman import DeviceFn
    from filterpy_b200.kalman.UKF import _device_hooks
    a, b = DeviceFn("A"), DeviceFn("B")
    mask, fns = _device_hooks(residual_z=a, z_mean_fn=a, state_add=b)
    assert mask == L.BKE_HOOK_RESIDUAL_Z | L.BKE_HOOK_Z_MEAN | L.BKE_HOOK_STATE_ADD
    assert len(fns) == 2 and fns[0] is a and fns[1] is b
    assert _device_hooks() == (0, ())
