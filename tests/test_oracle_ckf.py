"""CPU: the CKF oracle against the reference's golden vectors, the CKF program text through NVRTC, and the
mirror's packing of positional fx_args / hx_args."""
import numpy as np
import pytest

from oracle import ckf as ockf

GOLDEN = ["ckf_bank_rae", "ckf_bank_lin", "ckf_user_ct_rb", "ckf_call_order"]


def _models(name, g):
    from filterpy_b200.common import workloads as wl
    if name == "ckf_user_ct_rb":
        return (lambda s, dt, om: wl.ct_fx(s, dt, om)), wl.offset_rb_hx, ockf.FX_LINEAR, ockf.HX_LINEAR
    if name == "ckf_bank_rae":
        def fx(s, dt):
            o = s.copy(); o[0::2] = s[0::2] + dt * s[1::2]
            return o
        return fx, (lambda s: ockf.hx_apply(ockf.HX_RANGE_AZ_EL, s)), ockf.FX_CONST_VEL, ockf.HX_RANGE_AZ_EL
    F, H = g["F"], g["H"]
    return (lambda s, dt: F @ s), (lambda s: H @ s), ockf.FX_LINEAR, ockf.HX_LINEAR


def _ops(name, g):
    return [str(o) for o in g["ops"]] if "ops" in g else ["predict+update"] * g["zs"].shape[0]


def _close(a, b, what, tol=1e-9):
    # the literal restatement repeats the reference's operations but does not reproduce its rounding bit for
    # bit (differences of 1e-12 to 1e-10 relative, growing over the epochs: the raw moments amplify
    # last-bit differences by |x|^2 / P); 1e-9 is the bound the golden generator asserts
    scale = max(np.abs(b).max(), 1e-300)
    err = np.abs(np.asarray(a) - b).max() / scale
    assert err < tol, (what, err)


# the centred sums differ from the reference's raw moments by its cancellation error, which the golden
# generator (tests/golden/make_golden_ckf.py) bounds by 1e-9 (measured: below 1e-10)
CENTRED = 1e-9


@pytest.mark.parametrize("name", GOLDEN)
def test_single_oracle_matches_golden(golden, name):
    """The reference's literal call sequence (raw moments) against its own recorded results."""
    g = golden(name)
    fx, hx, _, _ = _models(name, g)
    N, n = g["x"].shape
    m = g["R"].shape[-1]
    dt = float(g["dt"])
    for f in range(N):
        x, P = g["x"][f][:, None], g["P"][f]
        sf = np.zeros((2 * n, n))
        for t, op in enumerate(_ops(name, g)):
            fa = (g["omega"][f],) if name == "ckf_user_ct_rb" else ()
            ha = tuple(g["sensor"]) if name == "ckf_user_ct_rb" else ()
            if op.startswith("predict"):
                x, P, sf = ockf.ckf_predict_single(x, P, g["Q"][f], fx, dt, fa)
                _close(x.ravel(), g["ref_x_prior"][t, f], "x_prior"); _close(P, g["ref_P_prior"][t, f], "P_prior")
            _close(sf, g["ref_sigmas_f"][t, f], "sigmas_f")
            if g["valid"][t, f] and op != "predict+none":
                R = 0.5 if op == "predict+update_R" else g["R"][f]
                x, P, y, K, S, SI = ockf.ckf_update_single(x, P, sf, g["zs"][t, f][:, None], R, hx, ha)
                _close(K, g["ref_K"][t, f], "K"); _close(S, g["ref_S"][t, f], "S"); _close(y.ravel(), g["ref_y"][t, f], "y")
            _close(x.ravel(), g["ref_x"][t, f], "x %s t=%d f=%d" % (name, t, f)); _close(P, g["ref_P"][t, f], "P")
            assert m == g["ref_S"].shape[-1]


@pytest.mark.parametrize("name", ["ckf_bank_rae", "ckf_bank_lin", "ckf_call_order"])
def test_bank_oracle_matches_golden(golden, name):
    """The vectorised, centred restatement (the kernel's arithmetic) against the reference."""
    g = golden(name)
    _, _, fxm, hxm = _models(name, g)
    N, n = g["x"].shape
    x, P = g["x"], g["P"]
    sf = np.zeros((N, 2 * n, n))
    for t, op in enumerate(_ops(name, g)):
        pred = op.startswith("predict")
        valid = g["valid"][t] & (op != "predict+none")
        R = 0.5 * np.eye(g["R"].shape[-1]) if op == "predict+update_R" else g["R"]
        o = ockf.ckf_step_bank(x, P, g["zs"][t], g["Q"], R, float(g["dt"]), fxm, hxm, F=g["F"], H=g["H"],
                               valid=valid, sigmas_f=sf, predict=pred)
        x, P, sf = o["x"], o["P"], o["sigmas_f"]
        _close(sf, g["ref_sigmas_f"][t], "sigmas_f", CENTRED)
        _close(x, g["ref_x"][t], "x %s t=%d" % (name, t), CENTRED); _close(P, g["ref_P"][t], "P", CENTRED)
        if valid.any():
            _close(o["K"][valid], g["ref_K"][t][valid], "K", CENTRED); _close(o["S"][valid], g["ref_S"][t][valid], "S", CENTRED)


def _lib():
    from filterpy_b200 import _lib
    return _lib, _lib.load()


@pytest.mark.parametrize("dtype", [0, 1])
def test_ckf_user_models_compile_with_nvrtc(dtype):
    from filterpy_b200.common import workloads as wl
    L, lib = _lib()
    inc = L.kernel_include_dirs().encode()
    both = (wl.CT_FX_SOURCE + "\n" + wl.OFFSET_RB_HX_SOURCE).encode()
    assert lib.bke_debug_ckf_model_cubin_bytes(4, 2, dtype, L.BKE_FX_USER, L.BKE_HX_USER, both, inc) > 0
    assert lib.bke_debug_ckf_model_cubin_bytes(4, 2, dtype, L.BKE_FX_USER, L.BKE_HX_LINEAR, wl.CT_FX_SOURCE.encode(), inc) > 0


def test_ckf_user_model_errors_before_and_from_nvrtc():
    L, lib = _lib()
    inc = L.kernel_include_dirs().encode()
    bad = b"__device__ void fx(const real *x, real *o, real dt, const real *a) { o[0] = no_such_thing; }"
    assert lib.bke_debug_ckf_model_cubin_bytes(4, 2, 1, L.BKE_FX_USER, L.BKE_HX_LINEAR, bad, inc) == 0
    msg = lib.bke_last_error().decode()
    assert "user_model.cu" in msg and "no_such_thing" in msg and "CKF" in msg
    # refused before NVRTC runs: no user function, a transcendental built-in partner, bad sizes
    for args in [(4, 2, 1, L.BKE_FX_LINEAR, L.BKE_HX_LINEAR), (4, 2, 1, L.BKE_FX_USER, L.BKE_HX_RANGE_BEARING),
                 (0, 2, 1, L.BKE_FX_USER, L.BKE_HX_LINEAR), (4, 2, 7, L.BKE_FX_USER, L.BKE_HX_LINEAR)]:
        assert lib.bke_debug_ckf_model_cubin_bytes(*args, b"garbage that would not compile", inc) == 0
        assert "bke_ckf_model_compile" in lib.bke_last_error().decode() or "dtype" in lib.bke_last_error().decode()


def test_positional_args_pack_onto_arg_names_in_order():
    import torch
    from filterpy_b200.kalman.CubatureKalmanFilter import _positional
    from filterpy_b200.kalman import DeviceFx, ConstVelFx
    m = DeviceFx("", arg_names=("a", "b"))
    assert _positional(m, (), "fx_args") is None
    assert _positional(m, 3.0, "fx_args") == {"a": 3.0}                     # a non-tuple is wrapped (:314-315)
    ov = _positional(m, (1.0, np.array([2.0, 3.0])), "fx_args")
    t, stride = m.pack(ov, 2, torch.float64, "cpu")
    assert stride == 2 and t.tolist() == [[1.0, 2.0], [1.0, 3.0]]
    with pytest.raises(TypeError):
        _positional(m, (1.0, 2.0, 3.0), "fx_args")
    with pytest.raises(NotImplementedError):
        _positional(ConstVelFx(), (1.0,), "fx_args")
