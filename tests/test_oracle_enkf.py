"""CPU: the EnKF noise-stream replica (Philox4x32-10 against the Random123 known-answer vectors, Box-Muller,
the semi-definite factor), the EnKF oracle against the reference's golden vectors, the C-ABI's
argument checks, the EnKF program text through NVRTC and the mirror's constructor errors."""
import ctypes

import numpy as np
import pytest

from oracle import enkf as oe

GOLDEN = ["enkf_cv_lin", "enkf_cv_rae", "enkf_user_ct_rb", "enkf_call_order", "enkf_rank_q", "enkf_n256"]


def fx_cv(s, dt):
    o = np.array(s, dtype=float)
    o[0::2] = s[0::2] + dt * s[1::2]
    return o


def hx_rae(s):
    px, py, pz = s[0], s[2], s[4]
    return np.array([np.sqrt(px * px + py * py + pz * pz), np.arctan2(py, px), np.arctan2(pz, np.sqrt(px * px + py * py))])


def golden_models(name, g, f):
    """The reference's fx(s, dt) / hx(s) of filter f of golden case `name`."""
    from filterpy_b200.common import workloads as wl
    if name == "enkf_user_ct_rb":
        om, sen = g["omega"][f], g["sensor"]
        return (lambda s, dt: wl.ct_fx(s, dt, om)), (lambda s: wl.offset_rb_hx(s, *sen))
    if name == "enkf_cv_rae":
        return fx_cv, hx_rae
    H = g["H"]
    return fx_cv, (lambda s: H @ s)


def update_R(g, op):
    upd = op.split("+")[-1]
    return 0.5 if upd == "update_R" else (g["Rcall"] if upd == "update_Rm" else None)


def oracle_replay(name, g):
    """The golden call sequence on one oracle EnKF per filter; yields (op index, [filters]) after every op."""
    F, n = g["x"].shape
    m = g["R"].shape[-1]
    N, seed = int(g["n_members"]), int(g["seed"])
    fs = []
    for f in range(F):
        fx, hx = golden_models(name, g, f)
        e = oe.EnKF(g["x"][f], g["P"][f], m, float(g["dt"]), N, hx, fx, oe.Stream(seed, f))
        e.Q, e.R = g["Q"][f], g["R"][f]
        fs.append(e)
    call, t_z = 1, 0
    for t, op in enumerate(str(o) for o in g["ops"]):
        if op.startswith("predict"):
            for e in fs:
                e.counter = call
                e.predict()
            call += 1
        upd = op.split("+")[-1]
        if upd.startswith("update"):
            for f, e in enumerate(fs):
                e.counter = call
                e.update(g["zs"][t_z, f] if g["valid"][t, f] else None, R=update_R(g, op))
            call += 1
            t_z = min(t_z + 1, g["zs"].shape[0] - 1)
        elif upd == "none":
            for e in fs:
                e.update(None)
        yield t, fs


# ------------------------------------------------------------------------------------------ noise stream
def test_philox_known_answers():
    """Random123's kat_vectors for philox4x32_10."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        assert tuple(int(v) for v in oe.philox4x32_10(ctr, key)) == want


def test_box_muller_uniforms_exclude_zero():
    z0, z1 = oe.box_muller([np.uint64(0)] * 4)                 # u1 = 2^-53: the largest radius, finite
    assert np.isfinite(z0) and z0 == pytest.approx(np.sqrt(-2 * np.log(2.0 ** -53)))
    full = [np.uint64(0xffffffff)] * 4                          # u1 = 1: radius 0
    assert oe.box_muller(full) == (0.0, -0.0) or max(abs(v) for v in oe.box_muller(full)) == 0.0


def test_box_muller_f32_uniforms_at_the_ends_of_the_word():
    """fp32: u1 = (float(c0) + 1) 2^-32 in (0, 1] and u2 = float(c2) 2^-32, both rounded to float; c2 = 2^32 - 1
    rounds u2 up to exactly 1 (angle 2 pi), which the fp64 uniforms never reach."""
    top = 0xffffffff
    z0, z1 = oe.box_muller([np.uint64(0)] * 4, np.float32)     # u1 = 2^-32 exactly: the largest fp32 radius
    assert z0 == np.sqrt(-2 * np.log(2.0 ** -32)) and z1 == 0.0
    z0, z1 = oe.box_muller([np.uint64(top), np.uint64(0), np.uint64(0), np.uint64(0)], np.float32)
    assert z0 == 0.0 and z1 == 0.0                              # float(2^32 - 1) + 1 = 2^32: u1 = 1, radius 0
    z0, z1 = oe.box_muller([np.uint64(0), np.uint64(0), np.uint64(top), np.uint64(0)], np.float32)
    assert z0 == np.sqrt(-2 * np.log(2.0 ** -32)) and abs(z1) < 1e-14 * z0     # u2 = 1: cos 2 pi, sin 2 pi
    # float(2^32 - 100) = 2^32: u1 = 1; float(2^32 - 200) = 2^32 - 256: u1 = 1 - 2^-24, the smallest radius > 0
    assert oe.box_muller([np.uint64(top - 100), np.uint64(0), np.uint64(0), np.uint64(0)], np.float32)[0] == 0.0
    z0, _ = oe.box_muller([np.uint64(top - 200), np.uint64(0), np.uint64(0), np.uint64(0)], np.float32)
    assert z0 == np.sqrt(-2 * np.log(1 - 2.0 ** -24))
    # the fp32 uniforms are float(word) + 1 (u1) and float(word) (u2), scaled: exact at small words
    for w in (1, 5, 1 << 20, 123456789):
        z0, z1 = oe.box_muller([np.uint64(w), np.uint64(0), np.uint64(w), np.uint64(0)], np.float32)
        u1 = float(np.float32(np.float32(w) + np.float32(1))) * 2.0 ** -32
        u2 = float(np.float32(w)) * 2.0 ** -32
        r = np.sqrt(-2 * np.log(u1))
        assert z0 == r * np.cos(2 * np.pi * u2) and z1 == r * np.sin(2 * np.pi * u2)


def test_f32_stream_agrees_with_the_f64_stream_to_the_24_bit_uniforms():
    """The fp32 normals differ from the fp64 ones only by the uniforms' lost bits: within 1e-3 absolute over 2^20
    draws of each of three keys (median below 1e-6).  They are not the same stream, though: at c0 = c1 = 0 the
    fp64 u1 is 2^-53 and the fp32 one 2^-32, radii 8.6 and 6.7, so an fp32 comparison needs the fp32 uniforms."""
    for seed, f, call in ((0, 0, 0), (0xffffffff, 37, 0xffffffff), (7, 3, 2)):
        a = oe.std_normals(seed, f, call, 1 << 18, 4)
        b = oe.std_normals(seed, f, call, 1 << 18, 4, np.float32)
        d = np.abs(a - b)
        assert d.max() < 1e-3 and np.median(d) < 1e-6, (seed, f, call, d.max(), np.median(d))
    zero = [np.uint64(0)] * 4
    assert oe.box_muller(zero)[0] - oe.box_muller(zero, np.float32)[0] > 1.9


def test_f32_stream_factors_with_the_f32_eps():
    """Stream(dtype=float32) zeroes a pivot below 16 k eps32 max diag C, as the fp32 kernel does: a rank-one C
    rounded to float, whose second pivot is float rounding rather than 0, draws inside its range."""
    v = np.array([1.0, 1.0 / 3.0, 0.7])
    C = np.outer(v, v).astype(np.float32).astype(np.float64)
    assert not oe.psd_factor(C)[1] or oe.psd_factor(C)[0][1, 1] != 0.0       # fp64 eps sees the rounding
    L, ok = oe.psd_factor(C, np.finfo(np.float32).eps)
    assert ok and L[1, 1] == 0.0 and L[2, 2] == 0.0
    e = oe.Stream(3, 1, np.float32).draw(0, np.zeros(3), C, 1000)
    u = v / np.linalg.norm(v)
    assert np.abs(e - np.outer(e @ u, u)).max() < 1e-6 * np.abs(e).max()
    assert oe.Stream(3, 1).dtype is np.float64 and oe.Stream(3, 1, np.float32).dtype is np.float32


def test_std_normals_statistics_and_keys():
    xi = oe.std_normals(7, 3, 0, 40000, 4)
    assert abs(xi.mean()) < 0.02 and abs(xi.var() - 1) < 0.02
    c = np.corrcoef(xi.T)
    assert np.abs(c - np.eye(4)).max() < 0.03
    # different filters, calls and seeds give different numbers; the same key repeats bit for bit
    assert not np.array_equal(xi, oe.std_normals(7, 4, 0, 40000, 4))
    assert not np.array_equal(xi, oe.std_normals(7, 3, 1, 40000, 4))
    assert not np.array_equal(xi, oe.std_normals(8, 3, 0, 40000, 4))
    assert np.array_equal(xi[:5], oe.std_normals(7, 3, 0, 5, 4))
    # an odd component count takes the first of the pair
    assert np.array_equal(oe.std_normals(7, 3, 0, 5, 3), xi[:5, :3])


def test_psd_factor():
    rng = np.random.default_rng(0)
    A = rng.standard_normal((5, 5))
    C = A @ A.T + np.eye(5)
    L, ok = oe.psd_factor(C)
    assert ok and np.allclose(L, np.linalg.cholesky(C), rtol=1e-12, atol=1e-12)
    dt, q = 0.1, 0.3
    blk = q * np.array([[dt ** 4 / 4, dt ** 3 / 2], [dt ** 3 / 2, dt ** 2]])      # rank 1
    Q = np.kron(np.eye(2), blk)
    L, ok = oe.psd_factor(Q)
    assert ok and np.allclose(L @ L.T, Q, rtol=0, atol=1e-15) and L[1, 1] == 0 and L[3, 3] == 0
    L, ok = oe.psd_factor(np.zeros((3, 3)))
    assert ok and not L.any()
    assert not oe.psd_factor(np.diag([1.0, -1.0]))[1]
    assert not oe.psd_factor(np.array([[0.0, 1.0], [1.0, 0.0]]))[1]
    assert not oe.psd_factor(np.array([[1.0, 2.0], [2.0, 1.0]]))[1]


# ------------------------------------------------------------------------------------------ oracle vs reference
@pytest.mark.parametrize("name", GOLDEN)
def test_oracle_matches_golden(golden, name):
    g = golden(name)
    for t, fs in oracle_replay(name, g):
        for k in ("x", "P", "x_prior", "P_prior", "K", "S", "SI", "sigmas"):
            got = np.array([getattr(e, k) for e in fs])
            ref = g["ref_" + k][t]
            err = np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)
            assert err < 1e-9, (name, t, k, err)


def test_golden_covers_rank_deficient_and_zero_q(golden):
    g = golden("enkf_rank_q")
    assert not g["Q"][3:].any()
    for f in range(3):
        assert np.linalg.matrix_rank(g["Q"][f]) < g["Q"].shape[-1]
        assert oe.psd_factor(g["Q"][f])[1]
    assert int(g["n_members"]) == 2
    assert sorted(int(golden(n)["n_members"]) for n in GOLDEN) == [2, 8, 8, 33, 33, 256]


# ------------------------------------------------------------------------------------------ the C-ABI
def _args(L):
    a = L.EnkfArgs()
    fake = 1 << 20                                   # never dereferenced: every call below fails before a launch
    a.n_filters, a.dim_x, a.dim_z, a.n_members, a.dtype = 8, 4, 2, 16, L.BKE_F32
    a.flags = L.BKE_DO_PREDICT | L.BKE_DO_UPDATE
    a.fx_model, a.hx_model = L.BKE_FX_LINEAR, L.BKE_HX_LINEAR
    a.x = a.P = a.x_out = a.P_out = a.sigmas = a.sigmas_out = a.Q = a.R = a.F = a.H = a.z = fake
    return a


@pytest.mark.parametrize("field,value,msg", [
    ("dim_x", 0, b"bad dimensions"), ("dim_x", 17, b"bad dimensions"), ("dim_z", 0, b"bad dimensions"),
    ("n_filters", -1, b"bad dimensions"), ("n_members", 1, b"n_members must be 2"), ("dtype", 7, b"dtype"),
    ("flags", 0, b"neither"), ("flags", 7, b"only BKE_DO_PREDICT"), ("sigmas", None, b"sigmas"),
    ("Q", None, b"predict needs Q"), ("z", None, b"update needs R and z"), ("P_out", None, b"x, P, x_out, P_out"),
    ("F", None, b"BKE_FX_LINEAR needs F"), ("H", None, b"BKE_HX_LINEAR needs H"), ("Q_stride", -1, b"stride"),
    ("hx_model", 2, b"BKE_HX_RANGE_BEARING needs"), ("fx_model", 9, b"unknown fx/hx")])
def test_enkf_step_validates_arguments(field, value, msg):
    from filterpy_b200 import _lib as L
    lib = L.load()
    a = _args(L)
    setattr(a, field, value)
    if field == "hx_model":
        a.dim_x, a.dim_z = 6, 3
    assert lib.bke_enkf_step(ctypes.byref(a), None) == L.BKE_ERR_BAD_ARG
    assert msg in lib.bke_last_error()


def test_enkf_initialize_validates_arguments():
    from filterpy_b200 import _lib as L
    lib = L.load()
    fake = 1 << 20
    for args, msg in [((8, 0, 16, 0), b"dim_x"), ((8, 17, 16, 0), b"dim_x"), ((8, 4, 1, 0), b"n_members"),
                      ((-1, 4, 16, 0), b"n_filters"), ((8, 4, 16, 5), b"dtype")]:
        assert lib.bke_enkf_initialize(*args, 1, 0, fake, fake, fake, None, None) == L.BKE_ERR_BAD_ARG
        assert msg in lib.bke_last_error()
    assert lib.bke_enkf_initialize(8, 4, 16, 0, 1, 0, None, fake, fake, None, None) == L.BKE_ERR_BAD_ARG


@pytest.mark.parametrize("dtype", [0, 1])
def test_enkf_user_models_compile_with_nvrtc(dtype):
    from filterpy_b200 import _lib as L
    from filterpy_b200.common import workloads as wl
    lib = L.load()
    inc = L.kernel_include_dirs().encode()
    both = (wl.CT_FX_SOURCE + "\n" + wl.OFFSET_RB_HX_SOURCE).encode()
    assert lib.bke_debug_enkf_model_cubin_bytes(4, 2, dtype, L.BKE_FX_USER, L.BKE_HX_USER, both, inc) > 0
    assert lib.bke_debug_enkf_model_cubin_bytes(16, 4, dtype, L.BKE_FX_USER, L.BKE_HX_LINEAR,
                                                b"__device__ void fx(const real *x, real *o, real dt, const real *a)"
                                                b" { for (int i = 0; i < 16; i++) o[i] = x[i]; }", inc) > 0
    bad = b"__device__ void fx(const real *x, real *o, real dt, const real *a) { o[0] = no_such_thing; }"
    assert lib.bke_debug_enkf_model_cubin_bytes(4, 2, dtype, L.BKE_FX_USER, L.BKE_HX_LINEAR, bad, inc) == 0
    assert b"EnKF" in lib.bke_last_error() and b"no_such_thing" in lib.bke_last_error()


# ------------------------------------------------------------------------------------------ mirror errors
def test_mirror_constructor_errors_need_no_gpu():
    from filterpy_b200.kalman import EnsembleKalmanFilter, ConstVelFx, LinearHx
    x, P, H = np.zeros(4), np.eye(4), np.eye(2, 4)
    fx, hx = ConstVelFx(), LinearHx(H)
    with pytest.raises(ValueError, match="dim_z"):
        EnsembleKalmanFilter(x, P, 0, 0.1, 8, hx, fx)
    with pytest.raises(ValueError, match="N must be greater than zero"):
        EnsembleKalmanFilter(x, P, 2, 0.1, 0, hx, fx)
    with pytest.raises(ValueError, match="N - 1"):
        EnsembleKalmanFilter(x, P, 2, 0.1, 1, hx, fx)
    with pytest.raises(ValueError, match="1D"):
        EnsembleKalmanFilter(x[:, None], P, 2, 0.1, 8, hx, fx)
    with pytest.raises(NotImplementedError):
        EnsembleKalmanFilter(x, P, 2, 0.1, 8, lambda s: H @ s, fx)
