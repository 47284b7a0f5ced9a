"""GPU parity of the UKF on SimplexSigmaPoints: every pre-built simplex instance against the fp64 oracle, the
reference's golden vectors in single and bank mode, update-only / update(None) / split steps, the stand-alone
sigma points, the smoother (built-in fx, user fx, hooks), user models with per-filter arguments, the unused
alpha, and the refusal of a compiled model stepped with the other point set."""
import ctypes

import numpy as np
import pytest

import ukf_simplex_oracle as osx
from gpu_harness import rel_close, RTOL
from test_gpu_sigma_instances import (INSTANCES, INSTANCE_IDS, DT, FX, HX, DTYPES, STEP_TOL, _problem, _take, _compare,
                                      _per_filter)

pytestmark = pytest.mark.gpu
BANKS = {"ukf_simplex_bank_rae": ("CONST_VEL", "RANGE_AZ_EL"), "ukf_simplex_bank_rb": ("CONST_VEL", "RANGE_BEARING"),
         "ukf_simplex_bank_lin": ("LINEAR", "LINEAR")}


def _models(fx, hx, F=None, H=None):
    from filterpy_b200.kalman import LinearFx, ConstVelFx, LinearHx, RangeAzElHx, RangeBearingHx
    f = LinearFx(F) if fx == "LINEAR" else ConstVelFx()
    h = LinearHx(H) if hx == "LINEAR" else (RangeAzElHx() if hx == "RANGE_AZ_EL" else RangeBearingHx())
    return f, h


def _ukf(n, m, fx, hx, mats, N, dtype, diagnostics=True, alpha=1, dt=DT, **kw):
    from filterpy_b200.kalman import UnscentedKalmanFilter, SimplexSigmaPoints
    f, h = (fx, hx) if not isinstance(fx, str) else _models(fx, hx, mats.get("F"), mats.get("H"))
    u = UnscentedKalmanFilter(n, m, dt, h, f, SimplexSigmaPoints(n, alpha=alpha), n_filters=N, dtype=dtype,
                              diagnostics=diagnostics, **kw)
    u.Q = mats["Q"]; u.R = mats["R"]
    return u


def _oracle(inst, x, P, z, mats, valid, R=None, dt=DT):
    _, _, fx, hx = inst
    return osx.ukf_step_bank(x, P, z, mats["Q"], mats["R"] if R is None else R, dt, FX[fx], HX[hx],
                             F=mats.get("F"), H=mats.get("H"), valid=valid)


# ----------------------------------------------------------------------------------------- instance matrix
@DTYPES
@pytest.mark.parametrize("inst", INSTANCES, ids=INSTANCE_IDS)
def test_simplex_instance_vs_oracle(inst, dtype):
    """Every pre-built instance on the simplex set: banks of 1 and 1037 filters (the last CTA holds 13), models
    shared and per filter, 3 epochs with ~20 % of the measurements missing; the same bank with diagnostics off."""
    n, m = inst[:2]
    pr = _problem(*inst, seed=300 + INSTANCES.index(inst))
    for N in (1, 1037):
        for layout in ("shared", "per"):
            mats = _take(pr[layout], N)
            f = _ukf(n, m, inst[2], inst[3], mats, N, dtype)
            g = _ukf(n, m, inst[2], inst[3], mats, N, dtype, diagnostics=False)
            x, P = pr["x"][:N], pr["P"][:N]
            f.x = g.x = x; f.P = g.P = P
            for t in range(pr["zs"].shape[0]):
                z, v = pr["zs"][t, :N], pr["valid"][t, :N]
                f.predict(); f.update(z, valid=v)
                g.predict(); g.update(z, valid=v)
                o = _oracle(inst, x, P, z, mats, v)
                x, P = o["x"], o["P"]
                _compare(f, o, z, v, dtype, "simplex %s N=%d t=%d" % (layout, N, t))
                assert int(f.status.sum().item()) == 0
            rel_close(g.x.cpu().numpy(), x, STEP_TOL[dtype][0], "x, diagnostics off")
            rel_close(g.P.cpu().numpy(), P, STEP_TOL[dtype][0], "P, diagnostics off")


@DTYPES
@pytest.mark.parametrize("inst", [INSTANCES[0], INSTANCES[4], INSTANCES[7]], ids=[INSTANCE_IDS[0], INSTANCE_IDS[4], INSTANCE_IDS[7]])
def test_update_only_none_and_split(inst, dtype):
    """update without predict draws the points from (x, P) (the mirror's documented difference); predict +
    update(None) leaves the prior; a predict flushed on its own then the update equal the fused step bit for
    bit; P = -I in one filter flags it (status 2) and changes no other filter."""
    from oracle import ukf as oukf
    n, m = inst[:2]
    pr = _problem(*inst, seed=400 + INSTANCES.index(inst))
    N, mats = pr["x"].shape[0], pr["per"]
    z, v = pr["zs"][0], pr["valid"][0]
    u = _ukf(n, m, inst[2], inst[3], mats, N, dtype)
    u.x = pr["x"]; u.P = pr["P"]
    u.update(z, valid=v)
    sig = osx.simplex_sigma_points(pr["x"], pr["P"])
    sh = oukf.hx_apply(HX[inst[3]], sig, mats["H"])
    Wm, Wc = osx.simplex_weights(n)
    zp, S = oukf.unscented_transform(sh, Wm, Wc, mats["R"])
    K = np.einsum("s,nsa,nsb->nab", Wc, sig - pr["x"][:, None], sh - zp[:, None]) @ np.linalg.inv(S)
    xw = np.where(v[:, None], pr["x"] + (K @ (z - zp)[..., None])[..., 0], pr["x"])
    Pw = np.where(v[:, None, None], pr["P"] - K @ S @ np.swapaxes(K, 1, 2), pr["P"])
    rel_close(u.x.cpu().numpy(), xw, STEP_TOL[dtype][0], "x update-only")
    rel_close(u.P.cpu().numpy(), Pw, STEP_TOL[dtype][0], "P update-only")

    u.x = pr["x"]; u.P = pr["P"]
    u.predict(); u.update(None)
    o = _oracle(inst, pr["x"], pr["P"], z, mats, np.zeros(N, bool))
    rel_close(u.x.cpu().numpy(), o["x_prior"], STEP_TOL[dtype][0], "x after update(None)")
    rel_close(u.P.cpu().numpy(), o["P_prior"], STEP_TOL[dtype][0], "P after update(None)")

    bad = list(range(5, N, 128))
    good = np.ones(N, bool); good[bad] = False
    Pbad = pr["P"].copy(); Pbad[bad] = -np.eye(n)
    fused, split, flagged = (_ukf(n, m, inst[2], inst[3], mats, N, dtype) for _ in range(3))
    for f, P0 in ((fused, pr["P"]), (split, pr["P"]), (flagged, Pbad)):
        f.x = pr["x"]; f.P = P0
    for t in range(pr["zs"].shape[0]):
        z, v = pr["zs"][t], pr["valid"][t]
        fused.predict(); fused.update(z, valid=v)
        split.predict(); split.x; split.update(z, valid=v)
        flagged.predict(); flagged.update(z, valid=v)
        xa, Pa = fused.x.cpu().numpy(), fused.P.cpu().numpy()
        assert np.array_equal(split.x.cpu().numpy(), xa) and np.array_equal(split.P.cpu().numpy(), Pa), t
        st = flagged.status.cpu().numpy()
        assert (st[bad] == 2).all() and (st[good] == 0).all(), t
        assert np.array_equal(flagged.x.cpu().numpy()[good], xa[good]) and np.array_equal(flagged.P.cpu().numpy()[good], Pa[good])


# ----------------------------------------------------------------------------------------- golden vectors

@pytest.mark.parametrize("name", sorted(BANKS))
def test_golden_banks(golden, name):
    """The reference on SimplexSigmaPoints, filter by filter: the whole bank at once, and the first filters
    one at a time in single-filter mode (NumPy attributes); the linear bank overrides R on odd epochs."""
    g = golden(name)
    N, T = g["x"].shape[0], g["zs"].shape[0]
    u = _ukf(g["x"].shape[1], g["R"].shape[-1], *BANKS[name], dict(Q=g["Q"], R=g["R"], F=g["F"], H=g["H"]), N, np.float64,
             dt=float(g["dt"]))
    u.x = g["x"]; u.P = g["P"]
    for t in range(T):
        v = g["valid"][t]
        u.predict(); u.update(g["zs"][t], R=g["R_override"] if ("R_override" in g and t % 2) else None, valid=v)
        for k in ("x", "P", "x_prior", "P_prior"):
            rel_close(getattr(u, k).cpu().numpy(), g["ref_" + k][t], RTOL[np.float64], "%s t=%d" % (k, t))
        for k in ("K", "S"):
            rel_close(getattr(u, k).cpu().numpy()[v], g["ref_" + k][t][v], RTOL[np.float64], "%s t=%d" % (k, t))
        rel_close(u.log_likelihood.cpu().numpy()[v], g["ref_loglik"][t][v], 10 * RTOL[np.float64], "loglik t=%d" % t)
    from filterpy_b200.kalman import UnscentedKalmanFilter, SimplexSigmaPoints
    for f in range(3):
        fx, hx = _models(*BANKS[name], F=g["F"], H=g["H"])
        s = UnscentedKalmanFilter(g["x"].shape[1], g["R"].shape[-1], float(g["dt"]), hx, fx, SimplexSigmaPoints(g["x"].shape[1]))
        s.x = g["x"][f]; s.P = g["P"][f]; s.Q = g["Q"][f]; s.R = g["R"][f]
        for t in range(T):
            s.predict()
            s.update(g["zs"][t, f] if g["valid"][t, f] else None, R=g["R_override"] if ("R_override" in g and t % 2) else None)
            assert isinstance(s.x, np.ndarray) and s.x.shape == (g["x"].shape[1],)
            rel_close(s.x, g["ref_x"][t, f], RTOL[np.float64], "single x f=%d t=%d" % (f, t))
            rel_close(s.P, g["ref_P"][t, f], RTOL[np.float64], "single P f=%d t=%d" % (f, t))


def test_golden_user_models_per_filter_args(golden):
    """DeviceFx (coordinated turn, a turn rate per filter) and DeviceHx (range / bearing from an offset sensor)."""
    from filterpy_b200.kalman import DeviceFx, DeviceHx
    from filterpy_b200.common import workloads as wl
    g = golden("ukf_simplex_user_ct_rb")
    N = g["x"].shape[0]
    sx, sy = (float(v) for v in g["sensor"])
    fx = DeviceFx(wl.CT_FX_SOURCE, arg_names=("omega",))
    hx = DeviceHx(wl.OFFSET_RB_HX_SOURCE, arg_names=("sx", "sy"), sx=sx, sy=sy)
    u = _ukf(4, 2, fx, hx, dict(Q=g["Q"], R=g["R"]), N, np.float64, dt=float(g["dt"]))
    u.x = g["x"]; u.P = g["P"]
    for t in range(g["zs"].shape[0]):
        u.predict(omega=g["omega"]); u.update(g["zs"][t], valid=g["valid"][t])
        rel_close(u.x.cpu().numpy(), g["ref_x"][t], RTOL[np.float64], "x t=%d" % t)
        rel_close(u.P.cpu().numpy(), g["ref_P"][t], RTOL[np.float64], "P t=%d" % t)


@pytest.mark.parametrize("mode", ["bank", "single"])
def test_golden_hooks(golden, mode):
    """residual_z / z_mean_fn as DeviceFn on targets crossing behind the sensor."""
    from filterpy_b200.kalman import DeviceFn, ConstVelFx, RangeBearingHx
    from filterpy_b200.common import workloads as wl
    g = golden("ukf_simplex_hooks_rb")
    rb = DeviceFn(wl.RB_HOOKS_SOURCE)
    sel = range(g["x"].shape[0]) if mode == "bank" else [0, 7]
    for f in ([None] if mode == "bank" else sel):
        idx = slice(None) if f is None else f
        u = _ukf(4, 2, ConstVelFx(), RangeBearingHx(), dict(Q=g["Q"][idx], R=g["R"][idx]), None if f is not None else g["x"].shape[0],
                 np.float64, dt=float(g["dt"]), residual_z=rb, z_mean_fn=rb)
        u.x = g["x"][idx]; u.P = g["P"][idx]
        for t in range(g["zs"].shape[0]):
            u.predict()
            if f is None:
                u.update(g["zs"][t], valid=g["valid"][t])
            else:
                u.update(g["zs"][t, f] if g["valid"][t, f] else None)
            got = (u.x.cpu().numpy(), u.P.cpu().numpy()) if f is None else (u.x, u.P)
            rel_close(got[0], g["ref_x"][t][idx], RTOL[np.float64], "x t=%d" % t)
            rel_close(got[1], g["ref_P"][t][idx], RTOL[np.float64], "P t=%d" % t)


# ----------------------------------------------------------------------------------------- smoother
@pytest.mark.parametrize("case", ["cv", "ct", "hooks"])
def test_golden_batch_filter_and_rts(golden, case):
    """batch_filter + rts_smoother: the built-in constant-velocity fx, the user coordinated turn (its turn rate
    the callable's default, UKF.py:712), and the built-in fx on a model compiled with hooks (the smoother runs
    the run-time compiled simplex instance; residual_z / z_mean_fn do not enter it)."""
    import torch
    from filterpy_b200.kalman import ConstVelFx, LinearHx, DeviceFx, DeviceFn
    from filterpy_b200.common import workloads as wl
    g = golden("ukf_simplex_rts")
    c = "ct" if case == "ct" else "cv"
    N = g[c + "_x0"].shape[0]
    fx = DeviceFx(wl.CT_FX_SOURCE, arg_names=("omega",), omega=float(g["omega"])) if case == "ct" else ConstVelFx()
    kw = {}
    if case == "hooks":
        kw = dict(residual_x=DeviceFn("__device__ void residual_x(const real *a, const real *b, real *o)"
                                      "{ for (int i = 0; i < BKE_DIM_X; i++) o[i] = a[i] - b[i]; }"))
    u = _ukf(4, 2, fx, LinearHx(g["H"]), dict(Q=g[c + "_Q"], R=g[c + "_R"]), N, np.float64, dt=float(g["dt"]), **kw)
    u.x = g[c + "_x0"]; u.P = g[c + "_P0"]
    mu, cov = u.batch_filter(torch.from_numpy(g[c + "_zs"]).cuda())
    rel_close(_per_filter(mu.cpu().numpy()), _per_filter(g[c + "_Xs"]), RTOL[np.float64], "Xs")
    rel_close(_per_filter(cov.cpu().numpy()), _per_filter(g[c + "_Ps"]), RTOL[np.float64], "Ps")
    xs, Ps, Ks = (a.cpu().numpy() for a in u.rts_smoother(torch.from_numpy(g[c + "_Xs"]).cuda(), torch.from_numpy(g[c + "_Ps"]).cuda()))
    rel_close(_per_filter(xs), _per_filter(g[c + "_ref_x"]), RTOL[np.float64], "xs")
    rel_close(_per_filter(Ps), _per_filter(g[c + "_ref_P"]), RTOL[np.float64], "Ps smoothed")
    rel_close(_per_filter(Ks[:-1]), _per_filter(g[c + "_ref_K"][:-1]), RTOL[np.float64], "Ks")


@DTYPES
@pytest.mark.parametrize("n", range(1, 9))
def test_rts_every_n_vs_oracle(n, dtype):
    """The built-in simplex smoother at every n <= 8 (linear fx, per-filter F), 65 filters, 9 epochs."""
    import torch
    from filterpy_b200.kalman import LinearFx, LinearHx
    rng = np.random.default_rng(n)
    N, T = 65, 9
    A = rng.standard_normal((T, N, n, n))
    Ps = A @ np.swapaxes(A, -1, -2) / n + 0.5 * np.eye(n)
    Xs = rng.normal(0, 3, (T, N, n))
    F = np.eye(n) + 0.1 * rng.standard_normal((N, n, n))
    B = rng.standard_normal((N, n, n))
    Q = B @ np.swapaxes(B, 1, 2) * 0.05 / n + 0.01 * np.eye(n)
    u = _ukf(n, 1, LinearFx(F), LinearHx(np.ones((1, n))), dict(Q=Q, R=np.eye(1)), N, dtype)
    xs, Pso, Ks = (a.cpu().numpy() for a in u.rts_smoother(torch.from_numpy(Xs), torch.from_numpy(Ps)))
    r = lambda a: a.astype(dtype).astype(np.float64)                                  # noqa: E731
    for i in range(N):
        wx, wP, wK = osx.ukf_rts_smoother(r(Xs[:, i]), r(Ps[:, i]), r(Q[i]), lambda s, dt, Fi=r(F[i]): Fi @ s, [DT] * T)
        tol = RTOL[dtype] if dtype == np.float64 else 3e-2
        rel_close(xs[:, i], wx, tol, "xs f=%d" % i)
        rel_close(Pso[:, i], wP, tol, "Ps f=%d" % i)
        rel_close(Ks[:-1, i], wK[:-1], tol, "Ks f=%d" % i)


# ----------------------------------------------------------------------------------------- stand-alone points
@DTYPES
@pytest.mark.parametrize("n", range(1, 33))
def test_sigma_points_vs_oracle(n, dtype):
    """bke_simplex_sigma_points at every n it accepts, for 1, 5 and 20011 filters (the grid-stride loop), with
    garbage in P's lower triangle (only the upper one is read); non-PD filters flagged alone."""
    import torch
    from filterpy_b200 import _lib
    from filterpy_b200._dev import bke_dtype
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(2000 + n)
    kw = dict(generator=g, device="cuda", dtype=torch.float64)
    lower = torch.tril(torch.ones(n, n, dtype=torch.bool, device="cuda"), -1)

    def raw(x, P):
        N = x.shape[0]
        sig = torch.empty(N, n + 1, n, dtype=x.dtype, device="cuda")
        st = torch.full((N,), -1, dtype=torch.int32, device="cuda")
        _lib.check(_lib.load().bke_simplex_sigma_points(N, n, bke_dtype(x.dtype), x.data_ptr(), P.data_ptr(), sig.data_ptr(),
                                                        st.data_ptr(), None))
        torch.cuda.synchronize()
        return sig, st.cpu().numpy()
    tol = 1e-10 if dtype == np.float64 else RTOL[dtype]
    for N in (1, 5, 20011):
        x = torch.randn(N, n, **kw).to(tdt).contiguous()
        A = torch.randn(N, n, n, **kw)
        P = A @ A.transpose(1, 2) / n + torch.eye(n, dtype=torch.float64, device="cuda")
        P = torch.where(lower, 100 * torch.randn(N, n, n, **kw), P).to(tdt).contiguous()
        sig, st = raw(x, P)
        assert not st.any(), N
        sel = torch.arange(N, device="cuda") if N <= 64 else torch.cat([torch.arange(0, 300, device="cuda"), torch.arange(N - 64, N, device="cuda")])
        want = osx.simplex_sigma_points(x[sel].double().cpu().numpy(), P[sel].double().cpu().numpy())
        rel_close(sig[sel].cpu().numpy(), want, tol, "sigmas N=%d" % N)
        if N == 5:
            Pb = P.clone()
            Pb[1] = -torch.eye(n, dtype=tdt, device="cuda")
            Pb[3, n - 1, n - 1] = -1.0
            sb, sst = raw(x, Pb)
            assert sst.tolist() == [0, 2, 0, 2, 0]
            assert torch.equal(sb[[0, 2, 4]], sig[[0, 2, 4]])


def test_sigma_points_mirror_golden(golden):
    """SimplexSigmaPoints.sigma_points: NumPy single, scalar P, a CUDA bank, and LinAlgError."""
    import torch
    from filterpy_b200.kalman import SimplexSigmaPoints
    g = golden("ukf_simplex_sigma")
    for n in (1, 2, 3, 4, 6, 9):
        got = SimplexSigmaPoints(n).sigma_points(g["x%d" % n], g["P%d" % n])
        assert got.shape == (n + 1, n)
        rel_close(got, g["sigmas%d" % n], 1e-12, "n=%d" % n)
    rel_close(SimplexSigmaPoints(3).sigma_points(g["x_scalar"], float(g["P_scalar"])), g["sigmas_scalar"], 1e-12, "scalar P")
    xb = torch.from_numpy(np.stack([g["x6"]] * 3)).cuda()
    Pb = torch.from_numpy(np.stack([g["P6"]] * 3)).cuda()
    bank = SimplexSigmaPoints(6).sigma_points(xb, Pb)
    assert bank.shape == (3, 7, 6)
    rel_close(bank.cpu().numpy(), np.stack([g["sigmas6"]] * 3), 1e-12, "bank")
    with pytest.raises(np.linalg.LinAlgError):
        SimplexSigmaPoints(3).sigma_points(np.zeros(3), -np.eye(3))


# ----------------------------------------------------------------------------------------- alpha, refusals, torch op
def test_alpha_has_no_effect():
    pr = _problem(6, 3, "CONST_VEL", "RANGE_AZ_EL", seed=9)
    N = pr["x"].shape[0]
    a, b = (_ukf(6, 3, "CONST_VEL", "RANGE_AZ_EL", pr["per"], N, np.float64, alpha=al) for al in (1, 0.3))
    for f in (a, b):
        f.x = pr["x"]; f.P = pr["P"]
        for t in range(pr["zs"].shape[0]):
            f.predict(); f.update(pr["zs"][t], valid=pr["valid"][t])
    assert np.array_equal(a.x.cpu().numpy(), b.x.cpu().numpy()) and np.array_equal(a.P.cpu().numpy(), b.P.cpu().numpy())


def test_model_point_set_mismatch_is_refused():
    """A compiled model remembers its point set: its step and its smoother refuse args asking for the other."""
    import torch
    from filterpy_b200 import _lib
    from filterpy_b200.kalman import DeviceFx, LinearHx, MerweScaledSigmaPoints, UnscentedKalmanFilter
    from filterpy_b200.common import workloads as wl
    lib = _lib.load()
    N = 8
    fx = DeviceFx(wl.CT_FX_SOURCE, arg_names=("omega",), omega=0.05)
    H = np.zeros((2, 4)); H[0, 0] = H[1, 2] = 1
    spx = _ukf(4, 2, fx, LinearHx(H), dict(Q=np.eye(4), R=np.eye(2)), N, np.float64)
    mrw = UnscentedKalmanFilter(4, 2, DT, LinearHx(H), fx, MerweScaledSigmaPoints(4, .5, 2., 0.), n_filters=N)
    z = torch.zeros(N, 2, dtype=torch.float64, device="cuda")
    for u, flags in ((spx, _lib.BKE_DO_UPDATE), (mrw, _lib.BKE_DO_UPDATE | _lib.BKE_UKF_SIMPLEX)):
        a = u._fill(_lib.UkfArgs(), flags, DT, z, None, None)
        a.alpha, a.beta, a.kappa = 0.5, 2.0, 0.0
        rc = lib.bke_ukf_step_model(ctypes.byref(a), u._user_model, u._fx_args[0].data_ptr(), u._fx_args[1], None, 0, None)
        assert rc == _lib.BKE_ERR_BAD_ARG and b"point set" in lib.bke_last_error()
        Xs = torch.zeros(3, N, 4, dtype=torch.float64, device="cuda"); Ps = torch.eye(4, dtype=torch.float64, device="cuda").repeat(3, N, 1, 1)
        r = _lib.UkfRtsArgs()
        r.n_filters, r.n_steps, r.dim_x, r.dtype, r.fx_model = N, 3, 4, _lib.BKE_F64, fx.model
        r.flags = 0 if u is spx else _lib.BKE_UKF_SIMPLEX
        r.alpha, r.beta, r.kappa, r.dt = 0.5, 2.0, 0.0, DT
        out = [torch.empty_like(Xs), torch.empty_like(Ps)]
        r.Xs, r.Ps, r.x_out, r.P_out = Xs.data_ptr(), Ps.data_ptr(), out[0].data_ptr(), out[1].data_ptr()
        r.Q, r.Q_stride = u._Q.data_ptr(), 0
        rc = lib.bke_ukf_rts_smoother_model(ctypes.byref(r), u._user_model, u._fx_args[0].data_ptr(), u._fx_args[1], None)
        assert rc == _lib.BKE_ERR_BAD_ARG and b"point set" in lib.bke_last_error()


def test_torch_op_simplex_matches_mirror():
    import torch
    from filterpy_b200 import torch_ops
    torch_ops.load()
    pr = _problem(6, 3, "CONST_VEL", "RANGE_AZ_EL", seed=11)
    N = pr["x"].shape[0]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()                     # noqa: E731
    x, P = torch.ops.bke.ukf_step(t(pr["x"]), t(pr["P"]), t(pr["per"]["Q"]), t(pr["per"]["R"]), t(pr["zs"][0]), DT, .5, 2., 0.,
                                  FX["CONST_VEL"], HX["RANGE_AZ_EL"], simplex=True)
    u = _ukf(6, 3, "CONST_VEL", "RANGE_AZ_EL", pr["per"], N, np.float64, diagnostics=False)
    u.x = pr["x"]; u.P = pr["P"]
    u.predict(); u.update(pr["zs"][0])
    assert torch.equal(x, u.x) and torch.equal(P, u.P)
