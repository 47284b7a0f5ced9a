"""GPU: EnKF bank (CUDA through the mirror, the C-ABI and the torch op) vs the reference's golden vectors,
the oracle on the replica noise stream, bank independence of the stream, sampling statistics against a
KalmanFilter bank, and the failure statuses."""
import numpy as np
import pytest

from gpu_harness import rel_close, RTOL
from test_oracle_enkf import GOLDEN, update_R
from oracle import enkf as oe

pytestmark = pytest.mark.gpu


def make(name, g, dtype, shared=False, single=False, diagnostics=True, **kw):
    from filterpy_b200.kalman import EnsembleKalmanFilter, LinearFx, ConstVelFx, LinearHx, RangeAzElHx, DeviceFx, DeviceHx
    from filterpy_b200.common import workloads as wl
    F = g["x"].shape[0]
    if name == "enkf_user_ct_rb":
        om = g["omega"][:1] if single else g["omega"]
        fx = DeviceFx(wl.CT_FX_SOURCE, arg_names=("omega",), omega=om[0] if single else om)
        hx = DeviceHx(wl.OFFSET_RB_HX_SOURCE, arg_names=("sx", "sy"), sx=float(g["sensor"][0]), sy=float(g["sensor"][1]))
    elif name == "enkf_cv_rae":
        fx, hx = ConstVelFx(), RangeAzElHx()
    else:
        fx, hx = ConstVelFx(), LinearHx(g["H"])
        if shared:                       # per-filter F through LinearFx, H and R shared by the bank
            n = g["x"].shape[1]
            Fm = np.eye(n)
            Fm[0, 1] = Fm[2, 3] = float(g["dt"])
            fx = LinearFx(np.broadcast_to(Fm, (F, n, n)).copy())
    m = g["R"].shape[-1]
    x, P = (g["x"][0], g["P"][0]) if single else (g["x"], g["P"])
    e = EnsembleKalmanFilter(x, P, m, float(g["dt"]), int(g["n_members"]), hx, fx, n_filters=None if single else F,
                             dtype=dtype, seed=int(g["seed"]), diagnostics=diagnostics, **kw)
    e.Q = g["Q"][0] if single else g["Q"]
    e.R = g["R"][0] if (single or shared) else g["R"]
    return e


def run_op(e, g, t, t_z, op, single=False):
    if op.startswith("predict"):
        e.predict()
    upd = op.split("+")[-1]
    if upd == "none":
        e.update(None)
    elif upd.startswith("update"):
        if single:                       # the bank's update launches (and draws) even where valid is 0
            e.update(g["zs"][t_z, 0], R=update_R(g, op), valid=g["valid"][t, :1])
        else:
            e.update(g["zs"][t_z], R=update_R(g, op), valid=g["valid"][t])
        return min(t_z + 1, g["zs"].shape[0] - 1)
    return t_z


KEYS = ("x", "P", "x_prior", "P_prior", "K", "S", "SI", "sigmas")


def _np(v):
    return v.cpu().numpy() if hasattr(v, "cpu") else np.asarray(v)


def _rtol(name, k, dtype):
    # fp32 members carry positions of ~100-600 to 6e-8 relative, while the covariances are formed from their
    # spreads of ~1: in the angle-measurement cases (R of (0.005 rad)^2) and the N = 2 case (P - K S K' of a
    # rank-one ensemble covariance, where most of P cancels) the covariance-like attributes drift past 1e-3
    # (measured on the H100: K 1.7e-3 and P_prior 1.3e-3 with angles, P 8.9e-3 at N = 2).  x and the members
    # hold RTOL.
    if dtype == np.float32 and k in ("K", "P", "P_prior", "S", "SI"):
        if name == "enkf_rank_q":
            return 2e-2
        if name in ("enkf_cv_rae", "enkf_user_ct_rb"):
            return 5e-3
    return RTOL[dtype]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", GOLDEN)
def test_enkf_vs_reference_golden(golden, name, dtype):
    """Every recorded attribute after every call: built-in and NVRTC models, valid masks, the call-order
    case (update after initialize, two updates, update(None), scalar and per-call R), rank-deficient and
    zero Q, N = 2 / 8 / 33 / 256."""
    g = golden(name)
    e = make(name, g, dtype)
    t_z = 0
    for t, op in enumerate(str(o) for o in g["ops"]):
        t_z = run_op(e, g, t, t_z, op)
        for k in KEYS:
            rel_close(_np(getattr(e, k)), g["ref_" + k][t], _rtol(name, k, dtype), "%s %s t=%d" % (name, k, t))
    e.check()


@pytest.mark.parametrize("name", ["enkf_cv_lin", "enkf_call_order", "enkf_rank_q"])
def test_enkf_shared_models_and_linear_fx(golden, name):
    g = golden(name)
    e = make(name, g, np.float64, shared=True)
    t_z = 0
    for t, op in enumerate(str(o) for o in g["ops"]):
        t_z = run_op(e, g, t, t_z, op)
        for k in KEYS:
            rel_close(_np(getattr(e, k)), g["ref_" + k][t], RTOL[np.float64], "%s %s t=%d" % (name, k, t))


@pytest.mark.parametrize("name", ["enkf_cv_lin", "enkf_user_ct_rb", "enkf_call_order"])
def test_enkf_single_mode_is_filter_zero(golden, name):
    g = golden(name)
    e = make(name, g, np.float64, single=True)
    t_z = 0
    for t, op in enumerate(str(o) for o in g["ops"]):
        t_z = run_op(e, g, t, t_z, op, single=True)
        assert isinstance(e.sigmas, np.ndarray) and e.sigmas.shape == (int(g["n_members"]), g["x"].shape[1])
        for k in KEYS:
            rel_close(_np(getattr(e, k)), g["ref_" + k][t][0], RTOL[np.float64], "%s %s t=%d" % (name, k, t))


def test_enkf_diagnostics_off_and_torch_op_match(golden):
    import torch
    from filterpy_b200 import _lib
    from filterpy_b200.torch_ops import load
    g = golden("enkf_cv_lin")
    a = make("enkf_cv_lin", g, np.float64)
    b = make("enkf_cv_lin", g, np.float64, diagnostics=False)
    load()
    x, P, s = a.x.clone(), a.P.clone(), a.sigmas.clone()
    counter = a.counter
    for t in range(3):
        a.predict(); a.update(g["zs"][t])
        b.predict(); b.update(g["zs"][t])
        z = torch.as_tensor(g["zs"][t], device=x.device)
        x, P, s = torch.ops.bke.enkf_step(x, P, s, a.Q, a.R, z, float(g["dt"]), _lib.BKE_FX_CONST_VEL,
                                          _lib.BKE_HX_LINEAR, a.seed, counter, H=torch.as_tensor(g["H"], device=x.device))
        counter += 2
        assert torch.equal(x, a.x) and torch.equal(P, a.P) and torch.equal(s, a.sigmas)
        rel_close(_np(b.x), _np(a.x), 1e-12, "diagnostics=False x")
        rel_close(_np(b.sigmas), _np(a.sigmas), 1e-12, "diagnostics=False sigmas")
    assert a.counter == counter


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_enkf_2048_members_stream_through_global_memory(dtype):
    """N = 2048 does not fit on chip at dim_x = 6: the passes run over the output array."""
    from filterpy_b200.common import workloads as wl
    from filterpy_b200.kalman import EnsembleKalmanFilter, ConstVelFx, RangeAzElHx
    F, N, seed = 4, 2048, 99
    w = wl.ukf_bank_cv3d(F, seed=5, steps=2, dt=0.1)
    e = EnsembleKalmanFilter(w["x"], w["P"], 3, 0.1, N, RangeAzElHx(), ConstVelFx(), n_filters=F, dtype=dtype, seed=seed)
    e.Q, e.R = w["Q"], w["R"]
    from test_oracle_enkf import fx_cv, hx_rae
    orc = []
    for f in range(F):
        o = oe.EnKF(w["x"][f], w["P"][f], 3, 0.1, N, hx_rae, fx_cv, oe.Stream(seed, f))
        o.Q, o.R = w["Q"][f], w["R"][f]
        orc.append(o)
    for t in range(2):
        e.predict(); e.update(w["zs"][t])
        for o in orc:
            o.predict(); o.update(w["zs"][t, orc.index(o)])
        for k in ("x", "P", "K", "sigmas"):
            rel_close(_np(getattr(e, k)), np.array([getattr(o, k) for o in orc]), RTOL[dtype], "%s t=%d" % (k, t))


def _bank(w, F, seed, N=32):
    from filterpy_b200.kalman import EnsembleKalmanFilter, ConstVelFx, LinearHx
    e = EnsembleKalmanFilter(w["x"][:F], w["P"][:F], 2, 0.5, N, LinearHx(w["H"][0]), ConstVelFx(), n_filters=F, seed=seed)
    e.Q, e.R = w["Q"][:F], w["R"][:F]
    for t in range(2):
        e.predict(); e.update(w["zs"][t, :F])
    return e


def test_enkf_stream_is_independent_of_bank_size_and_reproducible():
    import torch
    from filterpy_b200.common import workloads as wl
    w = wl.kf_bank_cv2d(1 << 16, seed=1, steps=2)
    big, small = _bank(w, 1 << 16, 5), _bank(w, 10, 5)
    for k in ("x", "P", "sigmas", "K"):
        assert torch.equal(getattr(big, k)[:10], getattr(small, k)), k
    assert torch.equal(_bank(w, 10, 5).sigmas, small.sigmas)
    assert not torch.equal(_bank(w, 10, 6).sigmas, small.sigmas)
    np.random.seed(3)
    a = _bank(w, 10, None)
    np.random.seed(3)
    assert torch.equal(_bank(w, 10, None).sigmas, a.sigmas)


def test_enkf_statistics_against_kalman_filter_bank():
    """Linear model, N = 4096 members over 2^12 filters: x and P within sampling tolerance of the KF."""
    import torch
    from filterpy_b200.kalman import EnsembleKalmanFilter, KalmanFilter, LinearFx, LinearHx
    from filterpy_b200.common import workloads as wl
    Fn, N, steps = 1 << 12, 4096, 4
    w = wl.ukf_bank_ct2d(Fn, seed=4, steps=steps, dt=0.5, linear_hx=True)
    Fm = np.eye(4); Fm[0, 1] = Fm[2, 3] = 0.5
    Q = w["Q"] + 0.01 * np.eye(4)                     # full rank, so that the KF's P stays comparable
    e = EnsembleKalmanFilter(w["x"], w["P"], 2, 0.5, N, LinearHx(w["H"]), LinearFx(Fm), n_filters=Fn, seed=11)
    e.Q, e.R = Q, w["R"]
    kf = KalmanFilter(4, 2, n_filters=Fn)
    kf.x = w["x"]; kf.P = w["P"]; kf.F = Fm; kf.H = w["H"]; kf.Q = Q; kf.R = w["R"]
    for t in range(steps):
        e.predict(); e.update(w["zs"][t])
        kf.predict(); kf.update(w["zs"][t])
    xk = kf.x.reshape(Fn, 4)
    Pk = kf.P
    sd = torch.sqrt(torch.diagonal(Pk, dim1=1, dim2=2))
    zsc = (e.x - xk) / sd
    # the ensemble mean errs by about sd / sqrt(N) per epoch of noise: rms z-score well below 0.1
    assert zsc.pow(2).mean().sqrt().item() < 0.1, zsc.pow(2).mean().sqrt().item()
    # no bias: the mean z-score over 2^12 filters is within a few of its standard errors
    assert zsc.mean(0).abs().max().item() < 0.01
    relP = (torch.diagonal(e.P, dim1=1, dim2=2) - torch.diagonal(Pk, dim1=1, dim2=2)) / torch.diagonal(Pk, dim1=1, dim2=2)
    assert relP.abs().median().item() < 0.05 and relP.mean(0).abs().max().item() < 0.02


def test_enkf_process_noise_lies_in_the_range_of_rank_deficient_q():
    import torch
    from filterpy_b200.kalman import EnsembleKalmanFilter, LinearFx, LinearHx
    Fn, N = 64, 4096
    dt, q = 0.5, 0.2
    blk = q * np.array([[dt ** 4 / 4, dt ** 3 / 2], [dt ** 3 / 2, dt ** 2]])
    Q = np.kron(np.eye(2), blk)
    e = EnsembleKalmanFilter(np.zeros(4), np.zeros((4, 4)), 2, dt, N, LinearHx(np.eye(2, 4)), LinearFx(np.eye(4)),
                             n_filters=Fn, seed=2)
    assert not e.sigmas.any()                         # P = 0: every member at x
    e.Q = Q
    e.predict()
    d = e.sigmas                                      # x = 0, F = I: the members are the drawn noise
    C = torch.einsum("fni,fnj->ij", d, d).cpu().numpy() / (Fn * N)
    assert np.abs(C - Q).max() < 0.03 * np.abs(Q).max()
    u, s, vt = np.linalg.svd(Q)
    null = vt[s < 1e-12 * s[0]]
    assert null.shape[0] == 2
    proj = d.reshape(-1, 4).cpu().numpy() @ null.T
    assert np.abs(proj).max() < 1e-10 * np.sqrt(np.abs(Q).max())
    e.Q = np.zeros((4, 4))
    before = e.sigmas.clone()
    e.predict(); e.x
    assert torch.equal(e.sigmas, before)              # Q = 0 draws exact zeros


def test_enkf_failures_set_status_and_raise():
    import torch
    from filterpy_b200.kalman import EnsembleKalmanFilter, ConstVelFx, LinearHx
    bad_q = np.diag([1.0, 1.0, -1.0, 1.0])
    e = EnsembleKalmanFilter(np.zeros((3, 4)), np.eye(4), 2, 0.1, 16, LinearHx(np.eye(2, 4)), ConstVelFx(), n_filters=3, seed=1)
    Qs = np.broadcast_to(np.eye(4), (3, 4, 4)).copy()
    Qs[1] = bad_q
    e.Q = Qs
    s0 = e.sigmas.clone()
    e.predict(); e.update(np.zeros((3, 2)))
    assert e.status.tolist() == [0, 2, 0]
    assert torch.equal(e.sigmas[1], s0[1])            # the failing filter keeps its members
    with pytest.raises(np.linalg.LinAlgError):
        e.check()
    single = EnsembleKalmanFilter(np.zeros(4), np.eye(4), 2, 0.1, 16, LinearHx(np.eye(2, 4)), ConstVelFx(), seed=1)
    single.Q = bad_q
    single.predict()
    with pytest.raises(np.linalg.LinAlgError):
        single.update(np.zeros(2))
    # singular S: H = 0 and R = 0
    s2 = EnsembleKalmanFilter(np.zeros(4), np.eye(4), 2, 0.1, 16, LinearHx(np.zeros((2, 4))), ConstVelFx(), seed=1)
    s2.R = np.zeros((2, 2))
    with pytest.raises(np.linalg.LinAlgError):
        s2.update(np.zeros(2))
    with pytest.raises(np.linalg.LinAlgError):
        EnsembleKalmanFilter(np.zeros(4), -np.eye(4), 2, 0.1, 16, LinearHx(np.eye(2, 4)), ConstVelFx(), seed=1)
    with pytest.raises(NotImplementedError):
        s2.inv = np.linalg.pinv
    for attr in ("y", "log_likelihood", "mahalanobis"):
        assert not hasattr(s2, attr)
    assert "EnsembleKalmanFilter object" in repr(s2)
