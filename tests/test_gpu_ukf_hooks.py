"""GPU parity: the UKF / CKF with DeviceFn hooks (wrapped residuals, circular means, a wrapping state_add)
against the reference's golden vectors and the vectorised hooked oracle."""
import numpy as np
import pytest

import ukf_hooks_oracle as oh
from oracle import ukf as oukf
from gpu_harness import rel_close, RTOL

pytestmark = pytest.mark.gpu


def _hooks(all_five):
    from filterpy_b200.kalman import DeviceFn
    from filterpy_b200.common import workloads as wl
    rb = DeviceFn(wl.RB_HOOKS_SOURCE)                     # one object for two hooks: its text is included once
    h = dict(residual_z=rb, z_mean_fn=rb)
    if all_five:
        x = DeviceFn(wl.CTRV_X_HOOKS_SOURCE)
        h.update(residual_x=x, x_mean_fn=x, state_add=x)
    return h


def make(name, g, dtype, N=None, diagnostics=True, hooks=True):
    from filterpy_b200.kalman import (UnscentedKalmanFilter, MerweScaledSigmaPoints, ConstVelFx, RangeBearingHx,
                                      DeviceFx, DeviceHx)
    from filterpy_b200.common import workloads as wl
    ab = (float(g["alpha"]), float(g["beta"]), float(g["kappa"])) if "alpha" in g else (0.8, 2.0, 0.0)
    if name.startswith("ukf_hooks_ctrv"):
        sx, sy = (float(v) for v in g["sensor"])
        fx, hx, n = DeviceFx(wl.CTRV_FX_SOURCE), DeviceHx(wl.CTRV_RB_HX_SOURCE, arg_names=("sx", "sy"), sx=sx, sy=sy), 5
    else:
        fx, hx, n = ConstVelFx(), RangeBearingHx(), 4
    N = g["x"].shape[0] if N is None else N
    u = UnscentedKalmanFilter(n, 2, float(g["dt"]), hx, fx, MerweScaledSigmaPoints(n, *ab), n_filters=N, dtype=dtype,
                              diagnostics=diagnostics, **(_hooks(n == 5) if hooks else {}))
    u.x = g["x"][:N]; u.P = g["P"][:N]; u.Q = g["Q"][:N]; u.R = g["R"][:N]
    return u


def _check_update(f, g, t, rtol):
    v = g["valid"][t]
    rel_close(f.x.cpu().numpy(), g["ref_x"][t], rtol, "x t=%d" % t)
    rel_close(f.P.cpu().numpy(), g["ref_P"][t], rtol, "P t=%d" % t)
    rel_close(f.x_prior.cpu().numpy(), g["ref_x_prior"][t], rtol, "x_prior t=%d" % t)
    rel_close(f.P_prior.cpu().numpy(), g["ref_P_prior"][t], rtol, "P_prior t=%d" % t)
    if v.any():
        rel_close(f.K.cpu().numpy()[v], g["ref_K"][t][v], rtol, "K t=%d" % t)
        rel_close(f.S.cpu().numpy()[v], g["ref_S"][t][v], rtol, "S t=%d" % t)
        # the wrapped y: compared as z - y (y = z - z^ cancels most digits of z)
        z = g["zs"][t]
        rel_close((z - f.y.cpu().numpy())[v], (z - g["ref_y"][t])[v], rtol, "z - y t=%d" % t)
        rel_close(f.log_likelihood.cpu().numpy()[v], g["ref_loglik"][t][v], 10 * rtol, "loglik t=%d" % t)
    assert int(f.status.sum().item()) == 0


@pytest.mark.parametrize("name", ["ukf_hooks_rb", "ukf_hooks_ctrv"])
def test_ukf_hooks_vs_reference_golden(golden, name):
    g = golden(name)
    u = make(name, g, np.float64)
    for t in range(g["zs"].shape[0]):
        u.predict()
        u.update(g["zs"][t], valid=g["valid"][t])
        _check_update(u, g, t, RTOL[np.float64])


def test_ckf_residual_z_vs_reference_golden(golden):
    from filterpy_b200.kalman import CubatureKalmanFilter, ConstVelFx, RangeBearingHx
    g = golden("ckf_hooks_rb")
    c = CubatureKalmanFilter(4, 2, float(g["dt"]), RangeBearingHx(), ConstVelFx(), residual_z=_hooks(False)["residual_z"],
                             n_filters=g["x"].shape[0])
    c.x = g["x"]; c.P = g["P"]; c.Q = g["Q"]; c.R = g["R"]
    for t in range(g["zs"].shape[0]):
        c.predict()
        c.update(g["zs"][t], valid=g["valid"][t])
        _check_update(c, g, t, RTOL[np.float64])


def test_rb_fp32_2p16_vs_vectorised_oracle():
    from filterpy_b200.common import workloads as wl
    N, steps, dt = 1 << 16, 6, 1.0
    w = wl.ukf_bank_rb_behind(N, seed=4242, steps=steps, dt=dt)
    w32 = {k: v.astype(np.float32).astype(np.float64) for k, v in w.items()}        # the inputs the GPU sees
    g = dict(w32, dt=dt, alpha=0.8, beta=2.0, kappa=0.0)
    u = make("ukf_hooks_rb", g, np.float32, diagnostics=False)
    x, P = w32["x"], w32["P"]
    for t in range(steps):
        u.predict(); u.update(w32["zs"][t])
        o = oh.ukf_step_bank_hooks(x, P, w32["zs"][t], w32["Q"], w32["R"], dt, 0.8, 2.0, 0.0, oukf.FX_CONST_VEL,
                                   oukf.HX_RANGE_BEARING, angle_z=(1,), z_mean=True)
        x, P = o["x"], o["P"]
        rel_close(u.x.cpu().numpy(), x, RTOL[np.float32], "x t=%d" % t)
        rel_close(u.P.cpu().numpy(), P, RTOL[np.float32], "P t=%d" % t)


def test_batch_filter_equals_loop_and_rts_vs_golden(golden):
    import torch
    g = golden("ukf_hooks_ctrv_rts")
    a, b = make("ukf_hooks_ctrv_rts", g, np.float64), make("ukf_hooks_ctrv_rts", g, np.float64)
    means, covs = a.batch_filter(g["zs"])
    for t in range(g["zs"].shape[0]):
        b.predict(); b.update(g["zs"][t])
        assert torch.equal(means[t], b.x) and torch.equal(covs[t], b.P)
    rel_close(means.cpu().numpy(), g["Xs"], RTOL[np.float64], "batch_filter means")
    rel_close(covs.cpu().numpy(), g["Ps"], RTOL[np.float64], "batch_filter covariances")
    xs, Ps, Ks = a.rts_smoother(torch.as_tensor(g["Xs"], device=a._device), torch.as_tensor(g["Ps"], device=a._device))
    rel_close(xs.cpu().numpy(), g["ref_x"], RTOL[np.float64], "rts x")
    rel_close(Ps.cpu().numpy(), g["ref_P"], RTOL[np.float64], "rts P")
    rel_close(Ks.cpu().numpy(), g["ref_K"], RTOL[np.float64], "rts K")


def test_hooked_rts_with_builtin_fx_equals_builtin_smoother(golden):
    """A hooked handle around ConstVelFx carries its own RTS kernel; with no x hooks it is the built-in smoother."""
    import torch
    g = golden("ukf_hooks_rb")
    a, b = make("ukf_hooks_rb", g, np.float64), make("ukf_hooks_rb", g, np.float64, hooks=False)
    means, covs = a.batch_filter(g["zs"])
    sa, sb = a.rts_smoother(means, covs), b.rts_smoother(means.clone(), covs.clone())
    for p, q in zip(sa, sb):
        rel_close(p.cpu().numpy(), q.cpu().numpy(), 1e-12, "rts")
    assert torch.isfinite(sa[0]).all()


def test_single_mode_and_failure_status(golden):
    g = golden("ukf_hooks_rb")
    from filterpy_b200.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, ConstVelFx, RangeBearingHx
    u = UnscentedKalmanFilter(4, 2, float(g["dt"]), RangeBearingHx(), ConstVelFx(), MerweScaledSigmaPoints(4, .8, 2., 0.),
                              **_hooks(False))
    u.x = g["x"][0]; u.P = g["P"][0]; u.Q = g["Q"][0]; u.R = g["R"][0]
    for t in range(g["zs"].shape[0]):                        # single mode: filter 0 of the bank, NumPy attributes
        u.predict(); u.update(g["zs"][t, 0] if g["valid"][t, 0] else None)
        rel_close(u.x, g["ref_x"][t, 0], RTOL[np.float64], "single x t=%d" % t)
        rel_close(u.P, g["ref_P"][t, 0], RTOL[np.float64], "single P t=%d" % t)
    # the status / LinAlgError path is unchanged: an indefinite P fails that filter only
    bank = make("ukf_hooks_rb", g, np.float64)
    P = g["P"].copy(); P[3] = -np.eye(4)
    bank.P = P
    bank.predict(); bank.update(g["zs"][0])
    st = bank.status.cpu().numpy()
    assert st[3] != 0 and (np.delete(st, 3) == 0).all()
    with pytest.raises(np.linalg.LinAlgError):
        bank.check()
    u.P = -np.eye(4)
    u.predict()
    with pytest.raises(np.linalg.LinAlgError):
        u.update(g["zs"][4, 0])
