#!/usr/bin/env python
"""Generate the golden vectors of the polynomial trackers (tests/golden/poly_*.npz) from the UNMODIFIED reference.

Run after ``build()`` has staged the reference in ``oracle/_ref`` (``make -C oracle ref``):

    python tests/golden/make_golden_poly.py

Every case is a bank of N reference objects, one per filter, of one family (gh, ghk, gho, lsq, fm) and order:
  x0[N, S]        the initial state (gh: x, dx; ghk: x, dx, ddx; the others x[0..order])
  g, h, k, dt, beta [N] the parameters (NaN where the family has none); zs[T, N] the measurements
  snap[S]         the states kept: every state (0 .. T) for the small cases, every 40th and the last for the banks
  upd_state[S, N, S] the state at snap under update(); upd_y / upd_xp / upd_dxp / upd_ddxp [S-1, N] y and the
                  predictions of the update that led to snap[1:] (gh, ghk; gho: y); upd_z gho's z; upd_K lsq's K
  bat_res[S, N, 2], bat_pred[S-1, N]  batch_filter(zs, save_predictions=True) from x0 (gh, ghk) at the same epochs
The helper cases hold the gain helpers' inputs and outputs.  The tests never import the reference.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import save                                                            # noqa: E402

from filterpy.gh import (GHFilter, GHKFilter, GHFilterOrder, optimal_noise_smoothing,   # noqa: E402
                         least_squares_parameters, critical_damping_parameters, benedict_bornder_constants)
from filterpy.leastsq import LeastSquaresFilter                                         # noqa: E402
from filterpy.memory import FadingMemoryFilter                                          # noqa: E402

NAN = np.nan


def run(name, family, order, x0, zs, g=None, h=None, k=None, dt=None, beta=None, batch=True, every=1, **extra):
    """every > 1 stores the per-epoch outputs at the states snap = 0, every, 2 every, ..., T only"""
    T, N = zs.shape
    par = {n: (np.full(N, NAN) if v is None else np.broadcast_to(np.asarray(v, np.float64), (N,)).copy())
           for n, v in dict(g=g, h=h, k=k, dt=dt, beta=beta).items()}
    S = x0.shape[1]
    W = order + 1
    st = np.zeros((T + 1, N, S))
    y, xp, dxp, ddxp, zz = (np.zeros((T, N)) for _ in range(5))
    K = np.zeros((T, N, W))
    bres, bpred = np.zeros((T + 1, N, 2)), np.zeros((T, N))
    for f in range(N):
        p = {n: float(v[f]) for n, v in par.items()}
        if family == "gh":
            flt = GHFilter(x0[f, 0], x0[f, 1], p["dt"], p["g"], p["h"])
        elif family == "ghk":
            flt = GHKFilter(x0[f, 0], x0[f, 1], x0[f, 2], p["dt"], p["g"], p["h"], p["k"])
        elif family == "gho":
            flt = GHFilterOrder(x0[f].copy(), p["dt"], order, p["g"], None if order < 1 else p["h"],
                                None if order < 2 else p["k"])
        elif family == "lsq":
            flt = LeastSquaresFilter(p["dt"], order)
        else:
            flt = FadingMemoryFilter(x0[f].copy(), p["dt"], order, p["beta"])
        if family in ("gh", "ghk") and batch:
            bres[:, f], bpred[:, f] = flt.batch_filter(list(zs[:, f]), save_predictions=True)

        def state():
            if family == "gh":
                return [flt.x, flt.dx]
            if family == "ghk":
                return [flt.x, flt.dx, flt.ddx]
            return np.asarray(flt.x, np.float64).reshape(-1)
        st[0, f] = state()
        for t in range(T):
            flt.update(float(zs[t, f]))
            st[t + 1, f] = state()
            if family in ("gh", "ghk", "gho"):
                y[t, f] = np.asarray(flt.y).reshape(-1)[0]
            if family in ("gh", "ghk"):
                xp[t, f], dxp[t, f] = flt.x_prediction, flt.dx_prediction
            if family == "ghk":
                ddxp[t, f] = flt.ddx_prediction
            if family == "gho":
                zz[t, f] = np.asarray(flt.z).reshape(-1)[0]
            if family == "lsq":
                K[t, f] = flt.K
    snap = np.unique(np.r_[np.arange(0, T + 1, every), T])
    ep = snap[1:] - 1                                     # the epoch after which each later snapshot is taken
    out = dict(family=family, order=order, x0=x0, zs=zs, snap=snap, upd_state=st[snap], **par, **extra)
    if family in ("gh", "ghk", "gho"):
        out["upd_y"] = y[ep]
    if family in ("gh", "ghk"):
        out.update(upd_xp=xp[ep], upd_dxp=dxp[ep])
        if batch:
            out.update(bat_res=bres[snap], bat_pred=bpred[ep])
    if family == "ghk":
        out["upd_ddxp"] = ddxp[ep]
    if family == "gho":
        out["upd_z"] = zz[ep]
    if family == "lsq":
        out["upd_K"] = K[ep]
    save(name, **out)


def state0(family, order, N, rng, scale=1.):
    S = {"gh": 2, "ghk": 3}.get(family, order + 1)
    x0 = rng.standard_normal((N, S)) * scale
    if family in ("lsq",):
        x0[:] = 0.                                         # LeastSquaresFilter starts from zeros (least_squares.py:108)
    return x0


def gen_lsq_big_data(H=1000):
    """leastsq/tests/test_lsq.py::test_big_data: 10^6 epochs of orders 0, 1, 2 on z = i + noise (seeded here).
    Stored per order: the first H epochs from a fresh filter (head_z, head_x[H, W], head_K[H, W]) and the last H
    (tail_z; tail_n0 / tail_x0, the reference's counter and state before them; tail_x, tail_K).  The tail is where
    n(n+1)(n+2) passes 2**53, so the int -> float conversions of the gains round."""
    Nbig = 1000000
    zbig = np.arange(Nbig) + np.random.default_rng(13).standard_normal(Nbig)
    big = dict(head_z=zbig[:H], tail_z=zbig[-H:])
    for order in (0, 1, 2):
        lsq = LeastSquaresFilter(dt=1, order=order)
        hx, hK, tx, tK = [], [], [], []
        for t, zz in enumerate(zbig):
            if t == Nbig - H:
                big["tail_n0_%d" % order], big["tail_x0_%d" % order] = lsq.n, lsq.x.copy()
            lsq.update(zz)
            if t < H:
                hx.append(lsq.x.copy()); hK.append(lsq.K.copy())
            elif t >= Nbig - H:
                tx.append(lsq.x.copy()); tK.append(lsq.K.copy())
        big.update({"head_x_%d" % order: np.array(hx), "head_K_%d" % order: np.array(hK),
                    "tail_x_%d" % order: np.array(tx), "tail_K_%d" % order: np.array(tK)})
    save("poly_lsq_big_data", n_steps=Nbig, **big)


def main():
    # ---------------------------------------------------------------- the reference's own tests
    # gh/tests/test_gh.py::test_1d_array / test_2d_array: x = [0, 1], dx = 0, dt = 1, g = .8, h = .2; z = i, i+3
    i = np.arange(1, 10, dtype=np.float64)
    run("poly_gh_test_2d_array", "gh", 1, np.array([[0., 0.], [1., 0.]]), np.stack([i, i + 3], 1), g=.8, h=.2, dt=1.)
    # test_GHFilterOrder: order 1, g = .6, h = .02 against GHFilter; z = 2i + 1 + noise (seeded here)
    z = (2 * np.arange(100) + 1 + np.random.default_rng(11).standard_normal(100)).reshape(-1, 1)
    run("poly_gho_test_order1", "gho", 1, np.zeros((1, 2)), z, g=.6, h=.02, dt=1.)
    run("poly_gh_test_order1", "gh", 1, np.zeros((1, 2)), z, g=.6, h=.02, dt=1.)
    # leastsq/tests/test_lsq.py: test_first_order / test_second_order (Zarchan p. 105-6, 114), fig 3.8, listing 3.4
    xs = np.array([[1.2], [.2], [2.9], [2.1]])
    run("poly_lsq_first_order", "lsq", 1, np.zeros((1, 2)), xs, dt=1.)
    run("poly_lsq_second_order", "lsq", 2, np.zeros((1, 3)), xs, dt=1.)
    rng = np.random.default_rng(12)
    a = np.arange(0, 10, 0.1)
    run("poly_lsq_fig_3_8", "lsq", 1, np.zeros((1, 2)), (a + 3 + rng.standard_normal(a.size)).reshape(-1, 1), dt=0.1)
    run("poly_lsq_listing_3_4", "lsq", 2, np.zeros((1, 3)),
        (5 * a * a - a + 2 + 30 * rng.standard_normal(a.size)).reshape(-1, 1), dt=0.1)
    gen_lsq_big_data()
    # memory/tests/test_fading_memory.py: dotest_1d(order, beta) for several betas, and test_ghk_formulation
    betas = np.array([.3, .6, .7, .9])
    for order in (0, 1, 2):
        zs = np.arange(50)[:, None] + 3 * np.random.default_rng(20 + order).standard_normal((50, betas.size))
        run("poly_fm_1d_order%d" % order, "fm", order, np.zeros((betas.size, order + 1)), zs, dt=1., beta=betas)
    beta = .6
    g, h, k = 1 - beta**3, 1.5 * (1 + beta) * (1 - beta)**2, 0.5 * (1 - beta)**3
    zs = np.array([.02 * i**2 + 2 * i - 3 for i in range(1, 100)], np.float64)[:, None]
    run("poly_fm_ghk_formulation", "fm", 2, np.zeros((1, 3)), zs, dt=1., beta=beta)
    run("poly_ghk_ghk_formulation", "ghk", 2, np.zeros((1, 3)), zs, g=g, h=h, k=k, dt=1.)

    # ---------------------------------------------------------------- seeded banks, per-filter parameters
    N, T, E = 256, 200, 40
    rng = np.random.default_rng(30)
    t = np.arange(T)[:, None]

    def track(rng, dt):
        p0, v0, a0 = rng.uniform(-50, 50, N), rng.uniform(-3, 3, N), rng.uniform(-.05, .05, N)
        tt = t * dt
        z = p0 + v0 * tt + a0 * tt**2 + rng.standard_normal((T, N)) * rng.uniform(.1, 5, N)
        return np.round(z * 256) / 256                    # short mantissas: the file compresses

    dt = np.round(rng.uniform(.05, 2., N) * 64) / 64
    g = rng.uniform(.05, .9, N)
    h = g**2 / (2 - g) * rng.uniform(.5, 1.5, N)
    k = rng.uniform(.001, .05, N)
    run("poly_gh_bank", "gh", 1, state0("gh", 1, N, rng, 5), track(rng, dt), g=g, h=h, dt=dt, every=E)
    run("poly_ghk_bank", "ghk", 2, state0("ghk", 2, N, rng, 2), track(rng, dt), g=g, h=h, k=k, dt=dt, every=E)
    for order in (0, 1, 2):
        run("poly_gho_bank_order%d" % order, "gho", order, state0("gho", order, N, rng, 3), track(rng, dt),
            g=g, h=h, k=k, dt=dt, every=E)
        run("poly_lsq_bank_order%d" % order, "lsq", order, state0("lsq", order, N, rng), track(rng, dt), dt=dt, every=E)
        run("poly_fm_bank_order%d" % order, "fm", order, state0("fm", order, N, rng, 3), track(rng, dt), dt=dt,
            beta=rng.uniform(.05, .95, N), every=E)

    # ---------------------------------------------------------------- the quirks, one case each
    # GHFilter.batch_filter multiplies by h_dt = h / dt (gh_filter.py:433), update() rounds h * y / dt (:374)
    rng = np.random.default_rng(40)
    run("poly_quirk_gh_h_dt", "gh", 1, np.zeros((64, 2)), rng.standard_normal((40, 64)) * 7, g=.4, h=.1 * np.arange(1, 65) / 7,
        dt=np.full(64, .3))
    # GHKFilter.batch_filter ignores k and ddx (:717-743): a nonzero ddx and k
    run("poly_quirk_ghk_batch", "ghk", 2, np.column_stack([np.zeros(16), np.ones(16), np.full(16, 3.)]),
        rng.standard_normal((30, 16)) + np.arange(30)[:, None], g=.5, h=.2, k=.05, dt=.5)
    # GHFilterOrder stores z only for order 1 (:161)
    for order in (0, 1, 2):
        run("poly_quirk_gho_z_order%d" % order, "gho", order, np.zeros((4, order + 1)), rng.standard_normal((10, 4)),
            g=.5, h=.3, k=.1, dt=1.)
    # LeastSquaresFilter order 0 takes y = z - x over the whole vector (:132-133)
    run("poly_quirk_lsq_order0", "lsq", 0, np.zeros((8, 1)), rng.standard_normal((25, 8)) + 4, dt=1.)

    # ---------------------------------------------------------------- gain helpers
    gs = np.linspace(.01, .99, 99)
    ons = np.array([optimal_noise_smoothing(float(v)) for v in gs])
    n = np.arange(0, 200)
    lsp = np.array([least_squares_parameters(int(v)) for v in n])
    th = np.linspace(0., 1., 101)
    cd2 = np.array([critical_damping_parameters(float(v)) for v in th])
    cd3 = np.array([critical_damping_parameters(float(v), order=3) for v in th])
    bb = np.array([benedict_bornder_constants(float(v)) for v in gs])
    bbc = np.array([benedict_bornder_constants(float(v), critical=True) for v in gs])
    vr = []
    for gv in gs[::7]:
        f2 = GHFilter(0., 0., .5, float(gv), float(gv**2 / (2 - gv)))
        f3 = GHKFilter(0., 0., 0., .5, *[float(v) for v in ons[int(np.argmin(abs(gs - gv)))]])
        vr.append([f2.VRF_prediction(), *f2.VRF(), f3.VRF_prediction(), *f3.VRF(), f3.bias_error(1.5)])
    save("poly_helpers", gs=gs, ons=ons, n=n, lsp=lsp, theta=th, cd2=cd2, cd3=cd3, bb=bb, bbc=bbc, vrf_g=gs[::7],
         vrf=np.array(vr))


if __name__ == "__main__":
    if sys.argv[1:] == ["lsq_big_data"]:          # regenerate that file alone
        gen_lsq_big_data()
    else:
        main()
