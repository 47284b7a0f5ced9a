"""GPU: the polynomial tracker banks (bke_poly_filter) on every (family, order, dtype) instance against the reference's
golden vectors (fp64 bit for bit, fp32 within 1e-3), T update() calls against one batch_filter, shared against
per-filter parameters, the reference's test_2d_array identity, single mode and its exceptions, the torch op against
the ctypes path, and banks whose size is not a multiple of the block."""
import numpy as np
import pytest
import torch

from filterpy_b200 import _lib
from filterpy_b200.gh import GHFilter, GHKFilter, GHFilterOrder
from filterpy_b200.leastsq import LeastSquaresFilter
from filterpy_b200.memory import FadingMemoryFilter

import poly_oracle as po
from test_oracle_poly import CASES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DTYPES = [np.float64, np.float32]


def _np(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, np.float64)


def _same(a, b, dtype, scale=0.):
    """fp64: equal; fp32: within 1e-3 of max|b|, or of `scale` for a quantity that cancels (a residual against the
    measurements it is the difference of)"""
    a, b = _np(a), np.asarray(b, np.float64)
    if dtype == np.float64:
        assert np.array_equal(a, b)
    else:
        assert np.abs(a - b).max(initial=0) <= 1e-3 * max(np.abs(b).max(initial=0), scale, 1e-30)


def _make(c, dtype, N=None, idx=None):
    fam, order = str(c["family"]), int(c["order"])
    sel = slice(None) if idx is None else idx
    x0 = c["x0"][sel]
    N = x0.shape[0]
    p = {k: c[k][sel] for k in ("g", "h", "k", "dt", "beta")}
    kw = dict(n_filters=N, dtype=dtype, device=DEV)
    if fam == "gh":
        return GHFilter(x0[:, 0], x0[:, 1], p["dt"], p["g"], p["h"], **kw)
    if fam == "ghk":
        return GHKFilter(x0[:, 0], x0[:, 1], x0[:, 2], p["dt"], p["g"], p["h"], p["k"], **kw)
    if fam == "gho":
        return GHFilterOrder(x0, p["dt"], order, p["g"], p["h"] if order >= 1 else None, p["k"] if order == 2 else None, **kw)
    if fam == "lsq":
        return LeastSquaresFilter(p["dt"], order, **kw)
    return FadingMemoryFilter(x0, p["dt"], order, p["beta"], **kw)


def _state(f, fam):
    if fam == "gh":
        return torch.stack([f.x, f.dx], 1)
    if fam == "ghk":
        return torch.stack([f.x, f.dx, f.ddx], 1)
    return f.x


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", CASES)
def test_bank_update_matches_golden(golden, name, dtype):
    c = golden(name)
    fam = str(c["family"])
    f = _make(c, dtype)
    snap = list(c["snap"])
    zs = torch.as_tensor(c["zs"], device=DEV)
    zmax = float(np.abs(c["zs"]).max())
    for t in range(c["zs"].shape[0]):
        f.update(zs[t].to(f._dtype))
        if t + 1 in snap:
            i = snap.index(t + 1)
            _same(_state(f, fam), c["upd_state"][i], dtype)
            if fam in ("gh", "ghk", "gho"):
                _same(f.y, c["upd_y"][i - 1], dtype, zmax)
            if fam in ("gh", "ghk"):
                _same(f.x_prediction, c["upd_xp"][i - 1], dtype, zmax)
                _same(f.dx_prediction, c["upd_dxp"][i - 1], dtype, zmax)
            if fam == "ghk":
                _same(f.ddx_prediction, c["upd_ddxp"][i - 1], dtype, zmax)
            if fam == "gho":
                _same(f.z if int(c["order"]) == 1 else torch.zeros(c["x0"].shape[0]), c["upd_z"][i - 1], dtype)
            if fam == "lsq":
                _same(f.K, c["upd_K"][i - 1], dtype)
                assert (f.n == t + 1).all()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", CASES)
def test_bank_batch_filter_matches_golden_and_updates(golden, name, dtype):
    """gh / ghk: batch_filter against the reference's (its own rounding, h / dt); the others: batch_filter is T
    update() calls on a copy, so it equals the golden update states and leaves the filter alone"""
    c = golden(name)
    fam = str(c["family"])
    f = _make(c, dtype)
    before = _np(_state(f, fam)).copy()
    zs = torch.as_tensor(c["zs"], device=DEV).to(f._dtype)
    if fam in ("gh", "ghk"):
        res, pred = f.batch_filter(zs, save_predictions=True)
        _same(_np(res)[c["snap"]], c["bat_res"], dtype)
        _same(_np(pred)[c["snap"][1:] - 1], c["bat_pred"], dtype)
    else:
        res = f.batch_filter(zs)
        _same(_np(res)[c["snap"]], c["upd_state"], dtype)
    assert np.array_equal(_np(_state(f, fam)), before)


def test_gh_update_and_batch_round_apart(golden):
    """the same bank through update() and batch_filter: each equals its own golden, and they differ (h*y/dt vs h/dt*y)"""
    c = golden("poly_quirk_gh_h_dt")
    f = _make(c, np.float64)
    res = _np(f.batch_filter(c["zs"]))
    for t in range(c["zs"].shape[0]):
        f.update(c["zs"][t])
    assert np.array_equal(_np(torch.stack([f.x, f.dx], 1)), c["upd_state"][-1])
    assert np.array_equal(res[-1], c["bat_res"][-1])
    assert not np.array_equal(res[-1], c["upd_state"][-1])


@pytest.mark.parametrize("name", ["poly_gh_bank", "poly_ghk_bank", "poly_gho_bank_order2", "poly_lsq_bank_order1",
                                  "poly_fm_bank_order2"])
def test_shared_parameters_equal_per_filter_copies(golden, name):
    c = dict(golden(name))
    for k in ("g", "h", "k", "dt", "beta"):
        c[k] = np.full_like(c[k], c[k][0])
    per = _make(c, np.float64)
    fam, order = str(c["family"]), int(c["order"])
    x0 = c["x0"]
    N = x0.shape[0]
    kw = dict(n_filters=N, dtype=np.float64, device=DEV)
    s = {k: float(c[k][0]) for k in ("g", "h", "k", "dt", "beta")}
    shared = {"gh": lambda: GHFilter(x0[:, 0], x0[:, 1], s["dt"], s["g"], s["h"], **kw),
              "ghk": lambda: GHKFilter(x0[:, 0], x0[:, 1], x0[:, 2], s["dt"], s["g"], s["h"], s["k"], **kw),
              "gho": lambda: GHFilterOrder(x0, s["dt"], order, s["g"], s["h"], s["k"], **kw),
              "lsq": lambda: LeastSquaresFilter(s["dt"], order, **kw),
              "fm": lambda: FadingMemoryFilter(x0, s["dt"], order, s["beta"], **kw)}[fam]()
    assert shared._p["dt"][2] == 0 and per._p["dt"][2] == 1
    for t in range(40):
        per.update(c["zs"][t])
        shared.update(c["zs"][t])
    assert torch.equal(_state(per, fam), _state(shared, fam))
    if fam in ("gh", "ghk"):               # per-call gains: a scalar and an (N,) tensor of it agree
        per.update(c["zs"][40], g=torch.full((N,), .3, dtype=torch.float64, device=DEV), h=.01)
        shared.update(c["zs"][40], g=.3, h=torch.full((N,), .01, dtype=torch.float64, device=DEV))
        assert torch.equal(_state(per, fam), _state(shared, fam))


def test_reference_2d_array_identity():
    """gh/tests/test_gh.py::test_2d_array on the GPU: an array filter equals scalar filters, with =="""
    for zs in ([(i, i) for i in range(1, 10)], [(i, i + 3) for i in range(1, 10)]):
        f = GHFilter(np.array([0, 1]), np.array([0, 0]), 1, .8, .2)
        f0 = GHFilter(0, 0, 1, .8, .2)
        f1 = GHFilter(1, 0, 1, .8, .2)
        for a, b in zs:
            f.update(np.array([a, b]) if b != a else a)
            f0.update(a)
            f1.update(b)
            assert f.x[0] == f0.x and f.x[1] == f1.x
            assert f.dx[0] == f0.dx and f.dx[1] == f1.dx
            assert f.VRF() == f0.VRF() == f1.VRF()


def test_single_mode_matches_golden(golden):
    c = golden("poly_gho_test_order1")
    f1 = GHFilterOrder(x0=np.array([0, 0]), dt=1, order=1, g=.6, h=.02)
    f2 = GHFilter(x=0, dx=0, dt=1, g=.6, h=.02)
    for z in c["zs"][:, 0]:
        f1.update(z)
        f2.update(z)
        assert f1.x[0] == f2.x                             # test_GHFilterOrder's identity, exactly
    assert np.array_equal(f1.x, c["upd_state"][-1, 0]) and f1.z == c["zs"][-1, 0]
    g = golden("poly_lsq_second_order")
    lsq = LeastSquaresFilter(1, order=2)
    for t, z in enumerate(g["zs"][:, 0]):
        x = lsq.update(z)
        assert np.array_equal(x, g["upd_state"][t + 1, 0]) and lsq.n == t + 1 and lsq.y == 0
    err, std = lsq.errors()
    assert err.shape == (3,) and std.shape == (3,)
    lsq.reset()
    assert lsq.n == 0 and not lsq.x.any()
    m = golden("poly_fm_ghk_formulation")
    fm = FadingMemoryFilter(x0=0, dt=1, order=2, beta=.6)
    k = GHKFilter(0, 0, 0, 1, *[float(m2) for m2 in (1 - .6**3, 1.5 * 1.6 * .4**2, .5 * .4**3)])
    for z in m["zs"][:, 0]:
        fm.update(z)
        k.update(z)
    assert np.array_equal(fm.x, m["upd_state"][-1, 0]) and fm.P.shape == (3,) and fm.e.shape == (3,)
    res, pred = GHFilter(0., 0., 1., .6, .02).batch_filter(list(c["zs"][:, 0]), save_predictions=True)
    assert res.shape == (c["zs"].shape[0] + 1, 2) and pred.shape == (c["zs"].shape[0],)


def test_single_mode_exceptions():
    for make in (lambda: GHFilterOrder(0., 1., 3, .5), lambda: LeastSquaresFilter(1., -1),
                 lambda: FadingMemoryFilter(0., 1., 5, .5)):
        with pytest.raises(ValueError, match='order must be between 0 and 2'):
            make()
    with pytest.raises(NotImplementedError):
        GHFilter(0., 0., 1., .5, .1).batch_filter([1., 2.], saver=object())
    lsq = LeastSquaresFilter(1., 1)
    lsq.update(1.)
    with pytest.raises(ZeroDivisionError):                # std[1] at n = 1 divides by n(n*n - 1) = 0
        lsq.errors()


@pytest.mark.parametrize("dtype", DTYPES)
def test_torch_op_matches_the_ctypes_path(golden, dtype):
    from filterpy_b200 import torch_ops
    torch_ops.load()
    td = torch.float64 if dtype == np.float64 else torch.float32
    c = golden("poly_ghk_bank")
    f = _make(c, dtype)
    z = torch.as_tensor(c["zs"][:20], device=DEV).to(td)
    P = lambda a: torch.as_tensor(a, device=DEV).to(td)                                  # noqa: E731
    x, dx, ddx, _, res, _ = torch.ops.bke.poly_filter(P(c["x0"][:, 0]), P(c["x0"][:, 1]), P(c["x0"][:, 2]), None, z,
                                                       f._p["g"][1], f._p["h"][1], f._p["k"][1], f._p["dt"][1],
                                                       f._p["dt2"][1], None, _lib.BKE_POLY_GHK, 2, False)
    for t in range(20):
        f.update(z[t])
    assert torch.equal(x, f.x) and torch.equal(dx, f.dx) and torch.equal(ddx, f.ddx)
    assert torch.equal(res[-1], torch.stack([f.x, f.dx], 1))
    c = golden("poly_lsq_bank_order2")
    f = _make(c, dtype)
    z = torch.as_tensor(c["zs"][:20], device=DEV).to(td)
    n0 = torch.zeros(z.shape[1], dtype=torch.int64, device=DEV)
    x, _, _, n, res, pred = torch.ops.bke.poly_filter(torch.zeros_like(f.x), None, None, n0, z, None, None, None,
                                                      f._p["dt"][1], f._p["dt2"][1], f._p["hdt2"][1],
                                                      _lib.BKE_POLY_LSQ, 2, False)
    for t in range(20):
        f.update(z[t])
    assert torch.equal(x, f.x) and torch.equal(n, f.n) and pred.numel() == 0 and not n0.any()


@pytest.mark.parametrize("N", [1, 255, 257, 1000])
def test_ragged_bank_sizes(golden, N):
    """N not a multiple of the 256-thread block: the first N filters of a bank, tiled"""
    c = golden("poly_fm_bank_order2")
    idx = np.arange(N) % c["x0"].shape[0]
    f = _make(c, np.float64, idx=idx)
    for t in range(c["zs"].shape[0]):
        f.update(c["zs"][t][idx])
    assert np.array_equal(_np(f.x), c["upd_state"][-1][idx])
    o = po.run(c)
    assert np.array_equal(o["upd_state"][-1][idx], c["upd_state"][-1][idx])


@pytest.mark.parametrize("family,order,shape", [
    (_lib.BKE_POLY_GH_ORDER, 1, (64,)),            # [N] for order 1: the kernel would index x[f * 2 + j]
    (_lib.BKE_POLY_LSQ, 2, (64,)),
    (_lib.BKE_POLY_FADING, 2, (64, 2)),            # W < order + 1
    (_lib.BKE_POLY_LSQ, 1, (64, 3)),               # W > order + 1
    (_lib.BKE_POLY_GH, 1, (64, 2)),                # GH keeps x, dx apart
    (_lib.BKE_POLY_GHK, 2, (64, 3)),
])
def test_torch_op_refuses_a_mis_shaped_x(family, order, shape):
    """the call carries no size for x, so the op checks its shape before any launch"""
    from filterpy_b200 import torch_ops
    ops = torch_ops.load()
    x = torch.zeros(shape, dtype=torch.float64, device=DEV)
    v = torch.zeros(64, dtype=torch.float64, device=DEV)
    z = torch.zeros((3, 64), dtype=torch.float64, device=DEV)
    s = torch.tensor(.5, dtype=torch.float64, device=DEV)
    n = torch.zeros(64, dtype=torch.int64, device=DEV)
    with pytest.raises(RuntimeError, match="x"):
        ops.poly_filter(x, v, v, n, z, s, s, s, s, s, s, family, order, False)
    torch.cuda.synchronize()


def test_lsq_big_data_tail_on_the_counter_past_2_53(golden):
    """the reference's test_big_data: the first epochs from a fresh bank, and the last ones from the reference's
    counter and state at epoch 10^6 - H, where the gains' int -> float conversions round"""
    c = golden("poly_lsq_big_data")
    H = c["head_z"].size
    for order in (0, 1, 2):
        f = LeastSquaresFilter(1., order, n_filters=1, dtype=np.float64, device=DEV)
        for t in range(H):
            f.update(c["head_z"][t:t + 1])
        assert np.array_equal(_np(f.x)[0], c["head_x_%d" % order][-1])
        f.n, f.x = int(c["tail_n0_%d" % order]), c["tail_x0_%d" % order][None]
        res = _np(f.batch_filter(c["tail_z"][:, None]))[1:, 0]
        assert np.array_equal(res, c["tail_x_%d" % order])
        for t in range(H):
            f.update(c["tail_z"][t:t + 1])
        assert np.array_equal(_np(f.x)[0], c["tail_x_%d" % order][-1])
        assert np.array_equal(_np(f.K)[0], c["tail_K_%d" % order][-1])
        assert int(f.n[0]) == int(c["n_steps"])
