"""CPU: the fp64 scoring oracle against the reference's stats golden vectors, the argument checks of
bke_score_measurements (made before any device is needed) and the stats mirrors' shape and exception checks
before any device is touched."""
import ctypes
import math

import numpy as np
import pytest

from filterpy_b200 import _lib

import stats_oracle as so

SHAPES = [(1, 1), (2, 1), (4, 2), (6, 3), (9, 3)]


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def test_oracle_matches_mahalanobis_golden(golden):
    g = golden("stats_mahalanobis")
    for i in range(int(g["n_cases"])):
        x, mean = np.atleast_1d(g["c%d_x" % i].squeeze()), np.atleast_1d(g["c%d_mean" % i].squeeze())
        S = np.atleast_2d(g["c%d_cov" % i])
        o = so.score(x.reshape(1, 1, -1), mean.reshape(1, -1), S[None])
        assert abs(math.sqrt(o["d2"][0, 0]) - float(g["c%d_out" % i])) <= 1e-10 * max(1.0, float(g["c%d_out" % i])), i
    # the reference's docstring examples
    assert [float(g["c%d_out" % i]) for i in (10, 11)] == [0.125, 3.0]
    assert abs(float(g["c12_out"]) - 0.42533327058913922) < 1e-15


@pytest.mark.parametrize("n,m", SHAPES)
@pytest.mark.parametrize("layout", ["own", "scan"])
def test_oracle_matches_bank_golden(golden, n, m, layout):
    g = golden("stats_bank_%d_%d" % (n, m))
    N, K = g["ll_own"].shape
    z = g["z_own"] if layout == "own" else np.broadcast_to(g["z_scan"], (N, K, m))
    zhat = np.einsum("fmn,fn->fm", g["H"], g["x"])
    o = so.score(z, zhat, so.innovation_cov(g["P"], g["H"], g["R"]))
    assert _rel(o["log_likelihood"], g["ll_" + layout]) < 1e-10
    assert _rel(o["log_likelihood"], g["logpdf_" + layout]) < 1e-10
    assert _rel(o["likelihood"], g["lk_" + layout]) < 1e-10
    assert _rel(o["mahalanobis"], g["maha_" + layout]) < 1e-10


def test_oracle_matches_kf_methods_golden(golden):
    """log_likelihood_of after update scores with the update's S; after predict it mixes the prior x with that S
    (before the first update S = 0: the reference's -inf, a singular S here)."""
    g = golden("stats_kf_methods")
    F, H, Q, R = g["F"], g["H"], g["Q"], g["R"]
    x, P = g["x0"][:, 0], g["P0"]
    S = np.zeros((2, 2))
    for t in range(g["zs"].shape[0]):
        x, P = F @ x, F @ P @ F.T + Q
        o = so.score(g["cands"][t][None], (H @ x)[None], S[None])
        if t == 0:
            assert o["status"][0] == 1 and np.isneginf(g["ll_pred"][0]).all()
        else:
            assert _rel(o["log_likelihood"][0], g["ll_pred"][t]) < 1e-10
        assert _rel(g["zs"][t] - H @ x, g["res_pred"][t][:, 0]) < 1e-12
        assert _rel(H @ x, g["mos"][t][:, 0]) < 1e-12
        S = H @ P @ H.T + R
        K = P @ H.T @ np.linalg.inv(S)
        xp = x
        x = x + K @ (g["zs"][t] - H @ x)
        I_KH = np.eye(4) - K @ H
        P = I_KH @ P @ I_KH.T + K @ R @ K.T
        o = so.score(g["cands"][t][None], (H @ x)[None], S[None])
        assert _rel(o["log_likelihood"][0], g["ll_upd"][t]) < 1e-10
        assert _rel(g["zs"][t] - H @ xp, g["res_upd"][t][:, 0]) < 1e-12
    assert float(g["ll_none"]) == so.LOG_DBL_MIN and np.isneginf(g["ll_before"])


def test_oracle_matches_nees_golden(golden):
    g = golden("stats_nees")
    T = g["nees"].shape[0]
    o = so.score((g["xs"] - g["est_xs"]).reshape(T, 1, -1), np.zeros((T, 4)), g["ps"])
    assert _rel(o["d2"][:, 0], g["nees"]) < 1e-10


def test_deviations_from_scipy(golden):
    """Each case is a documented deviation (INTEGRATION.md): the reference's value or raise against the rule."""
    g = golden("stats_deviations")
    z, mean = g["z"][None, None], g["mean"][None]
    assert np.isneginf(g["logpdf_sing"]) and so.score(z, mean, g["S_sing"][None])["status"][0] == 1
    o = so.score(z, mean, g["S_cut"][None])                   # scipy drops the 1e-14 eigenvalue, the rule does not
    assert np.isneginf(g["logpdf_cut"]) and o["status"][0] == 0 and np.isfinite(o["log_likelihood"][0, 0])
    assert str(g["raise_indef"]) == "ValueError"              # scipy refuses an indefinite S; the rule scores it
    o = so.score(z, mean, g["S_indef"][None])
    SI = np.linalg.inv(g["S_indef"])
    d2 = g["z"] @ SI @ g["z"]
    assert np.isclose(o["log_likelihood"][0, 0], -0.5 * (d2 + math.log(2.) + 2 * math.log(2 * math.pi)))
    assert str(g["raise_len"]) == "ValueError"
    assert str(g["raise_maha_sing"]) == "LinAlgError" and str(g["raise_nees_sing"]) == "LinAlgError"


def test_oracle_missing_candidates():
    z = np.ones((2, 3, 2))
    v = np.array([[1, 0, 1], [0, 0, 1]], bool)
    o = so.score(z, np.zeros((2, 2)), np.stack([np.eye(2), np.zeros((2, 2))]), v)
    assert o["log_likelihood"][0, 1] == so.LOG_DBL_MIN and o["d2"][1, 0] == 0 and (o["y"][1, 1] == 0).all()
    assert np.isnan(o["d2"][1, 2]) and o["status"].tolist() == [0, 1]


# ---------------------------------------------------------------------------------------------- the C-ABI
def _zeros(n, dtype=np.float64):
    """np.zeros(n), page-locked where there is a device: a call that passes the checks then runs its kernel, which
    reads and writes these buffers through their host addresses."""
    import torch
    z = np.zeros(n, dtype)
    return torch.from_numpy(z).pin_memory().numpy() if torch.cuda.is_available() else z


def _args(n=4, m=2, N=8, K=3):
    keep = {k: _zeros(N * K * max(n, m) ** 2 + 16) for k in ("x", "P", "H", "R", "z", "ll", "zhat")}
    a = _lib.ScoreArgs()
    a.n_tracks, a.n_candidates, a.dim_x, a.dim_z, a.dtype = N, K, n, m, _lib.BKE_F64
    a.x, a.P, a.H, a.R, a.z = (keep[k].ctypes.data for k in ("x", "P", "H", "R", "z"))
    a.H_stride, a.R_stride = m * n, m * m
    a.z_track_stride, a.z_cand_stride = K * m, m
    a.log_likelihood = keep["ll"].ctypes.data
    return a, keep


def _refused(a):
    return _lib.load().bke_score_measurements(ctypes.byref(a), None) == _lib.BKE_ERR_BAD_ARG


@pytest.mark.parametrize("field,value", [
    ("n_tracks", -1), ("n_candidates", -1), ("dtype", 3), ("dim_z", 0), ("dim_x", 0), ("dim_z", 1025),
    ("x", None), ("R", None), ("z", None), ("H_stride", 3), ("R_stride", 1), ("z_track_stride", -1),
    ("z_cand_stride", -2), ("log_likelihood", None),
])
def test_score_refuses_bad_arguments(field, value):
    a, keep = _args()
    setattr(a, field, value)
    assert _refused(a)


def test_score_refuses_combinations_that_do_not_fit():
    a, keep = _args()
    a.mean = keep["zhat"].ctypes.data                       # x and mean
    assert _refused(a)
    a, keep = _args()
    a.S, a.S_stride = keep["P"].ctypes.data, 4              # P and S
    assert _refused(a)
    a, keep = _args()
    a.H = None                                              # identity H with n != m
    assert _refused(a)
    a, keep = _args()
    a.P = None                                              # R without P, and no covariance for the scores
    assert _refused(a)
    a.R = None
    assert _refused(a)
    a.log_likelihood, a.zhat = None, keep["zhat"].ctypes.data
    a.status = keep["ll"].ctypes.data                       # status needs a covariance
    assert _refused(a)
    a, keep = _args()
    a.x, a.P, a.R = None, None, None
    a.mean, a.S, a.S_stride = keep["zhat"].ctypes.data, keep["P"].ctypes.data, 4
    assert _refused(a)                                      # H with neither x nor P
    a.H = None
    a.S_stride = 3
    assert _refused(a)
    a.S_stride = 0
    assert _lib.load().bke_score_measurements(ctypes.byref(a), None) != _lib.BKE_ERR_BAD_ARG
    a.log_likelihood = None                                 # nothing requested
    assert _refused(a)
    a, keep = _args()
    a.n_tracks, a.n_candidates = 2 ** 40, 2 ** 30           # N * K * m overflows int64
    assert _refused(a)
    assert _lib.load().bke_score_measurements(None, None) == _lib.BKE_ERR_BAD_ARG


def test_zhat_alone_needs_no_covariance_or_z():
    a, keep = _args()
    a.P = a.R = a.z = a.log_likelihood = None
    a.zhat = keep["zhat"].ctypes.data
    rc = _lib.load().bke_score_measurements(ctypes.byref(a), None)
    assert rc != _lib.BKE_ERR_BAD_ARG


def test_score_needs_a_device():
    lib = _lib.load()
    if lib.bke_device_count() > 0:
        pytest.skip("a device is present")
    a, keep = _args()
    assert lib.bke_score_measurements(ctypes.byref(a), None) == _lib.BKE_ERR_CUDA


# ---------------------------------------------------------------------------------------------- the mirrors
def test_single_calls_check_shapes_before_the_device():
    from filterpy_b200 import stats
    with pytest.raises(ValueError, match="length of input vectors"):
        stats.mahalanobis([1], [1.4, 1.2], [[1., 2.], [2., 4.001]])
    with pytest.raises(ValueError, match="1-D"):
        stats.mahalanobis(np.ones((2, 2)), np.ones((2, 2)), np.eye(2))
    with pytest.raises(ValueError):
        stats.mahalanobis([1., 2.], [0., 0.], np.eye(3))
    with pytest.raises(ValueError):
        stats.log_likelihood([1., 2., 3.], np.zeros(4), np.eye(4), np.ones((2, 4)), np.eye(2))
    with pytest.raises(ValueError):
        stats.logpdf([1., 2.], [0., 0., 0.], np.eye(3))
    with pytest.raises(ValueError):
        stats.NEES(np.ones((3, 2)), np.zeros((3, 2)), np.stack([np.eye(3)] * 3))
    assert stats.NEES([], [], []) == []
