"""The UKF measurement-score oracle (tests/ukf_score_oracle.py) against the reference's own numbers
(tests/golden/ukf_score_*.npz: log_likelihood and mahalanobis of a deepcopy updated with each candidate), and
the NVRTC programs of every kind of UKF handle carry the score kernel."""
import ctypes
import os

import numpy as np
import pytest

import ukf_score_oracle as uso
from oracle import ukf as oukf

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _hx_user(g):
    def hx(s, f):
        dx, dy = s[0] - g["sx"][f], s[2] - g["sy"][f]
        return np.array([np.sqrt(dx * dx + dy * dy), np.arctan2(dy, dx)])
    return hx


# name -> (point set, oracle keyword arguments from the golden)
CASES = {
    "cv_rae": (("merwe", .5, 2., 0.), lambda g: dict(hx_model=oukf.HX_RANGE_AZ_EL)),
    "julier": (("merwe", 1., 0., 1.5), lambda g: dict(hx_model=oukf.HX_RANGE_AZ_EL)),
    "hooks_rb": (("merwe", .8, 2., 0.), lambda g: dict(hx_model=oukf.HX_RANGE_BEARING, angle_z=(1,), z_mean=True)),
    "simplex_rb": (("simplex",), lambda g: dict(hx_model=oukf.HX_RANGE_BEARING)),
    "user_rb": (("merwe", .5, 2., 0.), lambda g: dict(hx=_hx_user(g))),
    "lin": (("merwe", .5, 2., 0.), lambda g: dict(hx_model=oukf.HX_LINEAR, H=np.array([[1., 0, 0, 0], [0, 0, 1, 0]]))),
}


def load(name):
    return np.load(os.path.join(GOLDEN, "ukf_score_%s.npz" % name))


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_reference(name):
    g = load(name)
    pts, kw = CASES[name]
    o = uso.ukf_score_bank(g["x_prior"], g["P_prior"], g["z"], g["R"], pts, **kw(g))
    assert (o["status"] == 0).all()
    np.testing.assert_allclose(o["log_likelihood"], g["ref_ll"], rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(o["mahalanobis"], g["ref_maha"], rtol=1e-9, atol=1e-9)


def test_hooks_change_the_scores():
    """Without the angle hooks the candidates across +-pi score differently by far more than any tolerance."""
    g = load("hooks_rb")
    pts, kw = CASES["hooks_rb"]
    o = uso.ukf_score_bank(g["x_prior"], g["P_prior"], g["z"], g["R"], pts, hx_model=oukf.HX_RANGE_BEARING)
    assert np.max(np.abs(o["log_likelihood"] - g["ref_ll"])) > 100


def test_oracle_status_rules():
    """A missing candidate scores 0 / log(DBL_MIN) whatever the track; a P without a Cholesky factor scores NaN
    with status 2."""
    g = load("lin")
    P = g["P_prior"].copy()
    P[1] = -np.eye(4)
    valid = np.ones(g["z"].shape[:2], bool)
    valid[:, 2] = False
    o = uso.ukf_score_bank(g["x_prior"], P, g["z"], g["R"], ("merwe", .5, 2., 0.), H=np.array([[1., 0, 0, 0], [0, 0, 1, 0]]),
                           valid=valid)
    assert o["status"].tolist() == [0, 2, 0, 0, 0, 0]
    assert np.isnan(o["log_likelihood"][1, valid[1]]).all()
    assert (o["log_likelihood"][:, 2] == uso.so.LOG_DBL_MIN).all() and (o["mahalanobis"][:, 2] == 0).all()
    assert np.isfinite(o["log_likelihood"][[0, 2, 3, 4, 5]]).all()


# ------------------------------------------------------------------------------------------------- NVRTC
USER_HX = """
__device__ void hx(const real *x, real *z, const real *args)
{
    const real dx = x[0] - args[0], dy = x[2] - args[1];
    z[0] = sqrt(dx * dx + dy * dy); z[1] = atan2(dy, dx);
}
"""
USER_FX = """
__device__ void fx(const real *x, real *o, real dt, const real *args) { for (int i = 0; i < 4; i++) o[i] = x[i]; }
"""


@pytest.mark.parametrize("kind", ["user_hx", "user_fx", "hooks", "simplex", "simplex_hooks"])
@pytest.mark.parametrize("dtype", [0, 1], ids=["f32", "f64"])
def test_every_ukf_handle_compiles_the_score_kernel(kind, dtype):
    """The score program of each kind of UKF handle (compiled on its first bke_ukf_score_model call) compiles for
    sm_90a and its one name expression, the score kernel, lowers (the call fails otherwise)."""
    from filterpy_b200 import _lib
    from filterpy_b200.common import workloads as wl
    lib = _lib.load()
    inc = _lib.kernel_include_dirs().encode()
    fx, hx, spx = _lib.BKE_FX_CONST_VEL, _lib.BKE_HX_RANGE_BEARING, _lib.BKE_UKF_SIMPLEX
    hooks = _lib.BKE_HOOK_RESIDUAL_Z | _lib.BKE_HOOK_Z_MEAN
    args = {"user_hx": (fx, _lib.BKE_HX_USER, 0, 0, USER_HX), "user_fx": (_lib.BKE_FX_USER, _lib.BKE_HX_LINEAR, 0, 0, USER_FX),
            "hooks": (fx, hx, hooks, 0, wl.RB_HOOKS_SOURCE), "simplex": (fx, _lib.BKE_HX_USER, 0, spx, USER_HX),
            "simplex_hooks": (fx, hx, hooks, spx, wl.RB_HOOKS_SOURCE)}[kind]
    n = lib.bke_debug_ukf_score_model_cubin_bytes(4, 2, dtype, args[0], args[1], args[2], args[3], args[4].encode(), inc)
    assert n > 0, lib.bke_last_error()
