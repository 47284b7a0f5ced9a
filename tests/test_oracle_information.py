"""CPU: the fp64 InformationFilter oracle against the reference's golden vectors, the argument checks of
bke_if_step / bke_inverse (made before any device is needed) and the mirror's host-side checks."""
import ctypes

import numpy as np
import pytest

from filterpy_b200 import _lib

import information_oracle as io

GOLDEN = ["if_test_1d", "if_test_1d_0P", "if_test_against_kf", "if_cv_4_2", "if_ll_2_2", "if_ll_4_4", "if_ll_2_1",
          "if_bank_6_3", "if_bank_9_3", "if_ctrl_3_2", "if_noinfo_2_2", "if_noinfo_4_2", "if_stale_F_inv",
          "if_raise_F", "if_raise_AIQ", "if_raise_S", "if_raise_ll_4_2"]

# how many steps of a file the singularity rule covers: in if_test_1d_0P (P_inv = 1e-21 I) A is singular at step 8
# by the rounding of one elimination order only, which is not the rule's; if_raise_ll_4_2 stops at its ValueError
STEPS = {"if_test_1d_0P": 8, "if_raise_ll_4_2": 1}
KEYS = ("x", "P_inv", "ni", "ll", "y", "K", "S", "x_prior", "P_inv_prior")


def ll_mode(g):
    n, m = g["x"].shape[1], g["H"].shape[1]
    if not bool(g["compute_ll"]):
        return io.LL_NONE
    return io.LL_FULL if m == n else (io.LL_BROADCAST if m == 1 else io.LL_NONE)


def _close(a, b, tol):
    """relative to max|b|, over b's finite entries: scipy's logpdf is -inf where its eigenvalue cutoff finds S
    singular (allow_singular), which no inverse here does (if_test_1d_0P's first S, 1e-21 against 0.2)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    fin = np.isfinite(b)
    scale = max(np.abs(b[fin]).max(initial=0), 1e-300)
    assert np.abs(a[fin] - b[fin]).max(initial=0) / scale < tol


@pytest.mark.parametrize("name", GOLDEN)
def test_oracle_matches_golden(golden, name):
    g = golden(name)
    T = STEPS.get(name, g["zs"].shape[0])
    o = io.run_bank(g, ll_mode(g), steps=T)
    for k in KEYS:
        _close(o[k], g["out_" + k][:T], 1e-12)
    raised = g["raise_step"] >= 0
    lin = raised & (g["raise_type"] == "LinAlgError")
    assert np.array_equal(o["status"][-1] != 0, lin)


def test_golden_cases_cover_both_branches_and_every_raise(golden):
    ni = np.concatenate([golden(n)["out_ni"].reshape(-1) for n in GOLDEN])
    assert ni.min() == 0 and ni.max() == 1
    kinds = {(str(golden(n)["raise_op"][0]), str(golden(n)["raise_type"][0])) for n in GOLDEN}
    assert {("p", "LinAlgError"), ("u", "LinAlgError"), ("u", "ValueError")} <= kinds
    g = golden("if_noinfo_2_2")
    assert g["out_ni"][0].all() and not g["out_ni"][1:].any()      # one step in the branch, informed after
    g = golden("if_noinfo_4_2")
    assert g["out_ni"].all()                                        # the zero block keeps A singular
    g = golden("if_stale_F_inv")
    assert not np.allclose(g["F_inv"], np.linalg.inv(g["F"]))        # the steps run on the stale inverse
    assert np.allclose(g["F_inv"], np.linalg.inv(g["F_set"]))


def test_singularity_rule():
    assert io.singular(np.zeros((3, 3)))
    assert io.singular(np.diag([1., 0., 2.]))
    assert io.singular(np.array([[.2, -.2], [-.2, .2]]))
    assert not io.singular(np.array([[0., 1.], [1., 0.]]))          # a pivot is searched for, not taken in place
    A = np.random.default_rng(0).standard_normal((5, 5))
    assert not io.singular(A)
    assert np.allclose(io.inv(A), np.linalg.inv(A))


def test_logpdf_broadcast_matches_scipy():
    from scipy.stats import multivariate_normal
    S = np.array([[2., .3], [.3, 1.]])
    assert np.isclose(io.logpdf_broadcast([.5, -1.], S), multivariate_normal.logpdf([.5, -1.], None, S))
    assert np.isclose(io.logpdf_broadcast([.5], S), multivariate_normal.logpdf([.5, .5], None, S))


# ---------------------------------------------------------------------------------------------- the C-ABI
def _args(n=4, m=2, N=8):
    keep = {k: np.zeros(N * max(n, m) ** 2 + 16) for k in ("x", "P", "F", "Fi", "Q", "H", "Ri", "z")}
    keep["ni"] = np.zeros(N, np.uint8)
    a = _lib.IfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dtype = N, n, m, _lib.BKE_F64
    a.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
    a.x = a.x_out = keep["x"].ctypes.data
    a.P_inv = a.P_inv_out = keep["P"].ctypes.data
    a.no_information = keep["ni"].ctypes.data
    a.F, a.F_inv, a.Q = keep["F"].ctypes.data, keep["Fi"].ctypes.data, keep["Q"].ctypes.data
    a.H, a.R_inv, a.z = keep["H"].ctypes.data, keep["Ri"].ctypes.data, keep["z"].ctypes.data
    return a, keep


def _refused(a):
    lib = _lib.load()
    return lib.bke_if_step(ctypes.byref(a), None) == _lib.BKE_ERR_BAD_ARG


@pytest.mark.parametrize("field,value", [
    ("dim_x", 0), ("dim_z", 0), ("dim_u", -1), ("n_filters", -1), ("dtype", 7), ("flags", 0),
    ("flags", _lib.BKE_DO_UPDATE | _lib.BKE_UPDATE_FIRST), ("no_information", None), ("x", None), ("P_inv_out", None),
    ("F_inv", None), ("R_inv", None), ("z", None), ("F_stride", 3), ("F_inv_stride", 15), ("Q_stride", 1),
    ("H_stride", 9), ("R_inv_stride", 2), ("ll_mode", 3),
])
def test_if_step_refuses_bad_arguments(field, value):
    a, keep = _args()
    setattr(a, field, value)
    assert _refused(a)


def test_if_step_refuses_a_log_likelihood_mode_that_does_not_fit():
    ll = np.zeros(8)
    a, keep = _args(4, 2)
    a.ll_mode, a.log_likelihood = _lib.BKE_IF_LL_FULL, ll.ctypes.data        # m != n
    assert _refused(a)
    a.ll_mode = _lib.BKE_IF_LL_BROADCAST                                     # m != 1
    assert _refused(a)
    a, keep = _args(2, 2)
    a.ll_mode = _lib.BKE_IF_LL_FULL                                          # no log_likelihood array
    assert _refused(a)
    a, keep = _args(2, 1)
    a.ll_mode, a.log_likelihood = _lib.BKE_IF_LL_FULL, ll.ctypes.data
    assert _refused(a)


def test_if_step_refuses_a_half_control_input():
    a, keep = _args()
    B = np.zeros(64)
    a.B, a.dim_u = B.ctypes.data, 1
    assert _refused(a)
    assert _lib.load().bke_if_step(None, None) == _lib.BKE_ERR_BAD_ARG


def test_inverse_refuses_bad_arguments():
    lib = _lib.load()
    A = np.zeros(64)
    for args in [(-1, 2, _lib.BKE_F64, A.ctypes.data, 0), (4, 0, _lib.BKE_F64, A.ctypes.data, 0),
                 (4, 2, 5, A.ctypes.data, 0), (4, 2, _lib.BKE_F64, A.ctypes.data, 3), (4, 2, _lib.BKE_F64, None, 4)]:
        assert lib.bke_inverse(*args, A.ctypes.data, None, None) == _lib.BKE_ERR_BAD_ARG


def test_compute_calls_need_a_device():
    """No CPU fallback: valid arguments on a machine without a device return BKE_ERR_CUDA."""
    lib = _lib.load()
    if lib.bke_device_count() > 0:
        pytest.skip("a device is present")
    a, keep = _args()
    assert lib.bke_if_step(ctypes.byref(a), None) == _lib.BKE_ERR_CUDA
    A = np.eye(2).reshape(-1)
    assert lib.bke_inverse(1, 2, _lib.BKE_F64, A.ctypes.data, 0, A.ctypes.data, None, None) == _lib.BKE_ERR_CUDA


def test_mirror_checks_dimensions_before_the_device():
    from filterpy_b200.kalman import InformationFilter
    with pytest.raises(ValueError, match="dim_x"):
        InformationFilter(0, 1)
    with pytest.raises(ValueError, match="dim_z"):
        InformationFilter(2, 0)
    with pytest.raises(ValueError, match="dim_u"):
        InformationFilter(2, 1, dim_u=-1)
