"""Argument checks of bke_ukf_step, bke_ckf_step and bke_enkf_step, one bad field per case, and of the *_step_model
entry points for a missing handle.  Needs no GPU: every check runs before the device is looked up, so a call
that passes them returns BKE_ERR_CUDA on a machine without one.  The banks are empty (n_filters = 0), so on a
machine with a device a call that passes them returns BKE_OK without launching and the fake pointers are
never read."""
import ctypes

import pytest

from filterpy_b200 import _lib as L

FAKE = 1 << 20
COMMON = ("x", "P", "x_out", "P_out", "Q", "R", "z", "F", "H")
STEP = {"ukf": ("bke_ukf_step", L.UkfArgs), "ckf": ("bke_ckf_step", L.CkfArgs), "enkf": ("bke_enkf_step", L.EnkfArgs)}


def _args(family, **over):
    a = STEP[family][1]()
    a.n_filters, a.dim_x, a.dim_z, a.dtype = 0, 4, 2, L.BKE_F32
    a.flags = L.BKE_DO_PREDICT | L.BKE_DO_UPDATE
    a.fx_model, a.hx_model = L.BKE_FX_LINEAR, L.BKE_HX_LINEAR
    a.dt = 0.1
    for k in COMMON:
        setattr(a, k, FAKE)
    if family == "ukf":
        a.alpha, a.beta, a.kappa = 0.5, 2.0, 0.0
    if family == "ckf":
        a.sigmas_f = FAKE
    if family == "enkf":
        a.n_members, a.sigmas, a.sigmas_out = 16, FAKE, FAKE
    for k, v in over.items():
        setattr(a, k, v)
    return a


UPDATE_ONLY = dict(flags=L.BKE_DO_UPDATE)
# (fields changed from the valid args, whether each family refuses them)
CASES = [({}, dict(ukf=False, ckf=False, enkf=False))]
CASES += [({k: None}, dict(ukf=True, ckf=True, enkf=True)) for k in COMMON]
CASES += [
    (dict(flags=0), dict(ukf=True, ckf=True, enkf=True)),
    (dict(n_filters=-1), dict(ukf=True, ckf=True, enkf=True)),
    (dict(dim_x=0), dict(ukf=True, ckf=True, enkf=True)),
    (dict(dim_z=0), dict(ukf=True, ckf=True, enkf=True)),
    (dict(dtype=7), dict(ukf=True, ckf=True, enkf=True)),
    (dict(fx_model=L.BKE_FX_CONST_VEL, dim_x=3, dim_z=1), dict(ukf=True, ckf=True, enkf=True)),
    (dict(fx_model=L.BKE_FX_CONST_VEL, dim_x=4, F=None), dict(ukf=False, ckf=False, enkf=False)),
    (dict(hx_model=L.BKE_HX_RANGE_AZ_EL), dict(ukf=True, ckf=True, enkf=True)),
    (dict(hx_model=L.BKE_HX_RANGE_BEARING, dim_x=6, dim_z=3), dict(ukf=True, ckf=True, enkf=True)),
    (dict(hx_model=L.BKE_HX_RANGE_BEARING, H=None), dict(ukf=False, ckf=False, enkf=False)),
    (dict(fx_model=-1), dict(ukf=True, ckf=True, enkf=True)),
    (dict(fx_model=2), dict(ukf=True, ckf=True, enkf=True)),
    (dict(hx_model=3), dict(ukf=True, ckf=True, enkf=True)),
    (dict(fx_model=L.BKE_FX_USER), dict(ukf=True, ckf=True, enkf=True)),
    (dict(hx_model=L.BKE_HX_USER), dict(ukf=True, ckf=True, enkf=True)),
    (dict(flags=L.BKE_DO_PREDICT, R=None, z=None, H=None), dict(ukf=False, ckf=False, enkf=False)),
    (dict(flags=L.BKE_DO_UPDATE, Q=None, F=None), dict(ukf=False, ckf=False, enkf=False)),
    # only the EnKF rejects negative strides and flag bits other than predict / update
    (dict(Q_stride=-1), dict(ukf=False, ckf=False, enkf=True)),
    (dict(R_stride=-1), dict(ukf=False, ckf=False, enkf=True)),
    (dict(F_stride=-1), dict(ukf=False, ckf=False, enkf=True)),
    (dict(H_stride=-1), dict(ukf=False, ckf=False, enkf=True)),
    (dict(flags=L.BKE_DO_PREDICT | L.BKE_DO_UPDATE | 8), dict(ukf=False, ckf=False, enkf=True)),
    # only the CKF needs sigmas_f for an update-only step
    (dict(UPDATE_ONLY, sigmas_f=None), dict(ukf=False, ckf=True, enkf=False)),
    (dict(UPDATE_ONLY, sigmas_f=FAKE), dict(ukf=False, ckf=False, enkf=False)),
    # the UKF's Merwe points need alpha^2 (n + kappa) != 0; the simplex set has no alpha
    (dict(alpha=0.0), dict(ukf=True, ckf=False, enkf=False)),
    (dict(alpha=0.0, flags=L.BKE_DO_PREDICT | L.BKE_DO_UPDATE | L.BKE_UKF_SIMPLEX), dict(ukf=False, ckf=False, enkf=False)),
    # the EnKF: dim_x <= 16, 2 <= n_members <= 2^24, both ensemble arrays
    (dict(dim_x=17, dim_z=1), dict(ukf=False, ckf=False, enkf=True)),
    (dict(n_members=1), dict(ukf=False, ckf=False, enkf=True)),
    (dict(n_members=(1 << 24) + 1), dict(ukf=False, ckf=False, enkf=True)),
    (dict(n_members=1 << 24), dict(ukf=False, ckf=False, enkf=False)),
    (dict(sigmas=None), dict(ukf=False, ckf=False, enkf=True)),
    (dict(sigmas_out=None), dict(ukf=False, ckf=False, enkf=True)),
]


def _id(over):
    return "-".join("%s=%s" % kv for kv in over.items()) or "valid"


@pytest.mark.parametrize("family", ["ukf", "ckf", "enkf"])
@pytest.mark.parametrize("over,bad", CASES, ids=[_id(o) for o, _ in CASES])
def test_step_validates_arguments(family, over, bad):
    lib = L.load()
    fields = {f for f, _ in STEP[family][1]._fields_}
    if not set(over) <= fields:
        pytest.skip("%s args have no field %s" % (family, sorted(set(over) - fields)))
    rc = getattr(lib, STEP[family][0])(ctypes.byref(_args(family, **over)), None)
    if bad[family]:
        assert rc == L.BKE_ERR_BAD_ARG, lib.bke_last_error()
    else:
        assert rc == (L.BKE_OK if lib.bke_device_count() > 0 else L.BKE_ERR_CUDA), lib.bke_last_error()


@pytest.mark.parametrize("family", ["ukf", "ckf", "enkf"])
def test_step_model_refuses_null_handle_and_args(family):
    lib = L.load()
    fn = getattr(lib, STEP[family][0] + "_model")
    assert fn(ctypes.byref(_args(family)), None, None, 0, None, 0, None) == L.BKE_ERR_BAD_ARG
    assert b"NULL" in lib.bke_last_error()
    assert fn(None, None, None, 0, None, 0, None) == L.BKE_ERR_BAD_ARG
    assert getattr(lib, STEP[family][0])(None, None) == L.BKE_ERR_BAD_ARG
