"""CPU: the fp64 oracle of the polynomial trackers against the reference's golden vectors, bit for bit; the argument
checks of bke_poly_filter (made before any device is needed); the gain helpers against the reference's values;
and that the fp64 kernels carry no contracted multiply-add."""
import ctypes
import glob
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from filterpy_b200 import _lib
from filterpy_b200 import gh

import poly_oracle as po

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(HERE, "golden", "poly_*.npz"))
               if not p.endswith(("poly_helpers.npz", "poly_lsq_big_data.npz")))
OUTPUTS = ("upd_state", "upd_y", "upd_xp", "upd_dxp", "upd_ddxp", "upd_z", "upd_K", "bat_res", "bat_pred")


def test_every_family_and_order_has_golden_cases():
    fams = {(n.split("_")[1], ) for n in CASES}
    assert {("gh",), ("ghk",), ("gho",), ("lsq",), ("fm",)} <= fams
    assert len(CASES) >= 25


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_golden_bit_for_bit(golden, name):
    c = golden(name)
    o = po.run(c)
    for k in OUTPUTS:
        if k in c:
            assert np.array_equal(o[k], c[k]), k


def test_oracle_lsq_big_data(golden):
    """the reference's test_big_data: its first epochs from a fresh filter, and its last ones from the reference's
    counter and state at epoch 10^6 - H, where n(n+1)(n+2) is past 2**53 and the gains' conversions round"""
    c = golden("poly_lsq_big_data")
    H = c["head_z"].size
    for order in (0, 1, 2):
        for part, X, n in (("head", np.zeros((1, order + 1)), np.zeros(1, np.int64)),
                           ("tail", c["tail_x0_%d" % order][None].copy(), np.array([c["tail_n0_%d" % order]], np.int64))):
            xs, Ks = [], []
            for t in range(H):
                X, n, K = po.lsq_update(order, X, n, c[part + "_z"][t:t + 1], 1., 1., .5)
                xs.append(X[0]); Ks.append(K[0])
            assert np.array_equal(np.array(xs), c["%s_x_%d" % (part, order)])
            assert np.array_equal(np.array(Ks), c["%s_K_%d" % (part, order)])
        assert int(c["tail_n0_%d" % order]) + H == int(c["n_steps"])
    assert int(c["tail_n0_2"]) ** 3 > 2**53


def test_quirk_cases_show_their_quirk(golden):
    q = golden("poly_quirk_gh_h_dt")                   # batch_filter's h / dt rounds apart from update's h * y / dt
    assert not np.array_equal(q["bat_res"][1:], q["upd_state"][1:])
    assert np.allclose(q["bat_res"][1:], q["upd_state"][1:], rtol=1e-9, atol=1e-9)
    k = golden("poly_quirk_ghk_batch")                 # GHKFilter.batch_filter is the g-h recursion: no k, no ddx
    assert k["x0"][:, 2].all() and k["k"].all()
    x, dx = k["x0"][:, 0], k["x0"][:, 1]
    h_dt = po.consts(k)["h_dt"]
    for t in range(k["zs"].shape[0]):
        x, dx, _ = po.gh_batch_step(x, dx, k["zs"][t], k["g"], h_dt, k["dt"])
    assert np.array_equal(np.stack([x, dx], 1), k["bat_res"][-1])
    for order in (0, 2):                               # z is stored for order 1 only
        assert not golden("poly_quirk_gho_z_order%d" % order)["upd_z"].any()
    z1 = golden("poly_quirk_gho_z_order1")
    assert np.array_equal(z1["upd_z"], z1["zs"][z1["snap"][1:] - 1])


# ---------------------------------------------------------------------------------------------- gain helpers
def test_gain_helpers_equal_the_reference(golden):
    c = golden("poly_helpers")
    assert np.array_equal(np.array([gh.optimal_noise_smoothing(float(v)) for v in c["gs"]]), c["ons"])
    assert np.array_equal(np.array([gh.least_squares_parameters(int(v)) for v in c["n"]]), c["lsp"])
    assert np.array_equal(np.array([gh.critical_damping_parameters(float(v)) for v in c["theta"]]), c["cd2"])
    assert np.array_equal(np.array([gh.critical_damping_parameters(float(v), order=3) for v in c["theta"]]), c["cd3"])
    assert np.array_equal(np.array([gh.benedict_bornder_constants(float(v)) for v in c["gs"]]), c["bb"])
    assert np.array_equal(np.array([gh.benedict_bornder_constants(float(v), critical=True) for v in c["gs"]]), c["bbc"])


def test_gain_helper_exceptions():
    with pytest.raises(ValueError, match='theta must be between 0 and 1'):
        gh.critical_damping_parameters(1.5)
    with pytest.raises(ValueError, match='theta must be between 0 and 1'):
        gh.critical_damping_parameters(-.1)
    with pytest.raises(ValueError, match='bad order specified: 4'):
        gh.critical_damping_parameters(.5, order=4)


# ---------------------------------------------------------------------------------------------- the C-ABI
def _zeros(n, dtype=np.float64):
    """np.zeros(n), page-locked where there is a device: a call that passes the checks then runs its kernel, which
    reads and writes these buffers through their host addresses."""
    import torch
    z = np.zeros(n, dtype)
    return torch.from_numpy(z).pin_memory().numpy() if torch.cuda.is_available() else z


def _args(family=_lib.BKE_POLY_GH, order=1, N=8, T=3, mode=_lib.BKE_POLY_UPDATE):
    keep = {k: _zeros(N * 3 * (T + 1) + 16) for k in ("x", "dx", "ddx", "p", "z", "o")}
    keep["n"] = _zeros(N, np.int64)
    a = _lib.PolyArgs()
    a.n_filters, a.n_steps, a.family, a.order, a.dtype, a.mode = N, T, family, order, _lib.BKE_F64, mode
    a.x, a.dx, a.ddx, a.z = (keep[k].ctypes.data for k in ("x", "dx", "ddx", "z"))
    for name in ("g", "h", "k", "dt", "dt2", "hdt2"):
        setattr(a, name, keep["p"].ctypes.data)
    a.n = keep["n"].ctypes.data
    return a, keep


def _rc(a):
    return _lib.load().bke_poly_filter(ctypes.byref(a), None)


def _refused(a):
    return _rc(a) == _lib.BKE_ERR_BAD_ARG


@pytest.mark.parametrize("field,value", [
    ("n_filters", -1), ("n_steps", 0), ("dtype", 3), ("family", 5), ("family", -1), ("mode", 2), ("x", None),
    ("dx", None), ("z", None), ("g", None), ("h", None), ("dt", None), ("g_stride", 2), ("h_stride", -1),
    ("dt_stride", 8), ("dt2_stride", 3),
])
def test_poly_refuses_bad_arguments(field, value):
    a, keep = _args()
    setattr(a, field, value)
    assert _refused(a)


@pytest.mark.parametrize("family", [_lib.BKE_POLY_GH_ORDER, _lib.BKE_POLY_LSQ, _lib.BKE_POLY_FADING])
@pytest.mark.parametrize("order", [-1, 3])
def test_poly_refuses_a_bad_order(family, order):
    a, keep = _args(family, order)
    assert _refused(a)


@pytest.mark.parametrize("family,order,mode,field", [
    (_lib.BKE_POLY_GH, 1, _lib.BKE_POLY_UPDATE, "predictions"),          # batch only
    (_lib.BKE_POLY_GH, 1, _lib.BKE_POLY_BATCH, "y"),
    (_lib.BKE_POLY_GH, 1, _lib.BKE_POLY_BATCH, "x_prediction"),
    (_lib.BKE_POLY_GH, 1, _lib.BKE_POLY_UPDATE, "ddx_prediction"),       # GHK only
    (_lib.BKE_POLY_GH, 1, _lib.BKE_POLY_UPDATE, "K"),                    # LSQ only
    (_lib.BKE_POLY_GH_ORDER, 1, _lib.BKE_POLY_UPDATE, "x_prediction"),
    (_lib.BKE_POLY_GH_ORDER, 1, _lib.BKE_POLY_BATCH, "predictions"),
    (_lib.BKE_POLY_LSQ, 2, _lib.BKE_POLY_UPDATE, "y"),                   # least_squares.py never stores y
    (_lib.BKE_POLY_LSQ, 2, _lib.BKE_POLY_BATCH, "K"),
    (_lib.BKE_POLY_FADING, 2, _lib.BKE_POLY_UPDATE, "y"),
    (_lib.BKE_POLY_FADING, 2, _lib.BKE_POLY_UPDATE, "dx_prediction"),
])
def test_poly_refuses_an_output_the_family_does_not_have(family, order, mode, field):
    a, keep = _args(family, order, mode=mode)
    setattr(a, field, keep["o"].ctypes.data)
    assert _refused(a)


def test_poly_refuses_what_an_instance_reads_when_null():
    a, keep = _args(_lib.BKE_POLY_GHK, 2)
    a.ddx = None                                                          # GHK update reads ddx ...
    assert _refused(a)
    a.mode = _lib.BKE_POLY_BATCH                                          # ... its batch_filter does not
    assert not _refused(a)
    a, keep = _args(_lib.BKE_POLY_LSQ, 2)
    a.hdt2 = None
    assert _refused(a)
    a, keep = _args(_lib.BKE_POLY_LSQ, 1)
    a.n = None
    assert _refused(a)


@pytest.mark.parametrize("order,limit", [(2, 2097150), (1, 3037000498)])
def test_poly_refuses_an_lsq_counter_that_could_overflow(order, limit):
    """order 2 forms n(n+1)(n+2), order 1 n(n+1): n_max + n_steps may not make them overflow int64"""
    a, keep = _args(_lib.BKE_POLY_LSQ, order, T=1)
    top = limit + 1
    while True:                                      # the largest counter whose product fits
        p = top * (top + 1) * (top + 2 if order == 2 else 1)
        if p <= 2**63 - 1:
            break
        top -= 1
    a.n_max = top - 1                                # reaches top: fits
    assert _rc(a) != _lib.BKE_ERR_BAD_ARG
    a.n_max = top                                    # reaches top + 1: overflows
    assert _refused(a)
    a.n_max = -1
    assert _refused(a)
    a.n_max, a.n_steps = 0, 2**62
    assert _refused(a)


def test_poly_needs_a_device():
    """No CPU fallback: valid arguments on a machine without a device return BKE_ERR_CUDA."""
    lib = _lib.load()
    if lib.bke_device_count() > 0:
        pytest.skip("a device is present")
    for fam, order in [(_lib.BKE_POLY_GH, 1), (_lib.BKE_POLY_GHK, 2), (_lib.BKE_POLY_GH_ORDER, 0),
                       (_lib.BKE_POLY_LSQ, 2), (_lib.BKE_POLY_FADING, 1)]:
        a, keep = _args(fam, order)
        assert _rc(a) == _lib.BKE_ERR_CUDA


def test_mirrors_check_their_order_before_the_device():
    from filterpy_b200.leastsq import LeastSquaresFilter
    from filterpy_b200.memory import FadingMemoryFilter
    for make in (lambda o: gh.GHFilterOrder(0., 1., o, .5), lambda o: LeastSquaresFilter(1., o),
                 lambda o: FadingMemoryFilter(0., 1., o, .5)):
        for o in (-1, 3):
            with pytest.raises(ValueError, match='order must be between 0 and 2'):
                make(o)


def _kernel_sass(nvcc, src, tmp):
    """{(family, order, batch, dtype): SASS text} of every poly_kernel instance"""
    cubin = os.path.join(str(tmp), "poly.cubin")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-cubin", src, "-o", cubin],
                   capture_output=True, text=True, check=True)
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    out = {}
    for part in sass.split("Function : ")[1:]:
        m = re.search(r"poly_kernelILi(\d)ELi(\d)ELb(\d)E([df])E", part.splitlines()[0])
        assert m, part.splitlines()[0]
        out[(int(m.group(1)), int(m.group(2)), bool(int(m.group(3))), m.group(4))] = part
    return out


def test_fp64_kernels_have_no_contracted_fma(tmp_path):
    """poly.cu's arithmetic is explicitly rounded: its PTX holds no fma or mad, the fp64 instances without a division
    (GH batch, GH_ORDER 0, every fading order) have no DFMA in SASS, and in the others every DFMA comes with the
    MUFU.RCP64H of ptxas's IEEE division / reciprocal sequence"""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc is not available")
    src = os.path.join(os.path.dirname(HERE), "filterpy_b200", "csrc", "poly.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ptx", src, "-o", "-"],
                         capture_output=True, text=True, check=True).stdout
    assert "fma." not in out and "mad." not in out
    assert "div.rn.f64" in out
    sass = _kernel_sass(nvcc, src, tmp_path)
    assert len(sass) == 24                                   # 12 instances per dtype
    fp64 = {k: v for k, v in sass.items() if k[3] == "d"}
    no_division = {(_lib.BKE_POLY_GH, 1, True), (_lib.BKE_POLY_GH_ORDER, 0, False)} | \
        {(_lib.BKE_POLY_FADING, o, False) for o in (0, 1, 2)}
    for (fam, order, batch, _), text in fp64.items():
        if (fam, order, batch) in no_division:
            assert "DFMA" not in text, (fam, order, batch)
        else:
            assert "MUFU.RCP64H" in text, (fam, order, batch)
    assert len(no_division) == 5 and all((f, o, b, "d") in fp64 for f, o, b in no_division)
