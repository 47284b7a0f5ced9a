"""IMMEstimator.batch_filter without a GPU: the NumPy restatement (tests/imm_oracle.py) against the reference's
IMMEstimator loop (tests/golden/imm_batch_*.npz, mm.npz, mm_missing.npz), the argument checks of
bke_imm_batch_filter and the register budget of every fused instance."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from filterpy_b200 import _lib
from imm_oracle import golden_inputs, imm_batch

CASES = ["m2_4_2", "m3_4_2", "m4_4_2", "m3_6_3", "m2_2_1", "m3_3_1", "m2_5_2"]
MM_MISSING = ["a", "b", "c", "d", "e", "f", "g", "h", "man"]


def close(a, b, tol=1e-12):
    a, b = np.asarray(a), np.asarray(b)
    scale = max(np.abs(b).max(), 1e-300)
    assert np.abs(a - b).max() <= tol * scale, np.abs(a - b).max() / scale


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference_imm_loop(golden, name):
    g = golden("imm_batch_" + name)
    o = imm_batch(*golden_inputs(g))
    for k in ("x", "P", "xp", "Pp", "mu", "cbar", "omega", "fx", "fP"):
        close(o[k], g[k])
    np.testing.assert_allclose(o["lik"], g["lik"], rtol=1e-10, atol=0)


def _mm_case(g, prefix, nm, per_epoch_valid):
    """the shared-model goldens of mm.npz / mm_missing.npz as imm_batch inputs (model j starts at x0 + j)."""
    x0, P0, Qs = g[prefix + "x0"], g[prefix + "P0"], g[prefix + "Qs"][:nm]
    NT, n = x0.shape
    F = np.broadcast_to(g[prefix + "F"], (NT, nm, n, n))
    Q = np.broadcast_to(Qs[None], (NT, nm, n, n))
    xs = np.stack([x0 + j for j in range(nm)], axis=1)
    Ps = np.stack([P0] * nm, axis=1)
    zs = g[prefix + "zs"]
    valid = per_epoch_valid if per_epoch_valid is not None else np.ones(zs.shape[:2], bool)
    return imm_batch(xs, Ps, F, Q, g[prefix + "H"], g[prefix + "R"], np.ones(nm), g[prefix + "mu0"],
                     g[prefix + "trans"], zs, valid)


@pytest.mark.parametrize("nm", [2, 3])
def test_oracle_reproduces_mm_golden(golden, nm):
    g = golden("mm")
    o = _mm_case(g, "m%d_" % nm, nm, None)
    for k in ("x", "P", "xp", "Pp", "mu", "fx", "fP"):
        close(o[k], g["imm%d_%s" % (nm, k)])


@pytest.mark.parametrize("name", MM_MISSING)
def test_oracle_reproduces_mm_missing_golden(golden, name):
    g = golden("mm_missing")
    p = name + "_"
    nm = g[p + "trans"].shape[0]
    o = _mm_case(g, p, nm, g[p + "valid"])
    for k in ("x", "P", "xp", "Pp", "mu", "cbar", "omega", "fx", "fP"):
        close(o[k], g[p + "imm_" + k])
    np.testing.assert_allclose(o["lik"], g[p + "imm_lik"], rtol=1e-10, atol=0)


# ------------------------------------------------------------------ the C-ABI without a device
def _args(N=8, T=3, n=4, m=2, M=3, dtype=_lib.BKE_F32):
    es = 4 if dtype == _lib.BKE_F32 else 8
    keep = []

    def buf(nbytes):
        b = np.zeros(nbytes // 8 + 4)
        keep.append(b)
        return b.ctypes.data + (-b.ctypes.data) % 16      # 16-byte aligned
    a = _lib.ImmBatchArgs()
    a.n_tracks, a.dim_x, a.dim_z, a.n_models, a.dtype, a.n_steps = N, n, m, M, dtype, T
    for j in range(M):
        a.x[j], a.P[j] = buf(N * n * es), buf(N * n * n * es)
        a.F[j], a.Q[j], a.H[j], a.R[j] = buf(n * n * es), buf(n * n * es), buf(m * n * es), buf(m * m * es)
        a.alpha_sq[j] = 1.0
        a.S[j], a.log_likelihood[j], a.K[j] = buf(N * m * m * es), buf(N * es), buf(N * n * m * es)
        a.y[j], a.SI[j], a.x_prior[j], a.P_prior[j] = buf(N * m * es), buf(N * m * m * es), buf(N * n * es), buf(N * n * n * es)
        a.status[j] = buf(N * 4)
    a.mu, a.cbar, a.omega, a.trans = buf(N * M * 8), buf(N * M * 8), buf(N * M * M * 8), buf(M * M * 8)
    a.zs = buf(T * N * m * es)
    a.means, a.covariances = buf(T * N * n * es), buf(T * N * n * n * es)
    a.means_p, a.covariances_p, a.mus = buf(T * N * n * es), buf(T * N * n * n * es), buf(T * N * M * 8)
    return a, keep


def _rc(a):
    return _lib.load().bke_imm_batch_filter(ctypes.byref(a), None)


@pytest.mark.parametrize("field,value", [
    ("n_tracks", -1), ("n_steps", -1), ("dim_x", 0), ("dim_z", 0), ("dtype", 3), ("n_models", 1), ("n_models", 9),
    ("flags", 1), ("mu", None), ("cbar", None), ("omega", None), ("trans", None), ("zs", None), ("means", None),
    ("covariances", None), ("means_p", None), ("covariances_p", None), ("mus", None),
])
def test_refuses_bad_arguments(field, value):
    a, keep = _args()
    setattr(a, field, value)
    assert _rc(a) == _lib.BKE_ERR_BAD_ARG


@pytest.mark.parametrize("field", ["x", "P", "F", "Q", "H", "R", "S", "log_likelihood", "K", "y", "SI", "x_prior",
                                   "P_prior", "status"])
def test_refuses_a_null_model_array(field):
    a, keep = _args()
    getattr(a, field)[2] = None
    assert _rc(a) == _lib.BKE_ERR_BAD_ARG


@pytest.mark.parametrize("field,value", [("F_stride", 4), ("Q_stride", -16), ("H_stride", 4), ("R_stride", 2)])
def test_refuses_a_bad_stride(field, value):
    a, keep = _args()
    getattr(a, field)[1] = value
    assert _rc(a) == _lib.BKE_ERR_BAD_ARG


@pytest.mark.parametrize("out,other", [("means", "zs"), ("covariances", "means_p"), ("mus", "mu"),
                                       ("means", ("x", 0)), (("P", 1), ("P", 2)), (("S", 0), "cbar"),
                                       (("status", 2), ("F", 0))])
def test_refuses_aliased_arrays(out, other):
    a, keep = _args()

    def get(f):
        return getattr(a, f[0])[f[1]] if isinstance(f, tuple) else getattr(a, f)
    if isinstance(out, tuple):
        getattr(a, out[0])[out[1]] = get(other)
    else:
        setattr(a, out, get(other))
    assert _rc(a) == _lib.BKE_ERR_BAD_ARG


@pytest.mark.parametrize("n,m,dtype", [(5, 2, _lib.BKE_F32), (6, 3, _lib.BKE_F32), (6, 3, _lib.BKE_F64),
                                       (4, 2, _lib.BKE_F64), (1, 1, _lib.BKE_F32), (4, 4, _lib.BKE_F32)])
def test_a_shape_without_a_fused_instance_is_unsupported(n, m, dtype):
    a, keep = _args(n=n, m=m, dtype=dtype)
    assert _rc(a) == _lib.BKE_ERR_UNSUPPORTED


def test_the_overlap_check_holds_every_array_of_the_largest_bank():
    """BKE_MM_MAX_MODELS models with zs_valid: the most arrays a call can pass all go through the overlap check.
    The shape has no fused instance, so no machine launches a kernel."""
    a, keep = _args(n=5, m=2, M=_lib.BKE_MM_MAX_MODELS)
    valid = np.ones(3 * 8, np.uint8)
    a.zs_valid = valid.ctypes.data
    assert _rc(a) == _lib.BKE_ERR_UNSUPPORTED
    a.zs_valid = a.means
    assert _rc(a) == _lib.BKE_ERR_BAD_ARG


@pytest.mark.parametrize("field", ["covariances", ("x", 1), ("S", 0)])
def test_a_misaligned_array_is_unsupported(field):
    a, keep = _args()
    if isinstance(field, tuple):
        getattr(a, field[0])[field[1]] += 4
    else:
        setattr(a, field, getattr(a, field) + 4)
    assert _rc(a) == _lib.BKE_ERR_UNSUPPORTED


def test_nothing_to_do_is_ok_without_a_device():
    a, keep = _args(T=0)
    assert _rc(a) == _lib.BKE_OK
    a, keep = _args(N=0)
    assert _rc(a) == _lib.BKE_OK


def test_every_fused_instance_is_free_of_spills():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc is not available")
    from filterpy_b200 import _build
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc] + _build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(_build.CSRC, "imm.cu"),
                                                         "-o", os.path.join(d, "imm.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    kernels = re.findall(r"Compiling entry function '(\w*imm_batch_kernel\w*)'", log)
    # (float, double) x (2/1, 3/1) x G in {2, 4, 8} and float 4/2 x G
    assert len(kernels) == 15, kernels
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    frames = re.findall(r"(\d+) bytes stack frame", log)
    assert len(spills) == 15 and all(s == ("0", "0") for s in spills), spills
    assert all(f == "0" for f in frames), frames
