"""bke_db_step's argument checks: every refusal is BKE_ERR_BAD_ARG with its reason, returned before any device is
touched (the pointers below are never dereferenced), and the workspace size separates the two paths at the
shared-memory bound."""
import ctypes

import pytest

from filterpy_b200 import _lib

B, M, K = 4, 64, 3


def args(**kw):
    a = _lib.DbArgs()
    a.n_rows, a.n_bins, a.dtype, a.flags = B, M, _lib.BKE_F64, _lib.BKE_DB_NORMALIZE
    a.kernel, a.kernel_len, a.kernel_stride = 0x100000, K, 0
    a.pdf, a.likelihood, a.out = 0x200000, 0x300000, 0x400000
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def refused(a, text):
    lib = _lib.load()
    assert lib.bke_db_step(ctypes.byref(a), None) == _lib.BKE_ERR_BAD_ARG
    assert text in lib.bke_last_error().decode()


@pytest.mark.parametrize("kw, text", [
    (dict(n_bins=0), "n_bins >= 1"),
    (dict(n_rows=-1), "n_rows must be >= 0"),
    (dict(n_bins=1 << 31), "< 2^31"),
    (dict(dtype=7), "dtype must be"),
    (dict(flags=4), "flags may only hold"),
    (dict(kernel_len=0), "kernel_len must be 1 or greater"),
    (dict(kernel_stride=2), "model strides"),
    (dict(sums=0x500000, flags=0), "sums is an output of BKE_DB_NORMALIZE only"),
    (dict(pdf=None), "pdf and out must be non-NULL"),
    (dict(out=None), "pdf and out must be non-NULL"),
    (dict(out=0x300000 + 8), "overlaps"),                       # out inside the likelihood
    (dict(out=0x200000 + 8), "overlaps"),                       # out partly over pdf (only out == pdf may alias)
    (dict(sums=0x400000 + 16), "overlaps"),                     # sums inside out
    (dict(kernel=0x400000, kernel_stride=K), "overlaps"),       # a per-row kernel inside out
])
def test_refusals(kw, text):
    refused(args(**kw), text)


def test_multi_pass_workspace_is_checked():
    lib = _lib.load()
    long_m = 14465                                               # one bin past the fp64 rows one CTA stages
    need = lib.bke_db_workspace_bytes(long_m, _lib.BKE_F64)
    assert need > 2 * long_m * 8
    refused(args(n_bins=long_m), "workspace must be non-NULL and 256-byte aligned")
    refused(args(n_bins=long_m, workspace=0x10000000 + 8, workspace_bytes=need), "256-byte aligned")
    refused(args(n_bins=long_m, workspace=0x10000000, workspace_bytes=need - 1), "workspace too small")
    refused(args(n_bins=long_m, workspace=0x400000, workspace_bytes=need), "overlaps")


def test_workspace_bytes_split_at_the_staged_row():
    lib = _lib.load()
    assert lib.bke_db_workspace_bytes(28928, _lib.BKE_F32) == 0            # 2 * 28928 * 4 = 226 KB
    assert lib.bke_db_workspace_bytes(28929, _lib.BKE_F32) > 0
    assert lib.bke_db_workspace_bytes(14464, _lib.BKE_F64) == 0
    assert lib.bke_db_workspace_bytes(14465, _lib.BKE_F64) > 0
    assert lib.bke_db_workspace_bytes(1 << 24, _lib.BKE_F32) > 2 * (1 << 24) * 8


def test_empty_bank_and_in_place_pass_validation():
    """n_rows = 0 is a no-op, and out == pdf is the one alias allowed (validation passes; the call then needs a
    device, which a CPU-only machine refuses with BKE_ERR_CUDA rather than computing on the CPU)."""
    lib = _lib.load()
    assert lib.bke_db_step(ctypes.byref(args(n_rows=0, pdf=None, out=None)), None) == _lib.BKE_OK
    import torch
    if torch.cuda.is_available():
        pytest.skip("the no-device refusal needs a machine without a GPU")
    rc = lib.bke_db_step(ctypes.byref(args(out=0x200000)), None)
    assert rc == _lib.BKE_ERR_CUDA and b"no CPU fallback" in lib.bke_last_error()
