"""The C-ABI of the fused ring of the 4/2 fp32 step (bke_kf_steps_packed) and of bke_capture_node_count:
the signature and the argument checks, without a GPU."""
import ctypes
import os
import re

from filterpy_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_the_ring_and_its_limit():
    hdr = open(os.path.join(ROOT, "include", "bke.h")).read()
    assert int(re.search(r"#define BKE_KF42_MAX_RING (\d+)", hdr).group(1)) == _lib.BKE_KF42_MAX_RING == 8
    sig = re.search(r"int bke_kf_steps_packed\(([^;]*)\);", hdr).group(1)
    assert [p.strip().split()[-1].lstrip("*") for p in sig.split(",")] == ["args", "record", "host_map", "zs", "n_steps", "stream"]


def _args(fake):
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags = 8, 4, 2, _lib.BKE_F32, 3
    a.x = a.x_out = fake
    a.P = a.P_out = 2 * fake
    a.F = a.Q = a.H = a.R = 3 * fake
    return a


def test_ring_rejects_bad_arguments():
    lib = _lib.load()
    fake = 1 << 20                                        # never dereferenced: every call fails before a launch
    zs = (ctypes.c_void_p * 9)(*[4 * fake] * 9)
    m = _lib.KfModelMap()
    a = _args(fake)
    a.dim_x = 0
    assert lib.bke_kf_steps_packed(a, fake, m, zs, 4, None) == _lib.BKE_ERR_BAD_ARG
    assert b"dim_x must be 1 or greater" in lib.bke_last_error()
    a = _args(fake)
    assert lib.bke_kf_steps_packed(None, fake, m, zs, 4, None) == _lib.BKE_ERR_BAD_ARG
    assert lib.bke_kf_steps_packed(a, fake, None, zs, 4, None) == _lib.BKE_ERR_BAD_ARG
    assert b"host_map is NULL" in lib.bke_last_error()
    assert lib.bke_kf_steps_packed(a, fake, m, None, 4, None) == _lib.BKE_ERR_BAD_ARG
    assert b"zs is NULL" in lib.bke_last_error()
    m.varying = 3
    assert lib.bke_kf_steps_packed(a, None, m, zs, 4, None) == _lib.BKE_ERR_BAD_ARG
    assert b"record is NULL" in lib.bke_last_error()
    m.varying = 1 << 37
    assert lib.bke_kf_steps_packed(a, fake, m, zs, 4, None) == _lib.BKE_ERR_BAD_ARG
    m.varying = 3
    holes = (ctypes.c_void_p * 2)(4 * fake, None)
    assert lib.bke_kf_steps_packed(a, fake, m, holes, 2, None) == _lib.BKE_ERR_BAD_ARG
    assert b"zs[1] is NULL" in lib.bke_last_error()


def test_ring_refuses_what_it_does_not_take():
    lib = _lib.load()
    fake = 1 << 20
    zs = (ctypes.c_void_p * 9)(*[4 * fake] * 9)
    m = _lib.KfModelMap()
    m.varying = 3

    def refused(text, n_steps=4, zs=zs, **kw):
        a = _args(fake)
        for k, v in kw.items():
            setattr(a, k, v)
        assert lib.bke_kf_steps_packed(a, fake, m, zs, n_steps, None) == _lib.BKE_ERR_UNSUPPORTED, text
        assert text in lib.bke_last_error(), lib.bke_last_error()
    refused(b"n_steps", n_steps=0)
    refused(b"n_steps", n_steps=9)
    refused(b"flags", flags=_lib.BKE_DO_UPDATE)
    refused(b"flags", flags=3 | _lib.BKE_UPDATE_FIRST)
    refused(b"z_valid", z_valid=fake)
    refused(b"control", B=fake, u=fake)
    refused(b"optional outputs", status=fake)
    refused(b"optional outputs", K=fake)
    refused(b"in place", x_out=5 * fake)
    refused(b"in place", P_out=5 * fake)
    refused(b"aligned", zs=(ctypes.c_void_p * 4)(*[4 * fake + 8] * 4))
    refused(b"overlaps", zs=(ctypes.c_void_p * 4)(4 * fake, 4 * fake, 2 * fake + 64, 4 * fake))
    refused(b"overlaps", zs=(ctypes.c_void_p * 4)(*[fake - 16] * 4))


def test_capture_node_count_checks_its_arguments():
    lib = _lib.load()
    assert lib.bke_capture_node_count(None, None) == _lib.BKE_ERR_BAD_ARG
    assert b"n_nodes is NULL" in lib.bke_last_error()
