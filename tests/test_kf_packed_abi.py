"""The C-ABI of the packed model words of the 4/2 fp32 step: the record's size and the argument
checks, without a GPU."""
from filterpy_b200 import _lib


def test_record_size_is_whole_tiles_of_the_varying_planes():
    assert _lib.BKE_KF42_MODEL_WORDS == 37
    lib = _lib.load()
    bench = (1 << 1) | (1 << 11) | sum(1 << e for e in (16, 17, 20, 23, 24, 25)) | (1 << 34) | (1 << 36)   # k = 10
    assert lib.bke_kf_packed_models_bytes(0, bench) == 0
    assert lib.bke_kf_packed_models_bytes(-5, bench) == 0
    assert lib.bke_kf_packed_models_bytes(1, bench) == 10 * 128 * 4
    assert lib.bke_kf_packed_models_bytes(300, bench) == 3 * 10 * 128 * 4
    assert lib.bke_kf_packed_models_bytes(1 << 20, bench) == (1 << 20) * 40
    assert lib.bke_kf_packed_models_bytes(1 << 20, (1 << 37) - 1) == (1 << 20) * 148
    assert lib.bke_kf_packed_models_bytes(1 << 20, 0) == 0
    assert lib.bke_kf_packed_models_bytes(1 << 20, 1 << 37) == 0          # no word 37


def test_scan_pack_and_step_reject_bad_arguments_and_other_shapes():
    lib = _lib.load()
    fake = 1 << 20                                        # never dereferenced: every call fails before a launch
    f4 = (fake,) * 4
    assert lib.bke_kf_scan_models(-1, 4, 2, _lib.BKE_F32, *f4, fake, None) == _lib.BKE_ERR_BAD_ARG
    assert lib.bke_kf_scan_models(8, 4, 2, _lib.BKE_F32, fake, fake, None, fake, fake, None) == _lib.BKE_ERR_BAD_ARG
    assert lib.bke_kf_scan_models(8, 4, 2, _lib.BKE_F32, *f4, None, None) == _lib.BKE_ERR_BAD_ARG
    assert b"map must be non-NULL" in lib.bke_last_error()
    assert lib.bke_kf_pack_models(8, 4, 2, _lib.BKE_F32, None, fake, fake, fake, 3, fake, None) == _lib.BKE_ERR_BAD_ARG
    assert lib.bke_kf_pack_models(8, 4, 2, _lib.BKE_F32, *f4, 3, None, None) == _lib.BKE_ERR_BAD_ARG
    assert lib.bke_kf_pack_models(8, 4, 2, _lib.BKE_F32, *f4, 1 << 40, fake, None) == _lib.BKE_ERR_BAD_ARG
    assert b"bits above word 36" in lib.bke_last_error()
    for dims in ((4, 3, _lib.BKE_F32), (3, 2, _lib.BKE_F32), (4, 2, _lib.BKE_F64)):
        assert lib.bke_kf_scan_models(8, *dims, *f4, fake, None) == _lib.BKE_ERR_UNSUPPORTED
        assert lib.bke_kf_pack_models(8, *dims, *f4, 3, fake, None) == _lib.BKE_ERR_UNSUPPORTED
    a = _lib.KfArgs()
    m = _lib.KfModelMap()
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags = 8, 0, 2, _lib.BKE_F32, 3
    assert lib.bke_kf_step_packed(a, fake, m, None) == _lib.BKE_ERR_BAD_ARG
    assert b"dim_x must be 1 or greater" in lib.bke_last_error()
    a.dim_x = 4
    a.x = a.P = a.x_out = a.P_out = a.F = a.Q = a.H = a.R = a.z = fake
    assert lib.bke_kf_step_packed(a, fake, None, None) == _lib.BKE_ERR_BAD_ARG
    assert b"host_map is NULL" in lib.bke_last_error()
    m.varying = 3
    assert lib.bke_kf_step_packed(a, None, m, None) == _lib.BKE_ERR_BAD_ARG
    assert b"record is NULL" in lib.bke_last_error()
    m.varying = 1 << 37
    assert lib.bke_kf_step_packed(a, fake, m, None) == _lib.BKE_ERR_BAD_ARG
