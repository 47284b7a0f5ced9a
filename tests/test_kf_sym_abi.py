"""The C-ABI of the packed symmetric Q / R record: its size and argument checks, without a GPU."""
from filterpy_b200 import _lib


def test_record_size_is_whole_tiles_of_13_planes():
    lib = _lib.load()
    assert lib.bke_kf_sym_models_bytes(0) == 0
    assert lib.bke_kf_sym_models_bytes(1) == 13 * 128 * 4
    assert lib.bke_kf_sym_models_bytes(300) == 3 * 13 * 128 * 4
    assert lib.bke_kf_sym_models_bytes(1 << 20) == (1 << 20) * 52


def test_pack_and_step_reject_bad_arguments_and_other_shapes():
    lib = _lib.load()
    fake = 1 << 20                                        # never dereferenced: every call fails before a launch
    assert lib.bke_kf_pack_sym_models(-1, 4, 2, _lib.BKE_F32, fake, fake, fake, fake, None) == _lib.BKE_ERR_BAD_ARG
    assert lib.bke_kf_pack_sym_models(8, 4, 2, _lib.BKE_F32, None, fake, fake, fake, None) == _lib.BKE_ERR_BAD_ARG
    assert lib.bke_kf_pack_sym_models(8, 4, 2, _lib.BKE_F32, fake, fake, fake, None, None) == _lib.BKE_ERR_BAD_ARG
    for dims in ((4, 3, _lib.BKE_F32), (3, 2, _lib.BKE_F32), (4, 2, _lib.BKE_F64)):
        assert lib.bke_kf_pack_sym_models(8, *dims, fake, fake, fake, fake, None) == _lib.BKE_ERR_UNSUPPORTED
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags = 8, 0, 2, _lib.BKE_F32, 3
    assert lib.bke_kf_step_sym(a, fake, None) == _lib.BKE_ERR_BAD_ARG
    assert b"dim_x must be 1 or greater" in lib.bke_last_error()
    a.dim_x = 4
    a.x = a.P = a.x_out = a.P_out = a.F = a.Q = a.H = a.R = a.z = fake
    assert lib.bke_kf_step_sym(a, None, None) == _lib.BKE_ERR_BAD_ARG
    assert b"record is NULL" in lib.bke_last_error()
