"""bke_kf_step_packed refuses a map whose `duplicate` bits do not follow the rule of bke.h before it
looks for a device, so these checks run without a GPU."""
from filterpy_b200 import _lib

BENCH = (1 << 1) | (1 << 11) | sum(1 << e for e in (16, 17, 20, 23, 24, 25)) | (1 << 34) | (1 << 36)   # 10 slots


def _call(n_filters, duplicate, words=None):
    lib = _lib.load()
    fake = 1 << 20                                        # never dereferenced: no filter is stepped
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags = n_filters, 4, 2, _lib.BKE_F32, 3
    a.x = a.P = a.x_out = a.P_out = a.F = a.Q = a.H = a.R = a.z = fake
    a.F_stride, a.Q_stride, a.H_stride, a.R_stride = 16, 16, 8, 4
    m = _lib.KfModelMap()
    m.varying, m.duplicate = BENCH, duplicate
    for e in range(_lib.BKE_KF42_MODEL_WORDS):
        m.words[e] = float(e)                            # every filter-0 word distinct...
    for e, v in (words or {}).items():
        m.words[e] = v                                   # ...unless the case sets some equal
    return lib.bke_kf_step_packed(a, fake, m, None), lib.bke_last_error()


def test_bit_beyond_the_varying_slots_is_refused():
    rc, err = _call(8, 1 << 10, {11: 1.0})
    assert rc == _lib.BKE_ERR_BAD_ARG
    assert b"duplicate flags slot 10, but only 10 words vary" in err


def test_bit_without_an_earlier_equal_word_is_refused():
    rc, err = _call(8, 1 << 1)                           # F23 (slot 1) differs from F01 (slot 0) in filter 0
    assert rc == _lib.BKE_ERR_BAD_ARG
    assert b"duplicate flags slot 1 (word 11), but no earlier slot has the same filter-0 word" in err
    rc, err = _call(8, 1 << 0)                           # slot 0 has no earlier slot at all
    assert rc == _lib.BKE_ERR_BAD_ARG
    assert b"slot 0 (word 1)" in err
    rc, err = _call(8, (1 << 1) | (1 << 5), {11: 1.0, 23: -0.0, 16: 0.0})    # Q22 = -0.0 is not Q00 = +0.0
    assert rc == _lib.BKE_ERR_BAD_ARG
    assert b"slot 5 (word 23)" in err


def test_consistent_bits_pass_the_check():
    # no filter: nothing is launched, so the call reaches the device check (and succeeds on a GPU)
    rc, _ = _call(0, (1 << 1) | (1 << 5), {11: 1.0, 23: 16.0})
    assert rc != _lib.BKE_ERR_BAD_ARG
