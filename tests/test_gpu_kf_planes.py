"""The copies among the packed model words of the 4/2 fp32 step: bke_kf_scan_models flags in
`duplicate` the planes that equal an earlier plane in every filter (checked against NumPy), and
bke_kf_step_packed never reads a flagged plane (poisoned with NaN, the step is still bit-identical to the
dense step) while it does read the representative planes."""
import numpy as np
import pytest

from test_gpu_kf_packed import (_all_words_bank, _bench_bank, _dev, _last_filter_bank, _scan_and_pack,
                                _signed_zero_bank, _words)
from test_gpu_kf_sym import MODES, NS, _args, _mirror, _outputs, _uses_record

pytestmark = pytest.mark.gpu

BENCH_DUPLICATE = sum(1 << s for s in (1, 5, 6, 7, 9))     # F23, Q22, Q23, Q33, R11 of kf_bank_cv2d


def _duplicate(w):
    """The `duplicate` mask by the rule of bke.h, from the words of every filter."""
    bits = _words(w).view(np.uint32)
    sel = [e for e in range(37) if (bits[:, e] != bits[0, e]).any()]
    dup = 0
    for s, e in enumerate(sel[:32]):
        c = next((t for t in range(s) if bits[0, sel[t]] == bits[0, e]), None)
        if c is not None and (bits[:, sel[c]] == bits[:, e]).all():
            dup |= 1 << s
    return dup


def _slot(hmap, e):
    assert hmap.varying >> e & 1
    return bin(hmap.varying & ((1 << e) - 1)).count("1")


def _one_differs_bank(N, seed):
    """kf_bank_cv2d where Q22 differs from Q00 (its copy everywhere else) in one filter."""
    w = _bench_bank(N, seed)
    w["Q"][N // 2, 2, 2] = np.nextafter(w["Q"][N // 2, 2, 2], np.float32(1.0))
    return w


def _nan_bank(N, seed):
    """kf_bank_cv2d where filter 5 holds NaNs in F02, F03 and F12 with the same payload, and in F13 with
    another: F03 and F12 are copies of F02, F13 is not."""
    w = _bench_bank(N, seed)
    a, b = np.array([0x7fc00001, 0x7fc00002], dtype=np.uint32).view(np.float32)
    w["F"][5, 0, 2] = w["F"][5, 0, 3] = w["F"][5, 1, 2] = a
    w["F"][5, 1, 3] = b
    return w


def _class_of_three_bank(N, seed):
    """kf_bank_cv2d with F02 = dt as well: F01, F02 and F23 form one class."""
    w = _bench_bank(N, seed)
    w["F"][:, 0, 2] = w["F"][:, 0, 1]
    return w


def _many_words_bank(N, seed):
    """Every word varies (37 slots), F11 is a copy of F00 (slot 5) and R11 one of R00 (slot 36, beyond
    the 32 bits of `duplicate`)."""
    w = _all_words_bank(N, seed)
    w["F"][:, 1, 1] = w["F"][:, 0, 0]
    w["R"][:, 1, 1] = w["R"][:, 0, 0]
    return w


def _shared_bank(N, seed):
    """Every filter has filter 0's models: no word varies."""
    w = _bench_bank(N, seed)
    for k in "FQHR":
        w[k] = np.ascontiguousarray(np.broadcast_to(w[k][:1], w[k].shape))
    return w


SCAN_BANKS = {"bench": _bench_bank, "last_filter": _last_filter_bank, "signed_zero": _signed_zero_bank,
              "one_differs": _one_differs_bank, "nan": _nan_bank, "class_of_three": _class_of_three_bank,
              "many_words": _many_words_bank, "shared": _shared_bank}


@pytest.mark.parametrize("kind", list(SCAN_BANKS))
def test_scan_flags_the_copies(kind):
    N = 1000
    w = SCAN_BANKS[kind](N, 3)
    _, hmap = _scan_and_pack(_dev(w), N)
    assert hmap.duplicate == _duplicate(w)
    if kind == "bench":
        assert hmap.duplicate == BENCH_DUPLICATE
    elif kind == "last_filter":
        assert hmap.duplicate >> _slot(hmap, 35) & 1                  # R01 is a copy of F02
        assert not hmap.duplicate >> _slot(hmap, 18) & 1              # Q02 is not
    elif kind == "one_differs":
        assert hmap.duplicate == BENCH_DUPLICATE & ~(1 << _slot(hmap, 23))
    elif kind == "nan":
        assert hmap.duplicate >> _slot(hmap, 3) & 1 and hmap.duplicate >> _slot(hmap, 6) & 1
        assert not hmap.duplicate >> _slot(hmap, 7) & 1
    elif kind == "class_of_three":
        assert hmap.duplicate >> _slot(hmap, 2) & 1 and hmap.duplicate >> _slot(hmap, 11) & 1
        assert not hmap.duplicate >> _slot(hmap, 1) & 1
    elif kind == "many_words":
        assert hmap.varying == (1 << 37) - 1 and hmap.duplicate == 1 << 5
    elif kind == "shared":
        assert hmap.varying == 0 and hmap.duplicate == 0


def _step_bits(d, N, flags, extras, zs, graphed, rec=None, hmap=None):
    """Two chained steps, dense (rec None) or packed, on a copy of the state: every output as bits."""
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    o = _outputs(d, N, extras)
    args = [_args(d, o, N, flags, extras, z) for z in zs]

    def run():
        s = torch.cuda.current_stream().cuda_stream
        for a in args:
            _lib.check(lib.bke_kf_step(a, s) if rec is None else lib.bke_kf_step_packed(a, rec.data_ptr(), hmap, s))
    if graphed:
        x0, P0 = o["x"].clone(), o["P"].clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            run()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            run()
        o["x"].copy_(x0); o["P"].copy_(P0)
        g.replay()
    else:
        run()
    torch.cuda.synchronize()
    return {k: v.cpu().numpy().view(np.uint32) for k, v in o.items()}


def _poison(rec, hmap, N, slots):
    k = bin(hmap.varying).count("1")
    rec[:(N + 127) // 128 * k * 128].view(-1, k, 128)[:, slots, :] = float("nan")


_cache = {}


def _bank(kind, N):
    if (kind, N) not in _cache:
        _cache.clear()                                   # one bank of 2^20 filters at a time
        w = {"bench": _bench_bank, "last_filter": _last_filter_bank}[kind](N, 7)
        _cache[(kind, N)] = (w, _dev(w))
    return _cache[(kind, N)]


@pytest.mark.parametrize("graphed", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("extras", [False, True], ids=["plain", "extras"])
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("kind", ["bench", "last_filter"])
def test_flagged_planes_are_not_read(kind, N, mode, extras, graphed):
    """Every flagged plane of the record overwritten with NaN: the packed step still equals the dense
    step bit for bit (last_filter: an update-only step reads R01 from F02's plane in the predict part)."""
    import torch
    w, d = _bank(kind, N)
    zs = [torch.from_numpy(w["zs"][t]).cuda() for t in range(2)]
    rec, hmap = _scan_and_pack(d, N)
    flagged = [s for s in range(32) if hmap.duplicate >> s & 1]
    assert len(flagged) == {"bench": 5, "last_filter": 6}[kind]
    _poison(rec, hmap, N, flagged)
    dense = _step_bits(d, N, MODES[mode], extras, zs, graphed)
    packed = _step_bits(d, N, MODES[mode], extras, zs, graphed, rec, hmap)
    for k in dense:
        np.testing.assert_array_equal(packed[k], dense[k], err_msg=k)


@pytest.mark.parametrize("mode", list(MODES))
def test_poisoned_representative_changes_the_outputs(mode):
    """The same poisoning applied to a representative plane (F01's for predict, R00's for update) does
    reach the outputs: the test above can fail."""
    import torch
    N = (1 << 18) + 1
    w, d = _bank("bench", N)
    zs = [torch.from_numpy(w["zs"][t]).cuda() for t in range(2)]
    rec, hmap = _scan_and_pack(d, N)
    _poison(rec, hmap, N, [_slot(hmap, 1 if mode != "update" else 34)])
    dense = _step_bits(d, N, MODES[mode], False, zs, False)
    packed = _step_bits(d, N, MODES[mode], False, zs, False, rec, hmap)
    assert not np.array_equal(packed["x"], dense["x"])


def test_zeroed_duplicate_gives_the_same_bits():
    """A map whose `duplicate` is cleared reads every plane of its own and computes the same bits."""
    import torch
    N = (1 << 18) + 1
    w, d = _bank("last_filter", N)
    zs = [torch.from_numpy(w["zs"][t]).cuda() for t in range(2)]
    rec, hmap = _scan_and_pack(d, N)
    assert hmap.duplicate
    flagged = _step_bits(d, N, 3, True, zs, False, rec, hmap)
    hmap.duplicate = 0
    every = _step_bits(d, N, 3, True, zs, False, rec, hmap)
    for k in flagged:
        np.testing.assert_array_equal(every[k], flagged[k], err_msg=k)


def test_inconsistent_map_is_refused_before_a_launch():
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    N = 1000
    w = _bench_bank(N, 5)
    d = _dev(w)
    rec, hmap = _scan_and_pack(d, N)
    o = _outputs(d, N, False)
    a = _args(d, o, N, 3, False, torch.from_numpy(w["zs"][0]).cuda())
    bad = _lib.KfModelMap.from_buffer_copy(bytes(hmap))
    bad.duplicate = 1 << 2                                   # Q00 (slot 2) has no earlier equal word
    x0 = o["x"].clone()
    assert lib.bke_kf_step_packed(a, rec.data_ptr(), bad, torch.cuda.current_stream().cuda_stream) == _lib.BKE_ERR_BAD_ARG
    torch.cuda.synchronize()
    assert torch.equal(o["x"], x0)


def test_mirror_reads_the_representatives():
    """Several steps of the bench bank through KalmanFilter use the record with the five copies flagged,
    and x and P equal those of a bank that never packs (F assigned before every step) bit for bit."""
    import torch
    N = (1 << 14) + 1
    w = _bench_bank(N, 13)
    z = torch.from_numpy(w["zs"][0]).cuda()
    kf, ref = _mirror(w), _mirror(w)
    for _ in range(3):
        kf.predict(); kf.update(z)
        ref.F = w["F"]
        ref.predict(); ref.update(z)
    assert _uses_record(kf) and ref._sym_buf is None
    assert kf._sym_host_map.duplicate == BENCH_DUPLICATE
    for k in "xP":
        np.testing.assert_array_equal(getattr(kf, k).cpu().numpy().view(np.uint32),
                                      getattr(ref, k).cpu().numpy().view(np.uint32), err_msg=k)

