"""The tile-order word of the fused ring (bke_kf_args.tile_order): every launch of bke_kf_steps_packed given the
word walks the bank in the order of its epoch's parity and advances the epoch, so a captured graph of one launch
alternates the order across replays.  The order is a scheduling choice: replays equal eager stepping bit for bit,
each bank counts only its own launches, a call without the word keeps BKE_REVERSE_TILES and leaves any word alone,
and a misaligned word is refused before anything is launched."""
import ctypes

import numpy as np
import pytest

from test_gpu_kf_ring import _CBank, _mirror, _replays_equal_eager, _same_bits, _workload, _zbufs


def _captured(N, K):
    w = _workload(N)
    kf, ref = _mirror(w, N), _mirror(w, N)
    zs = _zbufs(w, K)

    def steps(bank=kf):
        for z in zs:
            bank.predict(); bank.update(z)
    graph = kf.capture(steps)
    assert (graph.launches, graph.fused_steps) == ((K + 7) // 8, K)
    return w, kf, ref, graph, steps


def _word(kf):
    import torch
    torch.cuda.synchronize()
    return [int(v) for v in kf._tile_order.cpu()]


@pytest.mark.gpu
@pytest.mark.parametrize("replays", [3, 4])
@pytest.mark.parametrize("K", [1, 4, 8, 12])
@pytest.mark.parametrize("N", [127, 129, (1 << 18) + 3])
def test_replays_of_the_ordered_ring_equal_eager_steps_bit_for_bit(N, K, replays):
    """N: one ragged tile, a tile plus one odd filter that reads its own z, and several tiles per CTA; the
    replays run in both orders (K = 12 is two launches per replay)."""
    w, kf, ref, graph, steps = _captured(N, K)
    _replays_equal_eager(kf, graph, ref, lambda: steps(ref), w, replays=replays)
    assert _word(kf) == [graph.launches * (1 + replays), 0]


@pytest.mark.gpu
def test_each_bank_counts_only_its_own_ring_launches():
    N = (1 << 18) + 3
    _, kf, _, g12, steps12 = _captured(N, 12)
    _, other, _, g4, _ = _captured(N, 4)
    assert kf._tile_order.data_ptr() != other._tile_order.data_ptr()
    assert _word(kf) == [2, 0] and _word(other) == [1, 0]           # the first, eager, run of each ring
    for _ in range(5):
        g12.replay()
        g4.replay()
    assert _word(kf) == [12, 0] and _word(other) == [6, 0]
    steps12()                                                          # separate steps do not use the word
    assert _word(kf) == [12, 0]
    g12.replay()
    assert _word(kf) == [14, 0] and _word(other) == [6, 0]


@pytest.mark.gpu
def test_a_ring_without_the_word_keeps_the_flag_and_leaves_a_word_alone():
    import torch
    from torch.profiler import profile, ProfilerActivity
    from filterpy_b200 import _lib
    N = (1 << 19) + 1                                   # above the bound under which BKE_REVERSE_TILES is ignored
    b = _CBank(_workload(N), N)
    zs = b.zs[:4]
    xs, Ps = b.stepwise(zs)
    idle = torch.tensor([7, 3], dtype=torch.int32, device="cuda")
    for flags in (3, 3 | _lib.BKE_REVERSE_TILES):
        rc, x, P = b.ring(zs, a=lambda x, P: b.args(x, P, flags))
        assert rc == 0, b.lib.bke_last_error()
        _same_bits(x, xs, "x, flags %d" % flags); _same_bits(P, Ps, "P, flags %d" % flags)
    word = torch.zeros(2, dtype=torch.int32, device="cuda")

    def with_word(x, P):
        a = b.args(x, P, 3 | _lib.BKE_REVERSE_TILES)  # the word decides; the flag is ignored
        a.tile_order = word.data_ptr()
        return a
    for epoch in (1, 2):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            rc, x, P = b.ring(zs, a=with_word)
        assert rc == 0, b.lib.bke_last_error()
        assert [n for n in (e.name for e in prof.events()) if "kf42_f32_kernel" in n and "Cv2dPattern" in n]
        _same_bits(x, xs, "x, epoch %d" % epoch); _same_bits(P, Ps, "P, epoch %d" % epoch)
        assert [int(v) for v in word.cpu()] == [epoch, 0]
    assert [int(v) for v in idle.cpu()] == [7, 3]


def test_a_misaligned_word_is_refused_without_a_gpu():
    from filterpy_b200 import _lib
    lib = _lib.load()
    fake = 1 << 20                                      # never dereferenced: the call fails before a launch
    zs = (ctypes.c_void_p * 4)(*[4 * fake] * 4)
    m = _lib.KfModelMap()
    m.varying = 3
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags = 8, 4, 2, _lib.BKE_F32, 3
    a.x = a.x_out = fake
    a.P = a.P_out = 2 * fake
    a.F = a.Q = a.H = a.R = 3 * fake
    for off in (1, 2, 3, 6):
        a.tile_order = 5 * fake + off
        assert lib.bke_kf_steps_packed(a, fake, m, zs, 4, None) == _lib.BKE_ERR_BAD_ARG
        assert b"tile_order must be 4-byte aligned" in lib.bke_last_error()
