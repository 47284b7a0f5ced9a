"""The fused ring of the 4/2 fp32 step (bke_kf_steps_packed): K predict+update steps in one launch are bit
for bit K launches of bke_kf_step_packed; what the ring does not take is refused before anything is
launched; KalmanFilter.capture returns the fused form of an eligible ring and the graph of separate steps
of every other one, and either replays to the same bits as eager stepping."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STEPS = 8
_cache = {}


def _workload(N):
    from filterpy_b200.common import workloads as wl
    if N not in _cache:
        _cache.clear()                                   # one bank of 2^20 filters at a time
        _cache[N] = wl.kf_bank_cv2d(N, seed=21, steps=STEPS, dtype=np.float32)
    return {k: v.copy() for k, v in _cache[N].items()}


def _bench_bank(N):
    return _workload(N)


def _one_model_bank(N):
    """Per-filter arrays that all hold filter 0's models: no word varies, the record is NULL."""
    w = _workload(N)
    for k in "FQHR":
        w[k] = np.ascontiguousarray(np.broadcast_to(w[k][0], w[k].shape))
    return w


def _all_words_bank(N):
    """Every one of the 37 model words differs between filters; Q and R stay exactly symmetric."""
    w = _workload(N)
    rng = np.random.default_rng(5)
    for k, shape in (("F", (4, 4)), ("H", (2, 4))):
        w[k] = np.ascontiguousarray(w[k] + np.float32(1e-3) * rng.standard_normal((N,) + shape).astype(np.float32))
    for k, n in (("Q", 4), ("R", 2)):
        a = w[k] + np.float32(1e-3) * rng.standard_normal((N, n, n)).astype(np.float32)
        w[k] = np.ascontiguousarray(np.triu(a) + np.swapaxes(np.triu(a, 1), 1, 2))
    return w


BANKS = {"bench": (_bench_bank, 10), "one_model": (_one_model_bank, 0), "all_words": (_all_words_bank, 37)}


class _CBank(object):
    """Device arrays, packed record and host map of a bank, for calls through the C-ABI."""

    def __init__(self, w, N):
        import torch
        from filterpy_b200 import _lib
        self.lib, self.N = _lib.load(), N
        self.d = {k: torch.from_numpy(np.ascontiguousarray(w[k])).cuda() for k in "xPFQHR"}
        self.zs = [torch.from_numpy(np.ascontiguousarray(z)).cuda() for z in w["zs"]]
        s = torch.cuda.current_stream().cuda_stream
        m = [self.d[k].data_ptr() for k in "FQHR"]
        dmap = torch.empty(ctypes.sizeof(_lib.KfModelMap), dtype=torch.uint8, device="cuda")
        _lib.check(self.lib.bke_kf_scan_models(N, 4, 2, _lib.BKE_F32, *m, dmap.data_ptr(), s))
        self.hmap = _lib.KfModelMap.from_buffer_copy(dmap.cpu().numpy().tobytes())
        nb = self.lib.bke_kf_packed_models_bytes(N, self.hmap.varying)
        self.rec = torch.empty(nb // 4, dtype=torch.float32, device="cuda") if nb else None
        _lib.check(self.lib.bke_kf_pack_models(N, 4, 2, _lib.BKE_F32, *m, self.hmap.varying, self.recp, s))

    @property
    def recp(self):
        return None if self.rec is None else self.rec.data_ptr()

    def args(self, x, P, flags=3):
        from filterpy_b200 import _lib
        a, d = _lib.KfArgs(), self.d
        a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags, a.alpha_sq = self.N, 4, 2, _lib.BKE_F32, flags, 1.0
        a.x = a.x_out = x.data_ptr(); a.P = a.P_out = P.data_ptr()
        a.F, a.F_stride, a.Q, a.Q_stride = d["F"].data_ptr(), 16, d["Q"].data_ptr(), 16
        a.H, a.H_stride, a.R, a.R_stride = d["H"].data_ptr(), 8, d["R"].data_ptr(), 4
        return a

    def stepwise(self, zs):
        """x, P after one bke_kf_step_packed per z."""
        import torch
        from filterpy_b200 import _lib
        x, P = self.d["x"].clone(), self.d["P"].clone()
        a = self.args(x, P)
        for z in zs:
            a.z = z.data_ptr()
            _lib.check(self.lib.bke_kf_step_packed(a, self.recp, self.hmap, torch.cuda.current_stream().cuda_stream))
        return x, P

    def ring(self, zs, a=None, n_steps=None):
        """(rc, x, P) of one bke_kf_steps_packed over zs."""
        import torch
        x, P = self.d["x"].clone(), self.d["P"].clone()
        a = a(x, P) if a is not None else self.args(x, P)
        arr = (ctypes.c_void_p * max(len(zs), 1))(*[z if isinstance(z, int) else z.data_ptr() for z in zs])
        rc = self.lib.bke_kf_steps_packed(a, self.recp, self.hmap, arr, len(zs) if n_steps is None else n_steps,
                                          torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return rc, x, P


def _same_bits(a, b, what):
    np.testing.assert_array_equal(a.cpu().numpy().view(np.uint32), b.cpu().numpy().view(np.uint32), err_msg=what)


# ---------------------------------------------------------------------------------------------- C level
@pytest.mark.parametrize("K", [1, 2, 4, 8])
@pytest.mark.parametrize("N", [1, 127, 128, 129, 1001, (1 << 20) + 3])
def test_ring_equals_separate_steps_bit_for_bit(N, K):
    b = _CBank(_bench_bank(N), N)
    assert bin(b.hmap.varying).count("1") == (10 if N > 1 else 0)         # one filter: nothing varies
    rc, x, P = b.ring(b.zs[:K])
    assert rc == 0, b.lib.bke_last_error()
    xs, Ps = b.stepwise(b.zs[:K])
    _same_bits(x, xs, "x"); _same_bits(P, Ps, "P")


@pytest.mark.parametrize("kind", ["one_model", "all_words"])
def test_ring_of_a_bank_with_no_or_with_37_varying_words(kind):
    N = 1001
    make, k = BANKS[kind]
    b = _CBank(make(N), N)
    assert bin(b.hmap.varying).count("1") == k and (b.rec is None) == (k == 0)
    rc, x, P = b.ring(b.zs[:4])
    assert rc == 0, b.lib.bke_last_error()
    xs, Ps = b.stepwise(b.zs[:4])
    _same_bits(x, xs, "x"); _same_bits(P, Ps, "P")


def test_ring_may_repeat_a_measurement_buffer_and_honours_the_tile_order():
    from filterpy_b200 import _lib
    N = (1 << 19) + 1                                   # above the bound under which the tile order is ignored
    b = _CBank(_bench_bank(N), N)
    zs = [b.zs[0], b.zs[1], b.zs[0], b.zs[0], b.zs[1]]
    xs, Ps = b.stepwise(zs)
    for flags in (3, 3 | _lib.BKE_REVERSE_TILES):
        rc, x, P = b.ring(zs, a=lambda x, P: b.args(x, P, flags))
        assert rc == 0, b.lib.bke_last_error()
        _same_bits(x, xs, "x"); _same_bits(P, Ps, "P")


def test_ring_refuses_what_it_does_not_take_without_a_launch():
    import torch
    from filterpy_b200 import _lib
    N = 1001
    b = _CBank(_bench_bank(N), N)
    status = torch.zeros(N, dtype=torch.int32, device="cuda")
    valid = torch.ones(N, dtype=torch.uint8, device="cuda")
    other = torch.zeros(N, 4, device="cuda")

    def with_(**kw):
        def make(x, P):
            a = b.args(x, P)
            for k, v in kw.items():
                setattr(a, k, v(x, P) if callable(v) else v)
            return a
        return make
    cases = {
        "n_steps = 0": dict(zs=b.zs[:1], n_steps=0),
        "n_steps = 9": dict(zs=b.zs + b.zs[:1]),
        "z_valid": dict(zs=b.zs[:2], a=with_(z_valid=valid.data_ptr())),
        "status": dict(zs=b.zs[:2], a=with_(status=status.data_ptr())),
        "update only": dict(zs=b.zs[:2], a=with_(flags=_lib.BKE_DO_UPDATE)),
        "x_out != x": dict(zs=b.zs[:2], a=with_(x_out=other.data_ptr())),
        "misaligned z": dict(zs=[b.zs[0].data_ptr() + 8]),
    }
    for name, kw in cases.items():
        rc, x, P = b.ring(**kw)
        assert rc == _lib.BKE_ERR_UNSUPPORTED, name
        assert b.lib.bke_last_error(), name
        _same_bits(x, b.d["x"], name); _same_bits(P, b.d["P"], name)
    # a z inside P
    x, P = b.d["x"].clone(), b.d["P"].clone()
    arr = (ctypes.c_void_p * 1)(P.data_ptr() + 64)
    rc = b.lib.bke_kf_steps_packed(b.args(x, P), b.recp, b.hmap, arr, 1, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == _lib.BKE_ERR_UNSUPPORTED and b"overlaps" in b.lib.bke_last_error()
    _same_bits(P, b.d["P"], "z in P")


# ---------------------------------------------------------------------------------------------- mirror
def _mirror(w, N, **kw):
    from filterpy_b200.kalman import KalmanFilter
    kf = KalmanFilter(4, 2, n_filters=N, dtype=np.float32, device="cuda", diagnostics=kw.pop("diagnostics", False))
    for k in "xPFHQR":
        setattr(kf, k, kw.get(k, w[k]))
    return kf


def _zbufs(w, n):
    import torch
    return [torch.from_numpy(w["zs"][i % STEPS]).cuda() for i in range(n)]


def _replays_equal_eager(kf, graph, ref, ref_step, w, replays=3):
    """Put the captured bank back on the initial state in place, replay, and compare with `ref` stepped eagerly."""
    import torch
    kf.x.copy_(torch.from_numpy(w["x"])); kf.P.copy_(torch.from_numpy(w["P"]))
    for _ in range(replays):
        graph.replay()
        ref_step()
    torch.cuda.synchronize()
    _same_bits(kf.x, ref.x, "x"); _same_bits(kf.P, ref.P, "P")


@pytest.mark.parametrize("ring,launches", [(4, 1), (3, 1), (11, 2)])
def test_captured_ring_is_fused_and_replays_equal_eager_steps(ring, launches):
    import torch
    N = (1 << 19) + 5
    w = _workload(N)
    kf, ref = _mirror(w, N), _mirror(w, N)
    zs = _zbufs(w, ring)

    def steps(bank=kf):
        for z in zs:
            bank.predict(); bank.update(z)
    graph = kf.capture(steps)
    assert (graph.launches, graph.fused_steps) == (launches, ring)
    _replays_equal_eager(kf, graph, ref, lambda: steps(ref), w)
    # measurements, then the state, refilled in place between replays
    for z in zs:
        z.mul_(1.5)
    graph.replay(); steps(ref)
    kf.x.mul_(0.5); kf.P.mul_(2.0); ref.x.mul_(0.5); ref.P.mul_(2.0)
    graph.replay(); steps(ref)
    torch.cuda.synchronize()
    _same_bits(kf.x, ref.x, "x after refills"); _same_bits(kf.P, ref.P, "P after refills")


def _not_fused(kf, ref, w, steps, ref_steps, launches=4, refusal=None):
    graph = kf.capture(steps)
    assert graph.fused_steps == 0 and graph.launches == launches
    if refusal is not None:                             # the library refused the ring, not the mirror
        assert refusal in kf._lib.bke_last_error()
    _replays_equal_eager(kf, graph, ref, ref_steps, w, replays=2)


def test_a_torch_op_between_the_steps_keeps_the_separate_steps():
    import torch
    N = (1 << 18) + 1
    w = _workload(N)
    kf, ref = _mirror(w, N), _mirror(w, N)
    zs, z = _zbufs(w, 4), torch.empty(N, 2, device="cuda")

    def steps(bank):
        for t in range(4):
            bank.predict()
            torch.mul(zs[t], 2.0, out=z)
            bank.update(z)
    _not_fused(kf, ref, w, lambda: steps(kf), lambda: steps(ref))


def test_two_banks_in_one_capture_keep_the_separate_steps():
    import torch
    N = (1 << 18) + 1
    w = _workload(N)
    kf, ref, other, other_ref = (_mirror(w, N) for _ in range(4))
    zs = _zbufs(w, 4)

    def steps(a, b):
        for z in zs:
            a.predict(); a.update(z)
            b.predict(); b.update(z)
    graph = kf.capture(lambda: steps(kf, other))
    assert graph.fused_steps == 0 and graph.launches == 4 and graph.nodes == 8
    for bank in (kf, other):
        bank.x.copy_(torch.from_numpy(w["x"])); bank.P.copy_(torch.from_numpy(w["P"]))
    graph.replay(); steps(ref, other_ref)
    torch.cuda.synchronize()
    for got, want in ((kf, ref), (other, other_ref)):
        _same_bits(got.x, want.x, "x"); _same_bits(got.P, want.P, "P")


@pytest.mark.parametrize("case", ["valid", "R", "asymmetric_Q", "shared_models", "z_in_x"])
def test_rings_the_fused_launch_does_not_cover_keep_the_separate_steps(case):
    import torch
    # z_in_x: every z is a view of the bank's own x, which separate steps read as the previous step left it
    # and a ring, which keeps x on chip, could not.  One tile: each separate step loads z before it stores x.
    N = 100 if case == "z_in_x" else (1 << 18) + 1
    w = _workload(N)
    kw, upd = {}, {}
    if case == "valid":
        upd = dict(valid=torch.from_numpy(np.arange(N) % 3 != 0).cuda())
    elif case == "R":
        upd = dict(R=torch.from_numpy(2.0 * w["R"]).cuda())
    elif case == "asymmetric_Q":
        Q = w["Q"].copy()
        Q[N // 2, 0, 1] *= np.float32(1.5)
        kw = dict(Q=Q)
    elif case == "shared_models":
        kw = {k: w[k][0] for k in "FHQR"}
    kf, ref = _mirror(w, N, **kw), _mirror(w, N, **kw)
    zs = {bank: [bank.x.view(-1)[:2 * N].view(N, 2)] * 4 if case == "z_in_x" else _zbufs(w, 4) for bank in (kf, ref)}

    def steps(bank):
        for z in zs[bank]:
            bank.predict(); bank.update(z, **upd)
    _not_fused(kf, ref, w, lambda: steps(kf), lambda: steps(ref),
               refusal=b"bke_kf_steps_packed: a z overlaps x or P" if case == "z_in_x" else None)


def test_no_filter_of_a_long_ring_reads_a_refilled_stage():
    """Every CTA walks some forty tiles and refills each stage right after the barrier that follows the
    loads of x, P, the model words and all 8 measurements: a read of the stage after that barrier would pick
    up rows of a later tile.  Every filter of the replayed ring equals eager stepping."""
    import torch
    N = (1 << 21) + 77
    w = _workload(N)
    kf, ref = _mirror(w, N), _mirror(w, N)
    zs = _zbufs(w, 8)

    def steps(bank=kf):
        for z in zs:
            bank.predict(); bank.update(z)
    graph = kf.capture(steps)
    assert (graph.launches, graph.fused_steps) == (1, 8)
    _replays_equal_eager(kf, graph, ref, lambda: steps(ref), w, replays=2)
