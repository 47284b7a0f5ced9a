"""The fused ring's pattern instance (kf42_f32_kernel<..., Cv2dPattern>) takes the constant-velocity 2-D model's
structural words, +0 and 1 in every filter, as constants and drops or folds their products.  It runs exactly when
a bank holds all of them with those bits, and it is bit for bit the dense ring: through signed zeros, kept
products that underflow to -0 ahead of dropped ones, and filters with non-finite words, which it runs again on the
dense arithmetic."""
import numpy as np
import pytest

from test_gpu_kf_ring import STEPS, _CBank, _same_bits, _workload

pytestmark = pytest.mark.gpu


def _ring_kernels(b, zs):
    """(rc, x, P, names of the kf42_f32_kernel launches) of one bke_kf_steps_packed over zs."""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rc, x, P = b.ring(zs)
    return rc, x, P, [e.name for e in prof.events() if "kf42_f32_kernel" in e.name]


def _equals_separate_steps(w, N, K):
    b = _CBank(w, N)
    rc, x, P = b.ring(b.zs[:K])
    assert rc == 0, b.lib.bke_last_error()
    xs, Ps = b.stepwise(b.zs[:K])
    _same_bits(x, xs, "x"); _same_bits(P, Ps, "P")
    return b, x, P


@pytest.mark.parametrize("K", range(1, STEPS + 1))
@pytest.mark.parametrize("N", [127, 129, (1 << 16) + 3])
def test_pattern_ring_equals_separate_steps_bit_for_bit(N, K):
    _equals_separate_steps(_workload(N), N, K)


def test_the_pattern_instance_runs_exactly_on_banks_with_its_structural_words():
    N = 1001
    w = _workload(N)
    b = _CBank(w, N)
    rc, x, P, names = _ring_kernels(b, b.zs[:4])
    assert rc == 0 and len(names) == 1 and "Cv2dPattern" in names[0], names
    # F[0][2] is -0.0 in every filter (shared, but not the bits of +0), or differs in one filter (it varies)
    minus = {k: v.copy() for k, v in w.items()}
    minus["F"][:, 0, 2] = -0.0
    one = {k: v.copy() for k, v in w.items()}
    one["F"][7, 0, 2] = np.float32(1e-3)
    for what, wk in (("-0.0", minus), ("one filter", one)):
        b = _CBank(wk, N)
        rc, x, P, names = _ring_kernels(b, b.zs[:4])
        assert rc == 0, b.lib.bke_last_error()
        assert len(names) == 1 and "Cv2dPattern" not in names[0] and "NoPattern" in names[0], (what, names)
        xs, Ps = b.stepwise(b.zs[:4])
        _same_bits(x, xs, what + " x"); _same_bits(P, Ps, what + " P")


def _signed_zero_bank(N):
    """The cv2d pattern with +-0 entries in x, P and z, subnormal and 1e-30-scale entries of P off its diagonal,
    and dt so small that dt x1 underflows: kept products round to -0 ahead of dropped ones (x0 = -0 and dt x1
    underflowing negative, followed by the dropped 0 x2 and 0 x3)."""
    rng = np.random.default_rng(17)
    w = _workload(N)
    f32 = np.float32
    pick = lambda vals, shape: np.asarray(vals, dtype=f32)[rng.integers(0, len(vals), shape)]
    tiny = [0.0, -0.0, 1e-30, -1e-30, 1e-40, -1e-40, 1e-45, -1e-45]
    dt = pick([1e-30, -1e-30, 1e-38, 1e-45, 0.1], N)
    w["F"][:, 0, 1] = dt
    w["F"][:, 2, 3] = dt
    w["x"] = pick([0.0, -0.0, 1e-20, -1e-20, 1.0, -1.5] + tiny, (N, 4))
    P = pick(tiny + [0.25, -0.125], (N, 4, 4))
    P[:, np.arange(4), np.arange(4)] = pick([1.0, 2.5, 7.0], (N, 4))
    w["P"] = np.ascontiguousarray(P)
    w["zs"] = np.ascontiguousarray(pick([0.0, -0.0, 1e-30, -1e-30, 0.5, -2.0], (STEPS, N, 2)))
    return w


@pytest.mark.parametrize("K", [1, 2, 5, 8])
def test_signed_zeros_and_underflow_bit_for_bit(K):
    N = (1 << 16) + 3
    w = _signed_zero_bank(N)
    b, x, P = _equals_separate_steps(w, N, K)
    assert np.isfinite(x.cpu().numpy()).all() and np.isfinite(P.cpu().numpy()).all()


def test_filters_with_non_finite_words_and_their_neighbours_bit_for_bit():
    N = (1 << 16) + 3
    w = _workload(N)
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    w["x"][10, 2] = inf
    w["x"][N - 1, 0] = nan
    w["P"][200, 1, 3] = nan
    w["P"][201, 0, 0] = -inf
    w["zs"][2, 500, 1] = -inf
    w["zs"][0, 501, 0] = nan
    w["Q"][300, 0, 0] = inf                                  # a varying model word
    w["x"][400, :] = np.float32(3e38)                       # finite, overflows inside the ring
    for K in (1, 3, 8):
        b, x, P = _equals_separate_steps(w, N, K)
        assert np.isfinite(x.cpu().numpy()[[9, 11, 199, 202, 499, 502, 299, 301, 401]]).all()
