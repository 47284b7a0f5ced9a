"""The block path of the fused ring's pattern instance: a warp whose filters all enter with zeros in the 8 cross-axis
words of P (P02 P03 P12 P13 and their mirrors) steps the two axis blocks of the constant-velocity 2-D model and
carries each cross word as a signed zero.  It is bit for bit the dense ring: through every sign of those zeros,
in-block signed zeros and underflow, negative variances, warps in which one filter has a nonzero or non-finite
cross word (the warp runs the pattern path) and filters with non-finite words (run again on the dense arithmetic)."""
import numpy as np
import pytest

from test_gpu_kf_ring import STEPS, _workload
from test_gpu_kf_ring_pattern import _equals_separate_steps

pytestmark = pytest.mark.gpu

CROSS = [(0, 2), (0, 3), (1, 2), (1, 3), (2, 0), (3, 0), (2, 1), (3, 1)]
IN_BLOCK = [(0, 0), (0, 1), (1, 0), (1, 1), (2, 2), (2, 3), (3, 2), (3, 3)]


@pytest.mark.parametrize("K", range(1, STEPS + 1))
@pytest.mark.parametrize("N", [127, 129, (1 << 16) + 3])
def test_block_ring_equals_separate_steps_bit_for_bit(N, K):
    # kf_bank_cv2d: P0 diagonal, so every warp runs the two blocks
    w = _workload(N)
    assert not w["P"][:, [i for i, _ in CROSS], [j for _, j in CROSS]].any()
    _equals_separate_steps(w, N, K)


def _sign_bank(N):
    """Filter f holds the cross-word signs f mod 256 (bit c: CROSS[c] is -0, else +0).  Its in-block words are
    drawn from signed zeros, 1e-30-scale and subnormal values, with variances that may be -0 or negative; x, z
    and the per-filter dt, q, r likewise, dt small enough that dt x1 underflows.  Negative variances make S, SI
    and so K and K R negative, which is where the signs of the cross words reach x and P."""
    rng = np.random.default_rng(29)
    w = _workload(N)
    f32 = np.float32
    pick = lambda vals, shape: np.asarray(vals, dtype=f32)[rng.integers(0, len(vals), shape)]
    tiny = [0.0, -0.0, 1e-30, -1e-30, 1e-40, -1e-40, 1e-45, -1e-45]
    dt = pick([1e-30, -1e-30, 1e-38, 1e-45, -1e-45, 0.1, -0.0], N)
    w["F"][:, 0, 1] = dt
    w["F"][:, 2, 3] = dt
    w["x"] = pick([0.0, -0.0, 1e-20, -1e-20, 1.0, -1.5] + tiny, (N, 4))
    P = np.zeros((N, 4, 4), dtype=f32)
    for i, j in IN_BLOCK:
        P[:, i, j] = pick(tiny + [0.25, -0.125], N) if i != j else pick([1.0, 2.5, -7.0, 0.0, -0.0, 1e-30], N)
    signs = np.arange(N) % 256
    for c, (i, j) in enumerate(CROSS):
        P[:, i, j] = np.where((signs >> c) & 1, f32(-0.0), f32(0.0))
    w["P"] = P
    for i0 in (0, 2):                                        # Q stays symmetric, its cross words +0
        for i, j in ((i0, i0), (i0, i0 + 1), (i0 + 1, i0 + 1)):
            w["Q"][:, i, j] = w["Q"][:, j, i] = pick([0.0, -0.0, 1e-3, -1e-3, 1e-30], N)
    for a in (0, 1):
        w["R"][:, a, a] = pick([0.5, -0.75, 0.0, -0.0, 1e-30], N)
    w["zs"] = np.ascontiguousarray(pick([0.0, -0.0, 1e-30, -1e-30, 0.5, -2.0], (STEPS, N, 2)))
    return w


@pytest.mark.parametrize("K", [1, 2, 3, 5, 8])
def test_every_sign_of_the_cross_words_bit_for_bit(K):
    N = (1 << 16) + 3
    w = _sign_bank(N)
    assert (np.signbit(w["P"][:, 0, 2]) != np.signbit(w["P"][:, 2, 0])).any()
    _equals_separate_steps(w, N, K)


@pytest.mark.parametrize("word", [1e-30, -1e-45, np.nan])
def test_a_warp_with_one_nonzero_cross_word_runs_the_pattern_path_bit_for_bit(word):
    N = (1 << 16) + 3
    w = _sign_bank(N)
    lanes = np.arange(0, N, 32) + (np.arange(0, N, 32) // 32) % 32      # one lane per warp, a different one each
    lanes = lanes[lanes < N]
    i, j = CROSS[3]
    w["P"][lanes, i, j] = np.float32(word)
    for K in (1, 4, 8):
        _equals_separate_steps(w, N, K)


def test_filters_with_non_finite_words_and_their_neighbours_bit_for_bit():
    N = (1 << 16) + 3
    inf, nan = np.float32(np.inf), np.float32(np.nan)
    for w in (_workload(N), _sign_bank(N)):
        w["x"][10, 2] = inf
        w["x"][N - 1, 0] = nan
        w["P"][200, 1, 3] = nan                                  # a cross word: the warp runs the pattern path
        w["P"][201 + 32, 0, 0] = -inf                            # in-block words: the warps stay on the blocks
        w["P"][202 + 64, 2, 3] = nan
        w["zs"][2, 500, 1] = -inf
        w["zs"][0, 501, 0] = nan
        w["Q"][300, 0, 0] = inf                                  # a varying model word
        w["R"][301, 1, 1] = nan
        w["x"][400, :] = np.float32(3e38)                       # finite, overflows inside the ring
        for K in (1, 3, 8):
            _equals_separate_steps(w, N, K)
