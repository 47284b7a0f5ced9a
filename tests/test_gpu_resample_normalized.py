"""ResamplePlan.normalized (bke_resample_normalized: the multi-pass pipeline of csrc/resample.cu with every
weight divided by S where it is read): the indexes of systematic_resample(w / S) (stratified_resample with
uniforms), S the engine's sum of the weights, bit for bit; and weights_out == w / S."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U_SYS = 0.37454011884736254
SIZES = (1, 2, 15, 16, 17, 31, 33, 255, 2047, 4095, 4096, 4097, 8191, 8193, 65537, 300007)
KINDS = ("heavy", "uniform", "zeros", "degenerate", "dyadic")


def _expected(wn, positions):
    """The reference's indexes for the normalised weights and the number of positions at or beyond the
    last cumulative sum (where the reference raises IndexError; the engine writes the last particle
    there and reports the count in info[0])."""
    from oracle import resample as ors
    try:
        return ors.resample_vec(wn, positions), 0
    except IndexError:
        idx = np.searchsorted(np.cumsum(wn), positions, side="right")
        over = int((idx >= len(wn)).sum())
        return np.minimum(idx, len(wn) - 1).astype("i"), over


def _run(w, u=None, U=None, offset=0, with_wout=True):
    """One normalized call on a copy of w that starts `offset` doubles into its device buffer."""
    import torch
    from filterpy_b200.monte_carlo import ResamplePlan
    n = len(w)
    buf = torch.zeros(n + 2, dtype=torch.float64, device="cuda")
    wd = buf[offset:offset + n]
    wd.copy_(torch.from_numpy(w))
    plan = ResamplePlan(n)
    plan.indexes.fill_(-7)
    wout = torch.full((n,), -1.0, dtype=torch.float64, device="cuda")
    Ud = torch.from_numpy(U).cuda() if U is not None else None
    idx, S = plan.normalized(wd, u=u, uniforms=Ud, weights_out=wout if with_wout else None)
    return idx.cpu().numpy(), float(S.item()), wout.cpu().numpy(), plan.info(), float(plan.cumsum_last.item())


def _check(w, u=None, U=None, offset=0, with_wout=True):
    """Checks one call and returns its info."""
    from oracle import resample as ors
    n = len(w)
    idx, S, wout, info, clast = _run(w, u=u, U=U, offset=offset, with_wout=with_wout)
    wn = w / S
    if with_wout:
        assert np.array_equal(wout, wn), "weights_out != w / S"
    else:
        assert (wout == -1.0).all(), "a buffer that was not passed was written"
    pos = ors.positions_stratified(n, U) if U is not None else ors.positions_systematic(n, u)
    want, over = _expected(wn, pos)
    bad = np.flatnonzero(idx != want)[:4]
    assert len(bad) == 0, ("indexes differ at", bad.tolist(), info.tolist())
    assert info[0] == over and info[1] == 0, info.tolist()
    assert clast == np.cumsum(wn)[-1]
    return info


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", SIZES)
def test_systematic_sizes_and_kinds(n, kind):
    from filterpy_b200.common import workloads as wl
    _check(wl.resample_weights(n, kind, seed=n % 997), u=U_SYS)


@pytest.mark.parametrize("offset", [1])
def test_unaligned_weights(offset):
    """weights not 16-byte aligned: the tiles are staged without TMA"""
    from filterpy_b200.common import workloads as wl
    _check(wl.resample_weights(100003, "heavy", seed=3), u=0.25, offset=offset)


@pytest.mark.parametrize("u", [0.0, 0.9999999999])
def test_u_at_the_ends(u):
    from filterpy_b200.common import workloads as wl
    _check(wl.resample_weights(100003, "heavy", seed=3), u=u)


def _hard_sets():
    n = 1 << 18
    rng = np.random.default_rng(0)
    w = rng.random(n); w[: n // 2] *= 1e-3; w[1000] = 50.0
    yield "skewed", w                                  # windows overflow, long runs
    yield "ties", rng.integers(0, 8, n) * 2.0 ** -55 + rng.integers(0, 3, n) * 2.0 ** -20
    yield "leading_zeros", np.concatenate([np.zeros(n // 3), rng.random(n - n // 3)])
    yield "30_decades", 10.0 ** rng.uniform(-30, 0, n)


@pytest.mark.parametrize("name", ["skewed", "ties", "leading_zeros", "30_decades"])
def test_hard_weight_sets(name):
    w = dict(_hard_sets())[name]
    _check(w, u=0.123)


@pytest.mark.parametrize("n", [1000, 4097, 300007])
def test_stratified(n):
    from filterpy_b200.common import workloads as wl
    _check(wl.resample_weights(n, "heavy", seed=7), U=np.random.default_rng(n).random(n))


def test_negative_weight_takes_the_literal_fallback():
    from oracle import resample as ors
    rng = np.random.default_rng(0)
    w = rng.random(3000); w[100] = -0.2
    idx, S, wout, info, _ = _run(w, u=0.4)
    wn = w / S
    assert info[1] == 1, info.tolist()
    assert np.array_equal(wout, wn)
    assert np.array_equal(idx, ors.resample_loop(wn, ors.positions_systematic(3000, 0.4)))


TILE = 4096      # particles per tile of the pipeline (resample_common.cuh)


@pytest.mark.parametrize("stratified", [False, True])
def test_cluster_chain(stratified):
    """at least 2048 tiles: the exact chain over the tiles runs as a thread-block cluster"""
    from filterpy_b200.common import workloads as wl
    n = (1 << 23) + 1
    assert -(-n // TILE) >= 2048
    U = np.random.default_rng(5).random(n) if stratified else None
    _check(wl.resample_weights(n, "heavy", seed=11), u=None if stratified else U_SYS, U=U)


def test_sequential_tile():
    """A tile in which every add starts exactly on a binade boundary (w / S = 0.5 before it, each of its
    weights far below half an ulp there) is walked element by element (info[5] counts such tiles)."""
    w = np.concatenate([np.full(TILE, 2.0 ** -12), np.full(TILE, 2.0 ** -80), np.full(TILE, 2.0 ** -12)])
    info = _check(w, u=0.3)
    assert info[5] > 0, info.tolist()


def test_without_weights_out():
    from filterpy_b200.common import workloads as wl
    _check(wl.resample_weights(300007, "heavy", seed=5), u=U_SYS, with_wout=False)
