"""The gated bank resampler without a GPU: NumPy's pairwise sum restated, the golden file against the oracle
loop and its draw order, argument checks and no CPU fallback."""
import numpy as np
import pytest

from oracle import resample as ors
import resample_bank_gated_oracle as rgo


def _lengths():
    near = [m + d for m in range(128, 4097, 128) for d in (-9, -8, -1, 0, 1, 7, 8)]
    return sorted(set(list(range(1, 301)) + near + [10007, 65536, 100003]))


def test_pairwise_sum_is_numpys_sum():
    rng = np.random.default_rng(1)
    for M in _lengths():
        a = rng.random(M) * 10.0 ** rng.uniform(-10, 0, M)
        s = np.sum(a)
        assert rgo.np_pairwise_sum(a) == s, M
        sq = np.square(a / s)
        assert rgo.np_pairwise_sum(sq) == np.sum(sq), M


def test_pairwise_sum_special_values_and_rows():
    rng = np.random.default_rng(2)
    for M in (3, 8, 130, 1000):
        r = np.full(M, -0.0)
        assert rgo.np_pairwise_sum(r) == 0.0 and not np.signbit(rgo.np_pairwise_sum(r)) and not np.signbit(np.sum(r))
        for v in (np.nan, np.inf, -np.inf, 5e-324, -1e308):
            r = rng.random(M)
            r[M // 2] = v
            a, b = rgo.np_pairwise_sum(r), np.sum(r)
            assert (np.isnan(a) and np.isnan(b)) or a == b, (M, v)
        r = rng.standard_normal(M) * 1e15
        assert rgo.np_pairwise_sum(r) == np.sum(r), M          # cancellation: the order shows
    A = rng.random((7, 1001)) * 10.0 ** rng.uniform(-8, 8, (7, 1001))
    assert np.array_equal(np.sum(A, axis=1), [rgo.np_pairwise_sum(row) for row in A])


def test_golden_is_the_oracle_loop_with_banked_draws(golden):
    """Seeded, the resampled sets draw random() (random(M)) in row order; one draw of random(n_res)
    (random((n_res, M))) gives the same values, and the stream is where the loop leaves it."""
    g = golden("resample_bank_gated")
    for (k, B, M, seed, sys_fail, str_fail) in g["meta"]:
        w, p = g["w%d" % k], g["p%d" % k]
        for kind, fail in (("sys", sys_fail), ("str", str_fail)):
            method = "systematic" if kind == "sys" else "stratified"
            mask = g["%s_mask%d" % (kind, k)]
            n_res = int(mask.sum())
            np.random.seed(seed)
            draws = np.random.random(n_res) if kind == "sys" else np.random.random((n_res, M))
            after = np.random.random()
            o = rgo.resample_if_degenerate_loop(w, p, draws, method=method)
            assert o["n_draws"] == n_res
            assert np.array_equal(o["resampled"], mask), (kind, k)
            assert np.array_equal(o["neff"], g["%s_neff%d" % (kind, k)], equal_nan=True), (kind, k)
            assert np.array_equal(o["weights"], g["%s_w%d" % (kind, k)], equal_nan=True), (kind, k)
            assert np.array_equal(o["particles"], g["%s_p%d" % (kind, k)]), (kind, k)
            ok = mask.copy()
            ok[o["failed"]] = False
            assert np.array_equal(o["indexes"][ok], g["%s_idx%d" % (kind, k)][ok]), (kind, k)
            assert o["failed"] == ([] if fail < 0 else [fail]), (kind, k)
            if fail < 0:
                assert after == g["%s_next%d" % (kind, k)], (kind, k)


def test_golden_covers_the_gate_and_special_rows(golden):
    g = golden("resample_bank_gated")
    meta = g["meta"]
    assert (meta[:, 4] >= 0).any() and (meta[:, 5] >= 0).any()
    neff = g["sys_neff2"]
    M = 128
    assert (neff == M / 2).any() and (neff < M / 2).any() and (neff > M / 2).any() and np.isnan(neff).any()
    assert (g["sys_mask2"] == (neff < M / 2)).all()
    w = g["w2"]
    assert (np.signbit(w) & (w == 0)).any()
    sums = w.sum(axis=1)
    assert np.isclose(sums, 2.0).any() and ((sums > 0) & (sums < 1e-299)).any()
    k = meta[meta[:, 4] >= 0][0][0]
    wf = g["w%d" % k][meta[k][4]]
    assert np.cumsum(wf / np.sum(wf))[-1] < 1


def _args(L, **kw):
    lib = L.load()
    a = L.ResampleBankGatedArgs()
    fake = 1 << 20                                   # never dereferenced: every call below fails before a launch
    a.n_sets, a.n_particles = 4, 8
    a.weights = a.u = a.particles = a.indexes = a.neff = a.resampled = a.status = a.workspace = fake
    a.particle_bytes = 16
    a.threshold = 4.0
    a.workspace_bytes = int(lib.bke_resample_bank_gated_workspace_bytes(4))
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw,msg", [
    (dict(n_sets=-1), b"must be >= 0"), (dict(n_particles=-3), b"must be >= 0"),
    (dict(n_particles=1 << 31), b"2^31"), (dict(n_sets=1 << 31), b"2^31"),
    (dict(uniforms=1 << 20), b"exactly one of u"), (dict(u=None), b"exactly one of u"),
    (dict(weights=None), b"non-NULL"), (dict(neff=None), b"non-NULL"), (dict(particles=None), b"non-NULL"),
    (dict(particle_bytes=0), b"particle_bytes"),
    (dict(workspace_bytes=16 + 4 * 3), b"workspace too small"), (dict(workspace=None), b"workspace"),
    (dict(workspace=(1 << 20) + 2), b"aligned")])
def test_gated_validates_arguments(kw, msg):
    from filterpy_b200 import _lib as L
    lib = L.load()
    assert lib.bke_resample_bank_gated(_args(L, **kw), None) == L.BKE_ERR_BAD_ARG
    assert msg in lib.bke_last_error()
    for fn in (lib.bke_resample_bank_gated, lib.bke_resample_bank_gated_stats, lib.bke_resample_bank_gated_apply):
        assert fn(None, None) == L.BKE_ERR_BAD_ARG


def test_workspace_bytes_and_empty_banks():
    from filterpy_b200 import _lib as L
    lib = L.load()
    assert lib.bke_resample_bank_gated_workspace_bytes(0) == 0
    assert lib.bke_resample_bank_gated_workspace_bytes(1000) == 16 + 4 * 1000
    for B, M in ((0, 8), (4, 0), (0, 0)):
        a = _args(L, n_sets=B, n_particles=M, weights=None, particles=None, workspace=None, workspace_bytes=0)
        for fn in (lib.bke_resample_bank_gated, lib.bke_resample_bank_gated_stats, lib.bke_resample_bank_gated_apply):
            assert fn(a, None) == L.BKE_OK


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from filterpy_b200 import _lib as L
    from filterpy_b200.monte_carlo import (systematic_resample_bank_if_degenerate,
                                           stratified_resample_bank_if_degenerate)
    lib = L.load()
    assert lib.bke_resample_bank_gated(_args(L), None) == L.BKE_ERR_CUDA
    assert lib.bke_resample_bank_gated_stats(_args(L), None) == L.BKE_ERR_CUDA
    w = np.full((3, 4), 0.25)
    p = np.zeros((3, 4, 2), np.float32)
    for fn in (systematic_resample_bank_if_degenerate, stratified_resample_bank_if_degenerate):
        with pytest.raises(L.BkeError):
            fn(w, p)
    assert np.array_equal(w, np.full((3, 4), 0.25))
    assert ors.systematic_resample_loop(np.full(4, 0.25), 0.5).tolist() == [0, 1, 2, 3]
