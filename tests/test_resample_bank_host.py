"""Bank resampling without a GPU: the golden's draw order, argument checks and no CPU fallback."""
import numpy as np
import pytest

from oracle import resample as ors


def test_golden_is_the_loop_over_rows_with_banked_draws(golden):
    """A seeded bank draws u = random(B) (stratified: U = random((B, M))) and resamples row b with u[b]:
    that is the reference's loop over the rows, which draws random() (random(M)) once per row, and it
    leaves the global stream where the loop leaves it."""
    g = golden("resample_bank")
    for (k, B, M, seed, sys_fail, str_fail) in g["meta"]:
        w = g["w%d" % k]
        for kind, fail, loop_fn in (("sys", sys_fail, ors.systematic_resample_loop),
                                    ("str", str_fail, ors.stratified_resample_loop)):
            np.random.seed(seed)
            draws = np.random.random(B) if kind == "sys" else np.random.random((B, M))
            after = np.random.random()
            for b in range(B):
                if b == fail:
                    with pytest.raises(IndexError):
                        loop_fn(w[b], draws[b])
                    break
                assert np.array_equal(loop_fn(w[b], draws[b]), g["%s%d" % (kind, k)][b]), (kind, k, b)
            if fail < 0:
                assert after == g["%s_next%d" % (kind, k)], (kind, k)


def test_golden_covers_the_weight_kinds_and_a_failing_row(golden):
    g = golden("resample_bank")
    meta = g["meta"]
    assert (meta[:, 4] >= 0).any() and (meta[:, 5] >= 0).any()
    assert any(B >= 5 for B in meta[:, 1])               # rows run through every kind of workloads.resample_weights
    w = g["w%d" % meta[meta[:, 4] >= 0][0][0]]
    assert (w.sum(axis=1) < 1 - 1e-6).any()


def _args(L, **kw):
    a = L.ResampleBankArgs()
    fake = 1 << 20                                   # never dereferenced: every call below fails before a launch
    a.n_sets, a.n_particles = 4, 8
    a.weights = a.u = a.indexes = fake
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw,msg", [
    (dict(n_sets=-1), b"must be >= 0"), (dict(n_particles=-3), b"must be >= 0"),
    (dict(n_particles=1 << 31), b"2^31"),
    (dict(uniforms=1 << 20), b"exactly one of u"), (dict(u=None), b"exactly one of u"),
    (dict(weights=None), b"non-NULL"), (dict(indexes=None), b"non-NULL")])
def test_resample_bank_validates_arguments(kw, msg):
    from filterpy_b200 import _lib as L
    lib = L.load()
    assert lib.bke_resample_bank(_args(L, **kw), None) == L.BKE_ERR_BAD_ARG
    assert msg in lib.bke_last_error()
    assert lib.bke_resample_bank(None, None) == L.BKE_ERR_BAD_ARG


def test_empty_banks_do_nothing():
    from filterpy_b200 import _lib as L
    lib = L.load()
    for B, M in ((0, 8), (4, 0), (0, 0)):
        assert lib.bke_resample_bank(_args(L, n_sets=B, n_particles=M, weights=None, indexes=None), None) == L.BKE_OK
    assert lib.bke_gather_rows_bank(0, 8, 16, None, None, 0, None, None, None) == L.BKE_OK


def test_gather_rows_bank_validates_arguments():
    from filterpy_b200 import _lib as L
    lib = L.load()
    fake = 1 << 20
    assert lib.bke_gather_rows_bank(-1, 8, 16, fake, fake, 0, fake + 4096, None, None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_gather_rows_bank(2, -8, 16, fake, fake, 0, fake + 4096, None, None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_gather_rows_bank(2, 8, 0, fake, fake, 0, fake + 4096, None, None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_gather_rows_bank(2, 8, 16, None, fake, 0, fake + 4096, None, None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_gather_rows_bank(2, 8, 16, fake, fake, 0, fake, None, None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_gather_rows_bank(1 << 40, 1 << 40, 16, fake, fake, 0, fake + 4096, None, None) == L.BKE_ERR_BAD_ARG


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from filterpy_b200 import _lib as L
    from filterpy_b200.monte_carlo import (systematic_resample_bank, stratified_resample_bank, gather_particles_bank,
                                           BankResamplePlan)
    lib = L.load()
    assert lib.bke_resample_bank(_args(L), None) == L.BKE_ERR_CUDA
    fake = 1 << 20
    assert lib.bke_gather_rows_bank(2, 8, 16, fake, fake, 0, fake + 4096, None, None) == L.BKE_ERR_CUDA
    w = np.full((3, 4), 0.25)
    for fn in (systematic_resample_bank, stratified_resample_bank):
        with pytest.raises(L.BkeError):
            fn(w)
    with pytest.raises(L.BkeError):
        gather_particles_bank(np.zeros((3, 4, 2)), np.zeros((3, 4), np.int32))
    with pytest.raises(L.BkeError):
        BankResamplePlan(3, 4)
