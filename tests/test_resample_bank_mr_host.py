"""Multinomial / residual bank resampling without a GPU: the oracles against the reference's golden loop,
argument checks, no spills in the new kernels, and no CPU fallback."""
import os
import subprocess

import numpy as np
import pytest

from oracle import resample as ors
import resample_bank_mr_oracle as mro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _draw_loop(g, k, seed, kind, fail):
    """The reference loop's uniforms, drawn as the bank mirrors draw them: (per-row uniforms, next draw)."""
    w = g["w%d" % k]
    B, M = w.shape
    np.random.seed(seed)
    if kind == "mul":
        U = np.random.random((B, M))
        return [U[b] for b in range(B)], np.random.random()
    _, kk, _ = mro.residual_prepare_bank(w)
    rows = B if fail < 0 else fail
    flat = np.random.random(int((M - kk[:rows]).sum()))
    off = np.concatenate([[0], np.cumsum(M - kk[:rows])])
    return [flat[off[b]:off[b + 1]] for b in range(rows)], np.random.random()


def test_oracles_reproduce_golden(golden):
    """binsearch_left (the restated NumPy bisection) and the vectorised NumPy oracle both give the reference
    loop's indexes, failing row and next draw."""
    g = golden("resample_bank_mr")
    for (k, B, M, seed, mul_fail, res_fail) in g["meta"]:
        w = g["w%d" % k]
        assert mul_fail < 0
        Us, after = _draw_loop(g, k, seed, "mul", -1)
        assert after == g["mul_next%d" % k], k
        with np.errstate(all="ignore"):
            for b in range(B):
                c = np.cumsum(w[b]); c[-1] = 1.
                assert np.array_equal(ors.binsearch_left(c, Us[b]), g["mul%d" % k][b]), (k, b)
        assert np.array_equal(mro.multinomial_bank(w, np.stack(Us)), g["mul%d" % k]), k
        Us, after = _draw_loop(g, k, seed, "res", res_fail)
        idx, kk, bad = mro.residual_bank(w, np.stack([np.pad(u, (0, M - len(u))) for u in Us] +
                                                      [np.zeros(M)] * (B - len(Us))))
        if res_fail >= 0:
            assert bad[0] == res_fail, k
            with pytest.raises(IndexError), np.errstate(all="ignore"):
                ors.residual_prepare(w[res_fail])
        else:
            assert after == g["res_next%d" % k], k
        for b in range(len(Us)):
            with np.errstate(all="ignore"):
                assert np.array_equal(ors.residual_resample_vec(w[b], Us[b]), g["res%d" % k][b]), (k, b)
            assert np.array_equal(idx[b], g["res%d" % k][b]), (k, b)


def test_golden_covers_special_rows_and_failures(golden):
    g = golden("resample_bank_mr")
    meta = g["meta"]
    assert (meta[:, 5] >= 0).sum() >= 2 and (meta[:, 4] < 0).all()
    ws = [g["w%d" % k] for k in meta[:, 0]]
    assert any(np.isnan(w).any() for w in ws) and any(np.isposinf(w).any() for w in ws)
    assert any(np.isneginf(w).any() for w in ws) and any((w < 0).any() for w in ws)
    with np.errstate(all="ignore"):
        # a row whose cumulative sum passes 1 before its last element (c[M-2] > 1)
        assert any((np.cumsum(w, axis=1)[:, -2] > 1).any() for w in ws if w.shape[1] > 1)
        # residual's cumulative sum is not monotone on ordinary rows
        _, _, c = mro.residual_prepare_bank(g["w3"])
        assert (np.diff(c[:, :-1], axis=1) < 0).any()


FAKE = 1 << 20          # never dereferenced: every refused call below fails before a launch


def _margs(L, **kw):
    a = L.MultinomialResampleBankArgs()
    a.n_sets, a.n_particles = 4, 8
    a.weights = a.uniforms = a.indexes = a.status = a.workspace = FAKE
    a.workspace_bytes = 4 * 8 * 8
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _rargs(L, **kw):
    a = L.ResidualResampleBankArgs()
    a.n_sets, a.n_particles = 4, 8
    a.weights = a.uniforms = a.indexes = a.n_copies = a.status = a.workspace = FAKE
    a.workspace_bytes = 4 * 8 * 8
    for k, v in kw.items():
        setattr(a, k, v)
    return a


COMMON = [(dict(n_sets=-1), b"must be >= 0"), (dict(n_particles=-3), b"must be >= 0"),
          (dict(n_particles=1 << 31), b"2^31"), (dict(workspace=None), b"workspace"),
          (dict(workspace=FAKE + 4), b"aligned"), (dict(workspace_bytes=4 * 8 * 8 - 1), b"too small"),
          (dict(n_sets=1 << 62, n_particles=1 << 20), b"too large"), (dict(indexes=None), b"non-NULL"),
          (dict(status=None), b"non-NULL")]


@pytest.mark.parametrize("kw,msg", COMMON + [(dict(weights=None), b"non-NULL"), (dict(uniforms=None), b"non-NULL")])
def test_multinomial_bank_validates_arguments(kw, msg):
    from filterpy_b200 import _lib as L
    lib = L.load()
    assert lib.bke_multinomial_resample_bank(_margs(L, **kw), None) == L.BKE_ERR_BAD_ARG
    assert msg in lib.bke_last_error()
    assert lib.bke_multinomial_resample_bank(None, None) == L.BKE_ERR_BAD_ARG


@pytest.mark.parametrize("kw,msg", COMMON + [(dict(n_copies=None), b"non-NULL")])
def test_residual_bank_validates_arguments(kw, msg):
    from filterpy_b200 import _lib as L
    lib = L.load()
    for fn in (lib.bke_residual_resample_bank_prepare, lib.bke_residual_resample_bank_search):
        assert fn(_rargs(L, **kw), None) == L.BKE_ERR_BAD_ARG
        assert msg in lib.bke_last_error()
        assert fn(None, None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_residual_resample_bank_prepare(_rargs(L, weights=None), None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_residual_resample_bank_search(_rargs(L, uniforms=None), None) == L.BKE_ERR_BAD_ARG


def test_workspace_sizes_and_empty_banks():
    from filterpy_b200 import _lib as L
    lib = L.load()
    for fn in (lib.bke_multinomial_resample_bank_workspace_bytes, lib.bke_residual_resample_bank_workspace_bytes):
        assert fn(3, 7) == 3 * 7 * 8 and fn(0, 7) == 0 and fn(3, 0) == 0 and fn(-1, 4) == 0
    none = dict(weights=None, uniforms=None, indexes=None, status=None, workspace=None, workspace_bytes=0)
    for B, M in ((0, 8), (4, 0), (0, 0)):
        assert lib.bke_multinomial_resample_bank(_margs(L, n_sets=B, n_particles=M, **none), None) == L.BKE_OK
        for fn in (lib.bke_residual_resample_bank_prepare, lib.bke_residual_resample_bank_search):
            assert fn(_rargs(L, n_sets=B, n_particles=M, n_copies=None, **none), None) == L.BKE_OK


def test_new_kernels_do_not_spill(tmp_path):
    from filterpy_b200 import _build
    cmd = [_build._nvcc()] + _build.NVCC_FLAGS + ["-I", os.path.join(ROOT, "include"), "-Xptxas", "-v", "-c",
                                                   os.path.join(_build.CSRC, "resample_bank.cu"),
                                                   "-o", str(tmp_path / "rb.o")]
    if not os.path.exists(cmd[0]):
        pytest.skip("nvcc not available")
    log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    kernels = {}
    name = None
    for ln in log.splitlines():
        if "Compiling entry function" in ln:
            name = ln.split("'")[1]
        elif name and "spill" in ln:
            kernels[name] = ln
    new = {n: ln for n, ln in kernels.items() if "k_prepare_bank" in n or "k_search_bank" in n}
    assert len(new) == 4, kernels
    for n, ln in new.items():
        assert "0 bytes spill stores, 0 bytes spill loads" in ln, (n, ln)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from filterpy_b200 import _lib as L
    from filterpy_b200.monte_carlo import multinomial_resample_bank, residual_resample_bank, BankResamplePlan
    lib = L.load()
    assert lib.bke_multinomial_resample_bank(_margs(L), None) == L.BKE_ERR_CUDA
    assert lib.bke_residual_resample_bank_prepare(_rargs(L), None) == L.BKE_ERR_CUDA
    assert lib.bke_residual_resample_bank_search(_rargs(L), None) == L.BKE_ERR_CUDA
    w = np.full((3, 4), 0.25)
    for fn in (multinomial_resample_bank, residual_resample_bank):
        with pytest.raises(L.BkeError):
            fn(w)
    with pytest.raises(L.BkeError):
        BankResamplePlan(3, 4)
