"""GPU parity for the rows beyond the KF / UKF / systematic resample core: multinomial_resample + exact cumsum + particle
gather (rank 2) and the RTS smoother (rank 3).  Index work is bit-exact; x / P within 1e-6 (fp64)
and 1e-3 (fp32) relative, the tolerances north_star states."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def rel_close(a, b, rtol, atol_scale=1.0):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    scale = max(1.0, float(np.max(np.abs(b)))) if b.size else 1.0
    np.testing.assert_allclose(a, b, rtol=rtol, atol=rtol * scale * atol_scale)


# ------------------------------------------------------------------ exact cumsum / multinomial
def gpu_multinomial(w, U):
    import torch
    from filterpy_b200.monte_carlo import ResamplePlan
    plan = ResamplePlan(len(w))
    wd = torch.from_numpy(np.ascontiguousarray(w)).cuda()
    Ud = torch.from_numpy(np.ascontiguousarray(U)).cuda()
    idx = plan.multinomial(wd, Ud)
    return idx.cpu().numpy(), plan.info()


def test_multinomial_golden_vectors_from_reference(golden):
    g = golden("resample_multinomial")
    for (i, N, seed) in g["meta"]:
        idx, info = gpu_multinomial(g["w%d" % i], g["U%d" % i])
        assert idx.dtype == np.int64
        assert np.array_equal(idx, g["idx%d" % i]), (i, N, info)


@pytest.mark.parametrize("kind", ["heavy", "uniform", "zeros", "degenerate", "random"])
@pytest.mark.parametrize("N", [4095, 4097, 100003, 1 << 20])
def test_exact_cumsum_and_multinomial_vs_oracle(kind, N):
    import torch
    from filterpy_b200.common import workloads as wl
    from filterpy_b200.monte_carlo import ResamplePlan
    from oracle import resample as ors
    w = wl.resample_weights(N, kind, seed=N + 5)
    plan = ResamplePlan(N)
    wd = torch.from_numpy(w).cuda()
    c = plan.cumsum(wd).cpu().numpy()
    info = plan.info()
    assert info[1] == 0, info                                   # no sequential fallback
    assert np.array_equal(c.view(np.int64), np.cumsum(w).view(np.int64))     # bit for bit
    c1 = plan.cumsum(wd, last_one=True).cpu().numpy()
    assert c1[-1] == 1.0 and np.array_equal(c1[:-1], c[:-1])
    U = np.random.default_rng(N).random(N)
    idx, info = gpu_multinomial(w, U)
    ref = ors.multinomial_resample_c(w, U)
    assert np.array_equal(idx, ref)
    # the plain bisection (no bracket table) and keys at / outside the ends give the same answers
    Ud = torch.from_numpy(U).cuda()
    assert np.array_equal(plan.multinomial(wd, Ud, lut=False).cpu().numpy(), ref)
    edge = U.copy()
    edge[:6] = [0.0, np.nextafter(1.0, 0.0), c[0], c[N // 2], np.nextafter(c[N // 2], 1.0), 1e-300]
    got = plan.multinomial(wd, torch.from_numpy(edge).cuda()).cpu().numpy()
    assert np.array_equal(got, ors.multinomial_resample_c(w, edge))


def test_multinomial_public_function_reproduces_reference_rng_stream(golden):
    from filterpy_b200.monte_carlo import multinomial_resample, residual_resample
    g = golden("resample_multinomial")
    for (i, N, seed) in g["meta"]:
        np.random.seed(int(seed))
        got = multinomial_resample(g["w%d" % i])
        assert got.dtype == np.int64 and np.array_equal(got, g["idx%d" % i])


def test_residual_resample_vs_reference_golden(golden):
    """resampling.py:27-76 through the public mirror with the reference's RNG stream: bit-equal int32
    indexes on every golden case (23 of the 35 cumulative sums are not monotone)."""
    from filterpy_b200.monte_carlo import residual_resample
    g = golden("resample_residual")
    for (i, N, seed, k) in g["meta"]:
        np.random.seed(int(seed))
        got = residual_resample(g["w%d" % i])
        assert got.dtype == np.int32 and got.shape == (N,)
        assert np.array_equal(got, g["idx%d" % i]), (i, N)
    # the stream position afterwards is the reference's too: exactly N - k uniforms were drawn
    (i, N, seed, k) = g["meta"][10]
    np.random.seed(int(seed)); residual_resample(g["w%d" % i]); nxt = np.random.random()
    np.random.seed(int(seed)); np.random.random(int(N - k)); assert nxt == np.random.random()
    with pytest.raises(IndexError):
        residual_resample(np.zeros(0))


@pytest.mark.parametrize("kind", ["heavy", "uniform", "zeros", "degenerate"])
def test_residual_resample_large_vs_oracle(kind):
    """2^20 particles: the deterministic copies, sum(residual), the cumulative sum (bit patterns) and the
    bracket-carrying bisection against the oracle / NumPy's searchsorted on the oracle's cumulative sum."""
    import torch
    from filterpy_b200.monte_carlo import residual_resample_with_uniforms
    from filterpy_b200.common import workloads as wl
    from oracle import resample as ors
    N = 1 << 20
    w = wl.resample_weights(N, kind, seed=77)
    with np.errstate(all="ignore"):
        idx0, k, c, s = ors.residual_prepare(w)
    rng = np.random.default_rng(12)
    U = rng.random(N - k)
    got, info = residual_resample_with_uniforms(torch.from_numpy(w).cuda(), lambda m: U[:m])
    got = got.cpu().numpy()
    assert info["k"] == k
    assert info["residual_sum"] == s or (np.isnan(s) and np.isnan(info["residual_sum"]))
    assert np.array_equal(got[:k], idx0[:k])
    assert np.array_equal(got[k:], np.searchsorted(c, U).astype(np.int32))
    assert info["sweeps"] <= 64 and (info["sweeps"] >= 1 or k == N)


def test_residual_cumsum_bits_and_sweep_abi():
    """The C-ABI pieces directly: cumulative_sum bit for bit (incl. the forced last 1.0) and one
    bracket sweep from a deliberately wrong `prev` moves towards NumPy's answer."""
    import torch
    from filterpy_b200 import _lib
    from filterpy_b200._dev import stream_ptr
    from oracle import resample as ors
    lib = _lib.load()
    rng = np.random.default_rng(8)
    for N in [1, 2, 33, 1024, 1025, 5000]:
        w = rng.random(N) ** 5
        w /= w.sum()
        with np.errstate(all="ignore"):
            idx0, k, c, s = ors.residual_prepare(w)
        wd = torch.from_numpy(w).cuda()
        idx = torch.full((N,), -7, dtype=torch.int32, device="cuda")
        cs = torch.empty(N, dtype=torch.float64, device="cuda")
        kd = torch.zeros(1, dtype=torch.int64, device="cuda")
        sd = torch.zeros(1, dtype=torch.float64, device="cuda")
        nb = int(lib.bke_residual_workspace_bytes(N))
        ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
        _lib.check(lib.bke_residual_prepare(N, wd.data_ptr(), idx.data_ptr(), cs.data_ptr(), kd.data_ptr(), sd.data_ptr(),
                                            ws.data_ptr(), nb, stream_ptr(wd.device)))
        assert int(kd.item()) == k
        assert np.array_equal(idx.cpu().numpy()[:k], idx0[:k]) and np.all(idx.cpu().numpy()[k:] == -7)
        assert np.array_equal(cs.cpu().numpy().view(np.int64), c.view(np.int64))      # NaNs included
        m = N - k
        if m == 0:
            continue
        U = rng.random(m)
        ref = np.searchsorted(c, U)
        keys = torch.from_numpy(U).cuda()
        prev = torch.zeros(m, dtype=torch.int64, device="cuda")                       # wrong on purpose
        nxt = torch.empty_like(prev)
        ch = torch.zeros(1, dtype=torch.int32, device="cuda")
        for _ in range(m + 2):
            ch.zero_()
            _lib.check(lib.bke_searchsorted_bracket_sweep(N, cs.data_ptr(), m, keys.data_ptr(), prev.data_ptr(),
                                                          nxt.data_ptr(), None, ch.data_ptr(), stream_ptr(wd.device)))
            prev, nxt = nxt, prev
            if int(ch.item()) == 0:
                break
        assert np.array_equal(prev.cpu().numpy(), ref)


def test_searchsorted_matches_numpy_both_sides():
    import ctypes
    import torch
    from filterpy_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(3)
    a = np.sort(np.round(rng.random(10000), 3))                 # many ties
    keys = np.concatenate([rng.random(5000), a[::7], [-1.0, 2.0, 0.0, 1.0]])
    ad = torch.from_numpy(a).cuda(); kd = torch.from_numpy(keys).cuda()
    out = torch.empty(len(keys), dtype=torch.int64, device="cuda")
    for side, flag in [("left", 0), ("right", 1)]:
        _lib.check(lib.bke_searchsorted(len(a), ad.data_ptr(), len(keys), kd.data_ptr(), flag, out.data_ptr(), None))
        assert np.array_equal(out.cpu().numpy(), np.searchsorted(a, keys, side=side))


# ------------------------------------------------------------------ gather
@pytest.mark.parametrize("shape,dtype", [((1000, 4), np.float64), ((1000, 3), np.float32), ((777,), np.float64),
                                          ((500, 5), np.uint8), ((300, 2, 3), np.float32), ((64, 7), np.int16)])
@pytest.mark.parametrize("idx_dtype", [np.int32, np.int64])
def test_gather_particles_equals_numpy_fancy_indexing(shape, dtype, idx_dtype):
    from filterpy_b200.monte_carlo import gather_particles
    rng = np.random.default_rng(1)
    p = (rng.random(shape) * 100).astype(dtype)
    idx = rng.integers(0, shape[0], size=shape[0] + 13).astype(idx_dtype)
    got = gather_particles(p, idx)
    assert got.dtype == p.dtype and np.array_equal(got, p[idx])


def test_gather_after_resample_roundtrip_and_errors():
    import torch
    from filterpy_b200.monte_carlo import gather_particles, systematic_resample
    rng = np.random.default_rng(2)
    N = 50000
    w = rng.random(N) ** 4; w /= w.sum()
    particles = rng.normal(size=(N, 4))
    np.random.seed(3)
    idx = systematic_resample(w)
    assert np.array_equal(gather_particles(particles, idx), particles[idx])
    # device in, device out; the identity permutation is a copy
    pd = torch.from_numpy(particles).cuda()
    ident = torch.arange(N, dtype=torch.int32, device="cuda")
    assert torch.equal(gather_particles(pd, ident), pd)
    with pytest.raises(IndexError):
        gather_particles(particles, np.array([0, N], dtype=np.int32))
    with pytest.raises(IndexError):
        gather_particles(particles, np.array([-1], dtype=np.int64))


# ------------------------------------------------------------------ RTS smoother
def test_rts_single_filter_golden(golden):
    from filterpy_b200.kalman import KalmanFilter, rts_smoother
    g = golden("rts")
    kf = KalmanFilter(4, 2)
    kf.F, kf.Q = g["c1_F"], g["c1_Q"]
    out = kf.rts_smoother(g["c1_means"], g["c1_covs"])
    for got, key in zip(out, ["c1_x", "c1_P", "c1_K", "c1_Pp"]):
        assert got.shape == g[key].shape
        rel_close(got, g[key], 1e-6)
    # per-epoch models: method (Fs[k+1]) and procedural (Fs[k]) forms
    out = kf.rts_smoother(g["c1_means"], g["c1_covs"], Fs=list(g["tv_Fs"]), Qs=list(g["tv_Qs"]))
    for got, key in zip(out, ["x", "P", "K", "Pp"]):
        rel_close(got, g["tv_method_" + key], 1e-6)
    out = rts_smoother(g["c1_means"], g["c1_covs"], list(g["tv_Fs"]), list(g["tv_Qs"]))
    for got, key in zip(out, ["x", "P", "K", "Pp"]):
        rel_close(got, g["tv_proc_" + key], 1e-6)
    # column-vector means (T,n,1) keep their shape (kalman_filter.py:1065 copies Xs)
    out = kf.rts_smoother(g["c1_means"][..., None], g["c1_covs"])
    assert out[0].shape == g["c1_means"].shape + (1,)
    rel_close(out[0][..., 0], g["c1_x"], 1e-6)
    with pytest.raises(ValueError):
        kf.rts_smoother(g["c1_means"][:-1], g["c1_covs"])


@pytest.mark.parametrize("name,dtype,tol", [("b42", np.float64, 1e-6), ("b42", np.float32, 1e-3),
                                            ("b93", np.float64, 1e-6)])
def test_rts_bank_golden(golden, name, dtype, tol):
    import torch
    from filterpy_b200.kalman import KalmanFilter
    g = golden("rts")
    Xs, Ps = g[name + "_Xs"], g[name + "_Ps"]
    T, N, n = Xs.shape
    kf = KalmanFilter(n, 1, n_filters=N, dtype=dtype, diagnostics=False)
    kf.F, kf.Q = g[name + "_F"], g[name + "_Q"]
    out = kf.rts_smoother(torch.from_numpy(Xs), torch.from_numpy(Ps))
    for got, key in zip(out, ["x", "P", "K", "Pp"]):
        rel_close(got.cpu().numpy(), g[name + "_" + key], tol, atol_scale=4.0 if dtype == np.float32 else 1.0)


def test_rts_after_batch_filter_bank_vs_oracle():
    """batch_filter -> rts_smoother entirely on the GPU, 4/2 fp64 and 2/1 fp32 (register kernels)
    and 3/2 (generic kernel), against the oracle run on the GPU's own batch_filter output."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.common import workloads as wl
    from oracle import kf as okf
    rng = np.random.default_rng(4)
    N, T = 300, 40
    w = wl.kf_bank_cv2d(N, seed=8)
    zs = rng.normal(size=(T, N, 2)) + np.einsum("nij,nj->ni", w["H"], w["x"])[None]
    kf = KalmanFilter(4, 2, n_filters=N, dtype=np.float64, diagnostics=False)
    kf.x, kf.P, kf.F, kf.H, kf.Q, kf.R = w["x"], w["P"], w["F"], w["H"], w["Q"], w["R"]
    means, covs, _, _ = kf.batch_filter(zs)
    out = kf.rts_smoother(means, covs)
    ref = okf.rts_smoother_bank(means.cpu().numpy(), covs.cpu().numpy(), w["F"], w["Q"])
    for a, b in zip(out, ref):
        rel_close(a.cpu().numpy(), b, 1e-6)
    # shared models + fp32, dim_x = 2
    F = np.array([[1., .1], [0., 1.]]); Q = np.array([[1e-4, 1e-3], [1e-3, 1e-2]]); H = np.array([[1., 0.]])
    kf = KalmanFilter(2, 1, n_filters=N, dtype=np.float32, diagnostics=False)
    kf.x = rng.normal(size=(N, 2)); kf.P = np.tile(np.eye(2) * 3, (N, 1, 1)); kf.F, kf.Q, kf.H = F, Q, H
    kf.R = np.array([[0.5]])
    means, covs, _, _ = kf.batch_filter(rng.normal(size=(T, N, 1)))
    out = kf.rts_smoother(means, covs)
    ref = okf.rts_smoother_bank(means.cpu().numpy().astype(np.float64), covs.cpu().numpy().astype(np.float64), F, Q)
    for a, b in zip(out, ref):
        rel_close(a.cpu().numpy(), b, 1e-3, atol_scale=4.0)
    # generic kernel: dim_x = 3
    F3 = np.eye(3) + np.diag([.1, .1], 1); Q3 = np.eye(3) * .01
    kf = KalmanFilter(3, 2, n_filters=17, dtype=np.float64, diagnostics=False)
    kf.x = rng.normal(size=(17, 3)); kf.P = np.tile(np.eye(3) * 2, (17, 1, 1)); kf.F, kf.Q = F3, Q3
    kf.H = np.array([[1., 0, 0], [0, 0, 1.]]); kf.R = np.eye(2) * .3
    means, covs, _, _ = kf.batch_filter(rng.normal(size=(25, 17, 2)))
    out = kf.rts_smoother(means, covs)
    ref = okf.rts_smoother_bank(means.cpu().numpy(), covs.cpu().numpy(), F3, Q3)
    for a, b in zip(out, ref):
        rel_close(a.cpu().numpy(), b, 1e-6)


# ------------------------------------------------------------------ IMM / MMAE banks
MM_MISSING = ["a", "b", "c", "d", "e", "f", "g", "h", "man"]


def mm_case(golden, nm):
    """One IMM / MMAE golden case: nm = 2 or 3 is mm.npz (4/2, every track measured at every epoch); a name of
    MM_MISSING is a case of mm_missing.npz (4/2, 2/1, 6/3, 3/1 with 2..4 models and missed measurements)."""
    if isinstance(nm, str):
        g = golden("mm_missing")
        return {k[len(nm) + 1:]: v for k, v in g.items() if k.startswith(nm + "_")}
    g = golden("mm")
    c = {k: g["m%d_%s" % (nm, k)] for k in ("zs", "trans", "mu0", "F", "H", "R", "Qs", "x0", "P0")}
    c["valid"] = np.ones(c["zs"].shape[:2], bool)
    for k in ("x", "P", "xp", "Pp", "mu", "fx", "fP", "init_x", "init_P", "init_omega", "init_cbar"):
        c["imm_" + k] = g["imm%d_%s" % (nm, k)]
    for k in ("x", "P", "p"):
        c["mmae_" + k] = g["mmae%d_%s" % (nm, k)]
    return c


def mm_filters(c, dtype, single_track=None):
    from filterpy_b200.kalman import KalmanFilter
    nm, n, m = c["Qs"].shape[0], c["F"].shape[0], c["H"].shape[0]
    NT = c["x0"].shape[0]
    fs = []
    for j in range(nm):
        if single_track is None:
            f = KalmanFilter(n, m, n_filters=NT, dtype=dtype)
            f.x = c["x0"] + j; f.P = c["P0"]
        else:
            f = KalmanFilter(n, m, dtype=dtype)
            f.x = c["x0"][single_track] + j; f.P = c["P0"][single_track]
        f.F, f.H, f.R, f.Q = c["F"], c["H"], c["R"], c["Qs"][j]
        fs.append(f)
    return fs


def mm_update(est, c, k):
    """Epoch k's measurements: update(z), update(None) when every track misses, else update(z, valid=...)."""
    import torch
    v = c["valid"][k]
    z = torch.from_numpy(c["zs"][k])
    if v.all():
        est.update(z)
    elif not v.any():
        est.update(None)
    else:
        est.update(z, valid=torch.from_numpy(v))


@pytest.mark.parametrize("nm", [2, 3] + MM_MISSING)
@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-6), (np.float32, 2e-3)])
def test_imm_bank_golden(golden, nm, dtype, tol):
    from filterpy_b200.kalman import IMMEstimator
    c = mm_case(golden, nm)
    zs = c["zs"]
    T = zs.shape[0] if dtype == np.float64 else min(8, zs.shape[0])      # fp32 drifts with the recursion length
    imm = IMMEstimator(mm_filters(c, dtype), c["mu0"], c["trans"])
    if "imm_init_x" in c:
        rel_close(imm.x[0].cpu().numpy(), c["imm_init_x"], tol)
        rel_close(imm.P[0].cpu().numpy(), c["imm_init_P"], tol)
        rel_close(imm.omega[0].cpu().numpy(), c["imm_init_omega"], 1e-12)
        rel_close(imm.cbar[0].cpu().numpy(), c["imm_init_cbar"], 1e-12)
    for k in range(T):
        imm.predict()
        rel_close(imm.x.cpu().numpy(), c["imm_xp"][k], tol); rel_close(imm.P.cpu().numpy(), c["imm_Pp"][k], tol)
        rel_close(imm.x_prior.cpu().numpy(), c["imm_xp"][k], tol)
        mm_update(imm, c, k)
        rel_close(imm.x.cpu().numpy(), c["imm_x"][k], tol); rel_close(imm.P.cpu().numpy(), c["imm_P"][k], tol)
        rel_close(imm.mu.cpu().numpy(), c["imm_mu"][k], tol * 10)
        if "imm_omega" in c:
            rel_close(imm.cbar.cpu().numpy(), c["imm_cbar"][k], tol * 10)
            rel_close(imm.omega.cpu().numpy(), c["imm_omega"][k], tol * 10)
            if dtype == np.float64:
                np.testing.assert_allclose(imm.likelihood.cpu().numpy(), c["imm_lik"][k], rtol=1e-6, atol=0)
        for j, f in enumerate(imm.filters):
            rel_close(f.x.cpu().numpy(), c["imm_fx"][k][:, j], tol)
            rel_close(f.P.cpu().numpy(), c["imm_fP"][k][:, j], tol)
    assert abs(float(imm.mu.sum(dim=1).mean().item()) - 1.0) < 1e-12


@pytest.mark.parametrize("nm", [2, 3] + MM_MISSING)
def test_mmae_bank_golden(golden, nm):
    from filterpy_b200.kalman import MMAEFilterBank
    c = mm_case(golden, nm)
    zs = c["zs"]
    bank = MMAEFilterBank(mm_filters(c, np.float64), list(c["mu0"]), dim_x=c["F"].shape[0])
    for k in range(zs.shape[0]):
        bank.predict()
        mm_update(bank, c, k)
        rel_close(bank.x.cpu().numpy(), c["mmae_x"][k], 1e-6)
        rel_close(bank.P.cpu().numpy(), c["mmae_P"][k], 1e-6)
        np.testing.assert_allclose(bank.p.cpu().numpy(), c["mmae_p"][k], rtol=1e-5, atol=1e-300)
        if "mmae_fx" in c:
            for j, f in enumerate(bank.filters):
                rel_close(f.x.cpu().numpy(), c["mmae_fx"][k][:, j], 1e-6)
                rel_close(f.P.cpu().numpy(), c["mmae_fP"][k][:, j], 1e-6)
                np.testing.assert_allclose(f.likelihood.cpu().numpy(), c["mmae_lik"][k][:, j], rtol=1e-6, atol=0)


def test_imm_single_track_drop_in_and_errors(golden):
    from filterpy_b200.kalman import IMMEstimator, KalmanFilter, MMAEFilterBank
    c = mm_case(golden, 2)
    zs = c["zs"]
    imm = IMMEstimator(mm_filters(c, np.float64, single_track=3), c["mu0"], c["trans"])
    for k in range(6):
        imm.predict(); imm.update(zs[k, 3])
        assert imm.x.shape == (4,) and imm.P.shape == (4, 4) and imm.mu.shape == (2,)
        rel_close(imm.x, c["imm_x"][k, 3], 1e-6); rel_close(imm.P, c["imm_P"][k, 3], 1e-6)
        rel_close(imm.mu, c["imm_mu"][k, 3], 1e-5)
    # a manoeuvre to z = (12, -6), then update(None): the reference re-evaluates each model's likelihood as
    # logpdf(0, S) of the kept S, and the mode probabilities move back towards the low-noise model
    c = mm_case(golden, "man")
    imm = IMMEstimator(mm_filters(c, np.float64, single_track=0), c["mu0"], c["trans"])
    for k in range(c["zs"].shape[0]):
        imm.predict(); imm.update(c["zs"][k, 0] if c["valid"][k, 0] else None)
        rel_close(imm.x, c["imm_x"][k, 0], 1e-6); rel_close(imm.P, c["imm_P"][k, 0], 1e-6)
        rel_close(imm.mu, c["imm_mu"][k, 0], 1e-5)
        np.testing.assert_allclose(imm.likelihood, c["imm_lik"][k, 0], rtol=1e-6, atol=0)
    assert not c["valid"][-1, 0] and imm.mu[0] > 0.1
    with pytest.raises(ValueError):
        IMMEstimator([KalmanFilter(4, 2)], [1.0], np.eye(1))
    with pytest.raises(ValueError):
        IMMEstimator([KalmanFilter(4, 2), KalmanFilter(3, 2)], [.5, .5], np.eye(2))
    with pytest.raises(ValueError):
        MMAEFilterBank([KalmanFilter(4, 2), KalmanFilter(4, 2)], [1.0], dim_x=4)


# ------------------------------------------------------------------ UKF RTS smoother
@pytest.mark.parametrize("name", ["cv", "lin"])
@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-6), (np.float32, 2e-3)])
def test_ukf_rts_bank_golden(golden, name, dtype, tol):
    import torch
    from filterpy_b200.kalman import (UnscentedKalmanFilter, MerweScaledSigmaPoints, ConstVelFx, LinearFx, LinearHx)
    g = golden("ukf_rts")
    Xs, Ps = g[name + "_Xs"], g[name + "_Ps"]
    T, N, n = Xs.shape
    fx = ConstVelFx() if name == "cv" else LinearFx(g[name + "_F"])
    u = UnscentedKalmanFilter(6, 3, float(g[name + "_dt"]), LinearHx(np.eye(3, 6)), fx,
                              MerweScaledSigmaPoints(6, float(g["alpha"]), float(g["beta"]), float(g["kappa"])),
                              n_filters=N, dtype=dtype)
    u.Q = g[name + "_Q"]
    dts = list(g[name + "_dts"]) if name == "cv" else None
    x, P, K = u.rts_smoother(torch.from_numpy(Xs), torch.from_numpy(Ps), dts=dts)
    rel_close(x.cpu().numpy(), g[name + "_x"], tol)
    rel_close(P.cpu().numpy(), g[name + "_P"], tol, atol_scale=4.0 if dtype == np.float32 else 1.0)
    rel_close(K.cpu().numpy(), g[name + "_K"], tol * 10, atol_scale=4.0)
    with pytest.raises(ValueError):
        u.rts_smoother(torch.from_numpy(Xs[:-1]), torch.from_numpy(Ps))


def test_ukf_rts_single_filter_drop_in(golden):
    from filterpy_b200.kalman import UnscentedKalmanFilter, MerweScaledSigmaPoints, ConstVelFx, LinearHx
    g = golden("ukf_rts")
    u = UnscentedKalmanFilter(6, 3, float(g["cv_dt"]), LinearHx(np.eye(3, 6)), ConstVelFx(),
                              MerweScaledSigmaPoints(6, float(g["alpha"]), float(g["beta"]), float(g["kappa"])))
    u.Q = g["cv_Q"][2]
    x, P, K = u.rts_smoother(g["cv_Xs"][:, 2], g["cv_Ps"][:, 2], dts=list(g["cv_dts"]))
    assert x.shape == g["cv_x"][:, 2].shape and P.shape == g["cv_P"][:, 2].shape
    rel_close(x, g["cv_x"][:, 2], 1e-6); rel_close(P, g["cv_P"][:, 2], 1e-6); rel_close(K, g["cv_K"][:, 2], 1e-5)


def test_imm_cuda_graph_of_three_steps_equals_direct_steps(golden):
    """The model filters rotate three state buffers; a graph of 3 IMM steps must leave them where a
    replay expects them."""
    import torch
    from filterpy_b200.kalman import IMMEstimator
    c = mm_case(golden, 3)
    z = torch.from_numpy(c["zs"][0]).cuda()

    def make():
        return IMMEstimator(mm_filters(c, np.float64), c["mu0"], c["trans"])
    a, b = make(), make()

    def step(imm):
        imm.predict(); imm.update(z)
    graph = b.capture(lambda: [step(b) for _ in range(3)], warmup=2)     # 6 warm-up steps run, the capture itself does not
    graph.replay(); graph.replay()
    for _ in range(12):
        step(a)
    torch.cuda.synchronize()
    assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P) and torch.equal(a.mu, b.mu)
    for fa, fb in zip(a.filters, b.filters):
        assert torch.equal(fa.x, fb.x) and torch.equal(fa.x_post, fb.x_post)


def test_imm_cuda_graph_with_missed_measurements_equals_direct_steps(golden):
    """A captured IMM step list with update(None) and update(z, valid=mask): the log-likelihood of a missed
    measurement is computed on the device without a host synchronisation, so it replays like the rest."""
    import torch
    from filterpy_b200.kalman import IMMEstimator
    c = mm_case(golden, "b")
    z = torch.from_numpy(c["zs"][1]).cuda()
    valid = torch.from_numpy(c["valid"][1]).cuda()

    def make():
        return IMMEstimator(mm_filters(c, np.float64), c["mu0"], c["trans"])
    a, b = make(), make()

    def steps(imm):
        imm.predict(); imm.update(z)
        imm.predict(); imm.update(None)
        imm.predict(); imm.update(z, valid=valid)
    graph = b.capture(lambda: steps(b), warmup=2)
    graph.replay(); graph.replay()
    for _ in range(4):
        steps(a)
    torch.cuda.synchronize()
    assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P) and torch.equal(a.mu, b.mu)
    for fa, fb in zip(a.filters, b.filters):
        assert torch.equal(fa.x, fb.x) and torch.equal(fa.log_likelihood, fb.log_likelihood)
