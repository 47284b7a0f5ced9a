"""IMMEstimator.batch_filter on the GPU: every golden case (imm_batch_*.npz, mm.npz, mm_missing.npz) through the
fused kernel or, for shapes without one, the loop of separate launches; equality with a twin estimator stepped with
predict() / update(); continuation across calls; a bank of 2^20 + 3 tracks; the single-track drop-in; the torch op
and a CUDA graph."""
import numpy as np
import pytest
import torch

from imm_oracle import imm_batch

pytestmark = pytest.mark.gpu

NEW = ["m2_4_2", "m3_4_2", "m4_4_2", "m3_6_3", "m2_2_1", "m3_3_1", "m2_5_2"]
MM_MISSING = ["a", "b", "c", "d", "e", "f", "g", "h", "man"]
DTYPES = [(np.float64, 1e-6), (np.float32, 2e-3)]


def np_(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def close(a, b, tol):
    a, b = np_(a).astype(np.float64), np_(b).astype(np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    inf = np.isinf(b)
    assert np.array_equal(np.isinf(a), inf) and np.array_equal(a[inf], b[inf])
    a, b = a[~inf], b[~inf]
    if b.size:
        err = np.abs(a - b).max() / max(np.abs(b).max(), 1.0)
        assert err <= tol, err


def case(golden, name):
    """a golden case as per-track inputs: x0, P0 [N,M,n(,n)], F, Q [N,M,n,n], H, R, alpha [M], mu0, trans, zs, valid,
    and the reference's per-epoch x, P, xp, Pp, mu, fx, fP (cbar, omega, lik where recorded)."""
    if name in NEW:
        return golden("imm_batch_" + name)
    if name in (2, 3):
        g, p, r = golden("mm"), "m%d_" % name, "imm%d_" % name
        c = {"valid": np.ones(g[p + "zs"].shape[:2], bool)}
    else:
        g, p, r = golden("mm_missing"), name + "_", name + "_imm_"
        c = {"valid": g[p + "valid"]}
    nm = g[p + "trans"].shape[0]
    x0, P0 = g[p + "x0"], g[p + "P0"]
    NT, n = x0.shape
    c.update(zs=g[p + "zs"], trans=g[p + "trans"], mu0=g[p + "mu0"], H=g[p + "H"], R=g[p + "R"], alpha=np.ones(nm),
             x0=np.stack([x0 + j for j in range(nm)], axis=1), P0=np.stack([P0] * nm, axis=1),
             F=np.broadcast_to(g[p + "F"], (NT, nm, n, n)), Q=np.broadcast_to(g[p + "Qs"][:nm][None], (NT, nm, n, n)))
    for k in ("x", "P", "xp", "Pp", "mu", "fx", "fP", "cbar", "omega", "lik"):
        if r + k in g:
            c[k] = g[r + k]
    return c


def build(c, dtype, single_track=None):
    from filterpy_b200.kalman import IMMEstimator, KalmanFilter
    N, nm, n = c["x0"].shape
    m = c["H"].shape[0]
    fs = []
    for j in range(nm):
        if single_track is None:
            f = KalmanFilter(n, m, n_filters=N, dtype=dtype)
            f.x, f.P, f.F, f.Q = c["x0"][:, j], c["P0"][:, j], np.ascontiguousarray(c["F"][:, j]), np.ascontiguousarray(c["Q"][:, j])
        else:
            i = single_track
            f = KalmanFilter(n, m, dtype=dtype)
            f.x, f.P, f.F, f.Q = c["x0"][i, j], c["P0"][i, j], c["F"][i, j], c["Q"][i, j]
        f.H, f.R = c["H"], c["R"]
        f.alpha = float(c["alpha"][j])
        fs.append(f)
    return IMMEstimator(fs, c["mu0"], c["trans"])


def run(imm, c, T, k0=0):
    dt = imm._dtype
    return imm.batch_filter(torch.from_numpy(np.ascontiguousarray(c["zs"][k0:T])).to(dt).cuda(),
                            valid=torch.from_numpy(np.ascontiguousarray(c["valid"][k0:T])).cuda())


@pytest.mark.parametrize("name", NEW + [2, 3] + MM_MISSING)
@pytest.mark.parametrize("dtype,tol", DTYPES)
def test_batch_filter_reproduces_the_reference(golden, name, dtype, tol):
    c = case(golden, name)
    T = c["zs"].shape[0] if dtype == np.float64 else min(8, c["zs"].shape[0])      # fp32 drifts with the recursion length
    imm = build(c, dtype)
    means, covs, means_p, covs_p, mus = run(imm, c, T)
    assert mus.dtype == torch.float64 and tuple(mus.shape) == (T, c["x0"].shape[0], c["x0"].shape[1])
    close(means, c["x"][:T], tol); close(covs, c["P"][:T], tol)
    close(means_p, c["xp"][:T], tol); close(covs_p, c["Pp"][:T], tol)
    close(mus, c["mu"][:T], tol * 10)
    close(imm.x, c["x"][T - 1], tol); close(imm.P, c["P"][T - 1], tol)
    close(imm.x_prior, c["xp"][T - 1], tol); close(imm.P_prior, c["Pp"][T - 1], tol)
    close(imm.x_post, c["x"][T - 1], tol); close(imm.P_post, c["P"][T - 1], tol)
    close(imm.mu, c["mu"][T - 1], tol * 10)
    if "omega" in c:
        close(imm.cbar, c["cbar"][T - 1], tol * 10); close(imm.omega, c["omega"][T - 1], tol * 10)
        if dtype == np.float64:
            np.testing.assert_allclose(np_(imm.likelihood), c["lik"][T - 1], rtol=1e-6, atol=0)
    for j, f in enumerate(imm.filters):
        close(f.x, c["fx"][T - 1][:, j], tol); close(f.P, c["fP"][T - 1][:, j], tol)


def _attrs(imm):
    out = {k: np_(getattr(imm, k)) for k in ("x", "P", "x_prior", "P_prior", "x_post", "P_post", "mu", "cbar", "omega",
                                              "likelihood")}
    for j, f in enumerate(imm.filters):
        for k in ("x", "P", "x_prior", "P_prior", "x_post", "P_post", "K", "y", "S", "SI", "log_likelihood", "status", "z"):
            out["f%d_%s" % (j, k)] = np_(getattr(f, k))
    return out


def _same(a, b, tol):
    assert a.keys() == b.keys()
    for k in a:
        if k.endswith("status"):
            assert np.array_equal(a[k], b[k]), k
        elif k.endswith("likelihood"):
            la, lb = np.log(np.maximum(a[k], 1e-300)) if k == "likelihood" else a[k], \
                np.log(np.maximum(b[k], 1e-300)) if k == "likelihood" else b[k]
            close(la, lb, tol * 10)
        else:
            close(a[k], b[k], tol * (10 if k in ("mu", "cbar", "omega") else 1))


@pytest.mark.parametrize("name", ["m3_4_2", "m4_4_2", "m2_2_1", "m3_3_1", "m2_5_2", "m3_6_3", "man"])
@pytest.mark.parametrize("dtype,tol", DTYPES)
def test_batch_filter_equals_the_loop(golden, name, dtype, tol):
    c = case(golden, name)
    T = c["zs"].shape[0] if dtype == np.float64 else min(16, c["zs"].shape[0])
    a, b = build(c, dtype), build(c, dtype)
    means, covs, means_p, covs_p, mus = run(a, c, T)
    for k in range(T):
        b.predict()
        close(means_p[k], b.x, tol); close(covs_p[k], b.P, tol)
        b.update(torch.from_numpy(c["zs"][k]).to(b._dtype).cuda(), valid=torch.from_numpy(c["valid"][k]).cuda())
        close(means[k], b.x, tol); close(covs[k], b.P, tol); close(mus[k], b.mu, tol * 10)
    _same(_attrs(a), _attrs(b), tol)


@pytest.mark.parametrize("name,dtype", [("m3_4_2", np.float32), ("m2_2_1", np.float64), ("m2_5_2", np.float64)])
def test_batch_filter_continues_where_it_stopped(golden, name, dtype):
    c = dict(case(golden, name))
    tol = 1e-6 if dtype == np.float64 else 2e-3
    T, k0 = 10, 4
    c["valid"] = c["valid"].copy()
    c["valid"][k0, 1] = False                                   # a miss at the first epoch of the second call
    a, b, loop = build(c, dtype), build(c, dtype), build(c, dtype)
    whole = run(a, c, T)
    first, second = run(b, c, k0), run(b, c, T, k0)
    for w, f, s in zip(whole, first, second):
        close(w, torch.cat([f, s]), tol * 10)
    _same(_attrs(a), _attrs(b), tol)
    # batch_filter, then predict(); update(z) equals the loop
    z = torch.from_numpy(c["zs"][T]).to(a._dtype).cuda()
    a.predict(); a.update(z)
    for k in range(T):
        loop.predict()
        loop.update(torch.from_numpy(c["zs"][k]).to(loop._dtype).cuda(), valid=torch.from_numpy(c["valid"][k]).cuda())
    loop.predict(); loop.update(z)
    _same(_attrs(a), _attrs(loop), tol)


def test_a_large_bank_against_the_oracle():
    from filterpy_b200.kalman import IMMEstimator, KalmanFilter
    N, M, T, n, m = (1 << 20) + 3, 3, 4, 4, 2
    rng = np.random.default_rng(11)
    dt = rng.uniform(0.5, 1.5, N)
    F = np.zeros((N, n, n), np.float32); F[:] = np.eye(n)
    F[:, 0, 1] = F[:, 2, 3] = dt
    H = np.kron(np.eye(2), np.array([[1.0, 0.0]]))
    R = np.eye(2) * 0.5
    qs = [0.05, 1.0, 8.0]
    Q1 = np.zeros((N, n, n)); Q1[:, 0, 0] = Q1[:, 2, 2] = dt ** 3 / 3; Q1[:, 0, 1] = Q1[:, 1, 0] = Q1[:, 2, 3] = Q1[:, 3, 2] = dt ** 2 / 2
    Q1[:, 1, 1] = Q1[:, 3, 3] = dt
    x0 = (rng.normal(size=(N, n)) * 3).astype(np.float32)
    zs = (rng.normal(size=(T, N, m)) * 2).astype(np.float32)
    valid = rng.random((T, N)) >= 0.2
    fs = []
    for j in range(M):
        f = KalmanFilter(n, m, n_filters=N, dtype=np.float32)
        f.x, f.P, f.F, f.Q, f.H, f.R = x0 + j, np.eye(n) * 2.0, F, (Q1 * qs[j]).astype(np.float32), H, R
        fs.append(f)
    trans = np.array([[.9, .05, .05], [.1, .8, .1], [.05, .15, .8]])
    imm = IMMEstimator(fs, [0.5, 0.3, 0.2], trans)
    means, covs, means_p, covs_p, mus = imm.batch_filter(torch.from_numpy(zs).cuda(), valid=torch.from_numpy(valid).cuda())
    idx = np.concatenate([rng.choice(N - 3, 61, replace=False), [N - 3, N - 2, N - 1]])
    xs0 = np.stack([x0[idx] + j for j in range(M)], axis=1).astype(np.float64)
    Ps0 = np.broadcast_to(np.eye(n) * 2.0, (len(idx), M, n, n))
    Fo = np.broadcast_to(F[idx][:, None].astype(np.float64), (len(idx), M, n, n))
    Qo = np.stack([Q1[idx] * q for q in qs], axis=1)
    o = imm_batch(xs0, Ps0, Fo, Qo, H, R, np.ones(M), np.array([0.5, 0.3, 0.2]), trans, zs[:, idx].astype(np.float64),
                  valid[:, idx])
    close(means[:, idx], o["x"], 2e-3); close(covs[:, idx], o["P"], 2e-3)
    close(means_p[:, idx], o["xp"], 2e-3); close(covs_p[:, idx], o["Pp"], 2e-3)
    close(mus[:, idx], o["mu"], 2e-2)


def test_single_track_drop_in(golden):
    c = case(golden, "m2_2_1")
    i = 0                                                       # misses epoch 0
    imm = build(c, np.float64, single_track=i)
    zs = [c["zs"][k, i] if c["valid"][k, i] else None for k in range(c["zs"].shape[0])]
    assert zs[0] is None
    means, covs, means_p, covs_p, mus = imm.batch_filter(zs)
    T, nm, n = len(zs), c["x0"].shape[1], c["x0"].shape[2]
    assert means.shape == (T, n) and covs.shape == (T, n, n) and means_p.shape == (T, n) and mus.shape == (T, nm)
    close(means, c["x"][:, i], 1e-6); close(covs, c["P"][:, i], 1e-6)
    close(means_p, c["xp"][:, i], 1e-6); close(covs_p, c["Pp"][:, i], 1e-6); close(mus, c["mu"][:, i], 1e-5)
    close(imm.x, c["x"][-1, i], 1e-6); close(imm.mu, c["mu"][-1, i], 1e-5)
    np.testing.assert_allclose(imm.likelihood, c["lik"][-1, i], rtol=1e-6, atol=0)
    # H = 0 and R = 0 make S singular: the reference's inv(S) raises
    bad = build(c, np.float64, single_track=i)
    for f in bad.filters:
        f.H, f.R = np.zeros((1, 2)), np.zeros((1, 1))
    with pytest.raises(np.linalg.LinAlgError):
        bad.batch_filter([np.array([1.0]), np.array([2.0])])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_torch_op_equals_the_mirror(golden, dtype):
    from filterpy_b200 import torch_ops
    ops = torch_ops.load()
    c = case(golden, "m3_3_1")
    a, b = build(c, dtype), build(c, dtype)
    T = c["zs"].shape[0]
    zs = torch.from_numpy(c["zs"]).to(a._dtype).cuda()
    valid = torch.from_numpy(c["valid"]).cuda()
    ref = a.batch_filter(zs, valid=valid)
    fs = b.filters
    out = ops.imm_batch_filter([f._x for f in fs], [f._P for f in fs], [f._F for f in fs], [f._Q for f in fs],
                               [f._H for f in fs], [f._R for f in fs], [f._alpha_sq for f in fs], [f._S for f in fs],
                               [f._ll for f in fs], b._mu, b._cbar, b._M, zs, valid)
    for r, o in zip(ref, out):
        assert torch.equal(r, o)
    for fa, fb in zip(a.filters, fs):
        assert torch.equal(fa._x, fb._x) and torch.equal(fa._P, fb._P) and torch.equal(fa._S, fb._S)
    assert torch.equal(a._mu, b._mu) and torch.equal(a._cbar, b._cbar)
    assert T == ref[0].shape[0]


def test_a_captured_batch_filter_replays_as_direct_calls(golden):
    c = case(golden, "m3_4_2")
    a, b = build(c, np.float32), build(c, np.float32)
    zs = torch.from_numpy(c["zs"][:6]).float().cuda()
    for _ in range(3):
        ref = a.batch_filter(zs)
    held = []
    g = b.capture(lambda: held.append(b.batch_filter(zs)), warmup=2)
    g.replay()
    torch.cuda.synchronize()
    for r, o in zip(ref, held[-1]):
        assert torch.equal(r, o)
    _same(_attrs(a), _attrs(b), 0.0)
