"""GPU: bke_score_measurements on every register instance and the warp / any-m catch-all, fp32 and fp64, against the
fp64 oracle (tests/stats_oracle.py); the stats mirrors and KalmanFilter's scoring methods against the reference's
golden vectors; a captured graph; the torch op; and two cross-checks against the step kernels."""
import math

import numpy as np
import pytest
import torch

import stats_oracle as so

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TOL = {torch.float32: 1e-3, torch.float64: 1e-6}
# register phase A (n/m of dispatch_m), warp phase A with register phase B (m <= 4), and any m
SHAPES = [(1, 1), (2, 1), (2, 2), (3, 1), (3, 3), (4, 1), (4, 2), (4, 4), (6, 3),
          (7, 1), (5, 2), (9, 3), (8, 4), (6, 6), (12, 5)]
SOURCES = [("x", "P"), ("x", "S"), ("mean", "P"), ("mean", "S")]


def _close(a, b, tol, what=""):
    a = a.double().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.array_equal(np.isnan(a), np.isnan(b)), what
    f = ~np.isnan(b)
    scale = max(np.abs(b[f]).max(initial=0.0), 1.0)
    assert np.abs(a[f] - b[f]).max(initial=0.0) / scale < tol, (what, np.abs(a[f] - b[f]).max(initial=0.0))


def _problem(n, m, N, K, dtype, seed=0, shared=False, layout="own"):
    """Seeded, well-conditioned inputs rounded to `dtype`, as fp64 NumPy."""
    rng = np.random.default_rng(seed + 31 * n + m)
    np_dt = np.float32 if dtype == torch.float32 else np.float64
    lead = () if shared else (N,)
    x = rng.standard_normal((N, n))
    A = rng.standard_normal((N, n, n))
    P = A @ A.transpose(0, 2, 1) / n + np.eye(n)
    H = rng.standard_normal(lead + (m, n))
    B = rng.standard_normal(lead + (m, m))
    R = B @ np.swapaxes(B, -1, -2) / m + np.eye(m)
    z = rng.standard_normal(((1 if layout == "scan" else N), K, m)) * 2
    return {k: v.astype(np_dt).astype(np.float64) for k, v in dict(x=x, P=P, H=H, R=R, z=z).items()}


def _t(a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV).to(dtype).contiguous()


def _zhat(H, x):
    return x @ H.T if H.ndim == 2 else np.einsum("fmn,fn->fm", H, x)


def _run(p, dtype, mean_src, cov_src, valid=None, want=("zhat", "y", "d2", "mahalanobis", "log_likelihood",
                                                       "likelihood", "status")):
    from filterpy_b200.stats.stats import score
    n, m = p["x"].shape[1], p["R"].shape[-1]
    zhat = _zhat(p["H"], p["x"])
    S = so.innovation_cov(p["P"], p["H"], p["R"])
    kw = {}
    if mean_src == "x":
        kw.update(x=_t(p["x"], dtype), H=_t(p["H"], dtype))
    else:
        kw.update(mean=_t(zhat.astype(np.float32) if dtype == torch.float32 else zhat, dtype))
    if cov_src == "P":
        kw.update(P=_t(p["P"], dtype), R=_t(p["R"], dtype), H=_t(p["H"], dtype))
    else:
        kw.update(S=_t(S, dtype))
    if cov_src == "S":
        S = S.astype(np.float32).astype(np.float64) if dtype == torch.float32 else S
    if mean_src == "mean":
        zhat = zhat.astype(np.float32).astype(np.float64) if dtype == torch.float32 else zhat
    vt = None if valid is None else _t(valid, torch.uint8)
    out = score(_t(p["z"], dtype), valid=vt, want=want, **kw)
    N, K = zhat.shape[0], p["z"].shape[1]
    ref = so.score(np.broadcast_to(p["z"], (N, K, m)), zhat, np.broadcast_to(S, (N, m, m)), valid)
    ref["zhat"] = zhat
    return out, ref


def _check(out, ref, dtype, what=""):
    for k, v in out.items():
        if k == "status":
            assert np.array_equal(v.cpu().numpy(), ref["status"]), what
        else:
            _close(v, ref[k], TOL[dtype], "%s %s" % (what, k))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("mean_src,cov_src", SOURCES)
@pytest.mark.parametrize("n,m", SHAPES)
def test_every_instance_and_source(n, m, mean_src, cov_src, dtype):
    for layout, K, shared in (("own", 37, False), ("scan", 5, True), ("own", 1, False)):
        p = _problem(n, m, 300, K, dtype, shared=shared, layout=layout)
        out, ref = _run(p, dtype, mean_src, cov_src)
        _check(out, ref, dtype, "%s K=%d shared=%s" % (layout, K, shared))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n,m", [(4, 2), (9, 3), (6, 6)])
def test_missing_candidates(n, m, dtype):
    p = _problem(n, m, 200, 45, dtype)
    valid = np.random.default_rng(3).random((200, 45)) > 0.3
    out, ref = _run(p, dtype, "x", "P", valid=valid)
    _check(out, ref, dtype)
    assert (out["log_likelihood"][~torch.as_tensor(valid, device=DEV)] == math.log(2.2250738585072014e-308)).all() \
        or dtype == torch.float32


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n,m", [(4, 2), (3, 3), (9, 3), (6, 6)])
def test_singular_track_inside_a_healthy_tile(n, m, dtype):
    from filterpy_b200.stats.stats import score
    p = _problem(n, m, 300, 9, dtype)
    S = so.innovation_cov(p["P"], p["H"], p["R"])
    S[130] = 1.0                                            # rank one
    S[131] = 0.0
    zhat = np.einsum("fmn,fn->fm", p["H"], p["x"])
    valid = np.ones((300, 9), bool)
    valid[130, 4] = False
    out = score(_t(p["z"], dtype), mean=_t(zhat, dtype), S=_t(S, dtype), valid=_t(valid, torch.uint8),
                want=("d2", "mahalanobis", "log_likelihood", "likelihood", "status", "y"))
    st = out["status"].cpu().numpy()
    assert st[130] == 1 and st[131] == 1 and st[:130].sum() == 0 and st[132:].sum() == 0
    ll = out["log_likelihood"].double().cpu().numpy()
    assert np.isnan(np.delete(ll[130], 4)).all() and np.isnan(ll[131]).all()
    assert ll[130, 4] == np.float64(np.asarray(math.log(2.2250738585072014e-308), np.float32 if dtype == torch.float32
                                                else np.float64))
    ref = so.score(p["z"], zhat.astype(np.float32).astype(np.float64) if dtype == torch.float32 else zhat,
                   S.astype(np.float32).astype(np.float64) if dtype == torch.float32 else S, valid)
    for k in ("d2", "mahalanobis", "log_likelihood", "y"):
        _close(out[k], ref[k], TOL[dtype], k)


def test_empty_banks_launch_nothing():
    from filterpy_b200.stats.stats import score
    for N, K in ((0, 4), (5, 0)):
        out = score(torch.zeros(N, K, 2, dtype=torch.float64, device=DEV), mean=torch.zeros(N, 2, dtype=torch.float64,
                    device=DEV), S=torch.eye(2, dtype=torch.float64, device=DEV), want=("log_likelihood",))
        assert tuple(out["log_likelihood"].shape) == (N, K)
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- the mirrors
def test_single_calls_match_the_golden(golden):
    from filterpy_b200 import stats
    g = golden("stats_mahalanobis")
    for i in range(int(g["n_cases"])):
        got = stats.mahalanobis(g["c%d_x" % i], g["c%d_mean" % i], g["c%d_cov" % i])
        assert isinstance(got, float)
        assert abs(got - float(g["c%d_out" % i])) <= 1e-10 * max(1.0, float(g["c%d_out" % i])), i
    assert stats.mahalanobis(3., 3.5, 4. ** 2) == 0.125 and stats.mahalanobis(3., 6, 1) == 3.0
    b = golden("stats_bank_4_2")
    for f, k in ((0, 0), (5, 3), (47, 6)):
        args = (b["z_own"][f, k], b["x"][f], b["P"][f], b["H"][f], b["R"][f])
        assert abs(stats.log_likelihood(*args) - b["ll_own"][f, k]) < 1e-10 * abs(b["ll_own"][f, k])
        assert abs(stats.likelihood(*args) - b["lk_own"][f, k]) < 1e-10 * abs(b["lk_own"][f, k])
        S = b["H"][f] @ b["P"][f] @ b["H"][f].T + b["R"][f]
        assert abs(stats.logpdf(b["z_own"][f, k], b["H"][f] @ b["x"][f], S) - b["logpdf_own"][f, k]) < 1e-9
    n = golden("stats_nees")
    got = stats.NEES(n["xs"], n["est_xs"], n["ps"])
    assert isinstance(got, list) and len(got) == len(n["nees"])
    _close(np.array(got).reshape(-1), n["nees"], 1e-10)


def test_single_calls_raise_where_the_reference_does(golden):
    from filterpy_b200 import stats
    d = golden("stats_deviations")
    with pytest.raises(np.linalg.LinAlgError):
        stats.mahalanobis(d["z"], d["mean"], d["S_sing"])
    with pytest.raises(np.linalg.LinAlgError):
        stats.NEES(np.ones((2, 2)), np.zeros((2, 2)), np.stack([np.eye(2), d["S_sing"]]))
    with pytest.raises(np.linalg.LinAlgError):                 # scipy: -inf (documented deviation)
        stats.logpdf(d["z"], d["mean"], d["S_sing"])
    ll = stats.logpdf(d["z"], d["mean"], d["S_cut"])            # scipy: -inf (its eigenvalue cutoff)
    assert math.isfinite(ll)
    o = so.score(d["z"][None, None], d["mean"][None], d["S_indef"][None])
    assert abs(stats.logpdf(d["z"], d["mean"], d["S_indef"]) - o["log_likelihood"][0, 0]) < 1e-12  # scipy raises


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n,m", [(1, 1), (2, 1), (4, 2), (6, 3), (9, 3)])
def test_bank_calls_match_the_golden(golden, n, m, dtype):
    from filterpy_b200 import stats
    g = golden("stats_bank_%d_%d" % (n, m))
    tol = TOL[dtype] * 10
    T = lambda a: _t(a, dtype)                                  # noqa: E731
    for lay, z in (("own", g["z_own"]), ("scan", g["z_scan"][None])):
        ll = stats.log_likelihood(T(z), T(g["x"]), T(g["P"]), T(g["H"]), T(g["R"]))
        _close(ll, g["ll_" + lay], tol, "ll")
        _close(stats.likelihood(T(z), T(g["x"]), T(g["P"]), T(g["H"]), T(g["R"])), g["lk_" + lay], tol, "lk")
        ll2, d = stats.score_measurements(T(z), T(g["x"]), T(g["P"]), T(g["H"]), T(g["R"]))
        _close(ll2, g["ll_" + lay], tol)
        _close(d, g["maha_" + lay], tol)
        S = g["H"] @ g["P"] @ np.swapaxes(g["H"], 1, 2) + g["R"]
        zh = np.einsum("fmn,fn->fm", g["H"], g["x"])
        _close(stats.mahalanobis(T(z), T(zh), T(S)), g["maha_" + lay], tol, "maha")
        _close(stats.logpdf(T(z), T(zh), T(S)), g["logpdf_" + lay], tol, "logpdf")
    # NumPy in, NumPy out; [N, m] candidates give [N]
    got = stats.log_likelihood(g["z_own"][:, 0], g["x"], g["P"], g["H"], g["R"])
    assert isinstance(got, np.ndarray) and got.shape == (g["x"].shape[0],)
    _close(got, g["ll_own"][:, 0], 1e-10)


def test_nees_bank(golden):
    from filterpy_b200 import stats
    g = golden("stats_nees")
    T = g["nees"].shape[0]
    xs = np.repeat(g["xs"][:, None, :, 0], 3, axis=1)
    est = np.repeat(g["est_xs"][:, None, :, 0], 3, axis=1)
    ps = np.repeat(g["ps"][:, None], 3, axis=1)
    ps[5, 1] = 0.0
    got = stats.NEES(xs, est, ps)
    assert got.shape == (T, 3) and np.isnan(got[5, 1])
    got[5, 1] = g["nees"][5]
    _close(got, np.repeat(g["nees"][:, None], 3, axis=1), 1e-10)


def _kf_from_golden(g, n_filters=None, dtype=np.float64):
    from filterpy_b200.kalman import KalmanFilter
    kf = KalmanFilter(4, 2, n_filters=n_filters, dtype=dtype, device=DEV)
    kf.x = g["x0"] if n_filters is None else np.repeat(g["x0"][None, :, 0], n_filters, 0)
    kf.P = g["P0"]
    kf.F, kf.H, kf.Q, kf.R = g["F"], g["H"], g["Q"], g["R"]
    return kf


def test_kalman_filter_scoring_methods_single(golden):
    g = golden("stats_kf_methods")
    kf = _kf_from_golden(g)
    assert kf.log_likelihood_of(None) == float(g["ll_none"])
    with pytest.raises(np.linalg.LinAlgError):                 # S = 0 before the first update (scipy: -inf)
        kf.log_likelihood_of(g["cands"][0, 0])
    for t in range(g["zs"].shape[0]):
        kf.predict()
        if t > 0:
            got = [kf.log_likelihood_of(c) for c in g["cands"][t]]
            _close(got, g["ll_pred"][t], 1e-10, "stale S")
        r = kf.residual_of(g["zs"][t])
        assert r.shape == (2, 1)
        _close(r, g["res_pred"][t], 1e-12)
        _close(kf.measurement_of_state(kf.x), g["mos"][t], 1e-12)
        kf.update(g["zs"][t])
        _close([kf.log_likelihood_of(c) for c in g["cands"][t]], g["ll_upd"][t], 1e-10)
        _close(kf.residual_of(g["zs"][t]), g["res_upd"][t], 1e-12)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_kalman_filter_scoring_methods_bank(golden, dtype):
    g = golden("stats_kf_methods")
    N = 3
    kf = _kf_from_golden(g, N, dtype)
    tol = TOL[torch.float32 if dtype == np.float32 else torch.float64] * 10
    for t in range(g["zs"].shape[0]):
        kf.predict()
        res = kf.residual_of(_t(np.repeat(g["zs"][t][None], N, 0), kf.x.dtype))
        assert tuple(res.shape) == (N, 2)
        _close(res, np.repeat(g["res_pred"][t][None, :, 0], N, 0), tol)
        _close(kf.measurement_of_state(kf.x), np.repeat(g["mos"][t][None, :, 0], N, 0), tol)
        kf.update(_t(np.repeat(g["zs"][t][None], N, 0), kf.x.dtype))
        scan = _t(g["cands"][t][None], kf.x.dtype)              # [1, K, m]: one scan for the whole bank
        ll = kf.log_likelihood_of(scan)
        assert tuple(ll.shape) == (N, g["cands"].shape[1])
        _close(ll, np.repeat(g["ll_upd"][t][None], N, 0), tol)
        valid = np.ones((N, g["cands"].shape[1]), bool)
        valid[1, 2] = False
        ll = kf.log_likelihood_of(scan, valid=valid).double().cpu().numpy()
        assert ll[1, 2] == np.float64(np.asarray(so.LOG_DBL_MIN, dtype))
    assert (kf.log_likelihood_of(None) == so.LOG_DBL_MIN).all()


def test_diagnostics_off_raises_as_the_getters_do():
    from filterpy_b200.kalman import KalmanFilter
    kf = KalmanFilter(4, 2, n_filters=4, device=DEV, diagnostics=False)
    with pytest.raises(AttributeError):
        kf.log_likelihood_of(torch.zeros(4, 2, dtype=torch.float64, device=DEV))
    with pytest.raises(AttributeError):
        kf.residual_of(torch.zeros(4, 2, dtype=torch.float64, device=DEV))
    assert tuple(kf.measurement_of_state(kf.x).shape) == (4, 2)


# ---------------------------------------------------------------------------------------------- cross-checks
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("n,m", [(4, 2), (9, 3)])
def test_scores_equal_the_step_kernels(n, m, dtype):
    """stats.log_likelihood(z, x_prior, P_prior, H, R) is the step's stored log_likelihood for the same z, and
    score_measurements' distance is kf.mahalanobis after that update."""
    from filterpy_b200 import stats
    from filterpy_b200.kalman import KalmanFilter
    N = 500
    p = _problem(n, m, N, 1, torch.float64)
    kf = KalmanFilter(n, m, n_filters=N, dtype=dtype, device=DEV)
    kf.x, kf.P, kf.H, kf.R = p["x"], p["P"], p["H"][0], p["R"][0]
    kf.F = np.eye(n) + 0.1 * np.eye(n, k=1)
    kf.Q = np.eye(n) * 0.05
    z = _t(p["z"][:, 0], kf.x.dtype)
    kf.predict()
    kf.update(z)
    tol = TOL[torch.float32 if dtype == np.float32 else torch.float64]
    ll = stats.log_likelihood(z, kf.x_prior, kf.P_prior, kf.H, kf.R)
    _close(ll, kf.log_likelihood.double().cpu().numpy(), tol, "ll")
    _, d = stats.score_measurements(z, kf.x_prior, kf.P_prior, kf.H, kf.R)
    _close(d, kf.mahalanobis.double().cpu().numpy(), tol, "maha")


def test_graph_capture_and_replay():
    from filterpy_b200.stats.stats import score
    p = _problem(4, 2, 1000, 64, torch.float32, layout="scan")
    T = lambda a: _t(a, torch.float32)                          # noqa: E731
    x, P, H, R, z = T(p["x"]), T(p["P"]), T(p["H"]), T(p["R"]), T(p["z"])
    score(z, x=x, P=P, H=H, R=R, want=("log_likelihood",))      # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            out = score(z, x=x, P=P, H=H, R=R, want=("log_likelihood", "mahalanobis"))
    z2 = np.random.default_rng(9).standard_normal(p["z"].shape).astype(np.float32)
    z.copy_(T(z2))
    g.replay()
    torch.cuda.synchronize()
    ref = so.score(np.broadcast_to(z2.astype(np.float64), (1000, 64, 2)), np.einsum("fmn,fn->fm", p["H"], p["x"]),
                   so.innovation_cov(p["P"], p["H"], p["R"]))
    _close(out["log_likelihood"], ref["log_likelihood"], 1e-3)
    _close(out["mahalanobis"], ref["mahalanobis"], 1e-3)


def test_torch_op():
    from filterpy_b200 import torch_ops
    ops = torch_ops.load()
    p = _problem(6, 3, 257, 33, torch.float64)
    T = lambda a: _t(a, torch.float64)                          # noqa: E731
    ll, d, st = ops.score_measurements(T(p["z"]), T(p["x"]), None, T(p["P"]), None, T(p["H"]), T(p["R"]), None,
                                       ["log_likelihood", "mahalanobis", "status"])
    ref = so.score(p["z"], np.einsum("fmn,fn->fm", p["H"], p["x"]), so.innovation_cov(p["P"], p["H"], p["R"]))
    _close(ll, ref["log_likelihood"], 1e-6)
    _close(d, ref["mahalanobis"], 1e-6)
    assert int(st.sum().item()) == 0
    with pytest.raises(RuntimeError, match="device"):
        ops.score_measurements(T(p["z"]), T(p["x"]).cpu(), None, T(p["P"]), None, T(p["H"]), T(p["R"]), None,
                               ["log_likelihood"])
