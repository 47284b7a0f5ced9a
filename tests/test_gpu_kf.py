"""GPU parity: linear KF bank (CUDA through the C-ABI) vs the oracle and the reference's golden
vectors.  Tolerances are north_star's: 1e-6 rel for fp64, 1e-3 rel for fp32 (the fp32 kernel is
compared with the fp64 reference because the reference silently promotes)."""
import numpy as np
import pytest

from gpu_harness import RTOL, rel_close

pytestmark = pytest.mark.gpu


def make_bank(g, dtype, diagnostics=True):
    from filterpy_b200.kalman import KalmanFilter
    N, n = g["x"].shape
    m = g["H"].shape[-2]
    du = g["B"].shape[-1] if "B" in g else 0
    kf = KalmanFilter(n, m, dim_u=du, n_filters=N, dtype=dtype, diagnostics=diagnostics)
    kf.x = g["x"]; kf.P = g["P"]; kf.F = g["F"]; kf.H = g["H"]; kf.Q = g["Q"]; kf.R = g["R"]
    kf.alpha = float(g["alpha"])
    if "B" in g:
        kf.B = g["B"]
    return kf


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["kf_bank_4_2", "kf_bank_9_3", "kf_bank_1_1", "kf_bank_2_1",
                                  "kf_bank_3_2", "kf_bank_6_3", "kf_bank_5_5"])
def test_bank_vs_reference_golden(golden, name, dtype):
    g = golden(name)
    rtol = RTOL[dtype]       # measured in round 2 (BKE_TEST_ERRLOG): fp32 worst case 6.3e-5 (x), 5.5e-6 on the 9/3 bank
    kf = make_bank(g, dtype)
    for t in range(g["zs"].shape[0]):
        v = g["valid"][t]
        kf.predict(u=g["us"][t] if "us" in g else None)
        kf.update(g["zs"][t], valid=v)
        rel_close(kf.x.cpu().numpy(), g["ref_x"][t], rtol, "x t=%d" % t)
        rel_close(kf.P.cpu().numpy(), g["ref_P"][t], rtol, "P t=%d" % t)
        rel_close(kf.x_prior.cpu().numpy(), g["ref_x_prior"][t], rtol, "x_prior")
        rel_close(kf.P_prior.cpu().numpy(), g["ref_P_prior"][t], rtol, "P_prior")
        rel_close(kf.K.cpu().numpy()[v], g["ref_K"][t][v], rtol, "K")
        rel_close(kf.S.cpu().numpy()[v], g["ref_S"][t][v], rtol, "S")
        rel_close(kf.SI.cpu().numpy()[v], g["ref_SI"][t][v], rtol, "SI")
        rel_close(kf.y.cpu().numpy(), g["ref_y"][t], max(rtol, 1e-5), "y")      # y = z - Hx cancels: fp64 1e-5 of the filter's scale
        # every filter: after a missed measurement the reference evaluates logpdf(0, S) of the kept S (-inf while
        # S is still zero)
        ll = kf.log_likelihood.cpu().numpy()
        np.testing.assert_allclose(ll, g["ref_loglik"][t], rtol=rtol, atol=rtol)
        assert int(kf.status.sum().item()) == 0


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_separate_predict_update_calls_match_fused(golden, dtype):
    g = golden("kf_bank_4_2")
    a = make_bank(g, dtype); b = make_bank(g, dtype, diagnostics=False)
    for t in range(3):
        a.predict(); a.update(g["zs"][t])
        b.predict(); _ = b.x      # forces a stand-alone predict launch
        b.update(g["zs"][t])
        rel_close(b.x.cpu().numpy(), a.x.cpu().numpy(), 1e-6 if dtype is np.float64 else 1e-4)
        rel_close(b.P.cpu().numpy(), a.P.cpu().numpy(), 1e-6 if dtype is np.float64 else 1e-4)


def test_shared_models_match_per_filter():
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.common import workloads as wl
    from oracle import kf as okf
    w = wl.kf_bank_cv2d(1000, seed=3, steps=2)
    F, H, Q, R = w["F"][0], w["H"][0], w["Q"][0], w["R"][0]
    for dtype in (np.float32, np.float64):
        kf = KalmanFilter(4, 2, n_filters=1000, dtype=dtype, diagnostics=False)
        kf.x = w["x"]; kf.P = w["P"]; kf.F = F; kf.H = H; kf.Q = Q; kf.R = R
        x, P = w["x"], w["P"]
        for t in range(2):
            kf.predict(); kf.update(w["zs"][t])
            o = okf.kf_step_bank(x, P, w["zs"][t], F, H, Q, R); x, P = o["x"], o["P"]
        rel_close(kf.x.cpu().numpy(), x, RTOL[dtype]); rel_close(kf.P.cpu().numpy(), P, RTOL[dtype])


@pytest.mark.parametrize("N", [1, 127, 128, 129, 4099, 1 << 20])
def test_fast_4_2_f32_sizes_vs_oracle(N):
    """The TMA-staged register-tile kernel at ragged and full (BASELINE config 2) sizes."""
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.common import workloads as wl
    from oracle import kf as okf
    w = wl.kf_bank_cv2d(N, seed=1234, steps=2)
    kf = KalmanFilter(4, 2, n_filters=N, dtype=np.float32, diagnostics=False)
    for k in "xPFHQR":
        setattr(kf, k, w[k])
    x, P = w["x"], w["P"]
    for t in range(2):
        kf.predict(); kf.update(w["zs"][t])
        o = okf.kf_step_bank(x, P, w["zs"][t], w["F"], w["H"], w["Q"], w["R"]); x, P = o["x"], o["P"]
    rel_close(kf.x.cpu().numpy(), x, 1e-3, "x"); rel_close(kf.P.cpu().numpy(), P, 1e-3, "P")


def test_full_size_properties_f32():
    """Size-independent properties at N = 2^20: a bank is N independent filters, so (i) the result
    of any slice equals the result of that slice alone, (ii) with z = None the posterior is the
    prior, (iii) P stays symmetric to rounding."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.common import workloads as wl
    N = 1 << 20
    w = wl.kf_bank_cv2d(N, seed=77, steps=1, dtype=np.float32)
    kf = KalmanFilter(4, 2, n_filters=N, dtype=np.float32, diagnostics=False)
    for k in "xPFHQR":
        setattr(kf, k, w[k])
    kf.predict(); kf.update(w["zs"][0])
    sl = slice(N // 2 - 777, N // 2 + 1001)
    sub = KalmanFilter(4, 2, n_filters=sl.stop - sl.start, dtype=np.float32, diagnostics=False)
    for k in "xPFHQR":
        setattr(sub, k, w[k][sl])
    sub.predict(); sub.update(w["zs"][0][sl])
    dx = (kf.x[sl] - sub.x).abs().max().item(); dP = (kf.P[sl] - sub.P).abs().max().item()
    nbad = int(((kf.P[sl] != sub.P).any(dim=2).any(dim=1)).sum().item())
    assert torch.equal(kf.x[sl], sub.x) and torch.equal(kf.P[sl], sub.P), (dx, dP, nbad)
    P = kf.P
    assert float((P - P.transpose(1, 2)).abs().max() / P.abs().max()) < 1e-5
    kf2 = KalmanFilter(4, 2, n_filters=N, dtype=np.float32, diagnostics=False)
    for k in "xPFHQR":
        setattr(kf2, k, w[k])
    kf2.predict(); xp = kf2.x.clone(); Pp = kf2.P.clone()
    valid = np.zeros(N, dtype=bool); valid[::3] = True
    kf2.update(w["zs"][0], valid=valid)
    inv = torch.from_numpy(~valid).cuda()
    assert torch.equal(kf2.x[inv], xp[inv]) and torch.equal(kf2.P[inv], Pp[inv])
    v = torch.from_numpy(valid).cuda()
    assert torch.allclose(kf2.x[v], kf.x[v], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("shape", [(4, 2), (9, 3), (2, 1)])
@pytest.mark.parametrize("update_first", [False, True])
def test_batch_filter_bank_vs_oracle(dtype, shape, update_first):
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.common import workloads as wl
    from oracle import kf as okf
    n, m = shape
    N, T = 333, 12
    if (n, m) == (4, 2):
        w = wl.kf_bank_cv2d(N, seed=5, steps=T)
    elif (n, m) == (9, 3):
        w = wl.kf_bank_ca3d(N, seed=5, steps=T)
    else:
        rng = np.random.default_rng(0)
        w = dict(x=rng.standard_normal((N, 2)), P=np.eye(2) * 5 + np.zeros((N, 2, 2)),
                 F=np.array([[1, .1], [0, 1.]]) + np.zeros((N, 2, 2)), H=np.array([[1., 0]]) + np.zeros((N, 1, 2)),
                 Q=np.eye(2) * .01 + np.zeros((N, 2, 2)), R=np.ones((N, 1, 1)) * .5, zs=rng.standard_normal((T, N, 1)))
    rng = np.random.default_rng(1)
    valid = rng.random((T, N)) > 0.2
    kf = KalmanFilter(n, m, n_filters=N, dtype=dtype)
    for k in "xPFHQR":
        setattr(kf, k, w[k])
    got = kf.batch_filter(w["zs"], update_first=update_first, valid=valid)
    want = okf.kf_batch_filter_bank(w["x"], w["P"], w["zs"], w["F"], w["H"], w["Q"], w["R"], valid=valid,
                                    update_first=update_first)
    rtol = RTOL[dtype]       # fp32: 1e-3 (north_star); measured worst case 3.7e-4
    for a, b, nm in zip(got, want, ["means", "covs", "means_p", "covs_p"]):
        rel_close(a.cpu().numpy(), b, rtol, nm)
    last = want[2][-1] if update_first else want[0][-1]
    rel_close(kf.x.cpu().numpy(), last, rtol, "final x")


# ------------------------------------------------------------------ single-filter drop-in behaviour
def test_single_mode_c1_batch_filter(golden):
    """Config C1 through the reference-shaped API (kalman_filter.py:826): one filter, 1000 epochs."""
    from filterpy_b200.kalman import KalmanFilter
    g = golden("kf_c1")
    kf = KalmanFilter(dim_x=4, dim_z=2)
    kf.x = g["x"]; kf.P = g["P"]; kf.F = g["F"]; kf.H = g["H"]; kf.Q = g["Q"]; kf.R = g["R"]
    means, covs, means_p, covs_p = kf.batch_filter(list(g["zs"]))
    assert means.shape == (1000, 4) and covs.shape == (1000, 4, 4)
    np.testing.assert_allclose(means, g["means"], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(covs, g["covs"], rtol=1e-6, atol=1e-12)
    np.testing.assert_allclose(means_p, g["means_p"], rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(covs_p, g["covs_p"], rtol=1e-6, atol=1e-12)
    # known answers
    k2 = KalmanFilter(4, 2)
    k2.x = np.zeros(4); k2.P = 10 * np.eye(4); k2.F = g["F"]; k2.H = g["H"]; k2.Q = g["Q"]; k2.R = g["R"]
    k2.predict(); k2.update(np.array([1., 2.]))
    np.testing.assert_allclose(k2.x, g["one_x"], rtol=1e-9)
    np.testing.assert_allclose(k2.S, g["one_S"], rtol=1e-9)
    assert abs(k2.log_likelihood - float(g["one_loglik"])) < 1e-9
    assert abs(k2.mahalanobis - float(g["one_maha"])) < 1e-9


def test_single_mode_shapes_and_none():
    """Mirrors test_kf.py:347-362 (batch_filter with None) and the column-vector default."""
    from filterpy_b200.kalman import KalmanFilter
    f = KalmanFilter(dim_x=2, dim_z=1)
    f.x = np.array([[2.], [0.]])
    f.F = np.array([[1., 1.], [0., 1.]]); f.H = np.array([[1., 0.]])
    f.P *= 1000.; f.R = 5; f.Q = 0.0001 * np.eye(2)
    assert f.x.shape == (2, 1)
    zs = [None, 1., 2.]
    m, c, _, _ = f.batch_filter(zs, update_first=False)
    assert m.shape == (3, 2, 1) and c.shape == (3, 2, 2)
    m2, c2, _, _ = f.batch_filter(zs, update_first=True)
    assert np.all(np.isfinite(m2))
    f.predict(); f.update(None)
    assert f.z.shape == (1, 1) and f.z[0, 0] is None
    assert np.array_equal(f.x_post, f.x)
    with pytest.raises(ValueError):
        f.update(np.array([1., 2., 3.]))
    with pytest.raises(ValueError):
        KalmanFilter(0, 1)


def test_procedural_known_answers():
    """test_kf.py:663-696: procedural form with exact known answers."""
    from filterpy_b200.kalman import predict, update
    x, P = predict(x=np.array([10.]), P=np.array([[3.]]), u=np.array([1.]), B=np.array([[1.]]), Q=2. ** 2)
    assert x[0] == 11 and P[0, 0] == 7
    x = np.array([1., 1.]); P = np.eye(2) * 2
    x, P = update(x, P, z=np.array([3.]), R=np.array([[2.]]), H=np.array([[1., 0.]]))
    assert abs(x[0] - 2) < 1e-12 and abs(x[1] - 1) < 1e-12
    assert abs(P[0, 0] - 1) < 1e-12 and abs(P[1, 1] - 2) < 1e-12


def test_singular_S_reports_status():
    from filterpy_b200.kalman import KalmanFilter
    kf = KalmanFilter(2, 1, n_filters=4)
    kf.P = np.zeros((2, 2)); kf.R = np.zeros((1, 1)); kf.H = np.array([[1., 0.]]); kf.Q = np.zeros((2, 2))
    kf.predict(); kf.update(np.ones((4, 1)))
    assert kf.status.cpu().numpy().tolist() == [1, 1, 1, 1]
    with pytest.raises(np.linalg.LinAlgError):
        kf.check()


@pytest.mark.parametrize("shape,dtype", [((9, 3), np.float64), ((6, 3), np.float64)], ids=["shape0-float64", "shape2-float64"])
@pytest.mark.parametrize("N", [1, 9, 10, 11, 160, 40003])
def test_rowblock_kernel_vs_oracle(shape, dtype, N):
    """The sub-warp row-block kernel (TMA bulk-staged; config C3's 9/3 fp64 and friends), ragged
    sizes included (the tail shorter than a warp tile runs on the catch-all kernel), with missing
    measurements."""
    _two_steps_vs_oracle(shape, dtype, N)


@pytest.mark.parametrize("shape,dtype", [((4, 2), np.float64), ((6, 3), np.float32)], ids=["shape1-float64", "shape3-float32"])
@pytest.mark.parametrize("N", [1, 9, 10, 11, 160, 40003])
def test_direct_kernel_vs_oracle(shape, dtype, N):
    """The same two steps on shapes of the register-tile kernel kf_direct (4/2 fp64, 6/3 fp32), which takes every
    call of these shapes whose per-filter arrays are 16-byte aligned."""
    _two_steps_vs_oracle(shape, dtype, N)


def _two_steps_vs_oracle(shape, dtype, N):
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.common import workloads as wl
    from oracle import kf as okf
    n, m = shape
    rng = np.random.default_rng(N + n)
    if (n, m) == (9, 3):
        w = wl.kf_bank_ca3d(N, seed=N, steps=2)
    elif (n, m) == (4, 2):
        w = wl.kf_bank_cv2d(N, seed=N, steps=2)
    else:
        A = rng.standard_normal((N, n, n)) * 0.3
        w = dict(x=rng.standard_normal((N, n)), P=np.einsum("nij,nkj->nik", A, A) + np.eye(n),
                 F=np.eye(n) + 0.1 * rng.standard_normal((N, n, n)), H=rng.standard_normal((N, m, n)),
                 Q=0.01 * np.eye(n) + np.zeros((N, n, n)), R=np.eye(m) * rng.uniform(0.2, 1.0, (N, 1, 1)),
                 zs=rng.standard_normal((2, N, m)))
    valid = rng.random((2, N)) > 0.25
    kf = KalmanFilter(n, m, n_filters=N, dtype=dtype, diagnostics=False)
    for k in "xPFHQR":
        setattr(kf, k, w[k])
    kf.alpha = 1.01
    x, P = w["x"], w["P"]
    for t in range(2):
        kf.predict(); kf.update(w["zs"][t], valid=valid[t])
        o = okf.kf_step_bank(x, P, w["zs"][t], w["F"], w["H"], w["Q"], w["R"], 1.01 ** 2, valid[t]); x, P = o["x"], o["P"]
    rtol = RTOL[dtype]       # fp32: 1e-3 (north_star); measured worst case 3.7e-4
    rel_close(kf.x.cpu().numpy(), x, rtol, "x"); rel_close(kf.P.cpu().numpy(), P, rtol, "P")


def test_c3_size_slice_independence_f64():
    """Config C3 per-GPU size (1.25 M filters, 9/3 fp64): a slice of the bank equals the slice run alone
    bit for bit, and a 4096-filter subset matches the oracle."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    from filterpy_b200.common import workloads as wl
    from oracle import kf as okf
    N = 1250000
    small = wl.kf_bank_ca3d(50000, seed=4321, steps=1)        # tiled 25x: the full per-GPU size, cheap to generate
    w = {k: np.concatenate([v] * 25, axis=1 if k == "zs" else 0) for k, v in small.items()}
    kf = KalmanFilter(9, 3, n_filters=N, dtype=np.float64, diagnostics=False)
    for k in "xPFHQR":
        setattr(kf, k, w[k])
    kf.predict(); kf.update(w["zs"][0])
    sl = slice(600000, 604090)
    sub = KalmanFilter(9, 3, n_filters=sl.stop - sl.start, dtype=np.float64, diagnostics=False)
    for k in "xPFHQR":
        setattr(sub, k, w[k][sl])
    sub.predict(); sub.update(w["zs"][0][sl])
    assert torch.equal(kf.x[sl], sub.x) and torch.equal(kf.P[sl], sub.P)
    o = okf.kf_step_bank(w["x"][sl], w["P"][sl], w["zs"][0][sl], w["F"][sl], w["H"][sl], w["Q"][sl], w["R"][sl])
    rel_close(sub.x.cpu().numpy(), o["x"], 1e-6, "x"); rel_close(sub.P.cpu().numpy(), o["P"], 1e-6, "P")


def test_x_post_survives_predict_and_state_assignment(golden):
    """x_post / P_post are lazy views of the state after an update (no per-step copy); they must
    still hold the posterior once a predict has moved x, P (kalman_filter.py:560-561) or the user
    assigned a new state."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    g = golden("kf_bank_4_2")
    N = g["x"].shape[0]
    kf = KalmanFilter(4, 2, n_filters=N, dtype=np.float64)
    kf.x, kf.P, kf.F, kf.H, kf.Q, kf.R = g["x"], g["P"], g["F"], g["H"], g["Q"], g["R"]
    z = torch.from_numpy(g["zs"][0]).cuda()
    kf.predict(); kf.update(z)
    post_x = kf.x.clone(); post_P = kf.P.clone()
    assert torch.equal(kf.x_post, post_x) and torch.equal(kf.P_post, post_P)
    kf.predict()
    prior_x = kf.x.clone()                                  # forces the stand-alone predict
    assert not torch.equal(prior_x, post_x)
    assert torch.equal(kf.x_post, post_x) and torch.equal(kf.P_post, post_P)
    assert torch.equal(kf.x_prior, prior_x)
    kf.update(torch.from_numpy(g["zs"][1]).cuda())
    assert torch.equal(kf.x_post, kf.x)
    post2 = kf.x.clone()
    kf.x = np.zeros((N, 4))                                 # a new state does not rewrite the stored posterior
    assert torch.equal(kf.x_post, post2)
    kf.update(None)                                         # z=None: posterior := prior (:515-520)
    assert torch.equal(kf.x_post, kf.x)


@pytest.mark.parametrize("diagnostics", [False, True])
def test_shared_models_in_launch_parameters_equal_device_models(golden, diagnostics):
    """A bank that shares F/H/Q/R carries them in the launch parameters when the mirror still holds
    host copies (bke_kf_args.*_host); reading an attribute hands out the live tensor, drops the
    host copy and the kernel reads device memory instead.  Same arithmetic, same result."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    g = golden("kf_bank_4_2")
    N = g["x"].shape[0]
    outs = []
    for device_path in (False, True):
        kf = KalmanFilter(4, 2, n_filters=N, dtype=np.float32, diagnostics=diagnostics)
        kf.x, kf.P = g["x"], g["P"]
        kf.F, kf.H, kf.Q, kf.R = g["F"][0], g["H"][0], g["Q"][0], g["R"][0]
        assert len(kf._host) == 4
        if device_path:
            assert kf.F.shape == (4, 4) and kf.H.shape == (2, 4)         # getters invalidate the host copies
            assert len(kf._host) == 2
        for t in range(3):
            kf.predict(); kf.update(torch.from_numpy(g["zs"][t].astype(np.float32)).cuda())
        outs.append((kf.x.cpu().numpy(), kf.P.cpu().numpy()))
    np.testing.assert_array_equal(outs[0][0], outs[1][0])
    np.testing.assert_array_equal(outs[0][1], outs[1][1])
    # and both agree with the oracle on the same shared models
    from oracle import kf as okf
    x, P = g["x"].copy(), g["P"].copy()
    for t in range(3):
        o = okf.kf_step_bank(x, P, g["zs"][t], g["F"][0], g["H"][0], g["Q"][0], g["R"][0])
        x, P = o["x"], o["P"]
    np.testing.assert_allclose(outs[0][0], x, rtol=1e-3, atol=1e-3 * np.abs(x).max())


@pytest.mark.parametrize("n,m", [(1, 1), (2, 1), (2, 2), (3, 1), (4, 1), (4, 2), (4, 4), (6, 2), (6, 3), (9, 3),
                                 (16, 4), (16, 2), (12, 3), (32, 4)])      # 16/x, 32/4 fp32: row-block instances; 12/3: catch-all
@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-6), (np.float32, 1e-3)])
@pytest.mark.parametrize("shared", [False, True])
def test_small_shapes_random_models_vs_oracle(n, m, dtype, tol, shared):
    """Every register-tile and row-block instance (and whatever kernel takes the other shapes) against
    the oracle on random well-conditioned models: 3 fused steps, optional outputs included, a ragged bank."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    from oracle import kf as okf
    rng = np.random.default_rng(100 * n + m)
    N = 1000 + 37

    def spd(k, cnt, scale):
        a = rng.normal(size=(cnt, k, k))
        return scale * (a @ np.swapaxes(a, -1, -2) / k + np.eye(k))
    cnt = 1 if shared else N
    F = np.eye(n) + 0.1 * rng.normal(size=(cnt, n, n))
    H = rng.normal(size=(cnt, m, n))
    Q, R, P0 = spd(n, cnt, 0.05), spd(m, cnt, 0.5), spd(n, N, 2.0)
    x0 = rng.normal(size=(N, n))
    zs = rng.normal(size=(3, N, m))
    kf = KalmanFilter(n, m, n_filters=N, dtype=dtype, diagnostics=True)
    kf.x, kf.P = x0, P0
    kf.F, kf.H, kf.Q, kf.R = (F[0], H[0], Q[0], R[0]) if shared else (F, H, Q, R)
    x, P = x0, P0
    for t in range(3):
        kf.predict(); kf.update(torch.from_numpy(zs[t]))
        o = okf.kf_step_bank(x, P, zs[t], F[0] if shared else F, H[0] if shared else H, Q[0] if shared else Q,
                             R[0] if shared else R)
        x, P = o["x"], o["P"]
    kf.check()
    scale = np.abs(P).max(axis=(1, 2))
    for got, want in [(kf.x, x), (kf.P, P), (kf.K, o["K"]), (kf.S, o["S"]), (kf.y, o["y"]), (kf.x_prior, o["x_prior"])]:
        got = got.cpu().numpy().astype(np.float64)
        ref_mag = np.abs(want).reshape(N, -1).max(axis=1).reshape((N,) + (1,) * (want.ndim - 1))
        assert np.all(np.abs(got - want) <= tol * (np.abs(want) + 0.05 * ref_mag + 1e-12)), (n, m, dtype)


@pytest.mark.parametrize("n,m,dtype", [(9, 3, np.float64), (9, 3, np.float32), (6, 3, np.float64),
                                       (16, 4, np.float64), (16, 4, np.float32), (16, 2, np.float64)])
@pytest.mark.parametrize("diagnostics", [False, True])
@pytest.mark.parametrize("shared", [False, True])
def test_rowblock_separate_predict_and_update_match_fused(n, m, dtype, diagnostics, shared):
    """The row-block kernel's predict-only and update-only modes (a stand-alone predict happens
    whenever the state is read between predict() and update(), and in every IMM step) against
    its fused mode, with a measurement mask and a ragged bank."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    rng = np.random.default_rng(n * 10 + m)
    N = 1037

    def spd(k, scale):
        a = rng.normal(size=(N, k, k))
        return scale * (a @ np.swapaxes(a, -1, -2) / k + np.eye(k))
    F = np.eye(n) + 0.1 * rng.normal(size=(N, n, n)); H = rng.normal(size=(N, m, n))
    Q, R, P0, x0 = spd(n, 0.05), spd(m, 0.5), spd(n, 2.0), rng.normal(size=(N, n))
    zs = rng.normal(size=(3, N, m)); valid = rng.random((3, N)) > 0.2
    banks = []
    for separate in (False, True):
        kf = KalmanFilter(n, m, n_filters=N, dtype=dtype, diagnostics=diagnostics)
        kf.x, kf.P = x0, P0
        kf.F, kf.H, kf.Q, kf.R = (F[0], H[0], Q[0], R[0]) if shared else (F, H, Q, R)
        for t in range(3):
            kf.predict()
            if separate:
                prior = kf.x.clone()                       # forces the stand-alone predict launch
            kf.update(torch.from_numpy(zs[t]), valid=valid[t])
        banks.append(kf)
    tol = 1e-9 if dtype is np.float64 else 1e-4
    if n == 16 and shared and dtype is np.float32:
        # shared-model fp32 banks with dim_x = 16 run on the tensor cores (csrc/kf_tc.cu): the stand-alone predict as
        # three-term TF32 products, the fused step with the Joseph form expanded — different arithmetic from the
        # row-block update of the two-launch sequence, so each bank is held to north_star's fp32 bound against the fp64
        # oracle instead of to the other bank (fp32 itself sits at 3e-4 under this metric: x has cancelling entries)
        from oracle import kf as okf
        x, P = x0, P0
        for t in range(3):
            o = okf.kf_step_bank(x, P, zs[t], F[0], H[0], Q[0], R[0], valid=valid[t])
            x, P = o["x"], o["P"]
        for kf in banks:
            rel_close(kf.x.cpu().numpy(), x, 1e-3, "x vs oracle")
            rel_close(kf.P.cpu().numpy(), P, 1e-3, "P vs oracle")
        return
    a, b = banks
    rel_close(b.x.cpu().numpy(), a.x.cpu().numpy(), tol, "x")
    rel_close(b.P.cpu().numpy(), a.P.cpu().numpy(), tol, "P")
    if diagnostics:
        rel_close(b.K.cpu().numpy(), a.K.cpu().numpy(), tol * 10, "K")
        rel_close(b.x_prior.cpu().numpy(), a.x_prior.cpu().numpy(), tol, "x_prior")
        rel_close(b.P_prior.cpu().numpy(), a.P_prior.cpu().numpy(), tol, "P_prior")
        np.testing.assert_allclose(b.log_likelihood.cpu().numpy()[valid[2]], a.log_likelihood.cpu().numpy()[valid[2]],
                                   rtol=tol * 100, atol=tol * 100)
