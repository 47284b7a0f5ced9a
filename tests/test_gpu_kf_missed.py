"""Missed measurements (z_valid == 0, ``update(None)``) on every KF kernel path.

The reference's ``update(None)`` sets y = 0, keeps K, S and SI, and clears the cached log-likelihood, which
its property then recomputes as logpdf(0; 0, S) of the kept S (kalman_filter.py:511-520, :1203-1210).  The
kernels write y = 0 and leave K, S, SI and log_likelihood as they were (include/bke.h); KalmanFilter.update
computes the reference's log-likelihood from the kept S.  These tests pin both halves: the kept outputs on
every kernel behind bke_kf_step, and the log-likelihood the mirror reports after a miss."""
import ctypes
import math
import sys

import numpy as np
import pytest

from gpu_harness import rel_close, RTOL

pytestmark = pytest.mark.gpu
F32, F64 = np.float32, np.float64
SENTINEL = -3.25


def _problem(n, m, N, seed, du=0):
    rng = np.random.default_rng(seed)

    def spd(k, cnt, scale):
        a = rng.normal(size=(cnt, k, k))
        return scale * (a @ np.swapaxes(a, -1, -2) / k + np.eye(k))
    return dict(x=rng.normal(size=(N, n)), P=spd(n, N, 2.0),
                F=np.eye(n) + 0.1 * rng.normal(size=(N, n, n)), Q=spd(n, N, 0.05),
                H=rng.normal(size=(N, m, n)), R=spd(m, N, 0.5), z=rng.normal(size=(N, m)) * 2,
                B=rng.normal(size=(N, n, du)), u=rng.normal(size=(N, du)), valid=rng.random(N) < 0.5)


# (id, dim_x, dim_z, dtype, layout).  layout: "per" every model per filter; "shared" every model shared by the
# bank; "host" shared with host copies in the launch parameters; "shared_FQ" F and Q shared, H and R per
# filter; "misaligned" x one element past a 16-byte boundary; "control" a per-filter B u
PATHS = [
    ("tma_per", 4, 2, F32, "per"), ("tma_shared", 4, 2, F32, "shared"), ("tma_host", 4, 2, F32, "host"),
    ("direct_1_1", 1, 1, F64, "per"), ("direct_2_1", 2, 1, F64, "per"), ("direct_2_2", 2, 2, F64, "per"),
    ("direct_3_1", 3, 1, F64, "per"), ("direct_4_1", 4, 1, F64, "per"), ("direct_4_4", 4, 4, F64, "per"),
    ("direct_4_2_f64", 4, 2, F64, "per"), ("direct_6_3_f32", 6, 3, F32, "per"), ("direct_6_2_f32", 6, 2, F32, "per"),
    ("rowblock_9_3", 9, 3, F64, "per"), ("rowblock_9_3_f32", 9, 3, F32, "per"), ("rowblock_6_3_f64", 6, 3, F64, "per"),
    ("rowblock_16_4_f64", 16, 4, F64, "per"), ("rowblock_16_2", 16, 2, F32, "per"), ("rowblock_32_4", 32, 4, F32, "per"),
    ("tc_16_4_fused", 16, 4, F32, "shared"), ("tc_32_4_two_launches", 32, 4, F32, "shared_FQ"),
    ("generic_12_3", 12, 3, F64, "per"), ("generic_misaligned_x", 4, 2, F64, "misaligned"),
    ("generic_control", 3, 2, F64, "control"),
]


@pytest.mark.parametrize("name,n,m,dtype,layout", PATHS, ids=[p[0] for p in PATHS])
def test_masked_filters_keep_K_S_SI_and_log_likelihood(name, n, m, dtype, layout):
    """bke_kf_step (predict + update) with half the filters masked: for those, K, S, SI and log_likelihood are
    bit for bit what they held before, y == 0, x / P are the oracle's predict and status is 0; the others match
    the oracle's update."""
    import torch
    from filterpy_b200 import _lib
    from oracle import kf as okf
    N = 1037
    du = 2 if layout == "control" else 0
    p = _problem(n, m, N, seed=n * 31 + m, du=du)
    if layout in ("shared", "host"):
        for k in "FQHR":
            p[k] = p[k][0]
    elif layout == "shared_FQ":
        p["F"], p["Q"] = p["F"][0], p["Q"][0]
    p = {k: (v.astype(dtype).astype(F64) if k != "valid" else v) for k, v in p.items()}
    tdt = torch.float32 if dtype == F32 else torch.float64

    def dev(a, offset=0):
        a = np.ascontiguousarray(a, dtype=dtype)
        buf = torch.zeros(offset + a.size, dtype=tdt, device="cuda")
        buf[offset:] = torch.from_numpy(a.reshape(-1)).cuda()
        return buf[offset:].view(a.shape)
    x = dev(p["x"], 1 if layout == "misaligned" else 0)
    P = dev(p["P"])
    mats = {k: dev(p[k]) for k in "FQHR"}
    z = dev(p["z"])
    valid = torch.from_numpy(p["valid"].astype(np.uint8)).cuda()
    outs = {k: torch.full(s, SENTINEL, dtype=tdt, device="cuda")
            for k, s in dict(K=(N, n, m), y=(N, m), S=(N, m, m), SI=(N, m, m), ll=(N,)).items()}
    status = torch.zeros(N, dtype=torch.int32, device="cuda")
    a = _lib.KfArgs()
    a.n_filters, a.dim_x, a.dim_z, a.dim_u = N, n, m, du
    a.dtype = _lib.BKE_F32 if dtype == F32 else _lib.BKE_F64
    a.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
    a.alpha_sq = 1.0
    a.x = a.x_out = x.data_ptr(); a.P = a.P_out = P.data_ptr()
    for k in "FQHR":
        setattr(a, k, mats[k].data_ptr())
        setattr(a, k + "_stride", 0 if mats[k].dim() == 2 else mats[k].shape[1] * mats[k].shape[2])
    host = []
    if layout == "host":
        host = [np.ascontiguousarray(p[k], dtype=dtype) for k in "FQHR"]
        a.F_host, a.Q_host, a.H_host, a.R_host = (h.ctypes.data for h in host)
    if du:
        B, u = dev(p["B"]), dev(p["u"])
        a.B, a.B_stride, a.u, a.u_stride = B.data_ptr(), n * du, u.data_ptr(), du
    a.z, a.z_valid = z.data_ptr(), valid.data_ptr()
    a.K, a.y, a.S, a.SI, a.log_likelihood = (outs[k].data_ptr() for k in ("K", "y", "S", "SI", "ll"))
    a.status = status.data_ptr()
    lib = _lib.load()
    assert lib.bke_kf_step(ctypes.byref(a), torch.cuda.current_stream().cuda_stream) == _lib.BKE_OK, lib.bke_last_error()
    torch.cuda.synchronize()

    v = p["valid"]
    xp, Pp = okf.kf_predict_bank(p["x"], p["P"], p["F"], p["Q"], 1.0, p["B"] if du else None, p["u"] if du else None)
    o = okf.kf_update_bank(xp, Pp, p["z"], p["H"], p["R"], v)
    got = {k: t.cpu().numpy() for k, t in outs.items()}
    for k in ("K", "S", "SI", "ll"):
        assert np.all(got[k][~v] == dtype(SENTINEL)), "%s: %s written for a filter without a measurement" % (name, k)
    assert np.all(got["y"][~v] == 0)
    assert np.all(status.cpu().numpy() == 0)
    rtol = RTOL[dtype]
    xg, Pg = x.cpu().numpy(), P.cpu().numpy()
    rel_close(xg[~v], xp[~v], rtol, name + " x (masked: the prior)")
    rel_close(Pg[~v], Pp[~v], rtol, name + " P (masked: the prior)")
    rel_close(xg[v], o["x"][v], rtol, name + " x")
    rel_close(Pg[v], o["P"][v], rtol, name + " P")
    for k in ("K", "S", "SI"):
        rel_close(got[k][v], o[k][v], rtol, name + " " + k)
    rel_close(got["y"][v], o["y"][v], max(rtol, 1e-5), name + " y")
    ll = okf.log_likelihood_bank(o["y"][v], o["S"][v])
    np.testing.assert_allclose(got["ll"][v], ll, rtol=rtol, atol=rtol)


def _missed_ll(S):
    """log N(0; 0, S) in fp64, -inf where det S <= 0 (scipy's value for S = 0)."""
    from oracle import kf as okf
    return okf.missed_log_likelihood_bank(np.asarray(S, F64))


# one bank per kernel family: (id, dim_x, dim_z, dtype, models shared by the bank)
FAMILIES = [("tma", 4, 2, F32, False), ("direct", 4, 2, F64, False), ("rowblock", 9, 3, F64, False),
            ("tc", 16, 4, F32, True), ("generic", 12, 3, F64, False)]


@pytest.mark.parametrize("name,n,m,dtype,shared", FAMILIES, ids=[f[0] for f in FAMILIES])
def test_bank_log_likelihood_after_a_miss(name, n, m, dtype, shared):
    """Bank mode: a filter masked on its first epoch reports -inf (S is still zero); one masked later reports
    logpdf(0, S) of the S it kept; update(None) does so for the whole bank; a filter with a measurement
    reports its own log N(y; 0, S)."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    N = 37
    p = _problem(n, m, N, seed=n + 100 * m)
    kf = KalmanFilter(n, m, n_filters=N, dtype=dtype)
    kf.x, kf.P = p["x"], p["P"]
    for k in "FQHR":
        setattr(kf, k, p[k][0] if shared else p[k])
    tol = 1e-10 if dtype == F64 else 1e-4
    rng = np.random.default_rng(3)
    masks = [np.arange(N) % 3 != 0, rng.random(N) < 0.5, None]
    S_before = None
    for t, v in enumerate(masks):
        kf.predict()
        z = rng.normal(size=(N, m))
        if v is None:
            kf.update(None)
            v = np.zeros(N, bool)
        else:
            kf.update(torch.from_numpy(z), valid=torch.from_numpy(v))
        ll = kf.log_likelihood.cpu().numpy().astype(F64)
        S = kf.S.cpu().numpy()
        if S_before is not None:
            assert np.array_equal(S[~v], S_before[~v])                   # the kept S
        want = _missed_ll(S)
        if t == 0:
            assert np.all(np.isneginf(ll[~v])) and np.all(np.isneginf(want[~v]))
        else:
            np.testing.assert_allclose(ll[~v], want[~v], rtol=tol, atol=tol)
        assert np.all(np.isfinite(ll[v]))
        if dtype == F64:
            lk = kf.likelihood.cpu().numpy()
            np.testing.assert_allclose(lk[~v], np.maximum(np.exp(want[~v]), sys.float_info.min), rtol=1e-10, atol=0)
        S_before = S


@pytest.mark.parametrize("n,m", [(4, 2), (2, 1), (9, 3)])
def test_single_filter_log_likelihood_after_a_miss(n, m):
    """Single mode, as the reference: update(None) before any measurement gives -inf and likelihood float min;
    after a measurement, update(None) gives scipy's logpdf(0; 0, S) of the kept S."""
    from scipy.stats import multivariate_normal
    from filterpy_b200.kalman import KalmanFilter
    p = _problem(n, m, 1, seed=n * m)
    kf = KalmanFilter(n, m)
    kf.x, kf.P = p["x"][0], p["P"][0]
    kf.F, kf.Q, kf.H, kf.R = p["F"][0], p["Q"][0], p["H"][0], p["R"][0]
    kf.predict(); kf.update(None)
    assert kf.log_likelihood == -math.inf and kf.likelihood == sys.float_info.min
    kf.predict(); kf.update(p["z"][0])
    ll_z = kf.log_likelihood
    kf.predict(); kf.update(None)
    want = multivariate_normal.logpdf(np.zeros(m), None, kf.S, True)
    assert kf.log_likelihood != ll_z
    assert abs(kf.log_likelihood - want) <= 1e-12 * max(1.0, abs(want))
    assert abs(kf.likelihood - math.exp(want)) <= 1e-12 * math.exp(want)
    assert np.all(kf.y == 0)


def test_packed_record_keeps_outputs_of_masked_filters():
    """The 4/2 fp32 bank with per-filter models steps from the packed model record from its second launch
    with unchanged models on; masked filters keep K, S and SI there too, and report logpdf(0, S)."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    N = 1037
    p = _problem(4, 2, N, seed=11)
    kf = KalmanFilter(4, 2, n_filters=N, dtype=F32)
    kf.x, kf.P = p["x"], p["P"]
    for k in "FQHR":
        t = p[k]
        setattr(kf, k, (t + np.swapaxes(t, -1, -2)) / 2 if k in "QR" else t)      # exactly symmetric Q, R
    rng = np.random.default_rng(2)
    prev = None
    for t in range(4):
        v = np.ones(N, bool) if t == 0 else rng.random(N) < 0.5
        kf.predict(); kf.update(torch.from_numpy(rng.normal(size=(N, 2)).astype(F32)), valid=torch.from_numpy(v))
        cur = {k: getattr(kf, k).cpu().numpy() for k in ("K", "S", "SI", "y")}
        ll = kf.log_likelihood.cpu().numpy().astype(F64)
        if prev is not None:
            for k in ("K", "S", "SI"):
                assert np.array_equal(cur[k][~v], prev[k][~v]), k
            assert np.all(cur["y"][~v] == 0)
            np.testing.assert_allclose(ll[~v], _missed_ll(cur["S"][~v]), rtol=1e-4, atol=1e-4)
        prev = cur
    assert kf._sym_buf is not None                  # the steps after the first ran on the packed record
