"""GPU: KalmanFilter.update_sequential / update_correlated on every register-tile instance and on the catch-all
kernel, in fp32 and fp64, against the reference's golden vectors and the fp64 oracle; the fused predict, the valid
mask, status, single mode, capture and the torch ops."""
import numpy as np
import pytest
import torch

from filterpy_b200 import _lib
from filterpy_b200.kalman import KalmanFilter
from oracle import kf as okf

import kf_forms_oracle as kfo

from test_oracle_kf_forms import CORR, SEQ, _block_args, run_corr_bank, run_seq_bank

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {np.float64: 1e-6, np.float32: 1e-3}

# the register tiles of the correlated step (kf_direct.cu's shapes) and of the row block, (dim_x, L)
CORR_TILES = [(4, 2), (2, 1), (1, 1), (2, 2), (3, 1), (4, 1), (4, 4)]
CORR_TILES_F32 = [(6, 3), (6, 2)]
ROW_TILES = [(1, 1), (2, 1), (2, 2), (3, 1), (4, 1), (4, 2), (4, 3), (4, 4)]
ROW_TILES_F32 = [(6, 1), (6, 2), (6, 3)]


def _err(a, b):
    a = a.detach().double().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b)), "NaN pattern differs"
    fin = np.isfinite(b)
    return np.abs(a[fin] - b[fin]).max(initial=0) / max(np.abs(b[fin]).max(initial=0), 1e-300)


def _bank(g, dtype, control=False, M=False):
    N, n = g["x"].shape
    m = g["H"].shape[1]
    kf = KalmanFilter(n, m, n_filters=N, dtype=dtype, device=DEV)
    kf.x, kf.P, kf.F, kf.Q, kf.H, kf.R = g["x"], g["P"], g["F"], g["Q"], g["H"], g["R"]
    if M:
        kf.M = g["M"]
    return kf


def _predict(kf, control):
    # a zero control input leaves the arithmetic alone and sends the step to the catch-all kernel
    if control:
        kf.predict(u=np.zeros(1), B=np.zeros((kf.dim_x, 1)))
    else:
        kf.predict()


def _run_seq(kf, g, control=False):
    for t in range(g["zs"].shape[0]):
        _predict(kf, control)
        for k, (s, L) in enumerate(zip(g["starts"], g["lens"])):
            Ri, Hi = _block_args(g, k)
            kf.update_sequential(int(s), g["zs"][t][:, s:s + L], R_i=Ri, H_i=Hi, valid=g["valid"][t])


@pytest.mark.parametrize("control", [False, True], ids=["tile", "catchall"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", SEQ)
def test_sequential_golden(golden, name, dtype, control):
    g = golden(name)
    kf = _bank(g, dtype)
    _run_seq(kf, g, control)
    assert int((kf.status != 0).sum()) == 0
    for k, t in (("x", kf.x), ("P", kf.P), ("y", kf.y), ("K", kf.K), ("z", kf.z)):
        assert _err(t, g["out_" + k]) < TOL[dtype], k


@pytest.mark.parametrize("control", [False, True], ids=["tile", "catchall"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", CORR)
def test_correlated_golden(golden, name, dtype, control):
    g = golden(name)
    kf = _bank(g, dtype, M=True)
    status = torch.zeros(g["x"].shape[0], dtype=torch.int32, device=DEV)
    for t in range(g["zs"].shape[0]):
        _predict(kf, control)
        kf.update_correlated(g["zs"][t], valid=g["valid"][t])
        status |= kf.status
    np.testing.assert_array_equal(status.cpu().numpy(), g["out_status"])
    ok = g["out_status"] == 0
    assert _err(kf.x, g["out_x"]) < TOL[dtype] and _err(kf.P, g["out_P"]) < TOL[dtype]
    for k, t in (("y", kf.y), ("K", kf.K), ("S", kf.S), ("SI", kf.SI)):
        assert _err(t[torch.from_numpy(ok).to(DEV)], g["out_" + k][ok]) < TOL[dtype], k
    have = np.isfinite(g["out_ll"])
    assert _err(kf.log_likelihood[torch.from_numpy(have).to(DEV)], g["out_ll"][have]) < TOL[dtype]


def _random(n, m, N, seed):
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(N, n, n))
    B = rng.normal(size=(N, m, m))
    C = rng.normal(size=(N, n, n)) * .3
    return dict(x=rng.normal(size=(N, n)), P=A @ np.swapaxes(A, 1, 2) + np.eye(n), F=np.eye(n) + 0.1 * rng.normal(size=(N, n, n)),
                Q=C @ np.swapaxes(C, 1, 2) + .01 * np.eye(n), H=rng.normal(size=(N, m, n)),
                R=B @ np.swapaxes(B, 1, 2) + np.eye(m), M=0.05 * rng.normal(size=(N, n, m)),
                z=rng.normal(size=(N, m)), valid=rng.random(N) > 0.2)


def _instances(tiles, tiles_f32):
    out = [(n, m, d, c) for (n, m) in tiles for d in (np.float64, np.float32) for c in (False, True)]
    out += [(n, m, np.float32, c) for (n, m) in tiles_f32 for c in (False, True)]
    out += [(n, m, np.float64, False) for (n, m) in tiles_f32]        # fp64 6/x: the catch-all
    out += [(5, 3, d, False) for d in (np.float64, np.float32)]       # no register tile
    return out


@pytest.mark.parametrize("n,m,dtype,control", _instances(CORR_TILES, CORR_TILES_F32))
def test_correlated_instances_against_oracle(n, m, dtype, control):
    w = _random(n, m, 300, seed=n * 10 + m)
    kf = _bank(dict(w, x=w["x"]), dtype, M=True)
    _predict(kf, control)
    kf.update_correlated(w["z"], valid=w["valid"])
    xp, Pp = okf.kf_predict_bank(w["x"], w["P"], w["F"], w["Q"])
    o = kfo.kf_update_correlated_bank(xp, Pp, w["z"], w["H"], w["R"], w["M"], valid=w["valid"])
    assert _err(kf.x_prior, xp) < TOL[dtype]
    for k in ("x", "P", "y"):
        assert _err(getattr(kf, k), o[k]) < TOL[dtype], k
    v = torch.from_numpy(w["valid"]).to(DEV)
    for k in ("K", "S", "SI"):
        assert _err(getattr(kf, k)[v], o[k][w["valid"]]) < TOL[dtype], k
    ll = okf.log_likelihood_bank(o["y"], o["S"])
    assert _err(kf.log_likelihood[v], ll[w["valid"]]) < TOL[dtype]
    # shared M: stride 0
    kf2 = _bank(w, dtype)
    kf2.M = w["M"][0]
    kf2.update_correlated(w["z"])
    o2 = kfo.kf_update_correlated_bank(w["x"], w["P"], w["z"], w["H"], w["R"], w["M"][0])
    assert _err(kf2.P, o2["P"]) < TOL[dtype]


def _row_instances():
    out = []
    for (n, L) in ROW_TILES + ROW_TILES_F32:
        m = max(L + 1, 3)            # a block inside a larger z: start > 0 and rows after it
        for d in ((np.float64, np.float32) if (n, L) in ROW_TILES else (np.float32,)):
            for c in (False, True):
                out.append((n, m, L, d, c))
    out += [(5, 4, 2, np.float64, False), (5, 4, 1, np.float32, False), (6, 3, 2, np.float64, False)]
    return out


@pytest.mark.parametrize("n,m,L,dtype,control", _row_instances())
def test_row_instances_against_oracle(n, m, L, dtype, control):
    w = _random(n, m, 300, seed=n * 100 + m * 10 + L)
    start = m - L - 1 if m - L - 1 > 0 else 0
    kf = _bank(w, dtype)
    N = w["x"].shape[0]
    y0 = np.random.default_rng(1).normal(size=(N, m)); K0 = np.random.default_rng(2).normal(size=(N, n, m))
    kf.y.copy_(torch.from_numpy(y0)); kf.K.copy_(torch.from_numpy(K0))
    kf.update(w["z"])                          # gives the z record its starting rows
    z0 = w["z"]
    y0, K0 = kf.y.double().cpu().numpy(), kf.K.double().cpu().numpy()
    x0, P0 = kf.x.double().cpu().numpy(), kf.P.double().cpu().numpy()
    zi = w["z"][:, start:start + L] + 0.5
    _predict(kf, control)
    kf.update_sequential(start, zi, valid=w["valid"])
    xp, Pp = okf.kf_predict_bank(x0, P0, w["F"], w["Q"])
    o = kfo.kf_update_sequential_bank(xp, Pp, start, zi, w["H"], w["R"], y0, K0, z0, valid=w["valid"])
    for k in ("x", "P", "y", "K", "z"):
        assert _err(getattr(kf, k), o[k]) < TOL[dtype], k


def test_fused_predict_equals_predict_then_call():
    w = _random(4, 2, 500, seed=3)
    for form in ("seq", "corr"):
        a, b = _bank(w, np.float64, M=True), _bank(w, np.float64, M=True)
        a.predict()
        b.predict(); b.x                      # reading x runs the predict on its own
        for kf in (a, b):
            if form == "seq":
                kf.update_sequential(1, w["z"][:, 1:], valid=w["valid"])
            else:
                kf.update_correlated(w["z"], valid=w["valid"])
        assert torch.equal(a.x, b.x) and torch.equal(a.P, b.P)
        assert torch.equal(a.x_prior, b.x_prior)


def test_valid_mask_keeps_the_prior_and_the_block():
    w = _random(4, 2, 200, seed=4)
    kf = _bank(w, np.float64)
    kf.update(w["z"])
    y0, K0, z0 = kf.y.clone(), kf.K.clone(), kf.z.clone()
    kf.predict()
    v = torch.from_numpy(w["valid"]).to(DEV)
    kf.update_sequential(0, w["z"][:, :1] + 1.0, valid=w["valid"])
    assert torch.equal(kf.x[~v], kf.x_prior[~v])
    assert torch.equal(kf.y[~v], y0[~v]) and torch.equal(kf.K[~v], K0[~v]) and torch.equal(kf.z[~v], z0[~v])
    assert torch.equal(kf.y[v, 1], y0[v, 1]) and torch.equal(kf.K[v][:, :, 1], K0[v][:, :, 1])
    assert not torch.equal(kf.y[v, 0], y0[v, 0])


def test_status_singular_blocks():
    N = 8
    w = _random(3, 3, N, seed=5)
    kf = _bank(w, np.float64)
    Ri = np.zeros((N, 2, 2)); Ri[::2] = [[1., 1.], [1., 1.]]; Ri[1::2] = np.eye(2)
    Hi = np.zeros((N, 2, 3)); Hi[1::2] = w["H"][1::2, :2]
    kf.update_sequential(0, w["z"][:, :2], R_i=Ri, H_i=Hi)
    np.testing.assert_array_equal(kf.status.cpu().numpy(), np.tile([1, 0], N // 2))
    with pytest.raises(np.linalg.LinAlgError):
        kf.check()
    assert torch.equal(kf.x[::2], torch.from_numpy(w["x"][::2]).to(DEV))
    # L = 1 with S = 0: inf / nan, and no status
    kf.update_sequential(2, w["z"][:, 2:], R_i=0.0, H_i=np.zeros(3))
    assert int(kf.status.abs().sum()) == 0
    # a singular correlated S
    kf = _bank(w, np.float64)
    kf.H = np.zeros((3, 3)); kf.R = np.ones((3, 3))
    kf.update_correlated(w["z"])
    assert (kf.status == _lib.BKE_STATUS_SINGULAR_S).all()


def test_single_mode_shapes(golden):
    g = golden("kf_forms_corr_2_1")
    kf = KalmanFilter(2, 1)
    kf.x = g["x"][0].reshape(2, 1); kf.P = g["P"][0]; kf.F = g["F"][0]; kf.Q = g["Q"][0]
    kf.H = g["H"][0]; kf.R = g["R"][0]; kf.M = g["M"][0]
    assert kf.M.shape == (2, 1)
    for t in range(10):
        kf.predict()
        kf.update_correlated(3.)
    assert kf.x.shape == (2, 1) and kf.P.shape == (2, 2) and kf.K.shape == (2, 1) and kf.y.shape == (1, 1)
    assert _err(kf.x.reshape(-1), g["out_x"][0]) < 1e-6 and _err(kf.P, g["out_P"][0]) < 1e-6
    assert np.isfinite(kf.log_likelihood) and np.isfinite(kf.mahalanobis)
    assert np.array_equal(kf.x_post, kf.x)
    g = golden("kf_forms_seq_cv63_12")
    kf = KalmanFilter(6, 3)
    kf.x = np.zeros((6, 1)); kf.P = g["P"][0]; kf.F = g["F"][0]; kf.Q = g["Q"][0]; kf.H = g["H"][0]; kf.R = g["R"][0]
    assert np.zeros((6, 3)).shape == KalmanFilter(6, 3).M.shape
    for t in range(g["zs"].shape[0]):
        kf.predict()
        z = g["zs"][t, 0]
        kf.update_sequential(0, z[0])
        kf.update_sequential(1, z[1:])
    assert kf.x.shape == (6, 1) and kf.z.shape == (3, 1) and kf.y.shape == (3, 1)
    assert _err(kf.x.reshape(-1), g["out_x"][0]) < 1e-6 and _err(kf.P, g["out_P"][0]) < 1e-6
    assert _err(kf.x.reshape(-1), g["upd_x"][0]) < 1e-9
    with pytest.raises(ValueError):
        kf.update_sequential(2, [1., 2.])


@pytest.mark.parametrize("tag", ["111", "12", "21"])
def test_splits_agree_with_update_fp64(golden, tag):
    g = golden("kf_forms_seq_cv63_" + tag)
    a, b = _bank(g, np.float64), _bank(g, np.float64)
    _run_seq(a, g)
    for t in range(g["zs"].shape[0]):
        b.predict(); b.update(g["zs"][t])
    assert _err(a.x, b.x.double().cpu().numpy()) < 1e-9 and _err(a.P, b.P.double().cpu().numpy()) < 1e-9


def test_capture_keeps_separate_launches_and_replays_equal_eager():
    w = _random(4, 2, 4096, seed=6)
    zb = torch.from_numpy(w["z"]).float().to(DEV)

    def build():
        kf = KalmanFilter(4, 2, n_filters=4096, dtype=np.float32, device=DEV, diagnostics=False)
        for k in "xPFQHR":
            setattr(kf, k, w[k])
        kf.M = w["M"]
        return kf

    def fn(kf):
        kf.predict(); kf.update(zb)
        kf.predict(); kf.update_sequential(0, zb[:, :1])
        kf.predict(); kf.update_correlated(zb)

    kf = build()
    graph = kf.capture(lambda: fn(kf), warmup=1)
    assert not graph.fused_steps and graph.launches == 3
    kf.x.copy_(torch.from_numpy(w["x"])); kf.P.copy_(torch.from_numpy(w["P"]))
    ref = build()
    for _ in range(3):
        graph.replay()
        fn(ref)
    torch.cuda.synchronize()
    assert torch.equal(kf.x, ref.x) and torch.equal(kf.P, ref.P)


def test_torch_ops_equal_ctypes_path():
    from filterpy_b200 import torch_ops
    torch_ops.load()
    w = _random(4, 2, 1000, seed=7)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(DEV) for k, v in w.items() if k != "valid"}
    x, P = torch.ops.bke.kf_step_correlated(t["x"], t["P"], t["F"], t["H"], t["Q"], t["R"], t["M"], t["z"])
    kf = _bank(w, np.float64, M=True)
    kf.predict(); kf.update_correlated(w["z"])
    # (the bank writes its diagnostics, so it may run another instance of the same arithmetic)
    assert _err(x, kf.x.cpu().numpy()) < 1e-12 and _err(P, kf.P.cpu().numpy()) < 1e-12
    zi = t["z"][:, 1:].contiguous()
    x, P = torch.ops.bke.kf_update_rows(t["x"], t["P"], t["F"], t["H"], t["Q"], t["R"], zi, 1)
    kf = _bank(w, np.float64)
    kf.predict(); kf.update_sequential(1, zi)
    assert _err(x, kf.x.cpu().numpy()) < 1e-12 and _err(P, kf.P.cpu().numpy()) < 1e-12
