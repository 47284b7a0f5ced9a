"""GPU parity: fixed-lag smoother banks (CUDA through the mirror and the torch op) against the reference's golden
vectors and the vectorised oracle."""
import numpy as np
import pytest

from gpu_harness import rel_close, RTOL
from test_oracle_fls import BANKS, bank_inputs

pytestmark = pytest.mark.gpu

FUSED_CAP = 16                                   # BKE_FLS_FUSED_MAX_LAG


def per_filter(a):
    """[T, Nf, n] -> [Nf, T, n]: rel_close measures near-zero entries against each filter's own scale."""
    return np.swapaxes(np.asarray(a, np.float64), 0, 1)


def make(g, dtype, Nf=None, shared=False, N="golden", diagnostics=True):
    from filterpy_b200.kalman import FixedLagSmoother
    Nf = g["x"].shape[0] if Nf is None else Nf
    n, m = g["x"].shape[1], np.shape(g["H"])[-2]
    s = FixedLagSmoother(n, m, int(g["N"]) if N == "golden" else N, dim_u=g["B"].shape[-1] if "B" in g else 0,
                         n_filters=Nf, dtype=dtype, diagnostics=diagnostics)
    pick = (lambda a: a[0] if np.ndim(a) == 3 else a) if shared else (lambda a: a[:Nf] if np.ndim(a) == 3 else a)
    s.x = g["x"][:Nf]; s.P = g["P"][:Nf]
    s.F = pick(g["F"]); s.H = pick(g["H"]); s.Q = pick(g["Q"]); s.R = pick(g["R"])
    if "B" in g:
        s.B = g["B"]
    return s


def online(s, g, Nf=None):
    Nf = g["x"].shape[0] if Nf is None else Nf
    for t in range(g["zs"].shape[0]):
        s.smooth(g["zs"][t][:Nf], g["us"][t][:Nf] if "us" in g else None)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", BANKS)
def test_smooth_batch_vs_reference_golden(golden, name, dtype):
    """Every golden case through smooth_batch: 2/1, 4/2, 1/1 and the lags up to the cap run the fused kernel;
    6/3, 9/3, the control input, N = 20 and N >= T (above the cap) the per-epoch path."""
    g = golden(name)
    s = make(g, dtype)
    xs, xh = s.smooth_batch(g["zs"], int(g["N"]), us=g["us"] if "us" in g else None)
    rel_close(per_filter(xs.cpu().numpy()), per_filter(g["ref_xs"]), RTOL[dtype], "xSmooth " + name)
    rel_close(per_filter(xh.cpu().numpy()), per_filter(g["ref_xhat"]), RTOL[dtype], "xhat " + name)
    assert int(s.batch_status.sum().item()) == 0


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", BANKS)
def test_online_equals_batch_bit_for_bit(golden, name, dtype):
    """T calls of smooth() give smooth_batch's rows bit for bit on both paths; smooth_batch leaves the object's
    state and history as they were."""
    g = golden(name)
    s = make(g, dtype)
    online(s, g)
    b = make(g, dtype)
    x0, P0 = b.x.clone(), b.P.clone()
    xs, xh = b.smooth_batch(g["zs"], int(g["N"]), us=g["us"] if "us" in g else None)
    assert np.array_equal(s.xSmooth.cpu().numpy(), xs.cpu().numpy())
    assert np.array_equal(s.x.cpu().numpy(), xh[-1].cpu().numpy())
    assert b.count == 0 and b.xSmooth.shape[0] == 0
    assert np.array_equal(b.x.cpu().numpy(), x0.cpu().numpy()) and np.array_equal(b.P.cpu().numpy(), P0.cpu().numpy())
    rel_close(per_filter(s.xSmooth.cpu().numpy()), per_filter(g["ref_xs"]), RTOL[dtype], "online " + name)
    assert s.count == g["zs"].shape[0]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("lag", [4, FUSED_CAP + 2])
def test_online_sequence_golden(golden, dtype, lag):
    """The recorded smooth() sequence: xSmooth, x, P, y, S and count after calls 1, N-1, N, N+1 and the last;
    at lag 4 (the recorded N) on the fused kernel, and the same epochs at a lag above the cap (per-epoch path)
    against the oracle."""
    from oracle import fls as ofl
    g = golden("fls_online")
    s = make(g, dtype, N=lag)
    calls = [int(c) for c in g["rec_calls"]]
    for t in range(calls[-1]):
        s.smooth(g["zs"][t])
        c = t + 1
        if c not in calls:
            continue
        if lag == int(g["N"]):
            ref = dict(xs=g["ref_xs_%d" % c], x=g["ref_x_%d" % c], P=g["ref_P_%d" % c], y=g["ref_y_%d" % c],
                       S=g["ref_S_%d" % c])
            assert s.count == c and (g["ref_count_%d" % c] == c).all()
        else:
            ref = ofl.fls_bank(g["x"], g["P"], g["F"], g["H"], g["Q"], g["R"], g["zs"][:c], lag)
        rel_close(per_filter(s.xSmooth.cpu().numpy()), per_filter(ref["xs"]), RTOL[dtype], "xSmooth c=%d" % c)
        for k in ("x", "P", "y", "S"):
            rel_close(getattr(s, k).cpu().numpy(), ref[k], RTOL[dtype], "%s c=%d" % (k, c))


@pytest.mark.parametrize("name", ["fls_bank_2_1", "fls_scalar_1_1", "fls_ctrl_3_2"])
def test_single_mode_matches_reference(golden, name):
    """Single mode: NumPy in and out with the reference's shapes (scalar z and a column x for dim_z = 1), a list
    xSmooth, smooth_batch shaped (T, n) or (T, n, 1)."""
    from filterpy_b200.kalman import FixedLagSmoother
    g = golden(name)
    N = int(g["N"])
    col = bool(g["x_col"])
    n, m = g["x"].shape[1], np.shape(g["H"])[-2]
    pick = lambda a, f: a[f] if np.ndim(a) == 3 else a                  # noqa: E731
    for f in (0, 3):
        s = FixedLagSmoother(n, m, N)
        s.x = g["x"][f][:, None] if col else g["x"][f]
        s.P = g["P"][f]
        s.F, s.H, s.Q, s.R = (pick(g[k], f) for k in "FHQR")
        if "B" in g:
            s.B = g["B"]
        zs = [float(z[0]) if bool(g["scalar_z"]) else z for z in g["zs"][:, f]]
        us = g["us"][:, f] if "us" in g else None
        xs, xh = s.smooth_batch(zs, N, us=us)
        T = len(zs)
        assert xs.shape == ((T, n, 1) if col else (T, n)) and xh.shape == xs.shape
        rel_close(xs.reshape(T, n), g["ref_xs"][:, f], 1e-6, "single smooth_batch")
        for t, z in enumerate(zs):
            s.smooth(z, None if us is None else us[t])
        assert isinstance(s.xSmooth, list) and len(s.xSmooth) == T and s.count == T
        assert s.xSmooth[0].shape == ((n, 1) if col else (n,))
        rel_close(np.array(s.xSmooth).reshape(T, n), g["ref_xs"][:, f], 1e-6, "single xSmooth")
        assert s.x.shape == ((n, 1) if col else (n,)) and s.S.shape == (m, m)
        assert s.y.shape == ((m, 1) if col else (m,))
        assert s.K.shape == (n, 1) and not s.K.any() and not s.x_s.any()
        assert "FixedLagSmoother object" in repr(s)


def test_online_golden_in_single_mode(golden):
    from filterpy_b200.kalman import FixedLagSmoother
    g = golden("fls_online")
    N = int(g["N"])
    s = FixedLagSmoother(2, 1, N)
    s.x = g["x"][2]; s.P = g["P"][2]; s.F = g["F"]; s.H = g["H"]; s.Q = g["Q"]; s.R = g["R"]
    for t in range(int(g["rec_calls"][-1])):
        s.smooth(g["zs"][t, 2])
        c = t + 1
        if c in g["rec_calls"]:
            rel_close(np.array(s.xSmooth), g["ref_xs_%d" % c][:, 2], 1e-6, "xSmooth c=%d" % c)
            rel_close(s.x, g["ref_x_%d" % c][2], 1e-6, "x"); rel_close(s.P, g["ref_P_%d" % c][2], 1e-6, "P")
            rel_close(s.y, g["ref_y_%d" % c][2], 1e-6, "y"); rel_close(s.S, g["ref_S_%d" % c][2], 1e-6, "S")
            assert s.count == c


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["fls_bank_4_2", "fls_bank_9_3", "fls_lag_20"])
def test_shared_models_and_slices(golden, name, dtype):
    """Shared models (stride 0) agree bit for bit with the same models repeated per filter, and a bank with a
    slice of it, on the fused (4/2) and per-epoch (9/3, N = 20) paths."""
    g = dict(golden(name))
    Nf = g["x"].shape[0]
    for k in "FHQR":
        a = np.asarray(g[k])
        g[k] = np.broadcast_to(a[0] if a.ndim == 3 else a, (Nf,) + a.shape[-2:]).copy()
    N = int(g["N"])
    a, b = make(g, dtype), make(g, dtype, shared=True)
    xa, _ = a.smooth_batch(g["zs"], N)
    xb, _ = b.smooth_batch(g["zs"], N)
    assert np.array_equal(xa.cpu().numpy(), xb.cpu().numpy())
    c = make(g, dtype, Nf=5)
    xc, _ = c.smooth_batch(g["zs"][:, :5], N)
    if name == "fls_bank_9_3":
        # the 9/3 KF step runs the row-block kernel, which hands the filters past its last full block to another
        # instance: a bank and its slice agree to rounding there, not bit for bit
        rel_close(per_filter(xc.cpu().numpy()), per_filter(xa[:, :5].cpu().numpy()), RTOL[dtype], "slice")
    else:
        assert np.array_equal(xc.cpu().numpy(), xa[:, :5].cpu().numpy())


def test_history_grows_past_its_capacity(golden):
    """70 smooth() calls cross the reallocation of the 64-row history; the rows before it survive."""
    from oracle import fls as ofl
    g = golden("fls_bank_2_1")
    rng = np.random.default_rng(5)
    T = 70
    zs = (np.arange(T) / 2.)[:, None, None] + 1.1 * rng.standard_normal((T, 64, 1))
    for lag in (4, FUSED_CAP + 4):
        s = make(g, np.float64, N=lag)
        for t in range(T):
            s.smooth(zs[t])
        assert s.xSmooth.shape == (T, 64, 2) and s._hist.shape[0] >= T
        ref = ofl.fls_bank(g["x"], g["P"], g["F"], g["H"], g["Q"], g["R"], zs, lag)
        rel_close(per_filter(s.xSmooth.cpu().numpy()), per_filter(ref["xs"]), 1e-6, "lag %d" % lag)


@pytest.mark.parametrize("lag", [3, FUSED_CAP + 1])
def test_singular_S_status_and_single_mode_error(golden, lag):
    from filterpy_b200.kalman import FixedLagSmoother
    from oracle import fls as ofl
    g = golden("fls_bank_2_1")
    Nf = 6
    H = np.broadcast_to(g["H"], (Nf, 1, 2)).copy(); R = np.broadcast_to(g["R"], (Nf, 1, 1)).copy()
    H[2] = 0.; R[2] = 0.                                         # S = 0 for filter 2
    s = make(g, np.float64, Nf=Nf, N=lag)
    s.H = H; s.R = R
    zs = g["zs"][:, :Nf]
    for t in range(8):
        s.smooth(zs[t])
    assert s.status.cpu().numpy().tolist() == [0, 0, 1, 0, 0, 0]
    with pytest.raises(np.linalg.LinAlgError):
        s.check()
    ref = ofl.fls_bank(g["x"][:Nf], g["P"][:Nf], g["F"], H, g["Q"], R, zs[:8], lag)
    rel_close(per_filter(s.xSmooth.cpu().numpy()), per_filter(ref["xs"]), 1e-6, "singular bank")
    rel_close(s.x.cpu().numpy(), ref["x"], 1e-6, "x")
    b = make(g, np.float64, Nf=Nf, N=lag)                        # the neighbours, without the singular filter
    b.H = np.broadcast_to(g["H"], (Nf, 1, 2)).copy(); b.R = np.broadcast_to(g["R"], (Nf, 1, 1)).copy()
    xs, _ = b.smooth_batch(zs[:8], lag)
    keep = [0, 1, 3, 4, 5]
    assert np.array_equal(s.xSmooth.cpu().numpy()[:, keep], xs.cpu().numpy()[:, keep])
    single = FixedLagSmoother(2, 1, lag)
    single.H = np.zeros((1, 2)); single.R = np.zeros((1, 1))
    with pytest.raises(np.linalg.LinAlgError):
        single.smooth(1.0)
    assert single.count == 0 and len(single.xSmooth) == 0
    with pytest.raises(np.linalg.LinAlgError):
        single.smooth_batch([1.0, 2.0], lag)


def test_odd_bank_size_fp32():
    """33 filters, 2/1 fp32: a bank size that is no multiple of the block or of 16 bytes of rows."""
    from filterpy_b200.kalman import FixedLagSmoother
    from oracle import fls as ofl
    rng = np.random.default_rng(9)
    Nf, T, N = 33, 20, 5
    x = rng.standard_normal((Nf, 2)); P = np.tile(10. * np.eye(2), (Nf, 1, 1))
    F = np.array([[1., .1], [0., 1.]]); H = np.array([[1., 0.]]); Q = 0.01 * np.eye(2); R = np.eye(1)
    zs = rng.standard_normal((T, Nf, 1))
    s = FixedLagSmoother(2, 1, N, n_filters=Nf, dtype=np.float32)
    s.x, s.P, s.F, s.H, s.Q, s.R = x, P, F, H, Q, R
    for t in range(T):
        s.smooth(zs[t])
    ref = ofl.fls_bank(x, P, F, H, Q, R, zs, N)
    rel_close(per_filter(s.xSmooth.cpu().numpy()), per_filter(ref["xs"]), 1e-3, "33 filters")


def test_reference_errors():
    from filterpy_b200.kalman import FixedLagSmoother
    s = FixedLagSmoother(2, 1)
    with pytest.raises(AttributeError):
        s.xSmooth
    with pytest.raises(AttributeError):
        s.smooth(1.0)
    t = FixedLagSmoother(2, 1, 3)
    with pytest.raises(TypeError):
        t.smooth(None)
    with pytest.raises(NotImplementedError):
        t.B = 2.
    t.B = 0.
    assert t.B == 0.
    xs, xh = s.smooth_batch([1., 2., 3.], 2)                    # smooth_batch works without self.N
    assert xs.shape == (3, 2, 1)


def test_torch_op_equals_mirror(golden):
    import torch
    from filterpy_b200 import torch_ops
    ops = torch_ops.load()
    for name in ("fls_bank_4_2", "fls_bank_9_3"):
        g = golden(name)
        s = make(g, np.float64)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).cuda()      # noqa: E731
        N = int(g["N"])
        xs, xh = ops.fls_smooth_batch(dev(g["x"]), dev(g["P"]), dev(g["F"]), dev(g["H"]), dev(g["Q"]), dev(g["R"]),
                                      dev(g["zs"]), N)
        ms, mh = s.smooth_batch(g["zs"], N)
        assert np.array_equal(xs.cpu().numpy(), ms.cpu().numpy()) and np.array_equal(xh.cpu().numpy(), mh.cpu().numpy())


def test_1m_bank_vs_oracle_subset():
    """2^20 filters, 4/2 fp32 with per-filter models, smooth_batch on the fused kernel: a seeded 4096-filter
    subset against the fp64 vectorised oracle."""
    from filterpy_b200.common import workloads as wl
    from filterpy_b200.kalman import FixedLagSmoother
    from oracle import fls as ofl
    Nf, T, N = 1 << 20, 12, 4
    w = wl.kf_bank_cv2d(Nf, seed=1234, steps=T)
    s = FixedLagSmoother(4, 2, N, n_filters=Nf, dtype=np.float32)
    for k in ("x", "P", "F", "H", "Q", "R"):
        setattr(s, k, w[k])
    xs, xh = s.smooth_batch(w["zs"], N)
    sel = np.sort(np.random.default_rng(0).choice(Nf, 4096, replace=False))
    ref = ofl.fls_bank(w["x"][sel], w["P"][sel], w["F"][sel], w["H"][sel], w["Q"][sel], w["R"][sel], w["zs"][:, sel], N)
    rel_close(per_filter(xs.cpu().numpy()[:, sel]), per_filter(ref["xs"]), 1e-3, "xSmooth")
    rel_close(per_filter(xh.cpu().numpy()[:, sel]), per_filter(ref["xhat"]), 1e-3, "xhat")
