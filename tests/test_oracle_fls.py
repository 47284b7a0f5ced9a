"""CPU: the fixed-lag smoother's oracles against the reference's golden vectors, argument
validation of bke_fls_smooth and the absence of a CPU fallback."""
import numpy as np
import pytest

from oracle import fls as ofl

BANKS = ["fls_bank_2_1", "fls_bank_4_2", "fls_bank_6_3", "fls_bank_9_3", "fls_ctrl_3_2", "fls_lag_0", "fls_lag_1",
         "fls_lag_20", "fls_lag_ge_T", "fls_scalar_1_1"]


def _per(a, f, Nf):
    a = np.asarray(a)
    return a[f] if a.ndim == 3 and a.shape[0] == Nf else a


def _close(a, b, what, tol=1e-9):
    scale = max(np.abs(b).max(), 1e-300)
    err = np.abs(np.asarray(a, np.float64) - b).max() / scale
    assert err < tol, (what, err)


def bank_inputs(g, sel=None):
    """(x, P, F, H, Q, R, zs, B, us) of a golden case as [Nf, ...] arrays, optionally a subset of filters."""
    Nf = g["x"].shape[0]
    sel = np.arange(Nf) if sel is None else sel
    pick = lambda a: a[sel] if np.ndim(a) == 3 and np.shape(a)[0] == Nf else a     # noqa: E731
    us = g["us"][:, sel] if "us" in g else None
    return (g["x"][sel], pick(g["P"]), pick(g["F"]), pick(g["H"]), pick(g["Q"]), pick(g["R"]), g["zs"][:, sel],
            g["B"] if "B" in g else None, us)


@pytest.mark.parametrize("name", BANKS)
def test_single_oracle_matches_golden(golden, name):
    """The reference's statements, one filter at a time, reproduce its smooth_batch bit for bit."""
    g = golden(name)
    Nf, n = g["x"].shape
    N = int(g["N"])
    for f in range(Nf):
        x = g["x"][f][:, None] if bool(g["x_col"]) else g["x"][f].copy()
        zs = [float(z[0]) if bool(g["scalar_z"]) else z for z in g["zs"][:, f]]
        xs, xh = ofl.fls_smooth_batch_single(x, _per(g["P"], f, Nf), _per(g["F"], f, Nf), _per(g["H"], f, Nf),
                                             _per(g["Q"], f, Nf), _per(g["R"], f, Nf), zs, N,
                                             B=g["B"] if "B" in g else 0., us=g["us"][:, f] if "us" in g else None)
        T = len(zs)
        assert np.array_equal(xs.reshape(T, n), g["ref_xs"][:, f]), (name, f)
        assert np.array_equal(xh.reshape(T, n), g["ref_xhat"][:, f]), (name, f)


@pytest.mark.parametrize("name", BANKS)
def test_bank_oracle_matches_golden(golden, name):
    g = golden(name)
    x, P, F, H, Q, R, zs, B, us = bank_inputs(g)
    o = ofl.fls_bank(x, P, F, H, Q, R, zs, int(g["N"]), B=B, us=us)
    _close(o["xs"], g["ref_xs"], "xSmooth " + name)
    _close(o["xhat"], g["ref_xhat"], "xhat " + name)
    assert not o["status"].any()


def test_online_sequence(golden):
    """smooth() call by call: the recorded history, x, P, y, S and count after calls 1, N-1, N, N+1 and the last
    (the live rows k-N+2 .. k still change, the rows before are final), by both oracles, and the bank oracle
    continued from a recorded history (what a later smooth() call sees)."""
    g = golden("fls_online")
    N = int(g["N"])
    Nf = g["x"].shape[0]
    calls = [int(c) for c in g["rec_calls"]]
    st = [dict(x=g["x"][f].copy(), P=g["P"][f].copy(), F=g["F"], H=g["H"], Q=g["Q"], R=g["R"], B=0., N=N, count=0,
               xSmooth=[]) for f in range(Nf)]
    hist, x, P = None, g["x"], g["P"]
    for t in range(calls[-1]):
        for f in range(Nf):
            ofl.fls_smooth_single(st[f], g["zs"][t, f])
        o = ofl.fls_bank(x, P, g["F"], g["H"], g["Q"], g["R"], g["zs"][t:t + 1], N, count=t, hist=hist)
        hist, x, P = o["xs"], o["x"], o["P"]
        c = t + 1
        if c not in calls:
            continue
        ref = g["ref_xs_%d" % c]
        assert ref.shape[0] == c
        assert np.array_equal(np.stack([np.array(s["xSmooth"]) for s in st], 1), ref)
        assert np.array_equal(np.stack([s["y"] for s in st]), g["ref_y_%d" % c])
        assert np.array_equal(np.stack([s["S"] for s in st]), g["ref_S_%d" % c])
        assert (g["ref_count_%d" % c] == c).all()
        _close(hist, ref, "bank xSmooth after %d calls" % c)
        _close(x, g["ref_x_%d" % c], "x"); _close(P, g["ref_P_%d" % c], "P")
        _close(o["y"], g["ref_y_%d" % c], "y"); _close(o["S"], g["ref_S_%d" % c], "S")


def test_reassociated_correction_within_1e6_of_goldens(golden):
    """The kernels' order, P (A^i g) with A = (F - K H)' and g = H' (SI y), restated in fp64 NumPy, stays within
    1e-6 of the reference on every golden case (DESIGN.md §3.4b)."""
    for name in BANKS:
        g = golden(name)
        x, P, F, H, Q, R, zs, B, us = bank_inputs(g)
        Nf, n = x.shape
        N = int(g["N"])
        F3, H3, Q3, R3 = (np.broadcast_to(a, (Nf,) + np.shape(a)[-2:]) for a in (F, H, Q, R))
        xs = np.zeros((len(zs), Nf, n))
        for k in range(len(zs)):
            x_pre = np.einsum("fij,fj->fi", F3, x)
            if us is not None:
                x_pre = x_pre + np.einsum("ij,fj->fi", B, us[k])
            P = F3 @ P @ np.swapaxes(F3, 1, 2) + Q3
            y = zs[k] - np.einsum("fij,fj->fi", H3, x_pre)
            HT = np.swapaxes(H3, 1, 2)
            SI = np.linalg.inv(H3 @ P @ HT + R3)
            K = P @ HT @ SI
            x = x_pre + np.einsum("fia,fa->fi", K, y)
            IKH = np.eye(n) - K @ H3
            P = IKH @ P @ np.swapaxes(IKH, 1, 2) + K @ R3 @ np.swapaxes(K, 1, 2)
            xs[k] = x_pre
            if k >= N:
                v = np.einsum("fja,fab,fb->fj", HT, SI, y)
                A = np.swapaxes(F3 - K @ H3, 1, 2)
                for i in range(N):
                    xs[k - i] += np.einsum("fij,fj->fi", P, v)
                    v = np.einsum("fij,fj->fi", A, v)
            else:
                xs[k] = x
        _close(xs, g["ref_xs"], name, tol=1e-6)


def test_singular_S_keeps_the_prior_in_the_bank_oracle(golden):
    g = golden("fls_bank_2_1")
    x, P, F, H, Q, R, zs, _, _ = bank_inputs(g, np.arange(4))
    H3 = np.broadcast_to(H, (4,) + H.shape).copy()
    R3 = np.broadcast_to(R, (4,) + R.shape).copy()
    H3[1] = 0.; R3[1] = 0.                                    # S = 0 for filter 1
    o = ofl.fls_bank(x, P, F, H3, Q, R3, zs[:8], 2)
    assert o["status"].tolist() == [0, 1, 0, 0]
    Fx = x[1].copy()
    for k in range(8):
        Fx = F @ Fx
        assert np.array_equal(o["xs"][k, 1], Fx)              # never corrected: every row is x_pre
    ref = ofl.fls_bank(x[[0, 2, 3]], P[[0, 2, 3]], F, H, Q, R, zs[:8, [0, 2, 3]], 2)
    assert np.array_equal(ref["xs"], o["xs"][:, [0, 2, 3]])


# ------------------------------------------------------------------------------------------ the C-ABI
def _args(L):
    a = L.FlsArgs()
    fake = 1 << 20                                   # never dereferenced: every call below fails before a launch
    k = a.step
    k.n_filters, k.dim_x, k.dim_z, k.dtype = 8, 4, 2, L.BKE_F32
    k.x = k.P = k.x_out = k.P_out = k.F = k.H = k.Q = k.R = fake
    a.n_steps, a.lag, a.count = 4, 2, 0
    a.zs = a.xs_smooth = fake
    return a


@pytest.mark.parametrize("field,value,msg", [
    ("lag", -1, b"lag < 0"), ("count", -3, b"count < 0"), ("n_steps", 0, b"n_steps must be 1 or greater"),
    ("n_steps", -2, b"n_steps must be 1 or greater"), ("xs_smooth", None, b"xs_smooth (the history) is NULL"),
    ("zs", None, b"zs is NULL"), ("us", 1 << 20, b"control input")])
def test_fls_smooth_validates_arguments(field, value, msg):
    from filterpy_b200 import _lib as L
    lib = L.load()
    a = _args(L)
    setattr(a, field, value)
    assert lib.bke_fls_smooth(a, None) == L.BKE_ERR_BAD_ARG
    assert msg in lib.bke_last_error()


@pytest.mark.parametrize("field,value,msg", [
    ("dim_x", 0, b"dim_x must be 1 or greater"), ("dtype", 7, b"dtype"), ("Q", None, b"predict needs F and Q"),
    ("R", None, b"update needs H and R"), ("P_out", None, b"x, P, x_out, P_out"), ("F_stride", 3, b"strides")])
def test_fls_smooth_validates_the_step(field, value, msg):
    from filterpy_b200 import _lib as L
    lib = L.load()
    a = _args(L)
    setattr(a.step, field, value)
    assert lib.bke_fls_smooth(a, None) == L.BKE_ERR_BAD_ARG
    assert msg in lib.bke_last_error()


def test_workspace_bytes_zero_on_the_fused_path():
    from filterpy_b200 import _lib as L
    lib = L.load()
    cap = L.BKE_FLS_FUSED_MAX_LAG
    for n, m in ((1, 1), (2, 1), (4, 2)):
        for dt in (L.BKE_F32, L.BKE_F64):
            assert lib.bke_fls_workspace_bytes(1000, n, m, 0, dt, cap) == 0
            assert lib.bke_fls_workspace_bytes(1000, n, m, 0, dt, cap + 1) > 0
            assert lib.bke_fls_workspace_bytes(1000, n, m, 1, dt, 4) > 0      # a control input
    assert lib.bke_fls_workspace_bytes(1000, 6, 3, 0, L.BKE_F64, 4) >= 1000 * 8 * (6 + 18 + 3 + 9 + 6 + 6 + 3)
    assert lib.bke_fls_workspace_bytes(0, 6, 3, 0, L.BKE_F64, 4) == 0


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from filterpy_b200 import _lib as L
    from filterpy_b200.kalman import FixedLagSmoother
    lib = L.load()
    assert lib.bke_fls_smooth(_args(L), None) == L.BKE_ERR_CUDA
    with pytest.raises(L.BkeError):
        FixedLagSmoother(2, 1, 4)
    with pytest.raises(L.BkeError):
        FixedLagSmoother(4, 2, N=8, n_filters=16, dtype=np.float32)
