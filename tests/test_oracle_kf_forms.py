"""CPU: the oracles of KalmanFilter.update_sequential and update_correlated against the reference's golden vectors,
and the argument checks of bke_kf_update_rows / bke_kf_step_correlated, which run before any device is needed."""

import numpy as np
import pytest

from filterpy_b200 import _lib
from oracle import kf as okf

import kf_forms_oracle as kfo

SEQ = ["kf_forms_seq_cv63_111", "kf_forms_seq_cv63_12", "kf_forms_seq_cv63_21", "kf_forms_seq_4_2",
       "kf_forms_seq_6_3", "kf_forms_seq_given", "kf_forms_seq_given_4_4", "kf_forms_seq_s0"]
CORR = ["kf_forms_corr_2_1", "kf_forms_corr_4_2", "kf_forms_corr_singular"]


def _block_args(g, k):
    Ri, Hi = g.get("Ri_%d" % k), g.get("Hi_%d" % k)
    return (None if Ri is None else (float(Ri) if np.ndim(Ri) == 0 else Ri)), Hi


def run_seq_bank(g):
    """The golden file's steps through kf_update_sequential_bank (fp64)."""
    x, P = g["x"].copy(), g["P"].copy()
    N, n = x.shape
    m = g["H"].shape[1]
    y, K, z = np.zeros((N, m)), np.zeros((N, n, m)), np.full((N, m), np.nan)
    for t in range(g["zs"].shape[0]):
        x, P = okf.kf_predict_bank(x, P, g["F"], g["Q"])
        for k, (s, L) in enumerate(zip(g["starts"], g["lens"])):
            Ri, Hi = _block_args(g, k)
            o = kfo.kf_update_sequential_bank(x, P, int(s), g["zs"][t][:, s:s + L], g["H"], g["R"], y, K, z,
                                              R_i=Ri, H_i=Hi, valid=g["valid"][t])
            x, P, y, K, z = o["x"], o["P"], o["y"], o["K"], o["z"]
    return dict(x=x, P=P, y=y, K=K, z=z)


def run_corr_bank(g):
    x, P = g["x"].copy(), g["P"].copy()
    N = x.shape[0]
    n, m = x.shape[1], g["H"].shape[1]
    st = np.zeros(N, int)
    K, S = np.zeros((N, n, m)), np.zeros((N, m, m))
    for t in range(g["zs"].shape[0]):
        x, P = okf.kf_predict_bank(x, P, g["F"], g["Q"])
        o = kfo.kf_update_correlated_bank(x, P, g["zs"][t], g["H"], g["R"], g["M"], valid=g["valid"][t])
        st |= o["status"]
        v = g["valid"][t] & (o["status"] == 0)
        x, P = o["x"], o["P"]
        K = np.where(v[:, None, None], o["K"], K)           # a filter without a measurement keeps K and S
        S = np.where(v[:, None, None], o["S"], S)
    return dict(x=x, P=P, y=o["y"], K=K, S=S, status=st)


def _close(a, b, tol=1e-9):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b))
    fin = np.isfinite(b)
    scale = max(np.abs(b[fin]).max(initial=0), 1e-300)
    assert np.abs(a[fin] - b[fin]).max(initial=0) / scale < tol


@pytest.mark.parametrize("name", SEQ)
def test_sequential_oracle_matches_golden(golden, name):
    g = golden(name)
    o = run_seq_bank(g)
    for k in ("x", "P", "y", "K", "z"):
        _close(o[k], g["out_" + k])


@pytest.mark.parametrize("name", SEQ)
def test_sequential_single_oracle_matches_golden(golden, name):
    """The reference's np.dot sequence, one filter at a time."""
    g = golden(name)
    for f in range(g["x"].shape[0]):
        x, P = g["x"][f], g["P"][f]
        for t in range(g["zs"].shape[0]):
            x, P = okf.kf_predict_single(x, P, g["F"][f], g["Q"][f])
            if not g["valid"][t, f]:
                continue
            for k, (s, L) in enumerate(zip(g["starts"], g["lens"])):
                Ri, Hi = _block_args(g, k)
                x, P = kfo.kf_update_sequential_single(x, P, int(s), g["zs"][t, f, s:s + L], g["H"][f], g["R"][f],
                                                       R_i=Ri if Ri is None or np.isscalar(Ri) else Ri[f],
                                                       H_i=None if Hi is None else Hi[f])[:2]
        _close(x, g["out_x"][f]); _close(P, g["out_P"][f])


def test_sequential_splits_equal_update(golden):
    """The reference test's point: three block splittings of a 6/3 update give update()'s posterior."""
    for tag in ("111", "12", "21"):
        g = golden("kf_forms_seq_cv63_" + tag)
        _close(g["out_x"], g["upd_x"], 1e-9); _close(g["out_P"], g["upd_P"], 1e-9)


def test_sequential_zero_s_is_nan_not_an_error(golden):
    g = golden("kf_forms_seq_s0")
    assert np.isnan(g["out_x"]).all() and np.isnan(g["out_K"][:, :, 0]).all()


@pytest.mark.parametrize("name", CORR)
def test_correlated_oracle_matches_golden(golden, name):
    g = golden(name)
    o = run_corr_bank(g)
    np.testing.assert_array_equal(o["status"], g["out_status"])
    for k in ("x", "P"):
        _close(o[k], g["out_" + k])
    ok = g["out_status"] == 0
    for k in ("y", "K", "S"):
        _close(o[k][ok], g["out_" + k][ok])
    have = np.isfinite(g["out_ll"])
    valid = g["valid"][-1] & ok
    y, S = o["y"][have], o["S"][have]
    ll = np.where(valid[have], okf.log_likelihood_bank(y, S), okf.missed_log_likelihood_bank(S))
    _close(ll, g["out_ll"][have])


def test_correlated_single_oracle_matches_golden(golden):
    g = golden("kf_forms_corr_2_1")
    x, P = g["x"][0], g["P"][0]
    for t in range(g["zs"].shape[0]):
        x, P = okf.kf_predict_single(x, P, g["F"][0], g["Q"][0])
        x, P, y, K, S, SI = kfo.kf_update_correlated_single(x, P, g["zs"][t, 0], g["H"][0], g["R"][0], g["M"][0])
    _close(x, g["out_x"][0]); _close(P, g["out_P"][0]); _close(S, g["out_S"][0]); _close(K, g["out_K"][0])


def test_correlated_p_is_not_symmetrised(golden):
    """P = P - K (H P + M') of the reference drifts from symmetry with M != 0; the oracle keeps that."""
    g = golden("kf_forms_corr_4_2")
    assert np.abs(g["out_P"] - np.swapaxes(g["out_P"], 1, 2)).max() > 0


def _bank(N, n, m, seed):
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(N, n, n))
    B = rng.normal(size=(N, m, m))
    return dict(x=rng.normal(size=(N, n)), P=A @ np.swapaxes(A, 1, 2) + np.eye(n), H=rng.normal(size=(N, m, n)),
                R=B @ np.swapaxes(B, 1, 2) + np.eye(m), M=0.3 * rng.normal(size=(N, n, m)), z=rng.normal(size=(N, m)))


def test_sequential_bank_with_one_singular_block():
    """A singular S_i (L > 1) in one filter gives that filter status 1, its prior and no y, K or z, and leaves every
    other filter as a bank without it computes them (np.linalg.inv of the whole stack would raise)."""
    N, n, m, start, L = 6, 4, 4, 1, 2
    w = _bank(N, n, m, 0)
    y0, K0, z0 = np.full((N, m), 7.0), np.full((N, n, m), 7.0), np.full((N, m), 7.0)
    zi = w["z"][:, start:start + L]
    clean = kfo.kf_update_sequential_bank(w["x"], w["P"], start, zi, w["H"], w["R"], y0, K0, z0)
    H, R = w["H"].copy(), w["R"].copy()
    H[3, start + L - 1] = 0; R[3, start + L - 1] = 0; R[3, :, start + L - 1] = 0
    o = kfo.kf_update_sequential_bank(w["x"], w["P"], start, zi, H, R, y0, K0, z0)
    np.testing.assert_array_equal(o["status"], [0, 0, 0, 1, 0, 0])
    assert np.array_equal(o["x"][3], w["x"][3]) and np.array_equal(o["P"][3], w["P"][3])
    assert np.all(o["y"][3] == 7) and np.all(o["K"][3] == 7) and np.all(o["z"][3] == 7)
    ok = np.arange(N) != 3
    for k in ("x", "P", "y", "K", "z"):
        np.testing.assert_allclose(o[k][ok], clean[k][ok], rtol=1e-12, atol=1e-12)
    # BKE_STATUS_STICKY keeps the starting word where the update succeeds
    st = kfo.kf_update_sequential_bank(w["x"], w["P"], start, zi, H, R, y0, K0, z0, status=np.full(N, 5),
                                       sticky=True)["status"]
    np.testing.assert_array_equal(st, [5, 5, 5, 1, 5, 5])
    # L = 1 with S_i = 0: the reciprocal's inf / NaN, status 0
    Hi = np.zeros((N, 1, n)); Hi[:, 0, 0] = 1
    P = w["P"].copy(); P[:, 0, 0] = 2.0
    o = kfo.kf_update_sequential_bank(w["x"], P, 0, w["z"][:, :1], w["H"], w["R"], y0, K0, z0,
                                      R_i=np.full((N, 1, 1), -2.0), H_i=Hi)
    assert np.all(o["status"] == 0) and np.all(np.isinf(o["K"][:, 0, 0])) and np.isnan(o["P"]).any()


def test_zero_pivot_is_exact_singularity():
    """zero_pivot calls singular only an exact zero pivot: not an ill-conditioned or indefinite S, which
    np.linalg.matrix_rank's tolerance calls singular at cond 1e17."""
    U = np.linalg.qr(np.random.default_rng(1).normal(size=(3, 3)))[0]
    ill = (U * [1.0, 1e-9, 1e-17]) @ U.T
    assert np.linalg.matrix_rank(ill) < 3
    S = np.stack([ill, np.diag([1.0, -2.0, 3.0]), np.array([[1.0, 2.0, 0.0], [2.0, 4.0, 0.0], [0.0, 0.0, 1.0]]),
                  np.zeros((3, 3)), np.array([[0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])])
    np.testing.assert_array_equal(kfo.zero_pivot(S), [False, False, True, True, False])


def test_correlated_bank_singular_rule():
    """update_correlated's bank: an exactly singular S (a zero row of H, R and M') gives status 1, the prior and no y;
    an ill-conditioned S is inverted; a filter without a measurement gets y = 0 and status 0 whatever its S."""
    N, n, m = 5, 4, 3
    w = _bank(N, n, m, 2)
    H, R, M = w["H"].copy(), w["R"].copy(), w["M"].copy()
    H[1, -1] = 0; R[1, -1] = 0; R[1, :, -1] = 0; M[1, :, -1] = 0
    H[4] = H[1]; R[4] = R[1]; M[4] = M[1]
    U = np.linalg.qr(np.random.default_rng(3).normal(size=(m, m)))[0]
    HM = H[2] @ M[2]
    R[2] = (U * [1.0, 1e-6, 1e-12]) @ U.T - (H[2] @ w["P"][2] @ H[2].T + HM + HM.T)
    valid = np.array([True, True, True, True, False])
    o = kfo.kf_update_correlated_bank(w["x"], w["P"], w["z"], H, R, M, valid=valid)
    np.testing.assert_array_equal(o["status"], [0, 1, 0, 0, 0])
    assert np.array_equal(o["x"][1], w["x"][1]) and np.all(np.isnan(o["y"][1])) and np.all(o["y"][4] == 0)
    np.testing.assert_allclose(o["SI"][2] @ o["S"][2], np.eye(m), atol=1e-3)
    st = kfo.kf_update_correlated_bank(w["x"], w["P"], w["z"], H, R, M, valid=valid, status=np.full(N, 5),
                                       sticky=True)["status"]
    np.testing.assert_array_equal(st, [5, 1, 5, 5, 5])


# ---------------------------------------------------------------------------------------------- C-ABI checks
def _rows_args(N=4, n=4, m=3, start=0, rows=1):
    x = np.zeros((N, n)); P = np.zeros((N, n, n)); H = np.zeros((m, n)); R = np.eye(m); z = np.zeros((N, rows))
    r = _lib.KfRowsArgs()
    a = r.step
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags, a.alpha_sq = N, n, m, _lib.BKE_F64, _lib.BKE_DO_UPDATE, 1.0
    a.x = a.x_out = x.ctypes.data; a.P = a.P_out = P.ctypes.data
    a.H = H.ctypes.data; a.R = R.ctypes.data; a.z = z.ctypes.data
    r.start, r.rows = start, rows
    return r, (x, P, H, R, z)


@pytest.mark.parametrize("start,rows", [(-1, 1), (0, 0), (2, 2), (3, 1), (0, 4)])
def test_update_rows_refuses_a_block_outside_z(start, rows):
    lib = _lib.load()
    r, keep = _rows_args(start=start, rows=rows)
    assert lib.bke_kf_update_rows(r, None) == _lib.BKE_ERR_BAD_ARG
    assert b"not within" in lib.bke_last_error()


def test_update_rows_refuses_what_it_does_not_write():
    lib = _lib.load()
    for field in ("S", "SI", "log_likelihood"):
        r, keep = _rows_args()
        buf = np.zeros(64)
        setattr(r.step, field, buf.ctypes.data)
        assert lib.bke_kf_update_rows(r, None) == _lib.BKE_ERR_BAD_ARG
    r, keep = _rows_args()
    r.H_i_stride = 5
    assert lib.bke_kf_update_rows(r, None) == _lib.BKE_ERR_BAD_ARG
    r, keep = _rows_args()
    r.step.flags = _lib.BKE_DO_PREDICT
    assert lib.bke_kf_update_rows(r, None) == _lib.BKE_ERR_BAD_ARG
    assert lib.bke_kf_update_rows(None, None) == _lib.BKE_ERR_BAD_ARG


def test_step_correlated_refuses_a_bad_m():
    lib = _lib.load()
    r, keep = _rows_args()
    a = r.step
    Mc = np.zeros((4, 3))
    assert lib.bke_kf_step_correlated(a, None, 0, None) == _lib.BKE_ERR_BAD_ARG
    assert lib.bke_kf_step_correlated(a, Mc.ctypes.data, 7, None) == _lib.BKE_ERR_BAD_ARG
    a.flags = _lib.BKE_DO_UPDATE | _lib.BKE_UPDATE_FIRST
    assert lib.bke_kf_step_correlated(a, Mc.ctypes.data, 0, None) == _lib.BKE_ERR_BAD_ARG
    a.flags = _lib.BKE_DO_UPDATE
    a.dim_x = 0
    assert lib.bke_kf_step_correlated(a, Mc.ctypes.data, 0, None) == _lib.BKE_ERR_BAD_ARG
