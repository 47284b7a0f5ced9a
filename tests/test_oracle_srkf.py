"""CPU: the square-root filter's oracles against the reference's golden vectors, the dgeqr2 restatement against
scipy, argument validation of the new entries, and the fp32 accuracy contrast that motivates the filter."""
import numpy as np
import pytest
import scipy.linalg

from oracle import srkf as osr

BANKS = ["srkf_bank_4_2", "srkf_bank_6_3", "srkf_bank_9_3", "srkf_ctrl_3_2", "srkf_bank_1_1", "srkf_ill_4_2"]
GOLDEN = BANKS + ["srkf_call_order"]


def _ops(g):
    return [str(o) for o in g["ops"]] if "ops" in g else ["predict+update"] * g["zs"].shape[0]


def _per(a, f, N):
    a = np.asarray(a)
    return a[f] if a.ndim == 3 and a.shape[0] == N else a


def _close(a, b, what, tol=1e-9):
    scale = max(np.abs(b).max(), 1e-300)
    err = np.abs(np.asarray(a, np.float64) - b).max() / scale
    assert err < tol, (what, err)


@pytest.mark.parametrize("name", GOLDEN)
def test_single_oracle_matches_golden(golden, name):
    """The reference's literal call sequence (scipy qr, pinv), one filter at a time, against its recorded state."""
    g = golden(name)
    N, n = g["x"].shape
    m = np.shape(g["H"])[-2]
    rec = list(g["rec_steps"])
    for f in range(N):
        x, L = g["x"][f][:, None], np.linalg.cholesky(g["P"][f])
        Lq, Lr = np.linalg.cholesky(_per(g["Q"], f, N)), np.linalg.cholesky(_per(g["R"], f, N))
        F = _per(g["F"], f, N)
        H = np.zeros((m, n)) if "ops" in g else _per(g["H"], f, N)
        xp, Lp = np.zeros((n, 1)), np.eye(n)            # the reference's __init__ copies (:166-167)
        for t, op in enumerate(_ops(g)):
            if op.startswith("set_H"):
                H = _per(g["H"], f, N)
            for _ in range(op.count("predict")):
                if "us" in g:
                    x, L = osr.srkf_predict_single(x, L, F, Lq, g["B"], g["us"][t, f][:, None])
                else:
                    x, L = osr.srkf_predict_single(x, L, F, Lq)
                xp, Lp = x, L
            if g["valid"][t, f] and not op.endswith("none"):
                R2 = {"R0": np.zeros((m, m)), "Rs": float(g["R2s"]) * np.eye(m) if "R2s" in g else None,
                      "Rm": g["R2m"] if "R2m" in g else None}.get(op[-2:], Lr)
                o = osr.srkf_update_single(x, L, g["zs"][t, f][:, None], H, R2)
                x, L = o["x"], o["L"]
                if t in rec:
                    i = rec.index(t)
                    for k in ("K", "S1_2", "SI1_2"):
                        _close(o[k], g["ref_" + k][i, f], "%s %s t=%d f=%d" % (k, name, t, f))
                    _close(o["y"].ravel(), g["ref_y"][i, f], "y")
            if t in rec:
                i = rec.index(t)
                _close(x.ravel(), g["ref_x"][i, f], "x %s t=%d f=%d" % (name, t, f))
                _close(L, g["ref_P1_2"][i, f], "P1_2 %s t=%d f=%d" % (name, t, f))
                _close(xp.ravel(), g["ref_x_prior"][i, f], "x_prior")
                _close(Lp, g["ref_P1_2_prior"][i, f], "P1_2_prior")
                _close(Lp @ Lp.T, g["ref_P_post"][i, f], "P_post (the prior factor's product)")


def bank_replay(g, dtype=np.float64, sel=None):
    """Drive the vectorised dgeqr2 oracle through a golden case; yields (t, op, valid, out)."""
    N = g["x"].shape[0]
    sel = np.arange(N) if sel is None else sel
    cast = lambda a: np.asarray(a, dtype)                                    # noqa: E731
    pick = lambda a: cast(a[sel] if np.ndim(a) == 3 and np.shape(a)[0] == N else a)   # noqa: E731
    x, L = cast(g["x"][sel]), cast(np.linalg.cholesky(g["P"][sel]))
    Lq, Lr = cast(np.linalg.cholesky(pick(g["Q"]).astype(np.float64))), cast(np.linalg.cholesky(pick(g["R"]).astype(np.float64)))
    F = pick(g["F"])
    m, n = np.shape(g["H"])[-2:]
    H = cast(np.zeros((m, n))) if "ops" in g else pick(g["H"])
    for t, op in enumerate(_ops(g)):
        if op.startswith("set_H"):
            H = pick(g["H"])
        u = cast(g["us"][t][sel]) if "us" in g else None
        B = cast(g["B"]) if "B" in g else None
        for _ in range(op.count("predict")):
            o = osr.srkf_step_bank(x, L, None, F, H, Lq, Lr, predict=True, update=False, B=B, u=u)
            x, L = o["x"], o["L"]
        v = g["valid"][t][sel] & (not op.endswith("none"))
        R2 = {"R0": cast(np.zeros((m, m))), "Rs": cast(float(g["R2s"]) * np.eye(m)) if "R2s" in g else None,
              "Rm": cast(g["R2m"]) if "R2m" in g else None}.get(op[-2:], Lr)
        o = osr.srkf_step_bank(x, L, cast(g["zs"][t][sel]), F, H, Lq, R2, valid=v, predict=False)
        x, L = o["x"], o["L"]
        yield t, op, v, o


@pytest.mark.parametrize("name", GOLDEN)
def test_bank_oracle_matches_golden(golden, name):
    """The vectorised dgeqr2 restatement (the kernel's arithmetic) against the reference, P1_2 entrywise."""
    g = golden(name)
    rec = list(g["rec_steps"])
    for t, op, v, o in bank_replay(g):
        if t not in rec:
            continue
        i = rec.index(t)
        _close(o["x"], g["ref_x"][i], "x %s t=%d" % (name, t))
        _close(o["L"], g["ref_P1_2"][i], "P1_2 %s t=%d" % (name, t))
        if v.any() and not op.endswith("R0"):
            for k in ("K", "y", "S1_2", "SI1_2"):
                _close(o[k][v], g["ref_" + k][i][v], k)


def test_zero_R2_with_zero_H_is_the_singular_status(golden):
    """update(z, R2=0) on a fresh filter (H = 0): the reference's pinv(0) = 0 gives K = 0 and an unchanged
    posterior; the oracle (the kernel's rule) reports status 1 with the same result."""
    g = golden("srkf_call_order")
    t, op, v, o = next(bank_replay(g))
    assert op == "update_R0" and (o["status"] == osr.STATUS_SINGULAR_S).all()
    assert (o["K"] == 0).all() and (g["ref_K"][0] == 0).all() and (g["ref_S1_2"][0] == 0).all()
    _close(o["x"], g["ref_x"][0], "x"); _close(o["L"], g["ref_P1_2"][0], "P1_2")


def _random_cases():
    rng = np.random.default_rng(42)
    for _ in range(100):
        r, c = rng.integers(1, 11, 2)
        yield rng.standard_normal((r, c))
    A = rng.standard_normal((6, 4)); A[1:, 0] = 0; yield A                    # zero sub-column: tau = 0
    A = rng.standard_normal((6, 6)); A[3:, 2] = 0; A[3, 2] = -0.5; yield A
    yield np.triu(rng.standard_normal((5, 5)))                              # already triangular: no reflection
    yield np.zeros((3, 3))
    A = rng.standard_normal((8, 4)); A[:, 1] = -A[:, 1]; yield A
    yield np.vstack([np.eye(4), np.eye(4)])                                 # the fresh filter's predict matrix
    yield -np.eye(5)


def test_dgeqr2_matches_scipy_qr_with_signs():
    for A in _random_cases():
        R = osr.dgeqr2(A)
        Rs = scipy.linalg.qr(A)[1]
        assert R.shape == Rs.shape
        assert np.abs(R - Rs).max() <= 1e-13 * max(1.0, np.abs(Rs).max()), A.shape


def test_fp32_contrast_on_the_ill_conditioned_bank(golden):
    """On the ill-conditioned 4/2 bank the fp32 Joseph form loses more than 1e-3 of max|P| against the fp64
    Joseph form, and the fp32 square-root form (dgeqr2 in fp32) stays below it."""
    g = golden("srkf_ill_4_2")
    x64, P64 = g["x"], g["P"]
    x32, P32 = g["x"].astype(np.float32), g["P"].astype(np.float32)
    F32, H32, Q32, R32 = (g[k].astype(np.float32) for k in "FHQR")
    ej = es = 0.0
    srs = bank_replay(g, np.float32)
    for t in range(g["zs"].shape[0]):
        x64, P64, _, _ = osr.joseph_kf_bank(x64, P64, g["zs"][t], g["F"], g["H"], g["Q"], g["R"])
        x32, P32, _, _ = osr.joseph_kf_bank(x32, P32, g["zs"][t].astype(np.float32), F32, H32, Q32, R32)
        # bank_replay runs predict inside the update step of the next op: run one predict + update per step
        _, _, _, o = next(srs)
        ej = max(ej, osr.worst_relative_P_error(P32[None], P64[None]))
        es = max(es, osr.worst_relative_P_error((o["L"] @ np.swapaxes(o["L"], 1, 2))[None], P64[None]))
    assert ej > 1e-3, ej
    assert es < 1e-3, es


# ------------------------------------------------------------------------------------------ the C-ABI
def _args(L):
    a = L.SrkfArgs()
    fake = 1 << 20                                   # never dereferenced: every call below fails before a launch
    a.n_filters, a.dim_x, a.dim_z, a.dtype, a.flags = 8, 4, 2, L.BKE_F32, L.BKE_DO_PREDICT | L.BKE_DO_UPDATE
    a.x = a.L = a.x_out = a.L_out = a.F = a.H = a.Lq = a.Lr = a.z = fake
    return a


@pytest.mark.parametrize("field,value,msg", [
    ("dim_x", 0, b"dim_x must be 1 or greater"), ("dim_z", 0, b"dim_z must be 1 or greater"),
    ("dim_u", -1, b"dim_u must be 0 or greater"), ("dtype", 7, b"dtype"), ("flags", 0, b"neither"),
    ("flags", 7, b"may only hold"), ("Lq", None, b"predict needs F and Lq"), ("z", None, b"update needs H, Lr and z"),
    ("L_out", None, b"x, L, x_out, L_out"), ("F_stride", 3, b"strides"), ("B", 1 << 20, b"control input"),
    ("n_filters", -1, b"n_filters < 0")])
def test_srkf_step_validates_arguments(field, value, msg):
    from filterpy_b200 import _lib as L
    lib = L.load()
    a = _args(L)
    setattr(a, field, value)
    assert lib.bke_srkf_step(a, None) == L.BKE_ERR_BAD_ARG
    assert msg in lib.bke_last_error()


def test_cholesky_lower_validates_arguments():
    from filterpy_b200 import _lib as L
    lib = L.load()
    fake = 1 << 20
    assert lib.bke_cholesky_lower(-1, 4, L.BKE_F64, fake, 16, fake, None, None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_cholesky_lower(4, 0, L.BKE_F64, fake, 0, fake, None, None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_cholesky_lower(4, 4, 5, fake, 0, fake, None, None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_cholesky_lower(4, 4, L.BKE_F64, fake, 5, fake, None, None) == L.BKE_ERR_BAD_ARG
    assert lib.bke_cholesky_lower(4, 4, L.BKE_F64, None, 0, fake, None, None) == L.BKE_ERR_BAD_ARG
    k = L.BKE_CHOLESKY_MAX_DIM + 1
    assert lib.bke_cholesky_lower(4, k, L.BKE_F64, fake, 0, fake, None, None) == L.BKE_ERR_UNSUPPORTED
    assert b"BKE_CHOLESKY_MAX_DIM" in lib.bke_last_error()


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from filterpy_b200 import _lib as L
    from filterpy_b200.kalman import SquareRootKalmanFilter
    lib = L.load()
    assert lib.bke_srkf_step(_args(L), None) == L.BKE_ERR_CUDA
    assert lib.bke_cholesky_lower(1, 2, L.BKE_F64, 1 << 20, 0, 1 << 20, None, None) == L.BKE_ERR_CUDA
    with pytest.raises(L.BkeError):
        SquareRootKalmanFilter(4, 2)


def test_mirror_constructor_errors_are_the_references():
    from filterpy_b200.kalman import SquareRootKalmanFilter
    for dims in ((0, 2), (4, 0), (4, 2, -1)):
        with pytest.raises(ValueError):
            SquareRootKalmanFilter(*dims)
