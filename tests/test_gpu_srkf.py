"""GPU parity: square-root filter banks (CUDA through the mirror, the C-ABI and the torch op) against the
reference's golden vectors and the dgeqr2 oracle."""
import numpy as np
import pytest

from test_gpu_kf import rel_close, RTOL
from test_oracle_srkf import GOLDEN, _ops, bank_replay

pytestmark = pytest.mark.gpu


def make(g, dtype, N=None, diagnostics=True, shared=False):
    from filterpy_b200.kalman import SquareRootKalmanFilter
    N = g["x"].shape[0] if N is None else N
    n, m = g["x"].shape[1], np.shape(g["H"])[-2]
    s = SquareRootKalmanFilter(n, m, 0 if "B" not in g else g["B"].shape[-1], n_filters=N, dtype=dtype,
                               diagnostics=diagnostics)
    s.x = g["x"][:N]; s.P = g["P"][:N]
    pick = (lambda a: a[0] if np.ndim(a) == 3 else a) if shared else (lambda a: a[:N] if np.ndim(a) == 3 else a)
    s.Q = pick(g["Q"]); s.R = pick(g["R"]); s.F = pick(g["F"])
    if "ops" not in g:
        s.H = pick(g["H"])
    if "B" in g:
        s.B = g["B"]
    return s


def run_op(s, g, t, op, N=None):
    N = g["x"].shape[0] if N is None else N
    if op.startswith("set_H"):
        s.H = g["H"][:N] if np.ndim(g["H"]) == 3 else g["H"]
    for _ in range(op.count("predict")):
        s.predict(g["us"][t][:N] if "us" in g else 0)
    if op.endswith("none"):
        s.update(None)
        return
    R2 = {"R0": 0., "Rs": float(g["R2s"]) if "R2s" in g else None, "Rm": g["R2m"] if "R2m" in g else None}.get(op[-2:])
    s.update(g["zs"][t][:N], R2=R2, valid=g["valid"][t][:N])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", GOLDEN)
def test_srkf_vs_reference_golden(golden, name, dtype):
    """Every recorded output after every call: x, P, P1_2 entrywise (dgeqr2's signs), the priors, P_post (the
    prior factor's product), K, y, S, SI, S1_2, SI1_2.  4/2 and 1/1 run the register tile, 6/3, 9/3 and the
    control-input 3/2 the warp-per-filter kernel."""
    g = golden(name)
    s = make(g, dtype)
    rtol = RTOL[dtype]
    rec = list(g["rec_steps"])
    for t, op in enumerate(_ops(g)):
        run_op(s, g, t, op)
        if t not in rec:
            continue
        i = rec.index(t)
        get = lambda a: a.cpu().numpy()                                  # noqa: E731
        for k, got in (("x", s.x), ("P", s.P), ("P1_2", s.P1_2), ("x_prior", s.x_prior), ("P_prior", s.P_prior),
                       ("P_post", s.P_post), ("S1_2", s.S1_2), ("SI1_2", s.SI1_2), ("S", s.S), ("SI", s.SI)):
            rel_close(get(got), g["ref_" + k][i], rtol, "%s %s t=%d" % (k, name, t))
        # K and y only exist where a filter has ever been updated; y = z - H x cancels digits of z: compare H x
        rel_close(get(s.K), g["ref_K"][i], max(rtol, 1e-5) if dtype == np.float32 else rtol, "K t=%d" % t)
        if "ops" not in g:
            zf = g["zs"][t].astype(dtype).astype(np.float64)
            v = g["valid"][t]
            rel_close((zf - get(s.y))[v], (g["zs"][t] - g["ref_y"][i])[v], rtol, "z - y t=%d" % t)
    if "ops" in g:
        assert int(s.status.sum().item()) == 0          # the last update (R2 matrix) is regular


def test_split_equals_fused_valid_masks_and_diagnostics_off(golden):
    g = golden("srkf_bank_4_2")
    a, b = make(g, np.float64), make(g, np.float64)
    c = make(g, np.float64, diagnostics=False)
    for t in range(4):
        for s in (a, b, c):
            s.predict()
        b.x                                               # predict-only launch, then update-only launch
        for s in (a, b, c):
            s.update(g["zs"][t], valid=g["valid"][t])
        assert np.array_equal(a.x.cpu().numpy(), b.x.cpu().numpy())
        assert np.array_equal(a.P1_2.cpu().numpy(), b.P1_2.cpu().numpy())
        assert np.array_equal(a.P1_2.cpu().numpy(), c.P1_2.cpu().numpy())
    v = ~g["valid"][3]
    assert v.any()
    rel_close(a.x.cpu().numpy()[v], a.x_prior.cpu().numpy()[v], 0, "valid=0 keeps the prior")
    with pytest.raises(AttributeError):
        c.K


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["srkf_bank_4_2", "srkf_bank_9_3"])
def test_per_filter_vs_shared_models(golden, name, dtype):
    """The same models given once for the bank (stride 0) and repeated per filter give the same bank; 4/2 runs
    the register tile, 9/3 the warp kernel."""
    g = dict(golden(name))
    N = g["x"].shape[0]
    for k in "FHQR":
        a = np.asarray(g[k])
        g[k] = np.broadcast_to(a[0] if a.ndim == 3 else a, (N,) + a.shape[-2:]).copy()
    a, b = make(g, dtype), make(g, dtype, shared=True)
    for t in range(3):
        for s in (a, b):
            s.predict(); s.update(g["zs"][t])
    assert np.array_equal(a.x.cpu().numpy(), b.x.cpu().numpy())
    assert np.array_equal(a.P1_2.cpu().numpy(), b.P1_2.cpu().numpy())


def test_singular_S1_2_status_and_cholesky_errors():
    from filterpy_b200.kalman import SquareRootKalmanFilter
    from filterpy_b200.common import workloads as wl
    s = SquareRootKalmanFilter(4, 2, n_filters=3)
    s.H = np.array([[1., 0, 0, 0], [0, 0, 1, 0]])
    s.update(np.ones((3, 2)), R2=0.)                     # H = e_i rows, R2 = 0: S1_2 is regular (from L)
    assert s.status.cpu().numpy().tolist() == [0, 0, 0]
    t = SquareRootKalmanFilter(4, 2, n_filters=3)         # H = 0 and R2 = 0: S1_2 = 0
    x0 = t.x.clone(); L0 = t.P1_2.clone()
    t.update(np.ones((3, 2)), R2=0.)
    assert t.status.cpu().numpy().tolist() == [1, 1, 1]
    assert (t.K == 0).all() and (t.S1_2 == 0).all() and (t.SI1_2 == 0).all()
    assert np.array_equal(t.x.cpu().numpy(), x0.cpu().numpy()) and np.array_equal(t.P1_2.cpu().numpy(), L0.cpu().numpy())
    for v in (-np.eye(4), np.diag([1., 1., 0., 1.])):
        with pytest.raises(np.linalg.LinAlgError):
            s.P = v
    with pytest.raises(np.linalg.LinAlgError):
        s.R = np.array([[1., 2.], [2., 1.]])
    w = wl.kf_bank_cv2d(64, seed=1234)
    q = SquareRootKalmanFilter(4, 2, n_filters=64)
    with pytest.raises(np.linalg.LinAlgError, match=r"Q: \d+ of 64"):
        q.Q = w["Q"]                                      # rank-deficient white-noise Q: scipy refuses it too
    single = SquareRootKalmanFilter(2, 1)
    with pytest.raises(np.linalg.LinAlgError):
        single.Q = np.array([[1., 1.], [1., 1.]])
    single.Q = np.array([[4., 2.], [2., 5.]])
    rel_close(single.Q1_2, np.linalg.cholesky([[4., 2.], [2., 5.]]), 1e-12, "Q1_2")
    with pytest.raises(AttributeError):
        single.M
    with pytest.raises(NotImplementedError):
        single.residual_of(np.zeros(1))
    with pytest.raises(AttributeError):
        single.P1_2 = np.eye(2)


def test_single_mode_shapes_and_write_back(golden):
    from filterpy_b200.kalman import SquareRootKalmanFilter
    g = golden("srkf_bank_4_2")
    s = SquareRootKalmanFilter(4, 2)
    s.x = g["x"][0][:, None]; s.P = g["P"][0]; s.Q = g["Q"][0]; s.R = g["R"][0]; s.F = g["F"][0]; s.H = g["H"][0]
    assert s.x.shape == (4, 1) and s.P.shape == (4, 4) and s.z.shape == (2, 1)
    s.F[0, 1] = 0.5                                      # writes back, as on the reference's live array
    assert s.F[0, 1] == 0.5
    s.predict(); s.update(g["zs"][0][0])
    assert s.K.shape == (4, 2) and s.y.shape == (2, 1) and s.S1_2.shape == (2, 2) and s.x_prior.shape == (4, 1)
    assert np.allclose(s.P_post, s.P_prior)              # the reference's P_post reads the prior factor


def test_torch_op_equals_mirror(golden):
    import torch
    from filterpy_b200 import torch_ops
    ops = torch_ops.load()
    g = golden("srkf_bank_4_2")
    s = make(g, np.float64, diagnostics=False)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()      # noqa: E731
    L0, Lq, Lr = (dev(np.linalg.cholesky(g[k])) for k in ("P", "Q", "R"))
    x, L = ops.srkf_step(dev(g["x"]), L0, dev(g["F"]), dev(g["H"]), Lq, Lr, dev(g["zs"][0]))
    s.predict(); s.update(g["zs"][0])
    rel_close(x.cpu().numpy(), s.x.cpu().numpy(), 1e-12, "x"); rel_close(L.cpu().numpy(), s.P1_2.cpu().numpy(), 1e-12, "L")


@pytest.mark.parametrize("dtype", [np.float32])
def test_1m_bank_vs_oracle_subset(dtype):
    """2^20 filters, 4/2 CV with per-filter models (Q made positive definite), the register tile: a seeded
    4096-filter subset against the fp64 dgeqr2 oracle."""
    from filterpy_b200.common import workloads as wl
    from oracle import srkf as osr
    N, T = 1 << 20, 3
    w = wl.kf_bank_cv2d(N, seed=1234, steps=T)
    w["Q"] = osr.make_pd(w["Q"])
    g = dict(w, valid=np.ones((T, N), bool), rec_steps=np.arange(T))
    s = make(g, dtype, diagnostics=False)
    sel = np.sort(np.random.default_rng(0).choice(N, 4096, replace=False))
    sub = {k: (v[:, sel] if k == "zs" else (v[sel] if np.ndim(v) >= 2 and np.shape(v)[0] == N else v)) for k, v in w.items()}
    sub.update(valid=np.ones((T, 4096), bool))
    ref = list(bank_replay(sub))
    for t in range(T):
        s.predict(); s.update(w["zs"][t])
    o = ref[-1][3]
    rel_close(s.x.cpu().numpy()[sel], o["x"], RTOL[dtype], "x")
    rel_close(s.P1_2.cpu().numpy()[sel], o["L"], RTOL[dtype], "P1_2")


def test_ill_conditioned_bank_fp32_within_1e3_of_fp64_reference(golden):
    """The contrast that motivates the filter, on the GPU: the fp32 square-root bank's P stays within 1e-3 of
    max|P| of the fp64 Joseph-form filter over 300 steps (the fp32 Joseph form does not, test_oracle_srkf)."""
    from oracle import srkf as osr
    g = golden("srkf_ill_4_2")
    s = make(g, np.float32, diagnostics=False)
    x, P = g["x"], g["P"]
    worst = 0.0
    for t in range(g["zs"].shape[0]):
        s.predict(); s.update(g["zs"][t])
        x, P, _, _ = osr.joseph_kf_bank(x, P, g["zs"][t], g["F"], g["H"], g["Q"], g["R"])
        worst = max(worst, osr.worst_relative_P_error(s.P.cpu().numpy()[None], P[None]))
    assert worst < 1e-3, worst
