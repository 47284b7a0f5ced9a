"""GPU: InformationFilter banks, in fp32 and fp64, against the reference's golden vectors; status and
BKE_STATUS_STICKY through the mirror, fused against split launches, single mode's exceptions and the torch op.
Every kernel instance against the fp64 oracle: test_gpu_if_instances."""

import numpy as np
import pytest
import torch

from filterpy_b200 import _lib
from filterpy_b200.kalman import InformationFilter

from test_oracle_information import GOLDEN, STEPS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {np.float64: 1e-6, np.float32: 1e-3}
DIVERGING = "if_noinfo_4_2"           # x grows about tenfold per step: fp32 is held to the branch only


def _np(t):
    return t.detach().double().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t, np.float64)


def _err(a, b):
    a, b = _np(a), np.asarray(b, np.float64)
    fin = np.isfinite(b)
    return np.abs(a[fin] - b[fin]).max(initial=0) / max(np.abs(b[fin]).max(initial=0), 1e-300)


def _bank(g, dtype, N=None):
    N0, n = g["x"].shape
    m = g["H"].shape[-2]
    f = InformationFilter(n, m, dim_u=g["B"].shape[-1] if "B" in g else 0, compute_log_likelihood=bool(g["compute_ll"]),
                          n_filters=N0, dtype=dtype, device=DEV)
    f.x, f.P_inv, f.Q, f.H, f.R_inv = g["x"], g["P_inv"], g["Q"], g["H"], g["R_inv"]
    if "B" in g:
        f.B = g["B"]
    if "F_set" in g:
        f.F = g["F_set"]
        f.F.copy_(torch.as_tensor(g["F"], dtype=f.F.dtype, device=DEV))         # in place: F_inv stays
    elif "F_assigned" in g:
        f.F = g["F_assigned"]
        with pytest.raises(np.linalg.LinAlgError, match="4 of 4"):
            f.F = g["F"]
    else:
        f.F = g["F"]
    return f


def _step(f, g, t):
    u = g["us"][t] if "us" in g else 0
    valid = g["valid"][t]
    for op in str(g["order"]):
        if op == "p":
            f.predict(u)
        else:
            f.update(g["zs"][t], valid=valid)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", [n for n in GOLDEN if n not in ("if_raise_ll_4_2",)])
def test_bank_matches_golden(golden, name, dtype):
    if name == "if_test_1d_0P" and dtype == np.float32:
        pytest.skip("P_inv = 1e-21 I: det(A) = 1e-42 is below fp32's normal range")
    g = golden(name)
    T = STEPS.get(name, g["zs"].shape[0])
    f = _bank(g, dtype)
    for t in range(T):
        _step(f, g, t)
        raised = g["raise_step"] >= 0
        ok = ~raised | (g["raise_step"] > t)
        assert np.array_equal(_np(f._no_information)[ok], g["out_ni"][t][ok]), t
        if dtype == np.float32 and name == DIVERGING:
            continue
        for k in ("x", "P_inv"):
            got = getattr(f, k)
            assert _err(_np(got)[ok], g["out_" + k][t][ok]) < TOL[dtype], (k, t)
        if bool(g["compute_ll"]) and name != "if_test_1d_0P":
            assert _err(f.log_likelihood[ok], g["out_ll"][t][ok]) < TOL[dtype] * 10, t
        if str(g["order"]) == "pu":         # (update first: the predict after a failed update writes its own status)
            st = _np(f.status) != 0
            assert np.array_equal(st, raised & (g["raise_type"] == "LinAlgError") & (g["raise_step"] <= t))


def test_bank_status_of_a_singular_S(golden):
    g = golden("if_raise_S")
    f = _bank(g, np.float64)
    f.update(g["zs"][0])
    assert int(f.status[0]) == _lib.BKE_STATUS_SINGULAR_S
    assert _err(f.y, g["out_y"][0]) < 1e-12 and _err(f.S, g["out_S"][0]) < 1e-12
    assert _err(f.x, g["x"]) < 1e-12                        # x and P_inv are kept
    with pytest.raises(np.linalg.LinAlgError, match="1 of 1"):
        f.check()


def test_bank_raises_the_log_likelihood_error(golden):
    g = golden("if_raise_ll_4_2")
    f = _bank(g, np.float64)
    f.predict()
    with pytest.raises(ValueError, match="broadcast"):
        f.update(g["zs"][0])
    assert _err(f.x, g["out_x"][0]) < 1e-9 and _err(f.P_inv, g["out_P_inv"][0]) < 1e-9
    assert _err(f.z, g["zs"][0]) == 0                       # z is stored before the logpdf raises (:232)


@pytest.mark.parametrize("name", ["if_test_1d", "if_test_against_kf", "if_raise_F", "if_raise_AIQ", "if_raise_S",
                                  "if_raise_ll_4_2", "if_stale_F_inv"])
def test_single_mode_raises_where_the_reference_does(golden, name):
    g = golden(name)
    N, n = g["x"].shape
    m = g["H"].shape[1]
    T = STEPS.get(name, g["zs"].shape[0])
    for fi in range(min(N, 2)):
        f = InformationFilter(n, m, compute_log_likelihood=bool(g["compute_ll"]), device=DEV)
        f.x = g["x"][fi].reshape(n, 1); f.P_inv = g["P_inv"][fi]
        f.Q, f.H, f.R_inv = g["Q"][fi], g["H"][fi], g["R_inv"][fi]
        if "F_set" in g:
            f.F = g["F_set"][fi]
            f.F[...] = g["F"][fi]                          # write-back of an in-place edit: F_inv stays
        elif "F_assigned" in g:
            f.F = g["F_assigned"][fi]
            with pytest.raises(np.linalg.LinAlgError):
                f.F = g["F"][fi]
        else:
            f.F = g["F"][fi]
        rs, rop, rtype = int(g["raise_step"][fi]), str(g["raise_op"][fi]), str(g["raise_type"][fi])
        for t in range(T if rs < 0 else rs + 1):
            z = g["zs"][t, fi].reshape(m, 1) if g["valid"][t, fi] else None
            for op in str(g["order"]):
                if t == rs and op == rop:
                    exc = np.linalg.LinAlgError if rtype == "LinAlgError" else ValueError
                    with pytest.raises(exc):
                        f.predict() if op == "p" else f.update(z)
                    break
                f.predict() if op == "p" else f.update(z)
            assert _err(f.x.reshape(-1), g["out_x"][t, fi]) < 1e-9, t
            assert _err(f.P_inv, g["out_P_inv"][t, fi]) < 1e-9, t
            assert f._no_information == bool(g["out_ni"][t, fi])
            if t == rs and rtype == "ValueError":
                assert _err(f.z.reshape(-1), g["zs"][t, fi]) == 0      # stored before the logpdf raises (:232)
            if rs < 0 or t < rs:
                assert _err(f.y.reshape(-1), g["out_y"][t, fi]) < 1e-9
                assert _err(f.S, g["out_S"][t, fi]) < 1e-9


def test_single_mode_attributes():
    f = InformationFilter(2, 1, device=DEV)
    assert f.F == 0.
    with pytest.raises(AttributeError):
        f.predict()
    with pytest.raises(NotImplementedError):
        f.batch_filter([1., 2.])
    f.F = np.array([[1., 1.], [0., 1.]])
    f.P_inv = 0.
    with pytest.raises(np.linalg.LinAlgError):
        f.P
    f.P_inv = 4.
    assert np.allclose(f.P, np.eye(2) / 4)
    assert f.inv is np.linalg.inv
    f.update(None)
    assert f.z is None


# ---------------------------------------------------------------------------------------------- random banks
def _random(N, n, m, seed, shared=False, ni_frac=0.3):
    rng = np.random.default_rng(seed)
    F = np.eye(n) + 0.1 * rng.standard_normal((N, n, n))
    H = np.eye(m, n) + 0.3 * rng.standard_normal((N, m, n))     # H' H well conditioned where m >= n
    a = rng.standard_normal((N, n, n)); Q = 0.05 * (a @ a.transpose(0, 2, 1)) / n + 0.5 * np.eye(n)
    b = rng.standard_normal((N, m, m)); R = (b @ b.transpose(0, 2, 1)) / m + 0.5 * np.eye(m)
    c = rng.standard_normal((N, n, n)); P = (c @ c.transpose(0, 2, 1)) / n + np.eye(n)
    P_inv = np.linalg.inv(P)
    none = rng.random(N) < ni_frac
    P_inv[none] = 0.                                       # no information: both branches in every warp
    valid = rng.random((4, N)) > 0.2
    if m < n:
        valid[:, none] = False     # H' R_inv H alone would leave A singular by rounding, not by structure
    if shared:
        F, H, Q, R = F[0], H[0], Q[0], R[0]
    g = dict(x=rng.standard_normal((N, n)), P_inv=P_inv, F=F, H=H, Q=Q, R_inv=np.linalg.inv(R),
             zs=rng.standard_normal((4, N, m)), valid=valid, order=np.array("pu"),
             compute_ll=np.array(m in (1, n)))
    return g


@pytest.mark.parametrize("shape", [(4, 2), (5, 3)])
def test_status_and_sticky(shape):
    n, m = shape
    N = 64
    g = _random(N, n, m, seed=9, ni_frac=0.)
    g["Q"] = np.broadcast_to(g["Q"], (N, n, n)).copy()
    bad = np.arange(N) % 5 == 0
    # inv(AI + Q) singular: F = I, P_inv = I, Q = -I
    g["F"][bad] = np.eye(n); g["P_inv"][bad] = np.eye(n); g["Q"][bad] = -np.eye(n)
    f = _bank(g, np.float64)
    f.predict(); f.update(g["zs"][0])
    assert np.array_equal(_np(f.status) != 0, bad)
    with pytest.raises(np.linalg.LinAlgError, match="%d of %d" % (bad.sum(), N)):
        f.check()
    # sticky: a split predict keeps its failure through the update that follows
    f2 = _bank(g, np.float64)
    f2.predict()
    f2.F                                                    # flushes the predict on its own
    f2.update(g["zs"][0])
    assert np.array_equal(_np(f2.status) != 0, bad)
    # and the filters whose predict failed get no update, as in the fused launch
    assert torch.equal(f.x, f2.x) and torch.equal(f.P_inv, f2.P_inv) and torch.equal(f._ni, f2._ni)
    # update(None) completes the step: the next step's first launch writes status afresh
    f3 = _bank(g, np.float64)
    f3.predict(); f3.x
    f3.update(None)
    assert np.array_equal(_np(f3.status) != 0, bad)
    f3.Q = np.broadcast_to(np.eye(n), (N, n, n)).copy()      # no filter fails from here on
    f3.predict(); f3.update(g["zs"][1])
    assert not bool(f3.status.any())


def test_single_mode_raises_without_diagnostics():
    f = InformationFilter(2, 1, device=DEV, diagnostics=False)
    f.F = np.eye(2); f.P_inv = np.eye(2); f.Q = -np.eye(2)
    with pytest.raises(np.linalg.LinAlgError):
        f.predict()                                         # inv(AI + Q) = inv(0)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("shape", [(4, 2), (9, 3)])
def test_fused_equals_split_bit_for_bit(shape, dtype):
    n, m = shape
    g = _random(500, n, m, seed=11)
    fa, fb = _bank(g, dtype), _bank(g, dtype)
    for t in range(4):
        fa.predict(); fa.update(g["zs"][t], valid=g["valid"][t])
        fb.predict(); fb.x                                  # flush: a predict-only launch
        fb.update(g["zs"][t], valid=g["valid"][t])
    assert torch.equal(fa.x, fb.x) and torch.equal(fa.P_inv, fb.P_inv)
    assert torch.equal(fa._ni, fb._ni)


def test_bank_P_is_nan_where_P_inv_is_singular():
    g = _random(64, 4, 2, seed=3, ni_frac=0.5)
    f = _bank(g, np.float64)
    P = _np(f.P)
    zero = (g["P_inv"] == 0).all(axis=(1, 2))
    assert np.isnan(P[zero]).all() and np.isfinite(P[~zero]).all()
    assert np.allclose(P[~zero], np.linalg.inv(g["P_inv"][~zero]))


def test_torch_op_matches_mirror():
    from filterpy_b200 import torch_ops
    ops = torch_ops.load()
    g = _random(256, 4, 2, seed=13)
    f = _bank(g, np.float64)
    x, Pi, ni = f.x.clone(), f.P_inv.clone(), f._ni.clone()
    zs = torch.as_tensor(g["zs"][0], device=DEV)
    f.predict(); f.update(zs)
    x2, P2, ni2, st2 = ops.if_step(x, Pi, ni, f._F, f._F_inv, f._Q, f._H, f._R_inv, zs)
    assert torch.equal(x2, f.x) and torch.equal(P2, f.P_inv) and torch.equal(ni2, f._ni)
    assert torch.equal(st2, f.status) and not bool(st2.any())
    # a failing filter is reported: inv(AI + Q) = inv(0) with F = I, P_inv = I, Q = -I
    eye = torch.eye(4, dtype=torch.float64, device=DEV)
    x3, P3, ni3, st3 = ops.if_step(x[:2].contiguous(), eye.expand(2, 4, 4).contiguous(), ni[:2].contiguous(), eye, eye,
                                   -eye, f._H[:2].contiguous(), f._R_inv[:2].contiguous(), zs[:2].contiguous())
    assert st3.tolist() == [_lib.BKE_STATUS_SINGULAR_S] * 2
