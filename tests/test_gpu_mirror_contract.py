"""The attribute contract every filter mirror keeps, in single mode (n_filters=None) and bank mode: the shapes the
state, model, measurement and mask inputs accept or reject, the NumPy shapes single mode hands out, write-back
through the single-mode arrays, live tensors in bank mode, diagnostics, the deferred predict and status / check()."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KINDS = ["kf", "ukf", "ckf", "srkf", "fls"]
MODES = {"single": None, "bank": 5}
DT = 0.1
F4 = np.array([[1, DT, 0, 0], [0, 1, 0, 0], [0, 0, 1, DT], [0, 0, 0, 1]])
H42 = np.array([[1., 0, 0, 0], [0, 0, 1, 0]])


def make(kind, N, H=H42, dim_z=2, diagnostics=True, F=F4):
    from filterpy_b200.kalman import (KalmanFilter, UnscentedKalmanFilter, CubatureKalmanFilter, SquareRootKalmanFilter,
                                      FixedLagSmoother, MerweScaledSigmaPoints, LinearFx, LinearHx)
    kw = dict(n_filters=N, diagnostics=diagnostics)
    n = F.shape[0]
    if kind == "ukf":
        return UnscentedKalmanFilter(n, dim_z, DT, LinearHx(H), LinearFx(F), MerweScaledSigmaPoints(n, .5, 2., 0.), **kw)
    if kind == "ckf":
        return CubatureKalmanFilter(n, dim_z, DT, LinearHx(H), LinearFx(F), **kw)
    f = {"kf": KalmanFilter, "srkf": SquareRootKalmanFilter}.get(kind)
    f = f(n, dim_z, **kw) if f else FixedLagSmoother(n, dim_z, 3, **kw)
    f.F, f.H = F, H
    return f


def step(f, kind, z):
    if kind == "fls":
        f.smooth(z)
    else:
        f.predict()
        f.update(z)


def z_of(N, k=0):
    z = np.array([1.0 + k, 2.0 - k])
    return z if N is None else np.tile(z, (N, 1))


def sigma(kind):
    return kind in ("ukf", "ckf")


@pytest.fixture(params=KINDS)
def kind(request):
    return request.param


@pytest.fixture(params=list(MODES))
def mode(request):
    return MODES[request.param]


def test_x_shapes(kind, mode):
    import torch
    f, N = make(kind, mode), mode
    x = np.arange(4.0)
    if N is None:
        f.x = x
        assert isinstance(f.x, np.ndarray) and f.x.shape == (4,)
        if sigma(kind):
            with pytest.raises(ValueError):
                f.x = x.reshape(4, 1)                   # the reference UKF's x is 1-D
        else:
            f.x = x.reshape(4, 1)
            assert f.x.shape == (4, 1)
        np.testing.assert_allclose(np.ravel(f.x), x)
    else:
        for v in (x, np.tile(x, (N, 1)), np.tile(x, (N, 1))[..., None]):
            f.x = v
            assert isinstance(f.x, torch.Tensor) and tuple(f.x.shape) == (N, 4)
            np.testing.assert_allclose(f.x.cpu().numpy(), np.tile(x, (N, 1)))
        f.x[1, 2] = 9.0                                 # the live tensor
        assert float(f.x[1, 2]) == 9.0
        bad = np.zeros((N + 1, 4))
        with pytest.raises(ValueError):
            f.x = bad
    with pytest.raises(ValueError):
        f.x = np.zeros(5)


def test_P_shapes(kind, mode):
    f, N = make(kind, mode), mode
    P = np.diag([1.0, 2.0, 3.0, 4.0])
    for v, want in ((3.0, 3.0 * np.eye(4)), (P, P)):
        f.P = v
        got = f.P if N is None else f.P.cpu().numpy()
        np.testing.assert_allclose(got, want if N is None else np.broadcast_to(want, (N, 4, 4)), rtol=1e-12)
    if N is not None:
        f.P = np.broadcast_to(P, (N, 4, 4))
        np.testing.assert_allclose(f.P.cpu().numpy(), np.broadcast_to(P, (N, 4, 4)), rtol=1e-12)
        if kind != "srkf":                              # P is formed from its factor there
            f.P[0, 0, 0] = 7.0
            assert float(f.P[0, 0, 0]) == 7.0
    else:
        assert isinstance(f.P, np.ndarray) and f.P.shape == (4, 4)
    with pytest.raises(ValueError):
        f.P = np.eye(3)


def test_model_shapes(kind, mode):
    f, N = make(kind, mode), mode
    Q = np.diag([1.0, 2.0, 3.0, 4.0])
    f.Q = 2.0
    np.testing.assert_allclose(np.asarray(f.Q if N is None else f.Q.cpu().numpy()), 2.0 * np.eye(4), rtol=1e-12)
    f.Q = Q
    if N is not None:
        f.Q = np.broadcast_to(Q, (N, 4, 4))
        assert tuple(f.Q.shape) == (N, 4, 4)
    with pytest.raises(ValueError):
        f.Q = np.eye(3)
    if sigma(kind):
        with pytest.raises(ValueError):
            make(kind, N, H=np.eye(3))
        with pytest.raises(ValueError):
            make(kind, N, H=1.0)                        # a scalar H of a non-square model
    else:
        with pytest.raises(ValueError):
            f.H = np.eye(3)
        with pytest.raises(ValueError):
            f.H = 1.0
        if N is not None:
            f.H = np.broadcast_to(H42, (N, 2, 4))
            assert tuple(f.H.shape) == (N, 2, 4)


def test_one_row_model_takes_a_1d_row(kind, mode):
    row = np.array([1.0, 0])
    f = make(kind, mode, H=row, dim_z=1, F=np.array([[1, DT], [0, 1]]))
    step(f, kind, 1.5 if mode is None else np.full((mode, 1), 1.5))
    x = np.ravel(f.x) if mode is None else f.x.cpu().numpy()[0]
    assert 0.0 < x[0] < 1.5


def test_z_and_valid_shapes(kind, mode):
    f, N = make(kind, mode), mode
    if N is None:
        step(f, kind, [1.0, 2.0])
        step(f, kind, np.array([[1.0], [2.0]]))
        return
    z = z_of(N)
    step(f, kind, z)
    step(f, kind, z[..., None])                         # (N, m, 1)
    with pytest.raises(ValueError):
        step(f, kind, np.zeros((N, 3)))
    if kind == "fls":
        return
    f.predict()
    f.update(z, valid=np.ones(N, bool))


@pytest.mark.parametrize("shape", ["long", "column", "short"])
def test_valid_shape_is_checked(kind, shape):
    if kind == "fls":
        pytest.skip("FixedLagSmoother takes no valid mask")
    N = MODES["bank"]
    f = make(kind, N)
    valid = {"long": np.ones(N + 1, bool), "column": np.ones((N, 1), bool), "short": np.ones(N - 1, bool)}[shape]
    f.predict()
    with pytest.raises(ValueError):
        f.update(z_of(N), valid=valid)


def test_dims_are_checked(kind):
    with pytest.raises(ValueError):
        make(kind, -1)
    if sigma(kind):
        from filterpy_b200.kalman import UnscentedKalmanFilter, CubatureKalmanFilter, MerweScaledSigmaPoints, \
            LinearFx, LinearHx
        with pytest.raises(ValueError):
            if kind == "ukf":                           # (dim_x = 0 already fails the sigma points' size check)
                UnscentedKalmanFilter(4, 0, DT, LinearHx(None), LinearFx(None), MerweScaledSigmaPoints(4, .5, 2., 0.))
            else:
                CubatureKalmanFilter(4, 0, DT, LinearHx(None), LinearFx(None))
        if kind == "ckf":
            with pytest.raises(ValueError):
                CubatureKalmanFilter(0, 2, DT, LinearHx(None), LinearFx(None))


def test_single_mode_shapes_and_write_back(kind):
    f = make(kind, None)
    x_shape = (4,) if sigma(kind) else (4, 1)
    assert f.x.shape == x_shape and f.P.shape == (4, 4)
    if kind != "fls":
        assert f.z.shape == (2, 1) and f.z[0, 0] is None
    step(f, kind, [1.0, 2.0])
    m_shape = (2,) if sigma(kind) else (2, 1)
    assert isinstance(f.y, np.ndarray) and f.y.shape == m_shape
    assert f.S.shape == (2, 2) and f.K.shape == ((4, 1) if kind == "fls" else (4, 2))
    f.x[0] = 3.0
    assert np.ravel(f.x)[0] == 3.0
    if kind != "srkf":                                  # P is formed from its factor there, as in the reference
        P = np.array(f.P)
        f.P *= 2.0
        np.testing.assert_allclose(f.P, 2.0 * P, rtol=1e-12)
    if sigma(kind):
        f.Q[0, 0] = 5.0
        assert f.Q[0, 0] == 5.0
    else:
        f.F[0, 1] = 0.5
        assert f.F[0, 1] == 0.5


def test_bank_models_are_live(kind):
    import torch
    N = MODES["bank"]
    f = make(kind, N)
    names = ("Q", "R") if sigma(kind) else ("F", "H") if kind == "srkf" else ("F", "Q", "H", "R")
    for name in names:
        t = getattr(f, name)
        assert isinstance(t, torch.Tensor) and getattr(f, name) is t


def test_diagnostics_off(kind, mode):
    f = make(kind, mode, diagnostics=False)
    step(f, kind, z_of(mode))
    names = {"kf": "x_prior P_prior x_post P_post K y S SI log_likelihood likelihood mahalanobis status",
             "srkf": "x_prior P_prior x_post P_post K y S SI S1_2 SI1_2 status",
             "fls": "y S"}
    names["ukf"] = names["ckf"] = names["kf"]
    for name in names[kind].split():
        with pytest.raises(AttributeError):
            getattr(f, name)


def test_deferred_predict_uses_the_old_model(kind, mode):
    if kind == "fls":
        pytest.skip("FixedLagSmoother has no deferred predict")
    z = z_of(mode)
    late, ref = make(kind, mode), make(kind, mode)
    late.predict()
    late.Q = 5.0                                        # the reference has already predicted with Q = I
    late.update(z)
    step(ref, kind, z)
    ref.Q = 5.0
    for a, b in ((late.x, ref.x), (late.P, ref.P)):
        a, b = (np.asarray(a), np.asarray(b)) if mode is None else (a.cpu().numpy(), b.cpu().numpy())
        np.testing.assert_allclose(a, b, rtol=1e-12)
    if mode is not None and kind != "srkf":
        inplace = make(kind, mode)
        inplace.predict()
        inplace.Q.mul_(5.0)                             # an in-place edit through the live tensor
        inplace.update(z)
        np.testing.assert_allclose(inplace.P.cpu().numpy(), ref.P.cpu().numpy(), rtol=1e-12)


def test_status_and_check(kind):
    import torch
    N = MODES["bank"]
    f = make(kind, N)
    step(f, kind, z_of(N))
    st = f.status
    assert isinstance(st, torch.Tensor) and st.dtype == torch.int32 and tuple(st.shape) == (N,)
    assert int(st.abs().sum()) == 0
    f.check()
    # H = 0 and R = 0: S = 0, which the reference cannot invert
    g = make(kind, N, H=np.zeros((2, 4)))
    if kind == "srkf":
        g.predict()
        g.update(z_of(N), R2=0.0)
    else:
        g.R = 0.0
        step(g, kind, z_of(N))
    assert int((g.status != 0).sum()) == N
    with pytest.raises(np.linalg.LinAlgError):
        g.check()
