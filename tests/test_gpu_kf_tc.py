"""The tensor-core tile (csrc/kf_tc.cu): covariance propagation
P <- alpha^2 F P F' + Q, x <- F x (filterpy/kalman/kalman_filter.py:471-478) of shared-model fp32 banks with
dim_x = 16 / 32 on wgmma (three-term TF32 split, fp32 accumulation).  Reference: the same
arithmetic in fp64 on the fp32-rounded inputs; north_star's bound is 1e-3 relative, the split holds ~1e-6."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def bank(n, m, N, seed):
    rng = np.random.default_rng(seed)

    def spd(k, cnt, scale):
        a = rng.normal(size=(cnt, k, k))
        return scale * (a @ np.swapaxes(a, -1, -2) / k + np.eye(k))
    F = np.eye(n) + 0.1 * rng.normal(size=(n, n))
    H = rng.normal(size=(m, n))
    return dict(F=F, H=H, Q=spd(n, 1, 0.05)[0], R=spd(m, 1, 0.5)[0], P=spd(n, N, 2.0), x=rng.normal(size=(N, n)),
                zs=rng.normal(size=(3, N, m)))


@pytest.mark.parametrize("n", [16, 32])
@pytest.mark.parametrize("N", [1, 7, 9, 1037, 40003])
@pytest.mark.parametrize("alpha", [1.0, 1.02])
def test_tc_predict_vs_fp64(n, N, alpha):
    from filterpy_b200.kalman import KalmanFilter
    b = bank(n, 4, N, seed=n * 7 + N)
    kf = KalmanFilter(n, 4, n_filters=N, dtype=np.float32, diagnostics=True)
    kf.x, kf.P, kf.F, kf.H, kf.Q, kf.R = b["x"], b["P"], b["F"], b["H"], b["Q"], b["R"]
    kf.alpha = alpha
    kf.predict()
    F, Q, P, x = [b[k].astype(np.float32).astype(np.float64) for k in "FQPx"]
    Pr = alpha * alpha * (F @ P @ F.T) + Q
    xr = x @ F.T
    for got, want in [(kf.P, Pr), (kf.P_prior, Pr), (kf.x, xr), (kf.x_prior, xr)]:
        got = got.cpu().numpy().astype(np.float64)
        assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max()          # three-term split; one TF32 pass: ~5e-4
    kf.check()


@pytest.mark.parametrize("n,m", [(16, 4), (16, 2), (32, 4), (32, 6)])
def test_tc_fused_steps_vs_oracle(n, m):
    """Shared F, Q, H and R: 16/4, 16/2 and 32/4 run fused on the tensor cores (kf_cov_tc_kernel<NX, dim_z>); 32/6
    (dim_z > 4) runs its predict there and its update on the catch-all kernel.  Three steps with a measurement mask,
    against the fp64 oracle."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    from oracle import kf as okf
    N = 1037
    b = bank(n, m, N, seed=n + m)
    rng = np.random.default_rng(5)
    valid = rng.random((3, N)) > 0.2
    kf = KalmanFilter(n, m, n_filters=N, dtype=np.float32, diagnostics=True)
    kf.x, kf.P, kf.F, kf.H, kf.Q, kf.R = b["x"], b["P"], b["F"], b["H"], b["Q"], b["R"]
    x, P = b["x"], b["P"]
    for t in range(3):
        kf.predict(); kf.update(torch.from_numpy(b["zs"][t]), valid=valid[t])
        o = okf.kf_step_bank(x, P, b["zs"][t], b["F"], b["H"], b["Q"], b["R"], valid=valid[t])
        x, P = o["x"], o["P"]
    kf.check()
    v = valid[2]
    for got, want, mask in [(kf.x, x, None), (kf.P, P, None), (kf.x_prior, o["x_prior"], None), (kf.P_prior, o["P_prior"], None),
                            (kf.y, o["y"], None), (kf.K, o["K"], v), (kf.S, o["S"], v), (kf.SI, o["SI"], v)]:
        got = got.cpu().numpy().astype(np.float64)
        if mask is not None:                      # K, S, SI keep their old values where z is None (kalman_filter.py:515-520)
            got, want = got[mask], want[mask]
        M_ = want.shape[0]
        mag = np.abs(want).reshape(M_, -1).max(axis=1).reshape((M_,) + (1,) * (want.ndim - 1))
        assert np.all(np.abs(got - want) <= 1e-3 * (np.abs(want) + 0.05 * mag + 1e-12))
    # log-likelihood of the last step where there was a measurement: -0.5 (y' SI y + log det S + m log 2 pi)
    yv, Sv, SIv = o["y"][v], o["S"][v], o["SI"][v]
    ll = -0.5 * (np.einsum("na,nab,nb->n", yv, SIv, yv) + np.log(np.abs(np.linalg.det(Sv))) + m * np.log(2 * np.pi))
    got = kf.log_likelihood.cpu().numpy().astype(np.float64)[v]
    assert np.all(np.abs(got - ll) <= 1e-3 * (np.abs(ll) + 1.0))


def test_tc_fused_singular_S_reports_status_and_keeps_the_prior():
    """S = H P' H' + R singular for some filters (R = 0 and a zero row of H): status 1 there, posterior := prior, the
    other filters updated (np.linalg.inv raises LinAlgError in the reference, kalman_filter.py:541)."""
    import torch
    from filterpy_b200.kalman import KalmanFilter
    n, m, N = 16, 2, 200
    b = bank(n, m, N, seed=3)
    H = b["H"].copy(); H[1] = 0.0
    R = np.diag([0.5, 0.0])
    kf = KalmanFilter(n, m, n_filters=N, dtype=np.float32, diagnostics=True)
    kf.x, kf.P, kf.F, kf.H, kf.Q, kf.R = b["x"], b["P"], b["F"], H, b["Q"], R
    kf.predict(); kf.update(torch.from_numpy(b["zs"][0]))
    st = kf.status.cpu().numpy() if hasattr(kf, "status") else None
    assert torch.equal(kf.x, kf.x_prior) and torch.equal(kf.P, kf.P_prior)
    if st is not None:
        assert np.all(st == 1)
    with pytest.raises(np.linalg.LinAlgError):
        kf.check()
