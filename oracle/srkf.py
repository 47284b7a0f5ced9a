"""Oracle: square-root Kalman filter (TEST INFRASTRUCTURE).

Restates filterpy/kalman/square_root.py (reference @ 3b51149) twice:

* ``srkf_predict_single`` / ``srkf_update_single``: one filter, the reference's literal call sequence —
  ``predict`` :239-248 and ``update`` :189-224 with ``scipy.linalg.qr`` and ``pinv``.
* ``srkf_step_bank``: vectorised over N with ``dgeqr2``, a NumPy restatement of the QR that LAPACK runs for
  ``scipy.linalg.qr`` at these sizes (dgeqr2 / dlarfg, with their signs), in the dtype of its inputs.  A zero
  diagonal entry of S1_2 keeps the prior and sets K = SI1_2 = 0 (the CUDA kernel's rule, include/bke.h).

``joseph_kf_bank`` is the linear filter's Joseph form (kalman_filter.py:533-556) in the dtype of its inputs,
the accuracy yardstick of the square-root form.  ``make_pd`` lifts the workloads' rank-deficient white-noise
Q to a positive definite one, which the reference's ``cholesky`` setter accepts.

Parity: pinned by ``tests/golden/srkf_*.npz``.
"""
import numpy as np
import scipy.linalg

STATUS_OK, STATUS_SINGULAR_S = 0, 1


def _T(a):
    return np.swapaxes(a, -1, -2)


def make_pd(Q, eps=1e-3):
    """Q + eps * max|Q| * I per filter: the workloads' discrete white-noise Q is rank-deficient and
    scipy.linalg.cholesky refuses it."""
    Q = np.asarray(Q)
    scale = np.abs(Q).max(axis=(-1, -2), keepdims=True)
    return Q + eps * scale * np.eye(Q.shape[-1], dtype=Q.dtype)


# --------------------------------------------------------------------------- single filter, literal
def srkf_predict_single(x, L, F, Lq, B=0., u=0):
    """square_root.py:239-248 -> (x, L)."""
    n = L.shape[0]
    x = np.dot(F, x) + np.dot(B, u)
    _, P2 = scipy.linalg.qr(np.hstack([np.dot(F, L), Lq]).T)
    return x, P2[:n, :n].T


def srkf_update_single(x, L, z, H, Lr):
    """square_root.py:195-224 with R2 = Lr (an m x m matrix) -> dict(x, L, K, y, S1_2, SI1_2)."""
    m, n = H.shape
    M = np.zeros((m + n, m + n))
    M[0:m, 0:m] = Lr.T
    M[m:, 0:m] = np.dot(H, L).T
    M[m:, m:] = L.T
    _, r = scipy.linalg.qr(M)
    S1_2 = r[0:m, 0:m].T
    SI1_2 = scipy.linalg.pinv(S1_2)
    K = np.dot(r[0:m, m:].T, SI1_2)
    y = z - np.dot(H, x)
    x = x + np.dot(K, y)
    return dict(x=x, L=r[m:, m:].T, K=K, y=y, S1_2=S1_2, SI1_2=SI1_2)


# --------------------------------------------------------------------------- dgeqr2, batched
def dgeqr2(A):
    """R of A[..., r, c] as scipy.linalg.qr(A)[1] gives it (upper triangular, zeros below, r x c), computed the
    way LAPACK's dgeqr2 / dlarfg do: per column, tau = 0 when the sub-column is exactly zero, else
    beta = -copysign(sqrt(alpha^2 + |sub|^2), alpha) and H = I - tau v v' applied to the columns to the right."""
    return _dgeqr2(A)[0]


def dgeqr2_pivot_ratio(A):
    """(smallest |alpha| / norm, smallest |sub| / norm) over the reflections dgeqr2 applies to A, with
    norm = sqrt(alpha^2 + |sub|^2) (1.0 when it applies none).  Near 0, a rounding difference can flip the sign
    of a row of R: alpha near 0 changes the sign of beta, and a sub-column of rounding noise decides between a
    reflection (which negates the row) and none."""
    ra, rs = _dgeqr2(A)[1:]
    return float(np.min(ra)), float(np.min(rs))


def dgeqr2_pivot_ratios(A):
    """dgeqr2_pivot_ratio per matrix: two arrays of the leading shape of A[..., r, c]."""
    return _dgeqr2(A)[1:]


def _dgeqr2(A):
    A = np.array(A, copy=True)
    rows, cols = A.shape[-2:]
    one = A.dtype.type(1)
    ra, rs = np.ones(A.shape[:-2]), np.ones(A.shape[:-2])
    for j in range(min(rows - 1, cols)):
        sub = A[..., j + 1:, j]
        ss = np.sum(sub * sub, axis=-1)
        act = ss != 0
        alpha = A[..., j, j]
        with np.errstate(divide="ignore", invalid="ignore"):
            nrm = np.sqrt(alpha * alpha + ss)
            ra = np.where(act, np.minimum(ra, np.abs(alpha) / nrm), ra)
            rs = np.where(act, np.minimum(rs, np.sqrt(ss) / nrm), rs)
        beta = -np.copysign(np.sqrt(alpha * alpha + ss), alpha)
        with np.errstate(divide="ignore", invalid="ignore"):
            tau = np.where(act, (beta - alpha) / beta, 0)
            sc = np.where(act, one / (alpha - beta), 1)
        v = sub * sc[..., None]
        A[..., j + 1:, j] = np.where(act[..., None], v, sub)
        A[..., j, j] = np.where(act, beta, alpha)
        if j + 1 < cols:
            V = np.where(act[..., None], v, 0)
            blk = A[..., j:, j + 1:]
            w = blk[..., 0, :] + np.einsum("...i,...ik->...k", V, blk[..., 1:, :])
            w = w * tau[..., None]
            A[..., j, j + 1:] = blk[..., 0, :] - w
            A[..., j + 1:, j + 1:] = blk[..., 1:, :] - V[..., :, None] * w[..., None, :]
    return np.triu(A), ra, rs


def _tri_inv_lower(S):
    """S^-1 for lower-triangular S[..., m, m] by forward substitution."""
    m = S.shape[-1]
    X = np.zeros_like(S)
    for c in range(m):
        for i in range(c, m):
            s = (1.0 if i == c else 0.0) - np.einsum("...k,...k->...", S[..., i, c:i], X[..., c:i, c])
            X[..., i, c] = s / S[..., i, i]
    return X


def srkf_step_bank(x, L, z, F, H, Lq, Lr, valid=None, predict=True, update=True, B=None, u=None):
    """One (predict and/or update) step for x[N,n], L[N,n,n]; models [N,..] or shared; z[N,m]; valid bool[N].
    Arithmetic in the dtype of x.  Returns dict(x, L, x_prior, L_prior, K, y, S1_2, SI1_2, status) — the
    update outputs are NaN for filters without a measurement (the kernel leaves them untouched)."""
    x, L = np.array(x), np.array(L)
    N, n = x.shape
    dt = x.dtype
    out = {}
    if predict:
        x = np.matmul(F, x[..., None])[..., 0]
        if B is not None and u is not None:
            x = x + np.matmul(B, u[..., None])[..., 0]
        A = np.concatenate([_T(np.matmul(F, L)), np.broadcast_to(_T(Lq), (N, n, n))], axis=-2)
        L = _T(dgeqr2(A)[..., :n, :n])
        out["x_prior"], out["L_prior"] = x.copy(), L.copy()
    status = np.zeros(N, np.int32)
    if update:
        m = np.shape(H)[-2]
        v = np.ones(N, bool) if valid is None else np.asarray(valid, bool)
        Mx = np.zeros((N, m + n, m + n), dt)
        Mx[:, :m, :m] = _T(np.broadcast_to(Lr, (N, m, m)))
        Mx[:, m:, :m] = _T(np.matmul(H, L))
        Mx[:, m:, m:] = _T(L)
        r = dgeqr2(Mx)
        S1_2 = _T(r[:, :m, :m])
        diag = np.diagonal(S1_2, axis1=-2, axis2=-1)
        ok = np.all(diag != 0, axis=-1)
        with np.errstate(divide="ignore", invalid="ignore"):
            SI1_2 = np.where(ok[:, None, None], _tri_inv_lower(S1_2), 0).astype(dt)
        K = np.matmul(_T(r[:, :m, m:]), SI1_2)
        y = np.asarray(z, dt) - np.matmul(H, x[..., None])[..., 0]
        upd = v & ok
        x = np.where(upd[:, None], x + np.matmul(K, y[..., None])[..., 0], x)
        L = np.where(upd[:, None, None], _T(r[:, m:, m:]), L)
        status[v & ~ok] = STATUS_SINGULAR_S
        nan = lambda a: np.where(v.reshape((N,) + (1,) * (a.ndim - 1)), a, np.nan)   # noqa: E731
        out.update(K=nan(K), y=nan(y), S1_2=nan(S1_2), SI1_2=nan(SI1_2))
    out.update(x=x, L=L, status=status)
    return out


# --------------------------------------------------------------------------- the linear filter, Joseph form
def joseph_kf_bank(x, P, z, F, H, Q, R):
    """kalman_filter.py:471-478 then :533-556 for a bank, in the dtype of x (no up-cast) -> (x, P, x_prior, P_prior)."""
    n = x.shape[-1]
    xp = np.matmul(F, x[..., None])[..., 0]
    Pp = np.matmul(np.matmul(F, P), _T(F)) + Q
    y = z - np.matmul(H, xp[..., None])[..., 0]
    PHT = np.matmul(Pp, _T(H))
    S = np.matmul(H, PHT) + R
    K = np.matmul(PHT, np.linalg.inv(S))
    xn = xp + np.matmul(K, y[..., None])[..., 0]
    I_KH = np.eye(n, dtype=x.dtype) - np.matmul(K, H)
    Pn = np.matmul(np.matmul(I_KH, Pp), _T(I_KH)) + np.matmul(np.matmul(K, R), _T(K))
    return xn, Pn, xp, Pp


def ill_conditioned_bank(N=16, steps=300, q=1e-8, r=1e-4, p0=1e4, dt=0.1, seed=11):
    """The 4/2 constant-velocity bank on which fp32 Joseph form loses more than 1e-3 and the square-root
    form does not: Q = q I, R = r I, P0 = p0 I, dt = 0.1, a measured track of per-filter random walks."""
    rng = np.random.default_rng(seed)
    F1 = np.array([[1., dt], [0., 1.]])
    F = np.kron(np.eye(2), F1)
    H = np.zeros((2, 4)); H[0, 0] = 1; H[1, 2] = 1
    x0 = rng.standard_normal((N, 4))
    xt = x0 + rng.standard_normal((N, 4))
    zs = np.zeros((steps, N, 2))
    for t in range(steps):
        xt = xt @ F.T + np.sqrt(q) * rng.standard_normal((N, 4))
        zs[t] = xt @ H.T + np.sqrt(r) * rng.standard_normal((N, 2))
    return dict(x=x0, P=np.broadcast_to(p0 * np.eye(4), (N, 4, 4)).copy(), F=F, H=H, Q=q * np.eye(4),
                R=r * np.eye(2), zs=zs)


def worst_relative_P_error(Ps, Ps_ref):
    """max over steps of max|dP| / max|P_ref| (per step, over the whole bank)."""
    Ps, Ps_ref = np.asarray(Ps, np.float64), np.asarray(Ps_ref, np.float64)
    ax = tuple(range(1, Ps.ndim))
    return float((np.abs(Ps - Ps_ref).max(axis=ax) / np.abs(Ps_ref).max(axis=ax)).max())
