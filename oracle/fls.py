"""FixedLagSmoother oracles (filterpy/kalman/fixed_lag_smoother.py, reference @ 3b51149).

Two restatements of ``smooth`` (:133-215) / ``smooth_batch`` (:217-311):

* ``fls_smooth_single``: one filter, the reference's own statements in its own order (``scipy.linalg.inv``,
  the smoothed gain ``PS HTSI`` formed before it multiplies ``y``), appending to a Python list the way
  ``self.xSmooth`` grows.
* ``fls_bank``: vectorised over a bank of Nf filters, the same association as the reference (HTSI, F_LH and PS
  as matrices).  A singular S follows the kernel's rule (include/bke.h, ``bke_fls_args``): status 1, the
  filter keeps its prior for the epoch and no row is corrected, where the reference raises LinAlgError.

Both keep the reference's order of operations; the CUDA kernels reassociate the correction as P (A^i g)
(DESIGN.md §3.4b) and are held to these within the tests' tolerances.
"""
import numpy as np
import scipy.linalg

STATUS_SINGULAR_S = 1


def fls_smooth_single(state, z, u=None):
    """One ``smooth(z, u)`` call (:161-215) on ``state``, a dict with x, P, F, H, Q, R, B, N, count and the list
    xSmooth; updates it in place and sets y and S as the reference does."""
    H, R, F, P, x, Q, B, N = (state[k] for k in ("H", "R", "F", "P", "x", "Q", "B", "N"))
    k = state["count"]
    x_pre = np.dot(F, x)                                           # :174-178
    if u is not None:
        x_pre += np.dot(B, u)
    P = np.dot(F, P).dot(F.T) + Q
    state["y"] = z - np.dot(H, x_pre)                              # :181-191
    state["S"] = np.dot(H, P).dot(H.T) + R
    SI = scipy.linalg.inv(state["S"])
    K = np.dot(P, H.T).dot(SI)
    x = x_pre + np.dot(K, state["y"])
    I_KH = np.eye(len(x)) - np.dot(K, H)
    P = np.dot(I_KH, P).dot(I_KH.T) + np.dot(K, R).dot(K.T)
    state["xSmooth"].append(x_pre.copy())                          # :193
    HTSI = np.dot(H.T, SI)                                         # :196-197
    F_LH = (F - np.dot(K, H)).T
    if k >= N:                                                     # :199-206
        PS = P.copy()
        for i in range(N):
            K = np.dot(PS, HTSI)
            PS = np.dot(PS, F_LH)
            si = k - i
            state["xSmooth"][si] = state["xSmooth"][si] + np.dot(K, state["y"])
    else:                                                          # :207-211
        state["xSmooth"][k] = x.copy()
    state["count"] += 1
    state["x"], state["P"] = x, P


def fls_smooth_batch_single(x, P, F, H, Q, R, zs, N, B=0., us=None):
    """``smooth_batch(zs, N, us)`` (:253-311): returns (xSmooth, xhat); touches nothing it is given."""
    shape = (len(zs),) + np.shape(x)
    xSmooth, xhat = np.zeros(shape), np.zeros(shape)
    st = dict(x=x, P=P, F=F, H=H, Q=Q, R=R, B=B, N=N, count=0, xSmooth=[])
    for k, z in enumerate(zs):
        fls_smooth_single(st, z, None if us is None else us[k])
        xhat[k] = st["x"]
    xSmooth[:] = np.array(st["xSmooth"]).reshape(shape)
    return xSmooth, xhat


def _per(a, Nf):
    """a model given per filter ([Nf, r, c]) or shared ([r, c]) as a [Nf, r, c] view."""
    a = np.asarray(a)
    return a if a.ndim == 3 else np.broadcast_to(a, (Nf,) + a.shape)


def fls_bank(x, P, F, H, Q, R, zs, N, B=None, us=None, count=0, hist=None):
    """T epochs of ``smooth`` for Nf filters at once, continuing a run of ``count`` epochs whose history is
    ``hist`` ([count, Nf, n], or None when count is 0).  Returns dict(xs [count+T, Nf, n], xhat [T, Nf, n],
    x, P, y, S of the last epoch, status [Nf])."""
    x, P = np.array(x, np.float64), np.array(P, np.float64)
    Nf, n = x.shape
    F, H, Q, R = (_per(a, Nf) for a in (F, H, Q, R))
    T = len(zs)
    xs = np.zeros((count + T, Nf, n))
    if count:
        xs[:count] = hist
    xhat = np.zeros((T, Nf, n))
    status = np.zeros(Nf, np.int32)
    cond = np.ones(Nf)
    eye = np.eye(n)
    HT, FT = np.swapaxes(H, 1, 2), np.swapaxes(F, 1, 2)
    for t in range(T):
        k = count + t
        x_pre = np.einsum("fij,fj->fi", F, x)
        if us is not None:
            x_pre = x_pre + np.einsum("fij,fj->fi", _per(B, Nf), us[t])
        Pp = F @ P @ FT + Q
        y = zs[t] - np.einsum("fij,fj->fi", H, x_pre)
        S = H @ Pp @ HT + R
        ok = np.abs(np.linalg.det(S)) > 0
        SI = np.zeros_like(S)
        SI[ok] = np.linalg.inv(S[ok])
        if ok.any():
            cond[ok] = np.maximum(cond[ok], np.linalg.cond(S[ok]))
        K = Pp @ HT @ SI
        xn = x_pre + np.einsum("fia,fa->fi", K, y)
        I_KH = eye - K @ H
        Pn = I_KH @ Pp @ np.swapaxes(I_KH, 1, 2) + K @ R @ np.swapaxes(K, 1, 2)
        status[~ok] = STATUS_SINGULAR_S
        x = np.where(ok[:, None], xn, x_pre)
        P = np.where(ok[:, None, None], Pn, Pp)
        xhat[t] = x
        xs[k] = x_pre
        if k >= N:
            HTSI = HT @ SI
            F_LH = np.swapaxes(F - K @ H, 1, 2)
            PS = P.copy()
            for i in range(N):
                Ki = PS @ HTSI
                PS = PS @ F_LH
                xs[k - i, ok] += np.einsum("fia,fa->fi", Ki, y)[ok]
        else:
            xs[k] = x
    return dict(xs=xs, xhat=xhat, x=x, P=P, y=y, S=S, status=status, cond=cond)
