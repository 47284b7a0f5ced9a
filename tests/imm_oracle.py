"""IMMEstimator.batch_filter restated in NumPy fp64 for N tracks with per-track models: T epochs of predict();
update(z or None) as a loop over oracle.imm's bank forms (mixing, combined estimate, mode probabilities) and
oracle.kf's single-filter steps.  A model without a measurement keeps its prior and scores log N(0; 0, S) of the S
of its last real update."""
import numpy as np

from oracle import imm as oimm
from oracle import kf as okf


def imm_batch(x0, P0, F, Q, H, R, alpha_sq, mu0, trans, zs, valid):
    """x0 [N,M,n], P0 [N,M,n,n], F, Q [N,M,n,n], H [m,n] or [N,M,m,n], R [m,m] or [N,M,m,m], alpha_sq [M],
    mu0 [M] or [N,M], trans [M,M], zs [T,N,m], valid [T,N] (bool).  Returns a dict of per-epoch arrays
    x, P, xp, Pp [T,N,...], mu, cbar, lik [T,N,M], omega [T,N,M,M], fx [T,N,M,n], fP [T,N,M,n,n]."""
    N, M, n = x0.shape
    T, _, m = zs.shape
    H = np.broadcast_to(H, (N, M, m, n)); R = np.broadcast_to(R, (N, M, m, m))
    xs = np.array(x0.transpose(1, 0, 2), float)
    Ps = np.array(P0.transpose(1, 0, 2, 3), float)
    S = np.zeros((M, N, m, m))
    ll = np.zeros((M, N))
    mu = np.broadcast_to(np.asarray(mu0, float), (N, M))
    mu = mu / mu.sum(axis=1, keepdims=True)
    mu, cbar, omega = oimm.mm_probabilities_bank(mu, trans=trans)
    out = {k: [] for k in ("x", "P", "xp", "Pp", "mu", "cbar", "omega", "lik", "fx", "fP")}
    for k in range(T):
        x0m, P0m = oimm.mm_mix_bank(xs, Ps, omega)
        for j in range(M):
            for i in range(N):
                xs[j, i], Ps[j, i] = okf.kf_predict_single(x0m[j, i], P0m[j, i], F[i, j], Q[i, j], alpha_sq[j])
        xp, Pp = oimm.mm_estimate_bank(xs, Ps, mu)
        for j in range(M):
            for i in range(N):
                if valid[k, i]:
                    xs[j, i], Ps[j, i], y, _, S[j, i], _ = okf.kf_update_single(xs[j, i], Ps[j, i], zs[k, i], H[i, j], R[i, j])
                    ll[j, i] = okf.log_likelihood_bank(y[None], S[j, i][None])[0]
                else:
                    ll[j, i] = okf.missed_log_likelihood_bank(S[j, i][None])[0]
        mu, cbar, omega = oimm.mm_probabilities_bank(mu, ll.T, cbar, trans)
        x, P = oimm.mm_estimate_bank(xs, Ps, mu)
        lik = np.exp(ll.T)
        for name, v in (("x", x), ("P", P), ("xp", xp), ("Pp", Pp), ("mu", mu), ("cbar", cbar), ("omega", omega),
                        ("lik", np.where(lik == 0.0, oimm.FLOAT_MIN, lik)), ("fx", xs.transpose(1, 0, 2).copy()),
                        ("fP", Ps.transpose(1, 0, 2, 3).copy())):
            out[name].append(np.array(v))
    return {k: np.array(v) for k, v in out.items()}


def golden_inputs(g):
    """imm_batch's arguments from an imm_batch_*.npz case."""
    return (g["x0"], g["P0"], g["F"], g["Q"], g["H"], g["R"], g["alpha"] ** 2, g["mu0"], g["trans"], g["zs"], g["valid"])
