"""IMMEstimator.batch_filter restated in NumPy fp64 for N tracks with per-track models: T epochs of predict();
update(z or None) as a loop over oracle.imm's bank forms (mixing, combined estimate, mode probabilities) and
oracle.kf's bank steps, vectorised over the tracks.  A model without a measurement keeps its prior and scores
log N(0; 0, S) of the S of its last real update.  A model whose S is singular keeps its prior, its previous
log-likelihood, K, y and SI, stores the singular S and reports status 1 for that epoch (include/bke.h,
bke_imm_batch_args), where the reference's inv(S) raises."""
import numpy as np

from oracle import imm as oimm
from oracle import kf as okf

STATUS_SINGULAR_S = 1


def imm_batch(x0, P0, F, Q, H, R, alpha_sq, mu0, trans, zs, valid, S0=None, ll0=None, K0=None, y0=None, SI0=None,
              cbar0=None):
    """x0 [N,M,n], P0 [N,M,n,n], F, Q [N,M,n,n], H [m,n] or [N,M,m,n], R [m,m] or [N,M,m,m], alpha_sq [M],
    mu0 [M] or [N,M], trans [M,M], zs [T,N,m], valid [T,N] (bool).  The filters' starting diagnostics S0 [N,M,m,m],
    ll0 [N,M], K0 [N,M,n,m], y0 [N,M,m], SI0 [N,M,m,m] default to 0.  Without cbar0 [N,M], mu0 is normalised and
    cbar = mu0 . trans (the estimator's constructor); with it, mu0 and cbar0 are taken as they are (a run that
    continues).  Returns a dict of per-epoch arrays x, P, xp, Pp [T,N,...], mu, cbar, lik [T,N,M], omega
    [T,N,M,M], fx [T,N,M,n], fP [T,N,M,n,n], and per model at the end fxp, fPp, fS, fSI, fK, fy, fll [N,M,...],
    status (the last epoch's) and status_any (the first failure of the call) [N,M]; cond [N] is the largest
    cond(S) of a successful update of the track's models (1 where there is none)."""
    N, M, n = x0.shape
    T, _, m = zs.shape
    H = np.broadcast_to(H, (N, M, m, n)); R = np.broadcast_to(R, (N, M, m, m))
    xs = np.array(x0.transpose(1, 0, 2), float)
    Ps = np.array(P0.transpose(1, 0, 2, 3), float)

    def start(a, shape):
        return np.zeros((M, N) + shape) if a is None else np.array(np.moveaxis(np.asarray(a, float), 1, 0))
    S, SI, K, y = start(S0, (m, m)), start(SI0, (m, m)), start(K0, (n, m)), start(y0, (m,))
    ll = start(ll0, ())
    xpf, Ppf = np.zeros((M, N, n)), np.zeros((M, N, n, n))
    st_last = np.zeros((M, N), np.int32); st_any = np.zeros((M, N), np.int32)
    cond = np.ones(N)
    mu = np.broadcast_to(np.asarray(mu0, float), (N, M))
    if cbar0 is None:
        mu = mu / mu.sum(axis=1, keepdims=True)
        mu, cbar, omega = oimm.mm_probabilities_bank(mu, trans=trans)
    else:
        cbar = np.asarray(cbar0, float)
        omega = np.asarray(trans, float)[None] * mu[:, :, None] / cbar[:, None, :]
    out = {k: [] for k in ("x", "P", "xp", "Pp", "mu", "cbar", "omega", "lik", "fx", "fP")}
    for k in range(T):
        x0m, P0m = oimm.mm_mix_bank(xs, Ps, omega)
        for j in range(M):
            xs[j], Ps[j] = okf.kf_predict_bank(x0m[j], P0m[j], F[:, j], Q[:, j], alpha_sq[j])
        xpf[:], Ppf[:] = xs, Ps
        xp, Pp = oimm.mm_estimate_bank(xs, Ps, mu)
        v = np.asarray(valid[k], bool)
        for j in range(M):
            Sj = H[:, j] @ Ps[j] @ np.swapaxes(H[:, j], 1, 2) + R[:, j]
            S[j][v] = Sj[v]                                    # stored even when singular
            ok = v & (np.abs(np.linalg.det(Sj)) > 0)
            st = np.where(v & ~ok, STATUS_SINGULAR_S, 0).astype(np.int32)
            if ok.any():
                r = okf.kf_update_bank(xs[j][ok], Ps[j][ok], zs[k][ok], H[:, j][ok], R[:, j][ok])
                xs[j][ok], Ps[j][ok] = r["x"], r["P"]
                K[j][ok], y[j][ok], SI[j][ok] = r["K"], r["y"], r["SI"]
                ll[j][ok] = okf.log_likelihood_bank(r["y"], r["S"])
                cond[ok] = np.maximum(cond[ok], np.linalg.cond(r["S"]))
            if (~v).any():
                ll[j][~v] = okf.missed_log_likelihood_bank(S[j][~v])
                y[j][~v] = 0.0
            st_last[j] = st
            st_any[j] = np.where(st_any[j] != 0, st_any[j], st)
        mu, cbar, omega = oimm.mm_probabilities_bank(mu, ll.T, cbar, trans)
        x, P = oimm.mm_estimate_bank(xs, Ps, mu)
        lik = np.exp(ll.T)
        for name, val in (("x", x), ("P", P), ("xp", xp), ("Pp", Pp), ("mu", mu), ("cbar", cbar), ("omega", omega),
                          ("lik", np.where(lik == 0.0, oimm.FLOAT_MIN, lik)), ("fx", xs.transpose(1, 0, 2).copy()),
                          ("fP", Ps.transpose(1, 0, 2, 3).copy())):
            out[name].append(np.array(val))
    out = {k: np.array(v) for k, v in out.items()}
    sw = lambda a: np.ascontiguousarray(np.moveaxis(a, 0, 1))
    out.update(fxp=sw(xpf), fPp=sw(Ppf), fS=sw(S), fSI=sw(SI), fK=sw(K), fy=sw(y), fll=sw(ll), status=sw(st_last),
               status_any=sw(st_any), cond=cond)
    return out


def golden_inputs(g):
    """imm_batch's arguments from an imm_batch_*.npz case."""
    return (g["x0"], g["P0"], g["F"], g["Q"], g["H"], g["R"], g["alpha"] ** 2, g["mu0"], g["trans"], g["zs"], g["valid"])
