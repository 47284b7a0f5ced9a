"""fp64 NumPy restatement of filterpy's InformationFilter (filterpy/kalman/information_filter.py), filter by
filter, with the engine's singularity rule: a matrix is singular when a pivot of Gauss-Jordan elimination with
partial pivoting is exactly zero (reg_inverse / warp_inverse).  Where the reference's uncaught np.linalg.inv
raises, the filter gets status 1 and keeps what the reference has set by then."""
import math
import sys

import numpy as np

LOG_FLOAT_MIN = math.log(sys.float_info.min)
LL_NONE, LL_FULL, LL_BROADCAST = 0, 1, 2


def singular(A):
    """True when a pivot of the partially pivoted elimination of A is exactly zero."""
    A = np.array(A, dtype=np.float64)
    n = A.shape[0]
    for c in range(n):
        p = c + int(np.argmax(np.abs(A[c:, c])))
        if not abs(A[p, c]) > 0:
            return True
        A[[c, p]] = A[[p, c]]
        A[c] /= A[c, c]
        for r in range(n):
            if r != c:
                A[r] -= A[r, c] * A[c]
    return False


def inv(A):
    """np.linalg.inv(A), or None where the rule finds A singular."""
    return None if singular(A) else np.linalg.inv(A)


def logpdf_broadcast(y, S):
    """filterpy.stats.logpdf(x=y, cov=S) for m == n or m == 1 (scipy broadcasts y over the n of S)."""
    n = S.shape[0]
    yv = np.broadcast_to(np.asarray(y, np.float64).reshape(-1), (n,))
    _, logdet = np.linalg.slogdet(S)
    return -0.5 * (n * math.log(2 * math.pi) + logdet + yv @ np.linalg.solve(S, yv))


class Filter(object):
    """One reference filter's state: x (n,), P_inv (n,n), no_information, and its diagnostics."""

    def __init__(self, x, P_inv, F, F_inv, Q, H, R_inv, B=None, ll_mode=LL_NONE):
        n, m = len(x), H.shape[0]
        self.x, self.P_inv = np.array(x, np.float64), np.array(P_inv, np.float64)
        self.F, self.F_inv, self.Q, self.H, self.R_inv, self.B = F, F_inv, Q, H, R_inv, B
        self.ni = False
        self.ll_mode = ll_mode
        self.y, self.K, self.S = np.zeros(m), np.zeros((n, m)), np.zeros((n, n))
        self.ll = LOG_FLOAT_MIN
        self.x_prior, self.P_inv_prior = np.zeros(n), np.eye(n)        # the constructor's copies
        self.status = 0

    def predict(self, u=None):
        """information_filter.py:245-289; False where an uncaught inverse fails (status 1)."""
        n = len(self.x)
        A = self.F_inv.T @ self.P_inv @ self.F_inv
        AI = inv(A)
        if AI is not None:
            if self.ni:
                Pi = inv(self.P_inv)
                self.x = Pi @ self.x if Pi is not None else 0 * self.x
                self.ni = False
            self.x = self.F @ self.x
            if self.B is not None and u is not None:
                self.x = self.x + self.B @ u
            Pn = inv(AI + self.Q)
            if Pn is None:
                self.status = 1
                return False
            self.P_inv = Pn
            self.x_prior, self.P_inv_prior = self.x.copy(), self.P_inv.copy()
        else:
            self.ni = True
            I_PF = np.eye(n) - self.P_inv @ self.F_inv
            FTI = inv(self.F.T)
            AQI = inv(A + self.Q)
            if FTI is None or AQI is None:
                self.status = 1
                return False
            self.x = FTI @ ((I_PF @ AQI) @ (FTI @ self.x))
            self.x_prior, self.P_inv_prior = self.x.copy(), AQI.copy()
        return True

    def update(self, z, R_inv=None):
        """information_filter.py:178-243 for z given (z is None changes nothing); False where inv(S) fails."""
        if z is None:
            return True
        z = np.asarray(z, np.float64).reshape(-1)
        R_inv = self.R_inv if R_inv is None else R_inv
        H = self.H
        HR = H.T @ R_inv
        if self.ni:
            self.x = self.P_inv @ self.x + HR @ z
            self.P_inv = self.P_inv + HR @ H
            self.ll = LOG_FLOAT_MIN
            return True
        self.y = z - H @ self.x
        self.S = self.P_inv + HR @ H
        SI = inv(self.S)
        if SI is None:
            self.status = 1
            return False
        self.K = (SI @ H.T) @ R_inv
        self.x = self.x + self.K @ self.y
        self.P_inv = self.S.copy()
        if self.ll_mode != LL_NONE:
            self.ll = logpdf_broadcast(self.y, self.S)
        return True


def run_bank(g, ll_mode=LL_NONE, steps=None):
    """Every filter of a golden file through its steps (``order`` "pu": predict then update, "up": update then
    predict).  Returns the per-step state and diagnostics, [T, N, ...]; a filter whose step fails stops there
    and repeats its state at the failure."""
    x0 = g["x"]
    N, n = x0.shape
    T = g["zs"].shape[0] if steps is None else steps
    order = str(g.get("order", "pu"))
    keys = ("x", "P_inv", "ni", "ll", "y", "K", "S", "x_prior", "P_inv_prior", "status")
    out = {k: [] for k in keys}
    fl = []
    for f in range(N):
        B = g["B"][f] if "B" in g else None
        fl.append(Filter(x0[f], g["P_inv"][f], g["F"][f], g["F_inv"][f], g["Q"][f], g["H"][f], g["R_inv"][f], B, ll_mode))
    for t in range(T):
        rows = {k: [] for k in keys}
        for f, flt in enumerate(fl):
            if flt.status == 0:
                z = g["zs"][t, f] if g["valid"][t, f] else None
                u = g["us"][t, f] if "us" in g else None
                for op in order:
                    ok = flt.predict(u) if op == "p" else flt.update(z)
                    if not ok:
                        break
            for k in keys:
                rows[k].append(np.array(getattr(flt, k), np.float64))
        for k in keys:
            out[k].append(np.array(rows[k]))
    return {k: np.array(v) for k, v in out.items()}
