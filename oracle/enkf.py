"""NumPy oracle of the EnKF bank (filterpy/kalman/ensemble_kalman_filter.py:158-290) and the CPU replica of
its device noise stream (csrc/enkf_kernel.cuh).

``philox4x32_10`` / ``std_normals`` restate the kernel's generator in uint64-masked NumPy integer arithmetic;
``psd_factor`` its lower factor of a positive semi-definite covariance.  ``EnKF`` restates the reference's
arithmetic on an explicit noise source: ``draw(call, cov, size)`` returns ``size`` rows ``xi L'``.
"""
import numpy as np

M32 = np.uint64(0xffffffff)
_MUL = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57))
_WEYL = (0x9E3779B9, 0xBB67AE85)


def philox4x32_10(ctr, key):
    """Philox4x32-10 of counters ``ctr`` (4 arrays or ints, uint32 values) under ``key`` (k0, k1)."""
    c = [np.asarray(v, dtype=np.uint64) & M32 for v in ctr]
    c = np.broadcast_arrays(*c)
    c = [v.copy() for v in c]
    k0, k1 = int(key[0]) & 0xffffffff, int(key[1]) & 0xffffffff
    for _ in range(10):
        p0 = _MUL[0] * c[0]                     # < 2^64: exact in uint64
        p1 = _MUL[1] * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & M32
        hi1, lo1 = p1 >> np.uint64(32), p1 & M32
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0 = (k0 + _WEYL[0]) & 0xffffffff
        k1 = (k1 + _WEYL[1]) & 0xffffffff
    return c


def box_muller(c, dtype=np.float64):
    """The kernel's Box-Muller of one Philox output for element type ``dtype``: u1 in (0, 1]; u2 in [0, 1) in fp64,
    [0, 1] in fp32.

    fp64: u1 = (c0:c1 top 53 bits + 1) 2^-53, u2 = (c2:c3 top 53 bits) 2^-53.  fp32: u1 = (float(c0) + 1) 2^-32
    and u2 = float(c2) 2^-32 in float arithmetic (round to nearest), 24 bits from one word each, so u2 may round
    up to 1.  The radius and the angle are evaluated in fp64 either way: against the kernel's fp32 stream this
    measures its logf / sqrtf / sincospif, not the uniforms."""
    if np.dtype(dtype) == np.float32:
        f32 = np.float32
        u1 = ((np.asarray(c[0]).astype(np.float64).astype(f32) + f32(1.0)) * f32(2.0 ** -32)).astype(np.float64)
        u2 = (np.asarray(c[2]).astype(np.float64).astype(f32) * f32(2.0 ** -32)).astype(np.float64)
    else:
        u1 = (((c[0] << np.uint64(21)) | (c[1] >> np.uint64(11))) + np.uint64(1)).astype(np.float64) * 2.0 ** -53
        u2 = ((c[2] << np.uint64(21)) | (c[3] >> np.uint64(11))).astype(np.float64) * 2.0 ** -53
    r = np.sqrt(-2.0 * np.log(u1))
    return r * np.cos(2.0 * np.pi * u2), r * np.sin(2.0 * np.pi * u2)


def std_normals(seed, f, call, n_members, k, dtype=np.float64):
    """(n_members, k) standard normals of filter ``f``, draw call ``call`` (components 2q, 2q+1 from counter q),
    as the kernel of element type ``dtype`` draws them."""
    out = np.empty((n_members, k))
    member = np.arange(n_members, dtype=np.uint64)
    for q in range((k + 1) // 2):
        c = philox4x32_10((q, member, int(call) & 0xffffffff, int(f) >> 32), (seed, int(f) & 0xffffffff))
        z0, z1 = box_muller(c, dtype)
        out[:, 2 * q] = z0
        if 2 * q + 1 < k:
            out[:, 2 * q + 1] = z1
    return out


def psd_factor(C, eps=np.finfo(np.float64).eps):
    """Lower L with L L' = C for symmetric positive semi-definite C (lower triangle read): Cholesky, a pivot
    <= 16 k eps max(diag C) zeroes its column.  Returns (L, ok); ok is False for a clearly indefinite C."""
    C = np.asarray(C, dtype=np.float64)
    k = C.shape[0]
    mx = max(0.0, float(np.max(np.diag(C))))
    tol, tol_off = 16 * k * eps * mx, np.sqrt(16 * k * eps) * mx
    L = np.zeros((k, k))
    ok = True
    for j in range(k):
        d = C[j, j] - np.dot(L[j, :j], L[j, :j])
        piv = d > tol
        ok = ok and d >= -tol
        L[j, j] = np.sqrt(d) if piv else 0.0
        for i in range(j + 1, k):
            s = C[i, j] - np.dot(L[i, :j], L[j, :j])
            ok = ok and (piv or not abs(s) > tol_off)
            L[i, j] = s / L[j, j] if piv else 0.0
    return L, ok


class Stream(object):
    """The noise of one filter: ``draw(call, mean, cov, size)`` = mean + xi L' (what the golden generator
    substitutes for the reference's ``multivariate_normal``).  ``dtype`` is the element type of the kernel the
    stream stands for: its uniforms (box_muller) and the eps of its semi-definite factor (psd_factor)."""

    def __init__(self, seed, f, dtype=np.float64):
        self.seed, self.f, self.dtype = int(seed), int(f), np.dtype(dtype).type

    def draw(self, call, mean, cov, size):
        cov = np.atleast_2d(np.asarray(cov, dtype=np.float64))
        L, ok = psd_factor(cov, np.finfo(self.dtype).eps)
        if not ok:
            raise np.linalg.LinAlgError("covariance is not positive semi-definite")
        xi = std_normals(self.seed, self.f, call, size, cov.shape[0], self.dtype)
        return np.asarray(mean, dtype=np.float64) + xi @ L.T


class EnKF(object):
    """The reference's EnsembleKalmanFilter on a ``Stream``, with fx / hx as NumPy callables of one member.
    ``counter`` is the draw-call index, advanced once per draw."""

    def __init__(self, x, P, dim_z, dt, N, hx, fx, stream):
        self.dim_x, self.dim_z, self.dt, self.N = len(x), dim_z, dt, N
        self.hx, self.fx, self.stream = hx, fx, stream
        self.counter = 0
        self.K = np.zeros((self.dim_x, dim_z))
        self.S = np.zeros((dim_z, dim_z))
        self.SI = np.zeros((dim_z, dim_z))
        self.initialize(x, P)
        self.Q = np.eye(self.dim_x)
        self.R = np.eye(dim_z)

    def _draw(self, mean, cov):
        out = self.stream.draw(self.counter, mean, cov, self.N)
        self.counter += 1
        return out

    def initialize(self, x, P):
        self.sigmas = self._draw(x, P)
        self.x, self.P = np.array(x, dtype=np.float64), np.array(P, dtype=np.float64)
        self.x_prior, self.P_prior = self.x.copy(), self.P.copy()
        self.x_post, self.P_post = self.x.copy(), self.P.copy()

    def predict(self):
        N = self.N
        self.sigmas = np.array([self.fx(s, self.dt) for s in self.sigmas])
        self.sigmas = self.sigmas + self._draw(np.zeros(self.dim_x), self.Q)
        self.x = np.mean(self.sigmas, axis=0)
        d = self.sigmas - self.x
        self.P = d.T @ d / (N - 1)
        self.x_prior, self.P_prior = self.x.copy(), self.P.copy()

    def update(self, z, R=None):
        if z is None:
            self.x_post, self.P_post = self.x.copy(), self.P.copy()
            return
        if R is None:
            R = self.R
        if np.isscalar(R):
            R = np.eye(self.dim_z) * R
        N = self.N
        h = np.array([self.hx(s) for s in self.sigmas]).reshape(N, -1)
        zm = np.mean(h, axis=0)
        dz = h - zm
        self.S = dz.T @ dz / (N - 1) + R
        Pxz = (self.sigmas - self.x).T @ dz / (N - 1)
        self.SI = np.linalg.inv(self.S)
        self.K = Pxz @ self.SI
        e_r = self._draw(np.zeros(self.dim_z), R)
        self.sigmas = self.sigmas + (np.asarray(z) + e_r - h) @ self.K.T
        self.x = np.mean(self.sigmas, axis=0)
        self.P = self.P - self.K @ self.S @ self.K.T
        self.x_post, self.P_post = self.x.copy(), self.P.copy()
