"""Host mirrors of ``filterpy.kalman.MerweScaledSigmaPoints`` (filterpy/kalman/sigma_points.py:24-208),
``JulierSigmaPoints`` (:211-383) and ``SimplexSigmaPoints`` (:386-534).

The object carries its parameters and the weights.  Inside a UKF step the sigma points are generated
on chip by the fused kernel (csrc/ukf.cu); ``sigma_points(x, P)`` itself runs the stand-alone kernel
(csrc/ut.cu) — rows of the upper Cholesky factor of (n + lambda) P, exactly as sigma_points.py:167-175,
or the simplex points x + (U' sqrt(n) Istar)' of :499-513.
"""
import numpy as np
import torch

from .. import _lib
from .._dev import bke_dtype, require_cuda, stream_ptr

__all__ = ["MerweScaledSigmaPoints", "JulierSigmaPoints", "SimplexSigmaPoints"]


def _no_custom(sqrt_method, subtract):
    if sqrt_method is not None or subtract is not None:
        raise NotImplementedError(
            "custom sqrt_method / subtract are Python callables; the GPU path implements the "
            "defaults only (scipy.linalg.cholesky, np.subtract) and has no CPU fallback")


def _sigma_points(pts, x, P, launch):
    """The stand-alone sigma-point kernel of the point set ``pts`` on (x, P) or a bank of them.
    ``launch(lib, N, n, dtype, x, P, sigmas, status, stream)`` calls the set's C entry point."""
    n = pts.n
    is_t = isinstance(x, torch.Tensor)
    if not is_t and n != np.size(x) and np.ndim(x) < 2:
        raise ValueError("expected size(x) {}, but size is {}".format(n, np.size(x)))   # sigma_points.py:153-155
    dev = x.device if (is_t and x.is_cuda) else require_cuda(None)
    dt = x.dtype if (is_t and x.dtype in (torch.float32, torch.float64)) else torch.float64
    xt = (x if is_t else torch.from_numpy(np.atleast_1d(np.asarray(x, dtype=np.float64)))).to(device=dev, dtype=dt)
    single = xt.dim() == 1
    xt = xt.reshape(-1, n).contiguous()
    N = xt.shape[0]
    if np.isscalar(P):
        P = np.eye(n) * P
    Pt = (P if isinstance(P, torch.Tensor) else torch.from_numpy(np.atleast_2d(np.asarray(P, dtype=np.float64)))).to(device=dev, dtype=dt)
    Pt = Pt.expand(N, n, n).contiguous() if Pt.dim() == 2 else Pt.contiguous()
    if tuple(Pt.shape) != (N, n, n):
        raise ValueError("P must have shape (%d,%d) or (%d,%d,%d)" % (n, n, N, n, n))
    sig = torch.empty(N, pts.num_sigmas(), n, dtype=dt, device=dev)
    status = torch.zeros(N, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(launch(_lib.load(), N, n, bke_dtype(dt), xt.data_ptr(), Pt.data_ptr(), sig.data_ptr(),
                          status.data_ptr(), stream_ptr(dev)))
    if not is_t or single:
        if int(status.sum().item()):
            raise np.linalg.LinAlgError("%d-th leading minor of the array is not positive definite" % 1)
    if is_t:
        return sig[0] if single else sig
    out = sig.cpu().numpy()
    return out[0] if single else out


class MerweScaledSigmaPoints(object):
    def __init__(self, n, alpha, beta, kappa, sqrt_method=None, subtract=None):
        _no_custom(sqrt_method, subtract)
        self.n = int(n)
        self.alpha = float(alpha)
        self.beta = float(beta)
        self.kappa = float(kappa)
        self._compute_weights()

    def num_sigmas(self):
        """Number of sigma points (sigma_points.py:119-121)."""
        return 2 * self.n + 1

    def sigma_points(self, x, P):
        """sigma_points.py:124-177 on the GPU.  ``x`` (n,) with ``P`` (n,n) / scalar -> ndarray
        (2n+1, n); a bank ``x[N,n]``, ``P[N,n,n]`` (NumPy or CUDA tensors) -> ``[N, 2n+1, n]``.
        Raises ``LinAlgError`` where scipy's cholesky would (P not positive definite)."""
        return _sigma_points(self, x, P, lambda lib, N, n, dt, *ptrs: lib.bke_merwe_sigma_points(
            N, n, dt, self.alpha, self.beta, self.kappa, *ptrs))

    def _compute_weights(self):
        """sigma_points.py:180-192."""
        n = self.n
        lambda_ = self.alpha ** 2 * (n + self.kappa) - n
        c = .5 / (n + lambda_)
        self.Wc = np.full(2 * n + 1, c)
        self.Wm = np.full(2 * n + 1, c)
        self.Wc[0] = lambda_ / (n + lambda_) + (1 - self.alpha ** 2 + self.beta)
        self.Wm[0] = lambda_ / (n + lambda_)

    def __repr__(self):
        return "MerweScaledSigmaPoints(n=%d, alpha=%g, beta=%g, kappa=%g)" % (
            self.n, self.alpha, self.beta, self.kappa)


class JulierSigmaPoints(MerweScaledSigmaPoints):
    """Host mirror of ``filterpy.kalman.JulierSigmaPoints`` (filterpy/kalman/sigma_points.py:211-383):
    sigma offsets = rows of chol_upper((n + kappa) P) (:352-361), Wm = Wc = [kappa, .5, .5, ...] / (n + kappa)
    (:367-373).  That is the Merwe parameterisation with alpha = 1, beta = 0 (lambda = kappa), so the
    fused UKF kernel and the stand-alone sigma-point kernel serve it unchanged."""

    def __init__(self, n, kappa=0., sqrt_method=None, subtract=None):
        MerweScaledSigmaPoints.__init__(self, n, 1.0, 0.0, kappa, sqrt_method=sqrt_method, subtract=subtract)

    def _compute_weights(self):
        """sigma_points.py:367-373."""
        n, k = self.n, self.kappa
        self.Wm = np.full(2 * n + 1, .5 / (n + k))
        self.Wm[0] = k / (n + k)
        self.Wc = self.Wm

    def __repr__(self):
        return "JulierSigmaPoints(n=%d, kappa=%g)" % (self.n, self.kappa)


class SimplexSigmaPoints(object):
    """Host mirror of ``filterpy.kalman.SimplexSigmaPoints`` (filterpy/kalman/sigma_points.py:386-534): n + 1
    points x + D_j, D = (U' sqrt(n) Istar)' with U = chol_upper(P) unscaled and Istar of :502-507; Wm = Wc =
    1/(n+1), one array (:516-522).  ``alpha`` is stored and shown, and never used (as in the reference).
    A UKF built on this object runs the simplex instances of its kernels (the ``BKE_UKF_SIMPLEX`` flag)."""

    def __init__(self, n, alpha=1, sqrt_method=None, subtract=None):
        _no_custom(sqrt_method, subtract)
        self.n = int(n)
        self.alpha = alpha
        self._compute_weights()

    def num_sigmas(self):
        """Number of sigma points (sigma_points.py:449-451)."""
        return self.n + 1

    def sigma_points(self, x, P):
        """sigma_points.py:454-513 on the GPU.  ``x`` (n,) with ``P`` (n,n) / scalar -> ndarray (n+1, n),
        ordered Xi_0 .. Xi_n; a bank ``x[N,n]``, ``P[N,n,n]`` (NumPy or CUDA tensors) -> ``[N, n+1, n]``.
        Raises ``LinAlgError`` where scipy's cholesky would (P not positive definite)."""
        return _sigma_points(self, x, P, lambda lib, *a: lib.bke_simplex_sigma_points(*a))

    def _compute_weights(self):
        """sigma_points.py:516-522."""
        self.Wm = np.full(self.n + 1, 1. / (self.n + 1))
        self.Wc = self.Wm

    def __repr__(self):
        return "SimplexSigmaPoints(n=%d, alpha=%g)" % (self.n, self.alpha)
