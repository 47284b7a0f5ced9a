"""Host-side mirror of ``filterpy.kalman.IMMEstimator`` (filterpy/kalman/IMM.py:31-260) for a BANK
of tracks: ``filters`` is a list of M ``KalmanFilter`` banks (one per motion model, each with the
same ``n_filters`` tracks).  Every step of the reference's per-object Python loops — mode
probabilities (:178-184, :239-247), mixed initial conditions (:201-213), combined estimate
(:228-237) — is one CUDA launch over all tracks (csrc/mix.cu); the per-model predict / update are
the bank kernels.  Single-mode filters (``KalmanFilter(n, m)`` without ``n_filters``) give the
reference's one-track behaviour with NumPy attributes.  No CPU fallback.
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from .._dev import StepGraph, bke_dtype, ptr, stream_ptr, to_dev
from ..common.helpers import reshape_z

__all__ = ["IMMEstimator"]


def _check_bank(filters):
    f0 = filters[0]
    for f in filters:
        if (f.dim_x, f.n_filters, f._dtype, f._device, f._single) != \
                (f0.dim_x, f0.n_filters, f0._dtype, f0._device, f0._single):
            raise ValueError('All filters must have the same state dimension')     # IMM.py:143-146
        if not f.diagnostics:
            raise ValueError("the model filters must be built with diagnostics=True (likelihoods are read)")
    if len(filters) > _lib.BKE_MM_MAX_MODELS:
        raise NotImplementedError("at most %d models" % _lib.BKE_MM_MAX_MODELS)
    return f0


def _mm_args(filters, flags=0):
    f0 = filters[0]
    a = _lib.MmArgs()
    a.n_tracks, a.dim_x, a.n_models = f0.n_filters, f0.dim_x, len(filters)
    a.dtype, a.flags = bke_dtype(f0._dtype), flags
    for j, f in enumerate(filters):
        f._flush()
        a.x[j], a.P[j] = ptr(f._x), ptr(f._P)
        a.log_likelihood[j] = ptr(f._ll)
    return a


def _set_model_ptr(a, name, j, p, stride):
    """model ``name``'s pointer and stride of model j in an ImmBatchArgs."""
    getattr(a, name)[j] = p
    getattr(a, name + "_stride")[j] = stride


class IMMEstimator(object):
    """IMM.py:31-260.  ``mu``: (M,) initial mode probabilities shared by the tracks, or (N, M);
    ``M``: (M, M) Markov transition matrix."""

    def __init__(self, filters, mu, M):
        if len(filters) < 2:
            raise ValueError('filters must contain at least two filters')     # IMM.py:135-136
        f0 = _check_bank(filters)
        self.filters = filters
        self.N = len(filters)                                # number of models, as in the reference (:152)
        self.n_tracks = f0.n_filters
        self._single = f0._single
        self._dtype, self._device = f0._dtype, f0._device
        self._lib = _lib.load()
        nm, nt, n = self.N, self.n_tracks, f0.dim_x
        mu = np.asarray(mu, dtype=np.float64)
        mu = mu / np.sum(mu, axis=-1, keepdims=True)         # IMM.py:139
        if mu.shape == (nm,):
            mu = np.broadcast_to(mu, (nt, nm))
        if mu.shape != (nt, nm):
            raise ValueError("mu must have shape (%d,) or (%d,%d)" % (nm, nt, nm))
        kw = dict(dtype=torch.float64, device=self._device)
        self._mu = torch.from_numpy(np.array(mu, dtype=np.float64, order='C')).to(self._device)
        self._M = torch.from_numpy(np.ascontiguousarray(np.asarray(M, dtype=np.float64))).to(self._device)
        if tuple(self._M.shape) != (nm, nm):
            raise ValueError("M must have shape (%d,%d)" % (nm, nm))
        self._cbar = torch.zeros(nt, nm, **kw)
        self._omega = torch.zeros(nt, nm, nm, **kw)
        skw = dict(dtype=self._dtype, device=self._device)
        self._x = torch.zeros(nt, n, **skw)
        self._P = torch.zeros(nt, n, n, **skw)
        # spare state buffers for the mixing step (double-buffered with the filters' own)
        self._spare = [(torch.empty(nt, n, **skw), torch.empty(nt, n, n, **skw)) for _ in filters]
        self._compute_mixing_probabilities(initial=True)
        self._compute_state_estimate()
        self._x_prior = self._x.clone(); self._P_prior = self._P.clone()
        self._x_post = self._x.clone(); self._P_post = self._P.clone()

    # ------------------------------------------------------------------ outputs
    x = property(lambda self: self.filters[0]._vec_out(self._x))
    P = property(lambda self: self.filters[0]._out(self._P))
    x_prior = property(lambda self: self.filters[0]._vec_out(self._x_prior))
    P_prior = property(lambda self: self.filters[0]._out(self._P_prior))
    x_post = property(lambda self: self.filters[0]._vec_out(self._x_post))
    P_post = property(lambda self: self.filters[0]._out(self._P_post))
    mu = property(lambda self: self.filters[0]._out(self._mu))
    M = property(lambda self: self._M.cpu().numpy())
    cbar = property(lambda self: self.filters[0]._out(self._cbar))
    omega = property(lambda self: self.filters[0]._out(self._omega))

    @property
    def likelihood(self):
        """per-model likelihood of the last measurement (IMM.py:154, :174-176): (N, M), or (M,) for one track."""
        if self._single:
            return np.array([f.likelihood for f in self.filters])
        return torch.stack([f.likelihood for f in self.filters], dim=-1)

    # ------------------------------------------------------------------ steps
    def _call(self, fn, a):
        with torch.cuda.device(self._device):
            _lib.check(fn(ctypes.byref(a), stream_ptr(self._device)))

    def update(self, z, valid=None):
        """IMM.py:160-184: update every model, then mode probabilities and the combined estimate.
        ``z=None`` is a missed measurement for every track; ``valid`` (bool[N]) marks the tracks that
        have one, the others behave as the reference's ``update(None)``."""
        for f in self.filters:
            f.update(z, valid=valid)
        a = _mm_args(self.filters)
        a.mu, a.cbar, a.omega, a.trans = ptr(self._mu), ptr(self._cbar), ptr(self._omega), ptr(self._M)
        self._call(self._lib.bke_mm_probabilities, a)
        self._compute_state_estimate()
        self._x_post.copy_(self._x); self._P_post.copy_(self._P)

    def predict(self, u=None):
        """IMM.py:186-226: mixed initial conditions for every model, predict, combined prior."""
        a = _mm_args(self.filters)
        a.omega, a.weights_stride = ptr(self._omega), self.N * self.N
        for j, (xs, Ps) in enumerate(self._spare):
            a.x_out[j], a.P_out[j] = ptr(xs), ptr(Ps)
        self._call(self._lib.bke_mm_mix, a)
        for j, f in enumerate(self.filters):
            self._spare[j] = f._adopt_state(*self._spare[j])           # f.x = xs[i]; f.P = Ps[i] (:216-219)
            f.predict(u)
        self._compute_state_estimate()
        self._x_prior.copy_(self._x); self._P_prior.copy_(self._P)

    def _compute_state_estimate(self):
        """IMM.py:228-237."""
        a = _mm_args(self.filters)
        a.mu, a.weights_stride = ptr(self._mu), self.N
        a.x_out[0], a.P_out[0] = ptr(self._x), ptr(self._P)
        self._call(self._lib.bke_mm_estimate, a)

    def _compute_mixing_probabilities(self, initial=False):
        """IMM.py:239-247 (cbar = mu . M, omega); the likelihood step is part of update()."""
        a = _mm_args(self.filters, flags=_lib.BKE_MM_FROM_MU)
        a.mu, a.cbar, a.omega, a.trans = ptr(self._mu), ptr(self._cbar), ptr(self._omega), ptr(self._M)
        self._call(self._lib.bke_mm_probabilities, a)

    def batch_filter(self, zs, valid=None):
        """T epochs of ``predict(); update(zs[k], valid=valid[k])`` — the reference has no IMM batch_filter.

        Bank mode: ``zs[T,N,dim_z]`` (``valid[T,N]`` optional, False = that track misses the epoch) -> device
        tensors ``means[T,N,n] covariances[T,N,n,n] means_p covariances_p`` (the combined posterior and prior
        of each epoch) and ``mus[T,N,M]`` (fp64, the mode probabilities after each update).  Single mode: ``zs``
        is a sequence whose entries may be None; NumPy outputs ``(T,n) (T,n,n) (T,n) (T,n,n) (T,M)``.

        The estimator and its model filters are left as the loop leaves them.  Shapes with a fused instance
        (bke_imm_batch_filter: 2/1, 3/1 in fp32 and fp64, 4/2 in fp32) run in ONE launch; any other runs the
        loop of separate launches.  Neither synchronises the host in bank mode, so a graph can capture it."""
        fs = self.filters
        f0 = fs[0]
        N, n, m, nm = self.n_tracks, f0.dim_x, f0.dim_z, self.N
        if any(f.dim_z != m for f in fs):
            raise ValueError("batch_filter: every model must have the same dim_z")
        T = zs.shape[0] if isinstance(zs, torch.Tensor) else (len(zs) if isinstance(zs, (list, tuple)) else np.size(zs, 0))
        if self._single:
            zarr = np.zeros((T, 1, m))
            vmask = np.ones((T, 1), dtype=bool)
            for i, z in enumerate(zs):
                if z is None:
                    vmask[i, 0] = False
                else:
                    zarr[i, 0] = np.asarray(z, dtype=np.float64).reshape(-1)[:m] if np.size(z) == m else reshape_z(z, m, 1)
            zt = to_dev(zarr, self._dtype, self._device)
            vt = None if vmask.all() else torch.from_numpy(vmask.astype(np.uint8)).to(self._device)
        else:
            zt = to_dev(zs, self._dtype, self._device)
            if zt.dim() == 4 and zt.shape[-1] == 1:
                zt = zt[..., 0].contiguous()
            if tuple(zt.shape) != (T, N, m):
                raise ValueError("zs must have shape (T,%d,%d), got %s" % (N, m, tuple(zt.shape)))
            vt = None
            if valid is not None:
                vt = torch.as_tensor(valid, device=self._device).to(torch.uint8).contiguous()
                if tuple(vt.shape) != (T, N):
                    raise ValueError("valid must have shape (%d,%d)" % (T, N))
        kw = dict(dtype=self._dtype, device=self._device)
        means = torch.empty(T, N, n, **kw); means_p = torch.empty(T, N, n, **kw)
        covs = torch.empty(T, N, n, n, **kw); covs_p = torch.empty(T, N, n, n, **kw)
        mus = torch.empty(T, N, nm, dtype=torch.float64, device=self._device)
        for f in fs:
            f._flush()
        a = _lib.ImmBatchArgs()
        a.n_tracks, a.dim_x, a.dim_z, a.n_models, a.dtype = N, n, m, nm, bke_dtype(self._dtype)
        a.n_steps = T
        a.flags = _lib.BKE_STATUS_STICKY if self._single else 0
        keep = []
        for j, f in enumerate(fs):
            a.x[j], a.P[j] = ptr(f._x), ptr(f._P)
            for name in "FQHR":
                t = getattr(f, "_" + name)
                _set_model_ptr(a, name, j, ptr(t), f._stride(t))
            a.alpha_sq[j] = f._alpha_sq
            a.S[j], a.log_likelihood[j], a.K[j], a.y[j], a.SI[j] = ptr(f._S), ptr(f._ll), ptr(f._K), ptr(f._y), ptr(f._SI)
            a.x_prior[j], a.P_prior[j], a.status[j] = ptr(f._x_prior), ptr(f._P_prior), ptr(f._status)
        a.mu, a.cbar, a.omega, a.trans = ptr(self._mu), ptr(self._cbar), ptr(self._omega), ptr(self._M)
        a.zs, a.zs_valid = ptr(zt), ptr(vt)
        a.means, a.covariances, a.means_p, a.covariances_p, a.mus = ptr(means), ptr(covs), ptr(means_p), ptr(covs_p), ptr(mus)
        with torch.cuda.device(self._device):
            rc = self._lib.bke_imm_batch_filter(ctypes.byref(a), stream_ptr(self._device))
        if rc == _lib.BKE_ERR_UNSUPPORTED:
            # no fused instance for this shape / dtype: the same epochs on the separate launches
            for k in range(T):
                self.predict()
                means_p[k].copy_(self._x); covs_p[k].copy_(self._P)
                if self._single:
                    self.update(zarr[k, 0] if vmask[k, 0] else None)
                else:
                    self.update(zt[k], valid=None if vt is None else vt[k])
                means[k].copy_(self._x); covs[k].copy_(self._P); mus[k].copy_(self._mu)
        else:
            _lib.check(rc)
            if T > 0:
                self._x.copy_(means[T - 1]); self._P.copy_(covs[T - 1])
                self._x_prior.copy_(means_p[T - 1]); self._P_prior.copy_(covs_p[T - 1])
                self._x_post.copy_(means[T - 1]); self._P_post.copy_(covs[T - 1])
                last = None if (self._single and not vmask[T - 1, 0]) else zt[T - 1]
                for f in fs:
                    f._post_alias = True
                    f._z = last
                if self._single:
                    for f in fs:
                        f.check()
        if not self._single:
            return means, covs, means_p, covs_p, mus
        return (means[:, 0].cpu().numpy(), covs[:, 0].cpu().numpy(), means_p[:, 0].cpu().numpy(),
                covs_p[:, 0].cpu().numpy(), mus[:, 0].cpu().numpy())

    def capture(self, fn, warmup=2):
        """Capture ``fn`` — a fixed sequence of ``predict()`` / ``update(z_buffer)`` calls — into a CUDA
        graph (``.replay()``); one IMM step is ~15 small launches, so the host side dominates otherwise.
        The model filters' state buffers rotate with period 3 (state, stored posterior, spare), so
        ``fn`` must run a multiple of 3 steps for a replay to find the buffers where it left them."""
        return StepGraph(fn, self._device, warmup)

    def __repr__(self):
        return "IMMEstimator (H100): %d models x %d tracks, dim_x=%d" % (self.N, self.n_tracks, self.filters[0].dim_x)
