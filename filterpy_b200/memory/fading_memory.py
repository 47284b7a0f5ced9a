"""Mirror of filterpy.memory.FadingMemoryFilter (filterpy/memory/fading_memory.py) on bke_poly_filter.

``FadingMemoryFilter(x0, dt, order, beta, n_filters=None, dtype, device)``.  Single mode is one reference filter
(NumPy attributes, fp64).  Bank mode keeps x[N, order+1] on the device; ``dt`` and ``beta`` are scalars or one per
filter, and ``P`` / ``e`` are then [N, order+1].  ``update(z[N])`` is one launch and so is
``batch_filter(data[T, N])``, which returns results[T+1, N, order+1] and leaves the filter as it was (the reference
has no batch_filter: it equals T calls of update() on a copy).  Deviation: an integer x0 array is stored as float
(the reference keeps its dtype, so its order-1 and order-2 updates truncate into it).
"""
import numpy as np
import torch

from .. import _lib
from ..common.poly import PolyBank, host_const, to_numpy


def _P(order, beta, dt):
    """fading_memory.py:117-139: the diagonal of the unit-variance covariance"""
    if order == 0:
        return ((1 - beta) / (1 + beta),)
    if order == 1:
        return ((1 - beta) * (1 + 4 * beta + 5 * beta**2) / (1 + beta)**3, 2 * (1 - beta)**3 / (1 + beta)**3)
    return ((1 - beta) * ((1 + 6 * beta + 16 * beta**2 + 24 * beta**3 + 19 * beta**4) / (1 + beta)**5),
            (1 - beta)**3 * ((13 + 50 * beta + 49 * beta**2) / (2 * (1 + beta)**5 * dt**2)),
            6 * (1 - beta)**5 / ((1 + beta)**5 * dt**4))


def _e(order, beta, dt):
    """fading_memory.py:119-145: the truncation errors"""
    if order == 0:
        return (dt * beta / (1 - beta),)
    if order == 1:
        return (2 * dt * 2 * (beta / (1 - beta))**2, dt * ((1 + 3 * beta) / (1 - beta)))
    return (6 * dt**3 * (beta / (1 - beta))**3, dt**2 * (2 + 5 * beta + 11 * beta**2) / (1 - beta)**2,
            6 * dt * (1 + 2 * beta) / (1 - beta))


# the update's constants by order (fading_memory.py:165, 169-170, 180-182): g = G, h = H / dt, k = 2*K / dt**2
_G = {0: lambda b: 1 - b, 1: lambda b: 1 - b**2, 2: lambda b: 1 - b**3}
_H = {1: lambda b: (1 - b)**2, 2: lambda b: 1.5 * (1 + b) * (1 - b)**2}


class FadingMemoryFilter(PolyBank):
    def __init__(self, x0, dt, order, beta, n_filters=None, dtype=np.float64, device=None):
        if order < 0 or order > 2:
            raise ValueError('order must be between 0 and 2')                     # fading_memory.py:104-105
        self._init_mode(n_filters, 1, dtype, device)
        self.order = order
        W = order + 1
        if np.isscalar(x0):                                                        # :107-111
            x = np.zeros(W)
            x[0] = x0
        else:
            x = x0 if isinstance(x0, torch.Tensor) else np.asarray(x0, np.float64)
        self._x = self._tensor(x, (self.n_filters, W))
        self._beta, self._dt = self._host(beta), self._host(dt)
        self._constants()

    def _constants(self):
        o, b, dt = self.order, self._beta, self._dt
        self._set_param("g", host_const(_G[o], b))
        if o >= 1:
            self._set_param("h", host_const(lambda b, d: _H[o](b) / d, b, dt))
            self._set_param("dt", dt)
        if o == 2:
            self._set_param("k", host_const(lambda b, d: 2 * (0.5 * (1 - b)**3) / (d**2), b, dt))
            self._set_param("dt2", host_const(lambda d: d**2., dt))                      # :188 T2 = dt**2.
        self._Pv = np.stack(np.broadcast_arrays(*[host_const(lambda b, d, j=j: _P(o, b, d)[j], b, dt) for j in range(o + 1)]), -1)
        self._ev = np.stack(np.broadcast_arrays(*[host_const(lambda b, d, j=j: _e(o, b, d)[j], b, dt) for j in range(o + 1)]), -1)

    def _out(self, t):
        return t if not self._single else to_numpy(t)[0]

    def _host_out(self, v):
        if self._single:
            return np.array(v, dtype=float).reshape(-1)
        return torch.as_tensor(np.broadcast_to(v, (self.n_filters, self.order + 1)).copy(),
                               device=self._device).to(self._dtype)

    x = property(lambda self: self._out(self._x), lambda self, v: setattr(self, "_x", self._tensor(v, (self.n_filters, self.order + 1))))
    P = property(lambda self: self._host_out(self._Pv))
    e = property(lambda self: self._host_out(self._ev))

    @property
    def beta(self):
        return self._beta if self._single or np.ndim(self._beta) == 0 else torch.as_tensor(self._beta, device=self._device)

    @beta.setter
    def beta(self, v):
        self._beta = self._host(v)
        self._constants()

    @property
    def dt(self):
        return self._dt if self._single or np.ndim(self._dt) == 0 else torch.as_tensor(self._dt, device=self._device)

    @dt.setter
    def dt(self, v):
        self._dt = self._host(v)
        self._constants()

    def _params(self):
        return {k: self._call_param(None, k) for k in ("g", "h", "k", "dt", "dt2")}

    def update(self, z):
        """fading_memory.py:159-194: one launch"""
        self._launch(_lib.BKE_POLY_FADING, self.order, self._z(z), _lib.BKE_POLY_UPDATE, self._x, params=self._params())

    def batch_filter(self, data):
        """T epochs of update() in one launch on a copy of the state: results[T+1, N, order+1] (single mode:
        [T+1, order+1]); the filter itself is not changed"""
        z = self._z(data, T=len(data))
        T, N = z.shape
        res = torch.empty((T + 1, N, self.order + 1), dtype=self._dtype, device=self._device)
        self._launch(_lib.BKE_POLY_FADING, self.order, z, _lib.BKE_POLY_BATCH, self._x, params=self._params(), results=res)
        return to_numpy(res)[:, 0] if self._single else res
