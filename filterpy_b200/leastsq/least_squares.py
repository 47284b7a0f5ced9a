"""Mirror of filterpy.leastsq.LeastSquaresFilter (filterpy/leastsq/least_squares.py) on bke_poly_filter.

``LeastSquaresFilter(dt, order, noise_sigma=0., n_filters=None, dtype, device)``.  Single mode is one reference
filter (NumPy attributes, fp64).  Bank mode keeps x[N, order+1], K[N, order+1] and the counter n[N] (int64) on the
device; ``dt`` and ``noise_sigma`` are scalars or one per filter.  ``update(z[N])`` is one launch and so is
``batch_filter(data[T, N])``, which returns the states after every epoch, results[T+1, N, order+1], and leaves the
filter as it was (the reference has no batch_filter: it equals T calls of update() on a copy).
"""
import math

import numpy as np
import torch

from .. import _lib
from ..common.poly import PolyBank, host_const, to_numpy

_INT64_MAX = 2**63 - 1


class LeastSquaresFilter(PolyBank):
    def __init__(self, dt, order, noise_sigma=0., n_filters=None, dtype=np.float64, device=None):
        if order < 0 or order > 2:
            raise ValueError('order must be between 0 and 2')                     # least_squares.py:94-95
        self._init_mode(n_filters, 1, dtype, device)
        self._order = order
        self.dt = dt
        self.sigma = noise_sigma
        self.reset()

    def reset(self):
        """least_squares.py:104-110: n = 0, x = K = 0, y = 0"""
        N, W = self.n_filters, self._order + 1
        self._n = torch.zeros(N, dtype=torch.int64, device=self._device)
        self._n_max = 0
        self._x = torch.zeros((N, W), dtype=self._dtype, device=self._device)
        self._K = torch.zeros((N, W), dtype=self._dtype, device=self._device)
        self.y = 0       # update() never stores its residual (:128, :132): y stays 0

    def _out(self, t):
        return t if not self._single else to_numpy(t)[0]

    x = property(lambda self: self._out(self._x), lambda self, v: setattr(self, "_x", self._tensor(v, (self.n_filters, self._order + 1))))
    K = property(lambda self: self._out(self._K))
    sigma = property(lambda self: self._param_out("sigma"), lambda self, v: self._set_param("sigma", v))
    dt = property(lambda self: self._param_out("dt"), lambda self, v: self._set_dt(v))

    @property
    def n(self):
        return int(to_numpy(self._n)[0]) if self._single else self._n

    @n.setter
    def n(self, v):
        n = np.broadcast_to(np.asarray(to_numpy(v) if isinstance(v, torch.Tensor) else v, np.int64), (self.n_filters,))
        self._n = torch.as_tensor(n.copy(), device=self._device)
        self._n_max = int(n.max(initial=0))

    def _set_dt(self, v):
        self._set_param("dt", v)
        dt = self._p["dt"][0]
        self._set_param("dt2", host_const(lambda d: d**2, dt))                         # :148 den*dt**2
        self._set_param("hdt2", host_const(lambda d: 0.5 * d**2, dt))                  # :150-152 0.5 * dt**2

    def _params(self):
        return {k: self._call_param(None, k) for k in ("dt", "dt2", "hdt2")}

    def update(self, z):
        """least_squares.py:112-155: one launch; returns x"""
        self._launch(_lib.BKE_POLY_LSQ, self._order, self._z(z), _lib.BKE_POLY_UPDATE, self._x,
                     params=self._params(), n=self._n, n_max=self._n_max, K=self._K)
        self._n_max += 1
        return self.x

    def batch_filter(self, data):
        """T epochs of update() in one launch on a copy of the state: results[T+1, N, order+1] (single mode:
        [T+1, order+1]); the filter itself is not changed"""
        z = self._z(data, T=len(data))
        T, N = z.shape
        res = torch.empty((T + 1, N, self._order + 1), dtype=self._dtype, device=self._device)
        self._launch(_lib.BKE_POLY_LSQ, self._order, z, _lib.BKE_POLY_BATCH, self._x,
                     params=self._params(), n=self._n, n_max=self._n_max, results=res)
        return to_numpy(res)[:, 0] if self._single else res

    def errors(self):
        """least_squares.py:157-205: (error, std), each of order+1 (bank mode: [N, order+1] tensors), on the host"""
        order, W = self._order, self._order + 1
        ns = to_numpy(self._n)
        dts = np.broadcast_to(self._p["dt"][0], ns.shape)
        sig = np.broadcast_to(self._p["sigma"][0], ns.shape)
        error, std = np.zeros((len(ns), W)), np.zeros((len(ns), W))
        for f, (n, dt, sigma) in enumerate(zip(ns.tolist(), dts.tolist(), sig.tolist())):
            if n == 0:
                continue
            if order == 0:
                error[f, 0] = std[f, 0] = sigma / math.sqrt(n)
            elif order == 1:
                if n > 1:
                    error[f, 0] = sigma * math.sqrt(2 * (2 * n - 1) / (n * (n + 1)))
                    error[f, 1] = sigma * math.sqrt(12. / (n * (n * n - 1) * dt * dt))
                std[f, 0] = sigma * math.sqrt((2 * (2 * n - 1)) / (n * (n + 1)))
                std[f, 1] = (sigma / dt) * math.sqrt(12. / (n * (n * n - 1))) if n > 1 else _div0()
            else:
                dt2 = dt * dt
                if n >= 3:
                    error[f, 0] = sigma * math.sqrt(3 * (3 * n * n - 3 * n + 2) / (n * (n + 1) * (n + 2)))
                    error[f, 1] = sigma * math.sqrt(12 * (16 * n * n - 30 * n + 11) / (n * (n * n - 1) * (n * n - 4) * dt2))
                    error[f, 2] = sigma * math.sqrt(720 / (n * (n * n - 1) * (n * n - 4) * dt2 * dt2))
                std[f, 0] = sigma * math.sqrt((3 * (3 * n * n - 3 * n + 2)) / (n * (n + 1) * (n + 2)))
                if n < 3:
                    _div0()
                std[f, 1] = (sigma / dt) * math.sqrt((12 * (16 * n * n - 30 * n + 11)) / (n * (n * n - 1) * (n * n - 4)))
                std[f, 2] = (sigma / dt2) * math.sqrt(720 / (n * (n * n - 1) * (n * n - 4)))
        if self._single:
            return error[0], std[0]
        return (torch.as_tensor(error, device=self._device).to(self._dtype),
                torch.as_tensor(std, device=self._device).to(self._dtype))


def _div0():
    """what the reference's std raises for order 1 at n = 1 and order 2 at n < 3 (:189, :201): a zero divisor"""
    raise ZeroDivisionError('float division by zero')
