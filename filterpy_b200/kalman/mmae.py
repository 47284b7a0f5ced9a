"""Host-side mirror of ``filterpy.kalman.MMAEFilterBank`` (filterpy/kalman/mmae.py:29-230) for a
bank of tracks: ``filters`` is a list of M ``KalmanFilter`` banks with the same ``n_filters``.
``update`` runs every model's bank kernel, then one launch for ``p *= likelihood; p /= sum(p)``
(:180-184) and one for the combined estimate (:186-201, including the reference's element-wise
``zip`` over the mixed state — see ``bke_mm_estimate`` / ``BKE_MM_MMAE`` in include/bke.h).
"""
import ctypes
from copy import deepcopy

import numpy as np
import torch

from .. import _lib
from .._dev import ptr, stream_ptr
from .IMM import _check_bank, _mm_args

__all__ = ["MMAEFilterBank"]


class MMAEFilterBank(object):
    def __init__(self, filters, p, dim_x, H=None):
        if len(filters) != len(p):
            raise ValueError('length of filters and p must be the same')       # mmae.py:105-106
        if dim_x < 1:
            raise ValueError('dim_x must be >= 1')
        f0 = _check_bank(filters)
        self.filters = filters
        self.dim_x = dim_x
        self.H = None if H is None else np.copy(H)
        self._single = f0._single
        self._dtype, self._device = f0._dtype, f0._device
        self._lib = _lib.load()
        nt, nm, n = f0.n_filters, len(filters), f0.dim_x
        pa = np.asarray(p, dtype=np.float64)
        if pa.shape == (nm,):
            pa = np.broadcast_to(pa, (nt, nm))
        if pa.shape != (nt, nm):
            raise ValueError("p must have shape (%d,) or (%d,%d)" % (nm, nt, nm))
        self._p = torch.from_numpy(np.array(pa, dtype=np.float64, order='C')).to(self._device)
        self._x = f0._x.clone(); self._P = f0._P.clone()          # mmae.py:118-121
        self.z = f0.z
        self._x_prior = self._x.clone(); self._P_prior = self._P.clone()
        self._x_post = self._x.clone(); self._P_post = self._P.clone()

    x = property(lambda self: self.filters[0]._vec_out(self._x))
    P = property(lambda self: self.filters[0]._out(self._P))
    x_prior = property(lambda self: self.filters[0]._vec_out(self._x_prior))
    P_prior = property(lambda self: self.filters[0]._out(self._P_prior))
    x_post = property(lambda self: self.filters[0]._vec_out(self._x_post))
    P_post = property(lambda self: self.filters[0]._out(self._P_post))
    p = property(lambda self: self.filters[0]._out(self._p))

    def predict(self, u=0):
        """mmae.py:134-153."""
        for f in self.filters:
            f.predict(None if (np.isscalar(u) and u == 0) else u)
        self._x_prior.copy_(self._x); self._P_prior.copy_(self._P)

    def update(self, z, R=None, H=None, valid=None):
        """mmae.py:155-206.  ``valid`` (bool[N]) marks the tracks that have a measurement; the
        others behave as the reference's ``update(None)``."""
        if H is None:
            H = self.H
        for f in self.filters:
            f.update(z, R, H, valid=valid)
        a = _mm_args(self.filters, flags=_lib.BKE_MM_MMAE)
        a.mu = ptr(self._p)
        a.weights_stride = len(self.filters)
        a.x_out[0], a.P_out[0] = ptr(self._x), ptr(self._P)
        with torch.cuda.device(self._device):
            _lib.check(self._lib.bke_mm_probabilities(ctypes.byref(a), stream_ptr(self._device)))
            _lib.check(self._lib.bke_mm_estimate(ctypes.byref(a), stream_ptr(self._device)))
        self.z = deepcopy(z) if not isinstance(z, torch.Tensor) else z
        self._x_post.copy_(self._x); self._P_post.copy_(self._P)

    def __repr__(self):
        return "MMAEFilterBank (H100): %d models x %d tracks" % (len(self.filters), self.filters[0].n_filters)
