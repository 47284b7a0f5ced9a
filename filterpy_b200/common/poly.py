"""What the polynomial tracker mirrors (``filterpy_b200.gh``, ``.leastsq``, ``.memory``) share: the single / bank mode
switch, their parameters (host value and device copy), the constants the reference derives from its scalars and the
one launch of ``bke_poly_filter``.

Single mode (``n_filters=None``) is a drop-in for one reference object: NumPy attributes, fp64.  A ``GHFilter`` whose
``x`` is an array is a bank of ``x.size`` elements, as the reference's element-wise filter is.  Bank mode
(``n_filters=N``) keeps the state as device tensors with a leading N axis; a parameter is a scalar shared by the bank
or one value per filter.
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from .._dev import bke_dtype, require_cuda, resolve_dtype, stream_ptr


def host_const(fn, *vals):
    """``fn`` evaluated on Python floats, element by element over the broadcast of ``vals`` (scalars or arrays).

    The reference derives its constants (``dt**2``, ``h / dt``, ``1 - beta**3`` ...) from Python scalars, where ``**``
    is the C library's ``pow``; NumPy's vectorised power may round differently, so each distinct argument tuple is
    evaluated once as the reference evaluates it."""
    arrs = [np.asarray(v, np.float64) for v in vals]
    if all(a.ndim == 0 for a in arrs):
        return np.float64(fn(*[float(a) for a in arrs]))
    b = np.broadcast_arrays(*arrs)
    rows = np.stack([a.reshape(-1) for a in b], axis=1)
    uniq, inv = np.unique(rows, axis=0, return_inverse=True)
    vals = np.array([fn(*[float(v) for v in row]) for row in uniq], np.float64)
    return vals[np.asarray(inv).reshape(-1)].reshape(b[0].shape)


class PolyBank(object):
    """Mode, dtype and device of a tracker bank, and its parameters: ``self._p[name] = (host, device, stride)``."""

    def _init_mode(self, n_filters, size, dtype, device, saver=None):
        if saver is not None:
            raise NotImplementedError("saver is not supported (filterpy.common.Saver is out of scope)")
        self._single = n_filters is None
        self._device = require_cuda(device)
        self._dtype = torch.float64 if self._single else resolve_dtype(dtype)
        self.n_filters = int(size if self._single else n_filters)
        if self.n_filters < 0:
            raise ValueError('n_filters must be 0 or greater')
        self._p = {}

    # ------------------------------------------------------------------ conversions
    def _tensor(self, v, shape):
        """a device tensor of the bank's dtype broadcast to ``shape`` (a fresh copy)"""
        if isinstance(v, torch.Tensor):
            t = v.to(device=self._device, dtype=self._dtype)
        else:
            t = torch.as_tensor(np.asarray(v, np.float64), device=self._device).to(self._dtype)
        return t.expand(shape).contiguous().clone() if t.shape != torch.Size(shape) else t.contiguous().clone()

    def _host(self, v):
        """a parameter as the host sees it: a float64 scalar (shared) or an (N,) array (per filter)"""
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu().double().numpy()
        a = np.asarray(v, np.float64)
        if a.ndim == 0:
            return np.float64(a)
        a = a.reshape(-1)
        if a.size == 1 and self._single and self.n_filters != 1:
            return np.float64(a[0])
        if a.size != self.n_filters:
            raise ValueError("a parameter is a scalar or has one value per filter (%d), got %d" % (self.n_filters, a.size))
        return a.copy()

    def _dev_param(self, host):
        """(device tensor, stride) of a host parameter"""
        if np.ndim(host) == 0:
            return torch.tensor([float(host)], dtype=self._dtype, device=self._device), 0
        return torch.as_tensor(host, device=self._device).to(self._dtype).contiguous(), 1

    def _set_param(self, name, value):
        if value is None:
            self._p[name] = None
            return
        host = self._host(value)
        self._p[name] = (host,) + self._dev_param(host)

    def _param_out(self, name):
        """the attribute: the value as given in single mode, a device tensor in bank mode"""
        p = self._p.get(name)
        if p is None:
            return None
        if self._single:
            return p[0] if np.ndim(p[0]) == 0 or self.n_filters != 1 else np.float64(p[0][0])
        return p[1] if p[2] == 1 else p[1][0]

    def _call_param(self, value, name):
        """a per-call override (None: the attribute) as (device tensor, stride)"""
        if value is None:
            p = self._p.get(name)
            return (None, 0) if p is None else (p[1], p[2])
        if isinstance(value, torch.Tensor) and value.dim() == 1 and value.numel() == self.n_filters:
            return value.to(device=self._device, dtype=self._dtype).contiguous(), 1
        return self._dev_param(self._host(value))

    def _z(self, z, T=None):
        """the measurements as a [T, N] device tensor (T = 1 for update)"""
        shape = (1 if T is None else T, self.n_filters)
        if isinstance(z, torch.Tensor):
            t = z.to(device=self._device, dtype=self._dtype)
        else:
            t = torch.as_tensor(np.asarray(z, np.float64), device=self._device).to(self._dtype)
        if T is None:
            t = t.reshape(1, -1) if t.dim() > 0 else t.reshape(1, 1)
        elif t.dim() == 1:
            t = t.reshape(T, -1)
        return t.expand(shape).contiguous() if t.shape != torch.Size(shape) else t.contiguous()

    # ------------------------------------------------------------------ the launch
    def _launch(self, family, order, z, mode, x, dx=None, ddx=None, params=None, n=None, n_max=0, **outs):
        a = _lib.PolyArgs()
        a.n_filters, a.n_steps = self.n_filters, z.shape[0]
        a.family, a.order, a.dtype, a.mode = family, order, bke_dtype(self._dtype), mode
        keep = [z]
        a.x, a.z = x.data_ptr(), z.data_ptr()
        a.dx = dx.data_ptr() if dx is not None else None
        a.ddx = ddx.data_ptr() if ddx is not None else None
        for name, (t, stride) in (params or {}).items():
            if t is not None:
                keep.append(t)
                setattr(a, name, t.data_ptr())
                setattr(a, name + "_stride", stride)
        if n is not None:
            a.n, a.n_max = n.data_ptr(), int(n_max)
        for name, t in outs.items():
            if t is not None:
                setattr(a, name, t.data_ptr())
        if self.n_filters == 0:
            return
        with torch.cuda.device(self._device):          # the launch goes to the current device: make it the bank's
            _lib.check(_lib.load().bke_poly_filter(ctypes.byref(a), stream_ptr(self._device)))
        del keep


def to_numpy(t):
    return t.detach().cpu().numpy()
