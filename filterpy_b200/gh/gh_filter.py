"""Mirrors of filterpy.gh (filterpy/gh/gh_filter.py): GHFilter, GHKFilter and GHFilterOrder banks on bke_poly_filter,
and the gain helpers.

Single mode (no ``n_filters``) takes what the reference takes, fp64 with NumPy attributes; an array ``x`` is a bank
of ``x.size`` filters, as the reference's element-wise filter is.  Bank mode (``n_filters=N``, ``dtype``, ``device``)
keeps ``x``, ``dx`` (``ddx``) as device tensors [N]; ``update(z[N])`` and ``batch_filter(data[T, N])`` are one launch
each.  The gains may be scalars or one per filter, per call as well.  ``dt`` is a scalar or one per filter.
"""
import numpy as np
import torch

from .. import _lib
from ..common.poly import PolyBank, host_const, to_numpy


class _GHBase(PolyBank):
    _FAMILY = None
    _STATE = ()

    def _init_state(self, values, n_filters, dtype, device):
        arr = [np.asarray(v) if not isinstance(v, torch.Tensor) else v for v in values]
        self._scalar = n_filters is None and all(np.ndim(v) == 0 for v in arr)
        size = 1 if self._scalar else (max(int(np.size(v)) for v in arr) if n_filters is None else n_filters)
        self._init_mode(n_filters, size, dtype, device)
        N = self.n_filters
        for name, v in zip(self._STATE, arr):
            setattr(self, "_" + name, self._tensor(v, (N,)))
        for name in self._STATE:
            setattr(self, "_" + name + "_prediction", getattr(self, "_" + name).clone())   # gh_filter.py:311-312
        self._y = torch.zeros(N, dtype=self._dtype, device=self._device)                    # :314-319
        self._zlast = torch.zeros(N, dtype=self._dtype, device=self._device)

    def _out(self, t):
        if not self._single:
            return t
        a = to_numpy(t)
        return np.float64(a[0]) if self._scalar else a

    def _set_state(self, name, v):
        setattr(self, "_" + name, self._tensor(v, (self.n_filters,)))

    x = property(lambda self: self._out(self._x), lambda self, v: self._set_state("x", v))
    dx = property(lambda self: self._out(self._dx), lambda self, v: self._set_state("dx", v))
    x_prediction = property(lambda self: self._out(self._x_prediction))
    dx_prediction = property(lambda self: self._out(self._dx_prediction))
    y = property(lambda self: self._out(self._y))
    # GHFilter.update / GHKFilter.update never store z (:373, :674): it keeps its initial zeros
    z = property(lambda self: self._out(self._zlast))
    g = property(lambda self: self._param_out("g"), lambda self, v: self._set_param("g", v))
    h = property(lambda self: self._param_out("h"), lambda self, v: self._set_h(v))
    dt = property(lambda self: self._param_out("dt"), lambda self, v: self._set_dt(v))

    def _set_dt(self, v):
        self._set_param("dt", v)
        self._set_param("dt2", host_const(lambda dt: dt ** 2, self._p["dt"][0]))           # :667 dt_sqr = dt**2
        self._set_h_dt()

    def _set_h(self, v):
        self._set_param("h", v)
        self._set_h_dt()

    def _set_h_dt(self):
        """batch_filter's h_dt = self.h / self.dt (:433, :729): one IEEE division, NumPy's equals Python's"""
        if self._p.get("h") is not None and self._p.get("dt") is not None:
            self._set_param("h_dt", np.divide(self._p["h"][0], self._p["dt"][0]))

    def _pair(self):
        return (self.x, self.dx)

    def _closed(self, fn, *names, extra=()):
        """a closed form in the parameters, evaluated on the host as the reference evaluates it (Python floats)"""
        v = host_const(fn, *[self._p[n][0] for n in names], *[np.asarray(e, np.float64) if not isinstance(e, torch.Tensor)
                                                            else to_numpy(e) for e in extra])
        if self._single:
            return np.float64(v.reshape(-1)[0]) if self._scalar and np.ndim(v) else v
        return torch.as_tensor(np.asarray(v, np.float64), device=self._device).to(self._dtype)

    def batch_filter(self, data, save_predictions=False, saver=None):
        """GHFilter.batch_filter (gh_filter.py:380-455) / GHKFilter.batch_filter (:683-748): one launch over
        data[T] (single mode, scalar x) or data[T, N].  x and dx are read and not changed; GHKFilter's runs the
        g-h recursion and ignores k and ddx, as the reference does (:717-743)."""
        if saver is not None:
            raise NotImplementedError("saver is not supported (filterpy.common.Saver is out of scope)")
        z = self._z(data, T=len(data))
        T, N = z.shape
        res = torch.empty((T + 1, N, 2), dtype=self._dtype, device=self._device)
        pred = torch.empty((T, N), dtype=self._dtype, device=self._device) if save_predictions else None
        self._launch(_lib.BKE_POLY_GH, 1, z, _lib.BKE_POLY_BATCH, self._x, self._dx,
                     params=dict(g=self._call_param(None, "g"), h=self._call_param(None, "h_dt"), dt=self._call_param(None, "dt")),
                     results=res, predictions=pred)
        if self._single:
            res, pred = to_numpy(res), None if pred is None else to_numpy(pred)
            if self._scalar:
                res, pred = res[:, 0, :], None if pred is None else pred[:, 0]
        return (res, pred) if save_predictions else res


class GHFilter(_GHBase):
    """filterpy.gh.GHFilter (gh_filter.py:197-523): ``GHFilter(x, dx, dt, g, h, n_filters=None, dtype, device)``."""
    _STATE = ("x", "dx")

    def __init__(self, x, dx, dt, g, h, n_filters=None, dtype=np.float64, device=None):
        self._init_state((x, dx), n_filters, dtype, device)
        self.dt, self.g, self.h = dt, g, h

    def update(self, z, g=None, h=None):
        """gh_filter.py:322-377: one launch; returns (x, dx)."""
        self._launch(_lib.BKE_POLY_GH, 1, self._z(z), _lib.BKE_POLY_UPDATE, self._x, self._dx,
                     params=dict(g=self._call_param(g, "g"), h=self._call_param(h, "h"), dt=self._call_param(None, "dt")),
                     y=self._y, x_prediction=self._x_prediction, dx_prediction=self._dx_prediction)
        return self._pair()

    def VRF_prediction(self):
        """gh_filter.py:458-478, in the gains (host)"""
        return self._closed(lambda g, h: (2 * g**2 + 2 * h + g * h) / (g * (4 - 2 * g - h)), "g", "h")

    def VRF(self):
        """gh_filter.py:481-509: (vx, vdx)"""
        return (self._closed(lambda g, h: (2 * g**2 + 2 * h - 3 * g * h) / (g * (4 - 2 * g - h)), "g", "h"),
                self._closed(lambda g, h, dt: 2 * h**2 / (dt**2 * (g * (4 - 2 * g - h))), "g", "h", "dt"))


class GHKFilter(_GHBase):
    """filterpy.gh.GHKFilter (gh_filter.py:526-854): ``GHKFilter(x, dx, ddx, dt, g, h, k, n_filters=None, dtype, device)``."""
    _STATE = ("x", "dx", "ddx")

    def __init__(self, x, dx, ddx, dt, g, h, k, n_filters=None, dtype=np.float64, device=None):
        self._init_state((x, dx, ddx), n_filters, dtype, device)
        self.dt, self.g, self.h, self.k = dt, g, h, k

    ddx = property(lambda self: self._out(self._ddx), lambda self, v: self._set_state("ddx", v))
    ddx_prediction = property(lambda self: self._out(self._ddx_prediction))
    k = property(lambda self: self._param_out("k"), lambda self, v: self._set_param("k", v))

    def update(self, z, g=None, h=None, k=None):
        """gh_filter.py:630-680: one launch; returns (x, dx)."""
        self._launch(_lib.BKE_POLY_GHK, 2, self._z(z), _lib.BKE_POLY_UPDATE, self._x, self._dx, self._ddx,
                     params=dict(g=self._call_param(g, "g"), h=self._call_param(h, "h"), k=self._call_param(k, "k"),
                                 dt=self._call_param(None, "dt"), dt2=self._call_param(None, "dt2")),
                     y=self._y, x_prediction=self._x_prediction, dx_prediction=self._dx_prediction,
                     ddx_prediction=self._ddx_prediction)
        return self._pair()

    def VRF_prediction(self):
        """gh_filter.py:751-774"""
        def vrf(g, h, k):
            gh2 = 2 * g + h
            return (g * k * (gh2 - 4) + h * (g * gh2 + 2 * h)) / (2 * k - (g * (h + k) * (gh2 - 4)))
        return self._closed(vrf, "g", "h", "k")

    def bias_error(self, dddx):
        """gh_filter.py:777-794: the bias error for a constant jerk dddx"""
        return self._closed(lambda dt, k, j: -dt**3 * j / (2 * k), "dt", "k", extra=(dddx,))

    def VRF(self):
        """gh_filter.py:797-836: (vx, vdx, vddx)"""
        def hg4(g, h):
            return 4 - 2 * g - h

        def ghk(g, h, k):
            return g * h + g * k - 2 * k
        return (self._closed(lambda g, h, k: (2 * h * (2 * (g**2) + 2 * h - 3 * g * h) - 2 * g * k * hg4(g, h)) /
                             (2 * k - g * (h + k) * hg4(g, h)), "g", "h", "k"),
                self._closed(lambda g, h, k: (2 * (h**3) - 4 * (h**2) * k + 4 * (k**2) * (2 - g)) /
                             (2 * hg4(g, h) * ghk(g, h, k)), "g", "h", "k"),
                self._closed(lambda g, h, k, dt: 8 * h * (k**2) / ((dt**4) * hg4(g, h) * ghk(g, h, k)), "g", "h", "k", "dt"))


class GHFilterOrder(PolyBank):
    """filterpy.gh.GHFilterOrder (gh_filter.py:31-194): ``GHFilterOrder(x0, dt, order, g, h=None, k=None,
    n_filters=None, dtype, device)``.  Bank mode: x0 is a scalar, (order+1,) or (N, order+1); x is [N, order+1].
    ``batch_filter(data[T, N])`` returns the states after every epoch and leaves the filter as it was."""

    def __init__(self, x0, dt, order, g, h=None, k=None, n_filters=None, dtype=np.float64, device=None):
        if order < 0 or order > 2:
            raise ValueError('order must be between 0 and 2')                      # gh_filter.py:116-117
        self._init_mode(n_filters, 1, dtype, device)
        self.order = order
        W, N = order + 1, self.n_filters
        if np.isscalar(x0):                                                         # :119-123
            x = np.zeros(W)
            x[0] = x0
        else:
            x = x0 if isinstance(x0, torch.Tensor) else np.asarray(x0).astype(float)
        self._x = self._tensor(x, (N, W))
        self._y = torch.zeros(N, dtype=self._dtype, device=self._device)           # :131-132
        self._zlast = None
        self._updated = False
        self.dt, self.g, self.h, self.k = dt, g, h, k

    def _out(self, t):
        return t if not self._single else to_numpy(t)[0]

    x = property(lambda self: self._out(self._x), lambda self, v: setattr(self, "_x", self._tensor(v, (self.n_filters, self.order + 1))))
    g = property(lambda self: self._param_out("g"), lambda self, v: self._set_param("g", v))
    h = property(lambda self: self._param_out("h"), lambda self, v: self._set_param("h", v))
    k = property(lambda self: self._param_out("k"), lambda self, v: self._set_param("k", v))
    dt = property(lambda self: self._param_out("dt"), lambda self, v: self._set_dt(v))

    def _set_dt(self, v):
        self._set_param("dt", v)
        self._set_param("dt2", host_const(lambda dt: dt ** 2., self._p["dt"][0]))           # :175 T2 = dt**2.

    @property
    def y(self):
        """the last residual (a scalar per filter; zeros(order+1) before the first update, :131)"""
        if self._single and not self._updated:
            return np.zeros(self.order + 1)
        return self._out(self._y)

    @property
    def z(self):
        """the last measurement of an order-1 filter: update() stores z for order 1 only (:161)"""
        if self._zlast is None:
            return np.zeros(self.order + 1) if self._single else torch.zeros((self.n_filters, self.order + 1),
                                                                              dtype=self._dtype, device=self._device)
        return self._out(self._zlast)

    def update(self, z, g=None, h=None, k=None):
        """gh_filter.py:136-181: one launch"""
        zt = self._z(z)
        self._launch(_lib.BKE_POLY_GH_ORDER, self.order, zt, _lib.BKE_POLY_UPDATE, self._x,
                     params=dict(g=self._call_param(g, "g"), h=self._call_param(h, "h"), k=self._call_param(k, "k"),
                                 dt=self._call_param(None, "dt"), dt2=self._call_param(None, "dt2")), y=self._y)
        if self.order == 1:
            self._zlast = zt[0].clone()
        self._updated = True

    def batch_filter(self, data):
        """T epochs of update() in one launch on a copy of the state: results[T+1, N, order+1] (single mode:
        [T+1, order+1]); the filter itself is not changed (the reference has no batch_filter for this class)"""
        z = self._z(data, T=len(data))
        T, N = z.shape
        res = torch.empty((T + 1, N, self.order + 1), dtype=self._dtype, device=self._device)
        self._launch(_lib.BKE_POLY_GH_ORDER, self.order, z, _lib.BKE_POLY_BATCH, self._x,
                     params=dict(g=self._call_param(None, "g"), h=self._call_param(None, "h"), k=self._call_param(None, "k"),
                                 dt=self._call_param(None, "dt"), dt2=self._call_param(None, "dt2")), results=res)
        return to_numpy(res)[:, 0] if self._single else res


# ---------------------------------------------------------------------------------------------- gain helpers
def optimal_noise_smoothing(g):
    """(g, h, k) of the g-h-k filter that smooths noise optimally for the given g (Polge and Bhagavan, 1975)."""
    root = (4 * g**6 - 64 * g**5 + 64 * g**4) ** .5
    h = ((2 * g**3 - 4 * g**2) + root) / (8 * (1 - g))
    k = (h * (2 - g) - g**2) / g
    return (g, h, k)


def least_squares_parameters(n):
    """(g, h) that make a g-h filter the order-1 least-squares filter at measurement n (the first is n = 0)."""
    den = (n + 2) * (n + 1)
    return ((2 * (2 * n + 1)) / den, 6 / den)


def critical_damping_parameters(theta, order=2):
    """(g, h) for order 2, (g, h, k) for order 3, of the critically damped (fading-memory) filter with weight theta."""
    if theta < 0 or theta > 1:
        raise ValueError('theta must be between 0 and 1')
    if order == 2:
        return (1. - theta**2, (1. - theta)**2)
    if order == 3:
        return (1. - theta**3, 1.5 * (1. - theta**2) * (1. - theta), .5 * (1 - theta)**3)
    raise ValueError('bad order specified: {}'.format(order))


def benedict_bornder_constants(g, critical=False):
    """(g, h) of the Benedict-Bordner filter, which minimises the transient error for g; critical=True damps it
    nearly critically."""
    g2 = g**2
    if critical:
        return (g, 0.8 * (2. - g2 - 2 * (1 - g2)**.5) / g2)
    return (g, g2 / (2. - g))
