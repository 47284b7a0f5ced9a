"""Host-side mirror of ``filterpy.kalman.CubatureKalmanFilter`` for a BANK of filters on one H100
(filterpy/kalman/CubatureKalmanFilter.py: ``__init__`` :240-290, ``predict`` :292-327, ``update`` :329-389).

The process and measurement functions are the UKF mirror's device-side models (``LinearFx``,
``ConstVelFx``, ``LinearHx``, ``RangeAzElHx``, ``RangeBearingHx``, or ``DeviceFx`` / ``DeviceHx`` around
CUDA source text; see ``UKF.py``).  The kernel is ``csrc/ckf_kernel.cuh``.
"""
import numpy as np
import torch

from .. import _lib
from .._dev import bke_dtype, ptr, stream_ptr, to_dev
from .UKF import _DeviceModel, _SigmaPointBank, _compile_model, _no_hook

__all__ = ["CubatureKalmanFilter"]


def _positional(model, args, what):
    """The reference's positional ``fx_args`` / ``hx_args`` (a non-tuple is wrapped, :314-315, :354-355) as
    values of the model's ``arg_names``, in order; None when there are none."""
    if not isinstance(args, tuple):
        args = (args,)
    if not args:
        return None
    if not isinstance(model, _DeviceModel):
        raise NotImplementedError("%s are arguments of a Python callback; the built-in models take none" % what)
    if len(args) > len(model.arg_names):
        raise TypeError("%s has %d values but the model declares %d arguments %s"
                        % (what, len(args), len(model.arg_names), list(model.arg_names)))
    return dict(zip(model.arg_names, args))


class CubatureKalmanFilter(_SigmaPointBank):
    """``CubatureKalmanFilter(dim_x, dim_z, dt, hx, fx)`` for ``n_filters`` filters at once (``n_filters=None``:
    one filter with NumPy attributes, raising ``LinAlgError`` where the reference would).

    ``predict`` is deferred and runs fused with the next ``update`` in one launch.  The covariances are
    formed as centred sums instead of the reference's raw second moments (DESIGN.md §3.5b).

    ``sigmas_f`` (``[N, 2n, n]``) holds the propagated points of the last predict, zeros on a new filter,
    as in the reference: ``update`` reads its measurement points from them (:362-363), so an ``update``
    without a ``predict`` before it reuses the stale (or zero) points exactly like the reference.  With
    ``diagnostics=True`` every predict writes them.  With ``diagnostics=False`` the fused predict + update
    does not (it saves ``2n * n`` words per filter of memory traffic): an ``update`` whose points would come
    from such a fused step then raises ``NotImplementedError``.  A predict that runs on its own (flushed by
    reading ``x`` or by ``update(None)``) still writes them.
    """

    _compile_model = staticmethod(lambda *a: _compile_model(*a, entry="bke_ckf_model_compile"))

    def __init__(self, dim_x, dim_z, dt, hx, fx, x_mean_fn=None, z_mean_fn=None, residual_x=None,
                 residual_z=None, n_filters=None, dtype=np.float64, device=None, diagnostics=True):
        for nm, v in (("x_mean_fn", x_mean_fn), ("z_mean_fn", z_mean_fn), ("residual_x", residual_x),
                      ("residual_z", residual_z)):
            _no_hook(nm, v)
        if not hasattr(fx, "model") or not hasattr(hx, "model"):
            raise NotImplementedError(
                "fx / hx must be device-side models (LinearFx, ConstVelFx, LinearHx, RangeAzElHx, "
                "RangeBearingHx, or DeviceFx / DeviceHx around CUDA source text): Python callables cannot "
                "run inside the CUDA kernel and there is no CPU fallback")
        self._init_bank(dim_x, dim_z, fx, hx, n_filters, dtype, device, diagnostics)
        self._dt = dt
        self._num_sigmas = 2 * self._dim_x
        shape = (self.n_filters, self._num_sigmas, self._dim_x)
        self._sf = torch.zeros(shape, dtype=self._dtype, device=self._device) if self.diagnostics else None
        self._sf_lost = False        # a fused step without diagnostics left no points behind

    @property
    def sigmas_f(self):
        """The propagated points of the last predict, ``[N, 2n, n]`` (single mode: ``(2n, n)``)."""
        if not self.diagnostics:
            raise AttributeError("sigmas_f is only kept when the filter is built with diagnostics=True")
        self._flush()
        return self._out(self._sf)

    def _points(self):
        if self._sf is None:
            self._sf = torch.zeros((self.n_filters, self._num_sigmas, self._dim_x), dtype=self._dtype, device=self._device)
        return self._sf

    # ------------------------------------------------------------------ predict / update
    def predict(self, dt=None, fx_args=()):
        """CubatureKalmanFilter.py:292-327 (deferred and fused with the next ``update``).  ``fx_args`` are the
        values of the ``DeviceFx``'s ``arg_names`` in order; each is a scalar or one value per filter.  An
        empty ``fx_args`` keeps the values last given (or the model's defaults)."""
        ov = _positional(self.fx, fx_args, "fx_args")
        self._flush()
        if ov:
            self._fx_args = self.fx.pack(ov, self.n_filters, self._dtype, self._device)
        self._pending = self._dt if dt is None else dt

    def _flush(self):
        if self._pending is not None:
            dt, self._pending = self._pending, None
            self._launch(_lib.BKE_DO_PREDICT, dt, None, None, None)

    def update(self, z, R=None, hx_args=(), valid=None):
        """CubatureKalmanFilter.py:329-389.  ``z`` is ``(N, dim_z)`` in bank mode; ``z=None`` skips the update
        (:348-352); ``valid[N]`` (0 = no measurement) does so per filter.  A scalar ``R`` is ``R * I``."""
        ov = _positional(self.hx, hx_args, "hx_args")
        dt, self._pending = self._pending, None
        if z is None:
            if dt is not None:
                self._launch(_lib.BKE_DO_PREDICT, dt, None, None, None)
            self._z = None
            if self.diagnostics:
                self._x_post.copy_(self._x); self._P_post.copy_(self._P)
            return
        if ov:
            self._hx_args = self.hx.pack(ov, self.n_filters, self._dtype, self._device)
        if dt is None and self._sf_lost:
            raise NotImplementedError(
                "update() without predict() reads the propagated points of the last predict (sigmas_f), and "
                "the last predict ran fused with an update on a filter built with diagnostics=False, which does "
                "not keep them: build the filter with diagnostics=True to update twice without a predict")
        m = self._dim_z
        zt = to_dev(np.asarray(z, dtype=np.float64).reshape(1, -1) if self._single else z, self._dtype, self._device)
        if tuple(zt.shape) != (self.n_filters, m):
            raise ValueError("z must have shape (%d,%d), got %s" % (self.n_filters, m, tuple(zt.shape)))
        vt = None
        if valid is not None:
            vt = torch.as_tensor(valid, device=self._device).to(torch.uint8).contiguous()
        flags = _lib.BKE_DO_UPDATE | (_lib.BKE_DO_PREDICT if dt is not None else 0)
        self._launch(flags, self._dt if dt is None else dt, zt.contiguous(), vt, R)
        self._z = zt

    def _launch(self, flags, dt, zt, vt, R):
        a = _lib.CkfArgs()
        N, n, m = self.n_filters, self._dim_x, self._dim_z
        a.n_filters, a.dim_x, a.dim_z = N, n, m
        a.dtype = bke_dtype(self._dtype)
        a.flags = flags
        a.fx_model, a.hx_model = self.fx.model, self.hx.model
        a.dt = float(dt)
        a.x = a.x_out = ptr(self._x)
        a.P = a.P_out = ptr(self._P)
        a.Q, a.Q_stride = ptr(self._Q), self._stride(self._Q)
        Rm = self._R if R is None else self._model(R, m, m, "R")          # scalar R -> R*I (:359-360)
        a.R, a.R_stride = ptr(Rm), self._stride(Rm)
        if self._F is not None:
            a.F, a.F_stride = ptr(self._F), self._stride(self._F)
        if self._H is not None:
            a.H, a.H_stride = ptr(self._H), self._stride(self._H)
        a.z, a.z_valid = ptr(zt), ptr(vt)
        fused = (flags & _lib.BKE_DO_PREDICT) and (flags & _lib.BKE_DO_UPDATE)
        if self.diagnostics or not fused:
            a.sigmas_f = ptr(self._points())
        if self.diagnostics:
            if flags & _lib.BKE_DO_PREDICT:
                a.x_prior, a.P_prior = ptr(self._x_prior), ptr(self._P_prior)
            if flags & _lib.BKE_DO_UPDATE:
                a.K, a.y, a.S, a.SI = ptr(self._K), ptr(self._y), ptr(self._S), ptr(self._SI)
                a.log_likelihood = ptr(self._ll)
            a.status = ptr(self._status)
        with torch.cuda.device(self._device):
            if self._user_model is not None:
                for nm, mdl, (t, _) in (("fx", self.fx, self._fx_args), ("hx", self.hx, self._hx_args)):
                    if isinstance(mdl, _DeviceModel) and mdl.arg_names and t is None:
                        raise TypeError("%s needs values for its arguments %s" % (nm, list(mdl.arg_names)))
                _lib.check(self._lib.bke_ckf_step_model(a, self._user_model, ptr(self._fx_args[0]), self._fx_args[1],
                                                        ptr(self._hx_args[0]), self._hx_args[1], stream_ptr(self._device)))
            else:
                _lib.check(self._lib.bke_ckf_step(a, stream_ptr(self._device)))
        if flags & _lib.BKE_DO_PREDICT:
            self._sf_lost = bool(fused and not self.diagnostics)
        if self.diagnostics and (flags & _lib.BKE_DO_UPDATE):
            self._x_post.copy_(self._x); self._P_post.copy_(self._P)
        if self.diagnostics and self._single:
            self.check()
