"""Host-side mirror of ``filterpy.kalman.CubatureKalmanFilter`` for a BANK of filters on one H100
(filterpy/kalman/CubatureKalmanFilter.py: ``__init__`` :240-290, ``predict`` :292-327, ``update`` :329-389).

The process and measurement functions are the UKF mirror's device-side models (``LinearFx``,
``ConstVelFx``, ``LinearHx``, ``RangeAzElHx``, ``RangeBearingHx``, or ``DeviceFx`` / ``DeviceHx`` around
CUDA source text; see ``UKF.py``).  The kernel is ``csrc/ckf_kernel.cuh``.
"""
import numpy as np
import torch

from .. import _lib
from .._dev import ptr
from .UKF import _DeviceModel, _SigmaPointBank, _compile_model, _device_hooks, _no_hook, _require_device_models

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

    _compile_model = staticmethod(lambda *a, **k: _compile_model(*a, entry="bke_ckf_model_compile", **k))

    def __init__(self, dim_x, dim_z, dt, hx, fx, x_mean_fn=None, z_mean_fn=None, residual_x=None,
                 residual_z=None, n_filters=None, dtype=np.float64, device=None, diagnostics=True):
        # the reference stores x_mean_fn, z_mean_fn and residual_x but never calls them; residual_z forms
        # y = residual_z(z, z^) (:376) and may be a DeviceFn
        for nm, v in (("x_mean_fn", x_mean_fn), ("z_mean_fn", z_mean_fn), ("residual_x", residual_x)):
            _no_hook(nm, v)
        hooks = _device_hooks(residual_z=residual_z)
        _require_device_models(fx, hx)
        self._init_bank(dim_x, dim_z, fx, hx, n_filters, dtype, device, diagnostics, hooks)
        self._dt = dt
        self._num_sigmas = 2 * self.dim_x
        shape = (self.n_filters, self._num_sigmas, self.dim_x)
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
            self._sf = torch.zeros((self.n_filters, self._num_sigmas, self.dim_x), dtype=self._dtype, device=self._device)
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

    def update(self, z, R=None, hx_args=(), valid=None):
        """CubatureKalmanFilter.py:329-389.  ``z`` is ``(N, dim_z)`` in bank mode; ``z=None`` skips the update
        (:348-352); ``valid[N]`` (0 = no measurement) does so per filter.  A scalar ``R`` is ``R * I``."""
        ov = _positional(self.hx, hx_args, "hx_args")
        dt, self._pending = self._pending, None
        if z is None:
            self._skip_update(dt)
            return
        if ov:
            self._hx_args = self.hx.pack(ov, self.n_filters, self._dtype, self._device)
        if dt is None and self._sf_lost:
            raise NotImplementedError(
                "update() without predict() reads the propagated points of the last predict (sigmas_f), and "
                "the last predict ran fused with an update on a filter built with diagnostics=False, which does "
                "not keep them: build the filter with diagnostics=True to update twice without a predict")
        zt = self._z_rows(z)
        vt = self._valid_mask(valid)
        flags = _lib.BKE_DO_UPDATE | (_lib.BKE_DO_PREDICT if dt is not None else 0)
        self._launch(flags, self._dt if dt is None else dt, zt, vt, R)
        self._z = zt

    def _launch(self, flags, dt, zt, vt, R):
        a = self._fill(_lib.CkfArgs(), flags, dt, zt, vt, R)
        fused = (flags & _lib.BKE_DO_PREDICT) and (flags & _lib.BKE_DO_UPDATE)
        if self.diagnostics or not fused:
            a.sigmas_f = ptr(self._points())
        self._step(a, self._lib.bke_ckf_step, self._lib.bke_ckf_step_model)
        if flags & _lib.BKE_DO_PREDICT:
            self._sf_lost = bool(fused and not self.diagnostics)
