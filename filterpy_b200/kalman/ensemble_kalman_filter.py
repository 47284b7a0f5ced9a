"""Host-side mirror of ``filterpy.kalman.EnsembleKalmanFilter`` for a BANK of filters on one H100
(filterpy/kalman/ensemble_kalman_filter.py: ``__init__`` :158-185, ``initialize`` :187-215, ``update``
:218-273, ``predict`` :275-290).

The process and measurement functions are the UKF mirror's device-side models (``LinearFx``,
``ConstVelFx``, ``LinearHx``, ``RangeAzElHx``, ``RangeBearingHx``, or ``DeviceFx`` / ``DeviceHx`` around
CUDA source text; see ``UKF.py``).  The kernel is ``csrc/enkf_kernel.cuh``.

The reference draws its noise from NumPy's global generator.  Here every filter has its own
counter-based stream (Philox4x32-10 keyed with the seed and the filter index, DESIGN.md §3.5d), so a
filter draws the same numbers whatever the size of the bank.  ``seed=None`` takes the seed from
``np.random`` at construction: ``np.random.seed(k)`` before building the filter makes a run reproducible.

Deliberate differences from the reference:

- ``N == 1`` raises ``ValueError``: the reference divides by ``N - 1 = 0``.
- A clearly indefinite ``Q``, ``R`` or initial ``P`` is an error (``status``, ``check()``; single mode
  raises ``LinAlgError`` at once), where the reference's ``multivariate_normal`` only warns.  A
  positive SEMI-definite one (rank-deficient, or zero) is drawn from exactly.
- ``fx`` / ``hx`` must be device-side models and ``inv`` stays ``np.linalg.inv``.
"""
import numpy as np
import torch

from .. import _lib
from .._dev import bke_dtype, ptr, stream_ptr, to_dev
from ._bank import _Linked
from .UKF import _SigmaPointBank, _compile_model, _require_device_models

__all__ = ["EnsembleKalmanFilter"]


def _absent(name):
    def get(self):
        raise AttributeError("EnsembleKalmanFilter has no %s: the reference computes none" % name)
    return property(get)


class EnsembleKalmanFilter(_SigmaPointBank):
    """``EnsembleKalmanFilter(x, P, dim_z, dt, N, hx, fx)`` for ``n_filters`` filters at once
    (``n_filters=None``: one filter with NumPy attributes, raising ``LinAlgError`` where the reference would).

    ``x`` is ``(n,)`` or, in bank mode, ``(n_filters, n)``; ``P`` is ``(n, n)`` or ``(n_filters, n, n)``.
    ``predict`` is deferred and runs fused with the next ``update`` in one launch.  ``sigmas`` is the
    ensemble: ``(N, n)`` NumPy in single mode, the live ``(n_filters, N, n)`` tensor in bank mode; it is
    assignable.  ``update(z, R=None, valid=None)``: a scalar ``R`` is ``R * I``; ``valid[n_filters]``
    (0 = no measurement) skips the update of single filters, as ``z=None`` does for the whole bank.
    """

    _compile_model = staticmethod(lambda *a, **k: _compile_model(*a, entry="bke_enkf_model_compile", **k))
    _FAILURE = "covariance not positive semi-definite / singular S"

    def __init__(self, x, P, dim_z, dt, N, hx, fx, n_filters=None, dtype=np.float64, device=None,
                 diagnostics=True, seed=None):
        if dim_z <= 0:
            raise ValueError('dim_z must be greater than zero')           # :159-160
        if N <= 0:
            raise ValueError('N must be greater than zero')               # :162-163
        if N == 1:
            raise ValueError('N must be 2 or greater: the ensemble covariances divide by N - 1')
        _require_device_models(fx, hx)
        if n_filters is None and np.ndim(x) != 1:
            raise ValueError('x must be a 1D array')                      # :203-204
        dim_x = int(np.shape(x)[-1]) if not isinstance(x, torch.Tensor) else int(x.shape[-1])
        if seed is None:
            seed = int(np.random.randint(0, 2 ** 32, dtype=np.int64))
        self.seed = int(seed) & 0xffffffff
        self._counter = 0
        self._init_bank(dim_x, dim_z, fx, hx, n_filters, dtype, device, diagnostics)
        self.dt = dt
        self.N = int(N)
        self._sig = torch.zeros((self.n_filters, self.N, self.dim_x), dtype=self._dtype, device=self._device)
        self.initialize(x, P)

    y = _absent("y")
    log_likelihood = _absent("log_likelihood")
    likelihood = _absent("likelihood")
    mahalanobis = _absent("mahalanobis")

    @property
    def inv(self):
        return np.linalg.inv

    @inv.setter
    def inv(self, v):
        if v is not np.linalg.inv:
            raise NotImplementedError("the EnKF kernel inverts S as np.linalg.inv does; another inv is not supported")

    @property
    def counter(self):
        """The draw-call index of the next draw of the noise stream (one per initialize, predict and update)."""
        self._flush()
        return self._counter

    @property
    def sigmas(self):
        self._flush()
        if self._single:
            return _Linked(self._sig[0].cpu().numpy(), self, "sigmas")
        return self._sig

    @sigmas.setter
    def sigmas(self, v):
        self._flush()
        t = to_dev(v, self._dtype, self._device)
        if self._single:
            t = t.reshape((1,) + tuple(t.shape))
        if tuple(t.shape) != (self.n_filters, self.N, self.dim_x):
            raise ValueError("sigmas must have shape %s" % ((self.N, self.dim_x) if self._single
                                                           else (self.n_filters, self.N, self.dim_x),))
        self._sig = t.contiguous().clone()

    # ------------------------------------------------------------------ initialize / predict / update
    def initialize(self, x, P):
        """:187-215: members drawn from N(x, P); x and P are kept as given, the priors and posteriors copy them."""
        self._flush()
        if self._single and np.ndim(x) != 1:
            raise ValueError('x must be a 1D array')
        self.x = x
        self.P = P
        status = self._status if self.diagnostics else None
        self._run(self._lib.bke_enkf_initialize, self.n_filters, self.dim_x, self.N, bke_dtype(self._dtype),
                  self.seed, self._counter, ptr(self._x), ptr(self._P), ptr(self._sig), ptr(status),
                  stream_ptr(self._device))
        self._counter += 1
        if self.diagnostics:
            for t in (self._x_prior, self._x_post):
                t.copy_(self._x)
            for t in (self._P_prior, self._P_post):
                t.copy_(self._P)
            if self._single:
                self.check()

    def predict(self):
        """:275-290 (deferred and fused with the next ``update``)."""
        self._flush()
        self._pending = self.dt

    def update(self, z, R=None, valid=None):
        """:218-273.  ``z`` is ``(n_filters, dim_z)`` in bank mode; ``z=None`` leaves the members, x and P
        unchanged and copies them to the posteriors (:234-238)."""
        dt, self._pending = self._pending, None
        if z is None:
            self._skip_update(dt)
            return
        zt = self._z_rows(z)
        vt = self._valid_mask(valid)
        flags = _lib.BKE_DO_UPDATE | (_lib.BKE_DO_PREDICT if dt is not None else 0)
        self._launch(flags, self.dt if dt is None else dt, zt, vt, R)
        self._z = zt

    def _launch(self, flags, dt, zt, vt, R):
        a = self._fill(_lib.EnkfArgs(), flags, dt, zt, vt, R)
        a.n_members = self.N
        a.seed, a.counter = self.seed, self._counter
        a.sigmas = a.sigmas_out = ptr(self._sig)
        self._counter += (1 if flags & _lib.BKE_DO_PREDICT else 0) + (1 if flags & _lib.BKE_DO_UPDATE else 0)
        self._step(a, self._lib.bke_enkf_step, self._lib.bke_enkf_step_model)

    def __repr__(self):
        def show(name):
            try:
                v = getattr(self, name)
            except AttributeError:
                return "%s = (not kept)" % name
            return "%s = %s" % (name, v)
        return "\n".join(["EnsembleKalmanFilter object",
                          "dim_x = %d" % self.dim_x, "dim_z = %d" % self.dim_z, "dt = %s" % self.dt,
                          "N = %d" % self.N, "n_filters = %s" % (None if self._single else self.n_filters)]
                         + [show(k) for k in ("x", "P", "x_prior", "P_prior", "Q", "R", "K", "S", "sigmas")]
                         + ["hx = %r" % (self.hx,), "fx = %r" % (self.fx,)])
