"""Host-side mirror of ``filterpy.kalman.UnscentedKalmanFilter`` for a BANK of filters on one H100
(filterpy/kalman/UKF.py: ``__init__`` :284-362, ``predict`` :364-411, ``update`` :413-491,
``batch_filter`` :524-632).

The reference calls Python ``fx(x, dt)`` / ``hx(x)`` per sigma point (UKF.py:521-522, 463-464); a
device kernel cannot call back into Python, so ``fx`` / ``hx`` name a device-side model from the
closed set of include/bke.h instead:

    fx = LinearFx(F)        x' = F x                    (F: (n,n) shared or (N,n,n))
    fx = ConstVelFx()       (p0,v0,p1,v1,...): p += dt v
    hx = LinearHx(H)        z = H x
    hx = RangeAzElHx()      n=6 (x,vx,y,vy,z,vz) -> (range, azimuth, elevation)
    hx = RangeBearingHx()   n=4 (x,vx,y,vy)      -> (range, bearing)

The mean / residual / state-add hooks (x_mean_fn, z_mean_fn, residual_x, residual_z, state_add,
UKF.py:97-140), with which the reference wraps angles and takes circular means, are accepted as
``DeviceFn`` source text and compiled into the kernels.  Passing a Python callable for any hook or
model, sqrt_fn, or a per-call UT / fx / hx raises NotImplementedError: there is no CPU fallback.  As for the linear filter, ``n_filters=None`` gives a single-filter drop-in whose
attributes are NumPy arrays (``x`` is 1-D, UKF.py:298).
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from .._dev import bke_dtype, ptr, stream_ptr, to_dev
from ..stats.stats import _candidates, _valid
from ._bank import _BankMirror, _model_prop
from .sigma_points import SimplexSigmaPoints

__all__ = ["UnscentedKalmanFilter", "LinearFx", "ConstVelFx", "LinearHx", "RangeAzElHx", "RangeBearingHx",
           "DeviceFx", "DeviceHx", "DeviceFn"]


class LinearFx(object):
    model = _lib.BKE_FX_LINEAR

    def __init__(self, F):
        self.F = F


class ConstVelFx(object):
    model = _lib.BKE_FX_CONST_VEL
    F = None


class LinearHx(object):
    model = _lib.BKE_HX_LINEAR

    def __init__(self, H):
        self.H = H


class RangeAzElHx(object):
    model = _lib.BKE_HX_RANGE_AZ_EL
    H = None


class RangeBearingHx(object):
    model = _lib.BKE_HX_RANGE_BEARING
    H = None


class _DeviceModel(object):
    """A process / measurement function given as CUDA C++ source text (the reference takes Python callables:
    UKF.py:284-288, called per sigma point at :521-522 / :463-464).  The text defines, for the element
    type ``real`` (float or double, whichever the filter uses; ``BKE_DIM_X`` / ``BKE_DIM_Z`` are defined)::

        __device__ void fx(const real *x, real *x_out, real dt, const real *args)      # DeviceFx
        __device__ void hx(const real *x, real *z_out, const real *args)               # DeviceHx

    ``arg_names`` are the keyword arguments of the reference's callable (``predict(**fx_args)`` /
    ``update(z, **hx_args)``), delivered to the function as ``args[0..]`` in that order; ``defaults`` gives
    their values until a call overrides them.  A value is a scalar (whole bank) or an array ``(N,)``
    (one per filter).  The text is compiled at run time into an instance of the same kernel the built-in
    models use (NVRTC, sm_90a; ``csrc/ukf_rtc.cu``)."""
    F = None
    H = None

    def __init__(self, source, arg_names=(), **defaults):
        self.source = str(source)
        self.arg_names = tuple(arg_names)
        unknown = set(defaults) - set(self.arg_names)
        if unknown:
            raise TypeError("defaults for unknown arguments: %s" % sorted(unknown))
        self.values = dict(defaults)

    def pack(self, overrides, n_filters, dtype, device):
        """args vector(s) for the kernel: (tensor or None, stride)."""
        unknown = set(overrides) - set(self.arg_names)
        if unknown:
            raise TypeError("unexpected keyword arguments %s (declared: %s)" % (sorted(unknown), list(self.arg_names)))
        self.values.update(overrides)
        if not self.arg_names:
            return None, 0
        missing = [k for k in self.arg_names if k not in self.values]
        if missing:
            raise TypeError("missing values for the model arguments %s" % missing)
        vals = [self.values[k] for k in self.arg_names]
        if all(np.ndim(v) == 0 and not isinstance(v, torch.Tensor) for v in vals):
            return torch.tensor([float(v) for v in vals], dtype=dtype, device=device), 0
        cols = []
        for k, v in zip(self.arg_names, vals):
            t = torch.as_tensor(v, device=device).to(dtype).reshape(-1)
            if t.numel() == 1:
                t = t.expand(n_filters)
            if t.numel() != n_filters:
                raise ValueError("argument %s must be a scalar or have one value per filter (%d)" % (k, n_filters))
            cols.append(t)
        return torch.stack(cols, dim=1).contiguous(), len(cols)


class DeviceFx(_DeviceModel):
    model = _lib.BKE_FX_USER


class DeviceHx(_DeviceModel):
    model = _lib.BKE_HX_USER


class DeviceFn(object):
    """One of the reference's hooks (UKF.py:97-140) as CUDA C++ source text.  The keyword it is passed as
    names the ``__device__`` function the text defines, for the element type ``real`` (n = ``BKE_DIM_X``,
    m = ``BKE_DIM_Z``, ``BKE_N_SIGMAS`` points)::

        __device__ void residual_x(const real *a, const real *b, real *out);        # out = a - b, n
        __device__ void residual_z(const real *a, const real *b, real *out);        # out = a - b, m
        __device__ void state_add(const real *a, const real *b, real *out);         # out = a + b, n
        __device__ void x_mean_fn(const real *sigmas, const real *Wm, real *out);   # sigmas [BKE_N_SIGMAS][n]
        __device__ void z_mean_fn(const real *sigmas, const real *Wm, real *out);   # sigmas [BKE_N_SIGMAS][m]

    One object may define several of them and be passed for each: its text is included once."""

    def __init__(self, source):
        self.source = str(source)


_HOOK_BITS = (("x_mean_fn", _lib.BKE_HOOK_X_MEAN), ("z_mean_fn", _lib.BKE_HOOK_Z_MEAN),
              ("residual_x", _lib.BKE_HOOK_RESIDUAL_X), ("residual_z", _lib.BKE_HOOK_RESIDUAL_Z),
              ("state_add", _lib.BKE_HOOK_STATE_ADD))


def _device_hooks(**given):
    """The ``BKE_HOOK_*`` mask of the hooks given as ``DeviceFn`` and their distinct objects in keyword order;
    a Python callable raises NotImplementedError."""
    mask, fns = 0, []
    for nm, bit in _HOOK_BITS:
        v = given.get(nm)
        if v is None:
            continue
        if not isinstance(v, DeviceFn):
            _no_hook(nm, v)
        mask |= bit
        if not any(v is f for f in fns):
            fns.append(v)
    return mask, tuple(fns)


_compiled_models = {}


def _compile_model(lib, dim_x, dim_z, dtype_id, fx, hx, entry="bke_ukf_model_compile", hooks=(0, ()), points=0):
    """One NVRTC build per (filter family, shape, dtype, hooks, point set, source); shared by every filter object
    that uses it.  ``entry`` names the family's compile call (bke_ukf_model_compile / bke_ckf_model_compile);
    ``hooks`` is what ``_device_hooks`` returns; ``points`` is 0 or BKE_UKF_SIMPLEX (UKF only)."""
    mask, fns = hooks
    src = "\n".join([m.source for m in (fx, hx) if isinstance(m, _DeviceModel)] + [f.source for f in fns])
    key = (entry, dim_x, dim_z, dtype_id, fx.model, hx.model, mask, points, src)
    h = _compiled_models.get(key)
    if h is None:
        out = ctypes.c_void_p()
        inc = _lib.kernel_include_dirs().encode()
        if points:
            rc = lib.bke_ukf_model_compile_points(dim_x, dim_z, dtype_id, fx.model, hx.model, mask, points, src.encode(), inc,
                                                  ctypes.byref(out))
        elif mask:
            rc = getattr(lib, entry + "_hooks")(dim_x, dim_z, dtype_id, fx.model, hx.model, mask, src.encode(), inc,
                                                 ctypes.byref(out))
        else:
            rc = getattr(lib, entry)(dim_x, dim_z, dtype_id, fx.model, hx.model, src.encode(), inc, ctypes.byref(out))
        _lib.check(rc)
        h = _compiled_models[key] = out
    return h


def _no_hook(name, v):
    if v is not None:
        raise NotImplementedError(
            "%s is a Python callable hook; the GPU path implements the reference defaults only and "
            "has no CPU fallback (see filterpy_b200/kalman/UKF.py)" % name)


def _require_device_models(fx, hx):
    if not hasattr(fx, "model") or not hasattr(hx, "model"):
        raise NotImplementedError(
            "fx / hx must be device-side models (LinearFx, ConstVelFx, LinearHx, RangeAzElHx, "
            "RangeBearingHx, or DeviceFx / DeviceHx around CUDA source text): Python callables cannot "
            "run inside the CUDA kernel and there is no CPU fallback")


class _SigmaPointBank(_BankMirror):
    """What the UKF and CKF mirrors share on top of ``_BankMirror``: the device-side fx / hx models (and a
    compiled user model), the reference's Q and R, the deferred predict (``_pending`` holds its dt) and the
    fields and launch of their argument structs."""
    _compile_model = staticmethod(_compile_model)
    _COLUMN_X = False                                   # x is 1-D (UKF.py:298)
    _FAILURE = "matrix not positive definite / singular"

    def _init_bank(self, dim_x, dim_z, fx, hx, n_filters, dtype, device, diagnostics, hooks=(0, ()), points=0):
        """The state, models, compiled user model (around DeviceFx / DeviceHx or ``hooks``, for the point set
        ``points``) and diagnostic buffers of a bank (the reference's __init__ defaults: x = 0, P = I, Q = I, R = I)."""
        _BankMirror._init_bank(self, dim_x, dim_z, n_filters, dtype, device, diagnostics)
        self.fx, self.hx = fx, hx
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        kw = dict(dtype=self._dtype, device=self._device)
        self._x = torch.zeros(N, n, **kw)
        self._P = torch.eye(n, **kw).repeat(N, 1, 1)
        self._Q = torch.eye(n, **kw)
        self._R = torch.eye(m, **kw)
        self._F = None if fx.F is None else self._model(fx.F, n, n, "F")
        self._H = None if hx.H is None else self._model(hx.H, m, n, "H")
        self._pending = None
        self._z = None
        self._user_model = None
        self._fx_args = self._hx_args = (None, 0)
        self._hooks = hooks[0]
        if isinstance(fx, _DeviceModel) or isinstance(hx, _DeviceModel) or self._hooks:
            with torch.cuda.device(self._device):
                self._user_model = self._compile_model(self._lib, n, m, bke_dtype(self._dtype), fx, hx, hooks=hooks, points=points)
            if isinstance(fx, _DeviceModel):
                self._fx_args = fx.pack({}, N, self._dtype, self._device) if all(k in fx.values for k in fx.arg_names) else (None, 0)
            if isinstance(hx, _DeviceModel):
                self._hx_args = hx.pack({}, N, self._dtype, self._device) if all(k in hx.values for k in hx.arg_names) else (None, 0)
        if self.diagnostics:
            self._alloc_diagnostics()

    _dim_x = property(lambda self: self.dim_x)          # the reference's names
    _dim_z = property(lambda self: self.dim_z)
    Q = _model_prop("Q", "dim_x", "dim_x")
    R = _model_prop("R", "dim_z", "dim_z")

    def _flush(self):
        if self._pending is not None:
            dt, self._pending = self._pending, None
            self._launch(_lib.BKE_DO_PREDICT, dt, None, None, None)

    def _skip_update(self, dt):
        """``update(None)``: run a pending predict, and the posterior is the prior."""
        if dt is not None:
            self._launch(_lib.BKE_DO_PREDICT, dt, None, None, None)
        self._z = None
        if self.diagnostics:
            self._x_post.copy_(self._x); self._P_post.copy_(self._P)

    def _fill(self, a, flags, dt, zt, vt, R):
        """The fields the UKF and CKF argument structs share."""
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        a.n_filters, a.dim_x, a.dim_z = N, n, m
        a.dtype = bke_dtype(self._dtype)
        a.flags = flags
        a.fx_model, a.hx_model = self.fx.model, self.hx.model
        a.dt = float(dt)
        a.x = a.x_out = ptr(self._x)
        a.P = a.P_out = ptr(self._P)
        a.Q, a.Q_stride = ptr(self._Q), self._stride(self._Q)
        Rm = self._R if R is None else self._model(R, m, m, "R")          # scalar R -> R*I (UKF.py:456-457)
        a.R, a.R_stride = ptr(Rm), self._stride(Rm)
        if self._F is not None:
            a.F, a.F_stride = ptr(self._F), self._stride(self._F)
        if self._H is not None:
            a.H, a.H_stride = ptr(self._H), self._stride(self._H)
        a.z, a.z_valid = ptr(zt), ptr(vt)
        if self.diagnostics:
            if flags & _lib.BKE_DO_PREDICT:
                a.x_prior, a.P_prior = ptr(self._x_prior), ptr(self._P_prior)
            if flags & _lib.BKE_DO_UPDATE:
                a.K, a.y, a.S, a.SI = ptr(self._K), ptr(self._y), ptr(self._S), ptr(self._SI)
                a.log_likelihood = ptr(self._ll)
            a.status = ptr(self._status)
        return a

    def _step(self, a, step, step_model):
        """Launch a filled struct on the built-in models (``step``) or the compiled user model (``step_model``)."""
        if self._user_model is None:
            self._run(step, a, stream_ptr(self._device))
        else:
            for nm, mdl, (t, _) in (("fx", self.fx, self._fx_args), ("hx", self.hx, self._hx_args)):
                if isinstance(mdl, _DeviceModel) and mdl.arg_names and t is None:
                    raise TypeError("%s needs values for its arguments %s" % (nm, list(mdl.arg_names)))
            self._run(step_model, a, self._user_model, ptr(self._fx_args[0]), self._fx_args[1],
                      ptr(self._hx_args[0]), self._hx_args[1], stream_ptr(self._device))
        if self.diagnostics and (a.flags & _lib.BKE_DO_UPDATE):
            self._x_post.copy_(self._x); self._P_post.copy_(self._P)
        if self.diagnostics and self._single:
            self.check()


class UnscentedKalmanFilter(_SigmaPointBank):
    def __init__(self, dim_x, dim_z, dt, hx, fx, points, sqrt_fn=None, x_mean_fn=None, z_mean_fn=None,
                 residual_x=None, residual_z=None, state_add=None,
                 n_filters=None, dtype=np.float64, device=None, diagnostics=True):
        _no_hook("sqrt_fn", sqrt_fn)
        hooks = _device_hooks(x_mean_fn=x_mean_fn, z_mean_fn=z_mean_fn, residual_x=residual_x,
                              residual_z=residual_z, state_add=state_add)
        _require_device_models(fx, hx)
        if points.n != dim_x:
            raise ValueError("expected size(x) {}, but size is {}".format(points.n, dim_x))   # sigma_points.py:153
        # the point set selects the kernel instances: SimplexSigmaPoints runs the simplex ones (n + 1 points)
        self._point_flag = _lib.BKE_UKF_SIMPLEX if isinstance(points, SimplexSigmaPoints) else 0
        self._init_bank(dim_x, dim_z, fx, hx, n_filters, dtype, device, diagnostics, hooks, self._point_flag)
        self.points_fn = points
        self._dt = dt
        self._num_sigmas = points.num_sigmas()
        self.Wm, self.Wc = points.Wm, points.Wc

    # ------------------------------------------------------------------ predict / update
    def predict(self, dt=None, UT=None, fx=None, **fx_args):
        """UKF.py:364-411 (deferred and fused with the next ``update``)."""
        _no_hook("UT", UT); _no_hook("fx", fx)
        if fx_args:
            if not isinstance(self.fx, _DeviceModel):
                raise NotImplementedError("fx_args are arguments of a Python callback; the built-in process models take none")
        self._flush()
        if fx_args:
            self._fx_args = self.fx.pack(fx_args, self.n_filters, self._dtype, self._device)
        self._pending = self._dt if dt is None else dt

    def update(self, z, R=None, UT=None, hx=None, valid=None, **hx_args):
        """UKF.py:413-491.  ``z`` is ``(N, dim_z)`` in bank mode; ``z=None`` skips the update.

        Difference from the reference: an ``update`` WITHOUT a preceding ``predict`` draws its sigma
        points from the current (x, P) — what ``predict`` leaves behind (UKF.py:407) — whereas the
        reference would silently reuse the stale ``self.sigmas_f`` of the last predict (zeros on a
        fresh object).  After ``predict(); update(z)`` the two agree."""
        _no_hook("UT", UT); _no_hook("hx", hx)
        if hx_args:
            if not isinstance(self.hx, _DeviceModel):
                raise NotImplementedError("hx_args are arguments of a Python callback; the built-in measurement models take none")
            self._hx_args = self.hx.pack(hx_args, self.n_filters, self._dtype, self._device)
        dt, self._pending = self._pending, None
        if z is None:                                            # UKF.py:442-446
            self._skip_update(dt)
            return
        zt = self._z_rows(z)
        vt = self._valid_mask(valid)
        flags = _lib.BKE_DO_UPDATE | (_lib.BKE_DO_PREDICT if dt is not None else 0)
        self._launch(flags, self._dt if dt is None else dt, zt, vt, R)
        self._z = zt

    def _launch(self, flags, dt, zt, vt, R):
        a = self._fill(_lib.UkfArgs(), flags | self._point_flag, dt, zt, vt, R)
        if not self._point_flag:
            a.alpha, a.beta, a.kappa = self.points_fn.alpha, self.points_fn.beta, self.points_fn.kappa
        self._step(a, self._lib.bke_ukf_step, self._lib.bke_ukf_step_model)

    # ------------------------------------------------------------------ scores without a step
    def score_measurements(self, z, valid=None, **hx_args):
        """Gate candidates against the bank: for every track and candidate, the ``log_likelihood`` and
        ``mahalanobis`` the reference reports right after ``update(z)`` from the track's current state
        (UKF.py:459-477, 742-777), computed without updating: the sigma points of (x, P), hx, the unscented
        transform with R (and z_mean_fn / residual_z when given), then the scores of each candidate.  A pending
        ``predict`` is committed first, so the scores are against the prior the next ``update`` uses; x, P and
        the diagnostics are otherwise left exactly as they were.

        Bank mode: ``z`` is ``[N, m]`` (results ``[N]``), ``[N, K, m]`` or ``[1, K, m]`` (one scan for the whole
        bank; results ``[N, K]``); ``valid`` (bool, one per pair) marks missing candidates, which score
        log(DBL_MIN) and distance 0.  Returns device tensors ``(log_likelihood, mahalanobis)`` from one launch;
        a track whose P is not positive definite or whose S is singular scores NaN.  Single mode: ``z`` holds
        ``m`` values and the result is two floats; those failures raise ``LinAlgError``.  ``hx_args`` are the
        DeviceHx arguments for this call only."""
        self._flush()
        N, m = self.n_filters, self.dim_z
        if self._single:
            zt, sq = to_dev(np.asarray(z, dtype=np.float64).reshape(1, 1, -1), self._dtype, self._device), True
            if zt.shape[-1] != m:
                raise ValueError("z must hold %d values, got %d" % (m, zt.shape[-1]))
        else:
            zt, sq = _candidates(z, N, m, self._dtype, self._device)
        K = zt.shape[1]
        vt = _valid(valid, N, K, self._device)
        hx_t, hx_stride = self._hx_args
        if hx_args:
            if not isinstance(self.hx, _DeviceModel):
                raise NotImplementedError("hx_args are arguments of a Python callback; the built-in measurement models take none")
            kept = dict(self.hx.values)
            try:
                hx_t, hx_stride = self.hx.pack(hx_args, N, self._dtype, self._device)
            finally:
                self.hx.values = kept
        if isinstance(self.hx, _DeviceModel) and self.hx.arg_names and hx_t is None:
            raise TypeError("hx needs values for its arguments %s" % list(self.hx.arg_names))
        kw = dict(dtype=self._dtype, device=self._device)
        ll, maha = torch.empty(N, K, **kw), torch.empty(N, K, **kw)
        status = torch.empty(N, dtype=torch.int32, device=self._device)
        a = _lib.UkfScoreArgs()
        a.n_filters, a.n_candidates, a.dim_x, a.dim_z = N, K, self.dim_x, m
        a.dtype, a.flags, a.hx_model = bke_dtype(self._dtype), self._point_flag, self.hx.model
        if not self._point_flag:
            a.alpha, a.beta, a.kappa = self.points_fn.alpha, self.points_fn.beta, self.points_fn.kappa
        a.x, a.P = ptr(self._x), ptr(self._P)
        a.R, a.R_stride = ptr(self._R), self._stride(self._R)
        if self._H is not None:
            a.H, a.H_stride = ptr(self._H), self._stride(self._H)
        a.z, a.z_track_stride, a.z_cand_stride = ptr(zt), (0 if zt.shape[0] == 1 else K * m), m
        a.z_valid = ptr(vt)
        a.log_likelihood, a.mahalanobis, a.status = ptr(ll), ptr(maha), ptr(status)
        if K > 0:
            if self._user_model is None:
                self._run(self._lib.bke_ukf_score, ctypes.byref(a), stream_ptr(self._device))
            else:
                self._run(self._lib.bke_ukf_score_model, ctypes.byref(a), self._user_model, ptr(hx_t), hx_stride,
                          stream_ptr(self._device))
        if self._single:
            if int(status[0].item()) != 0:
                raise np.linalg.LinAlgError(self._FAILURE)
            return float(ll[0, 0].item()), float(maha[0, 0].item())
        return (ll[:, 0], maha[:, 0]) if sq else (ll, maha)

    def rts_smoother(self, Xs, Ps, Qs=None, dts=None, UT=None):
        """UKF.py:634-739 on the GPU.  Bank mode: ``Xs[T,N,n]``, ``Ps[T,N,n,n]`` (what
        ``batch_filter`` returns) -> ``(xs, Ps, Ks)`` tensors; single mode NumPy ``(T,n)`` /
        ``(T,n,n)``.  ``dts``: None (the filter's dt), a scalar, or one value per epoch.  ``Qs`` is
        accepted and, exactly like the reference (:715 uses ``self.Q``), not used."""
        _no_hook("UT", UT)
        if len(Xs) != len(Ps):
            raise ValueError('Xs and Ps must have the same length')
        self._flush()
        N, n = self.n_filters, self.dim_x
        is_np = not isinstance(Xs, torch.Tensor)
        Xt, Pt, _ = self._history(Xs, Ps)
        T = Xt.shape[0]
        kw = dict(dtype=self._dtype, device=self._device)
        xs = torch.empty(T, N, n, **kw); Pso = torch.empty(T, N, n, n, **kw); Ks = torch.empty(T, N, n, n, **kw)
        status = torch.zeros(N, dtype=torch.int32, device=self._device)
        a = _lib.UkfRtsArgs()
        a.n_filters, a.n_steps, a.dim_x, a.dtype = N, T, n, bke_dtype(self._dtype)
        a.fx_model = self.fx.model
        a.flags = self._point_flag
        if not self._point_flag:
            a.alpha, a.beta, a.kappa = self.points_fn.alpha, self.points_fn.beta, self.points_fn.kappa
        a.dt = float(self._dt)
        dts_t = None
        if dts is not None:
            if np.isscalar(dts):
                a.dt = float(dts)
            else:
                d = np.asarray(dts, dtype=np.float64).reshape(-1)
                if d.shape[0] != T:
                    raise ValueError("dts must have one entry per epoch (%d)" % T)
                dts_t = torch.from_numpy(np.ascontiguousarray(d)).to(self._device)
                a.dts = ptr(dts_t)
        a.Xs, a.Ps = ptr(Xt), ptr(Pt)
        a.Q, a.Q_stride = ptr(self._Q), self._stride(self._Q)
        if self._F is not None:
            a.F, a.F_stride = ptr(self._F), self._stride(self._F)
        a.x_out, a.P_out, a.K = ptr(xs), ptr(Pso), ptr(Ks)
        a.status = ptr(status)
        if isinstance(self.fx, _DeviceModel) or self._hooks:
            # the reference calls self.fx(sigma, dt) without keyword arguments here (UKF.py:712): the model's
            # current argument values stand in for the defaults of its callable
            if isinstance(self.fx, _DeviceModel) and self.fx.arg_names and self._fx_args[0] is None:
                raise TypeError("fx needs values for its arguments %s" % list(self.fx.arg_names))
            self._run(self._lib.bke_ukf_rts_smoother_model, ctypes.byref(a), self._user_model, ptr(self._fx_args[0]),
                      self._fx_args[1], stream_ptr(self._device))
        else:
            self._run(self._lib.bke_ukf_rts_smoother, ctypes.byref(a), stream_ptr(self._device))
        if not self._single:
            return xs, Pso, Ks
        if int(status[0].item()) != 0:
            raise np.linalg.LinAlgError("matrix not positive definite / singular")
        out = (xs[:, 0], Pso[:, 0], Ks[:, 0])
        return tuple(o.cpu().numpy() for o in out) if is_np else out

    def batch_filter(self, zs, Rs=None, dts=None, UT=None, saver=None, valid=None):
        """UKF.py:524-632: predict/update over the epochs of ``zs`` (bank: ``zs[T,N,m]``), one fused
        launch per epoch.  Returns ``(means, covariances)``."""
        _no_hook("UT", UT)
        try:
            z0 = zs[0]
        except TypeError:
            raise TypeError('zs must be list-like')                       # UKF.py:593-596
        m = self.dim_z
        if self._single:
            if m == 1:
                if not (np.isscalar(z0) or (np.ndim(z0) == 1 and len(z0) == 1)):
                    raise TypeError('zs must be a list of scalars or 1D, 1 element arrays')
            elif z0 is not None and len(z0) != m:
                raise TypeError('each element in zs must be a 1D array of length {}'.format(m))
        T = len(zs)
        N, n = self.n_filters, self.dim_x
        kw = dict(dtype=self._dtype, device=self._device)
        means = torch.empty(T, N, n, **kw); covs = torch.empty(T, N, n, n, **kw)
        for i in range(T):
            self.predict(dt=None if dts is None else dts[i])
            z = zs[i]
            v = None if valid is None else valid[i]
            self.update(z, None if Rs is None else Rs[i], valid=v)
            means[i].copy_(self._x); covs[i].copy_(self._P)
            if saver is not None:
                saver.save()
        if not self._single:
            return means, covs
        return means[:, 0].cpu().numpy(), covs[:, 0].cpu().numpy()
