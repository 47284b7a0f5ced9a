"""What every filter mirror shares: the single / bank mode switch, the state and model attributes with their
NumPy write-back views, the diagnostic attributes and the conversion of the caller's inputs to device tensors.

A mirror derives from ``_BankMirror``, calls ``_init_bank`` and adds its argument struct, its launch and the
attributes only its reference has.  Single mode (``n_filters=None``) is a drop-in for one reference object:
attributes are NumPy arrays with the reference's shapes.  Bank mode (``n_filters=N``) hands out the live device
tensors with a leading N axis; a model given un-batched is shared by the bank.
"""
import math
import sys

import numpy as np
import torch

from .. import _lib
from .._dev import require_cuda, resolve_dtype, to_dev


class _Linked(np.ndarray):
    """What the single-mode attribute getters hand out: a host copy of a device array that WRITES
    BACK.  The reference's attributes are the live arrays, so the usual idioms ``kf.P[2, 2] = 100``,
    ``kf.x[0] = z``, ``kf.F[0, 1] = dt``, ``kf.P *= 10`` must reach the filter; here they re-assign
    the attribute (which uploads it).  Views derived from it (``kf.P[2]``) do not write back."""

    def __new__(cls, arr, owner, name):
        obj = np.array(arr, copy=True).view(cls)
        obj._owner, obj._name = owner, name
        return obj

    def __array_finalize__(self, obj):
        self._owner, self._name = None, None

    def _push(self):
        if self._owner is not None:
            setattr(self._owner, self._name, np.array(self, copy=True).view(np.ndarray))

    def __setitem__(self, key, value):
        np.ndarray.__setitem__(self, key, value)
        self._push()

    def _inplace(self, op, other):
        res = op(self.view(np.ndarray), other)
        np.ndarray.__setitem__(self, Ellipsis, res)
        self._push()
        return self

    def __iadd__(self, o): return self._inplace(np.add, o)
    def __isub__(self, o): return self._inplace(np.subtract, o)
    def __imul__(self, o): return self._inplace(np.multiply, o)
    def __itruediv__(self, o): return self._inplace(np.true_divide, o)


def _model_prop(name, rows_attr, cols_attr):
    """A model matrix attribute (F, Q, H, R): write-back NumPy in single mode, the live tensor in bank mode."""
    return property(lambda self: self._get_model(name),
                    lambda self, v: self._set_model(name, v, getattr(self, rows_attr), getattr(self, cols_attr)))


class _BankMirror(object):
    """The state ``_x[N, n]`` / ``_P[N, n, n]``, the models ``_F``, ``_Q``, ``_H``, ``_R``, ``_B`` and the
    diagnostics of a bank, and the attributes over them.

    A mirror whose ``predict`` is deferred overrides ``_flush`` to run it: every setter, and every getter that
    hands out a live tensor, flushes first, so ``predict(); kf.F = F2; update(z)`` predicts with the old F,
    as the reference (whose predict has already happened) does."""

    _COLUMN_X = True     # single mode takes x as (n, 1) as well as (n,); the sigma-point filters' x is 1-D
    _FAILURE = "Singular matrix"        # what a nonzero status means, for check()

    def _init_bank(self, dim_x, dim_z, n_filters, dtype, device, diagnostics):
        if dim_x < 1:
            raise ValueError('dim_x must be 1 or greater')      # kalman_filter.py:388-393
        if dim_z < 1:
            raise ValueError('dim_z must be 1 or greater')
        self.dim_x, self.dim_z = int(dim_x), int(dim_z)
        self._single = n_filters is None
        self.n_filters = 1 if self._single else int(n_filters)
        if self.n_filters < 0:
            raise ValueError('n_filters must be 0 or greater')
        self._dtype = resolve_dtype(dtype)
        self._device = require_cuda(device)
        self._lib = _lib.load()
        self.diagnostics = bool(diagnostics)
        self._x_col = self._COLUMN_X        # single mode: x is (n,1) like the reference default

    def _alloc_diagnostics(self):
        """The per-filter outputs of a step; ``_x`` and ``_P`` must already be set."""
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        kw = dict(dtype=self._dtype, device=self._device)
        self._x_prior = self._x.clone(); self._P_prior = self._P.clone()
        self._x_post = self._x.clone(); self._P_post = self._P.clone()
        self._K = torch.zeros(N, n, m, **kw)
        self._y = torch.zeros(N, m, **kw)
        self._S = torch.zeros(N, m, m, **kw)
        self._SI = torch.zeros(N, m, m, **kw)
        self._ll = torch.full((N,), math.log(sys.float_info.min), **kw)
        self._status = torch.zeros(N, dtype=torch.int32, device=self._device)

    # ------------------------------------------------------------------ hooks
    def _flush(self):
        """Run a deferred predict, if the mirror defers one."""

    def _state_rebound(self):
        """``_x`` or ``_P`` is about to be re-bound to a new tensor."""

    def _model_hook(self, name, assigned):
        """Model ``name`` was re-assigned (``assigned``) or its live tensor handed out for in-place edits."""

    # ------------------------------------------------------------------ helpers
    def _model(self, a, rows, cols, name):
        """(rows,cols) -> shared; (N,rows,cols) -> per filter; a scalar -> scalar * I.  Returns a device tensor."""
        if np.isscalar(a):
            if rows != cols:
                raise ValueError("%s: a scalar needs a square matrix" % name)
            return torch.eye(rows, dtype=self._dtype, device=self._device) * float(a)
        t = to_dev(a, self._dtype, self._device)
        if t.dim() == 2 and tuple(t.shape) == (rows, cols):
            return t
        if t.dim() == 3 and tuple(t.shape) == (self.n_filters, rows, cols):
            return t
        if t.dim() == 1 and rows == 1 and t.shape[0] == cols:
            return t.reshape(1, cols)
        raise ValueError("%s must have shape (%d,%d) or (%d,%d,%d), got %s"
                         % (name, rows, cols, self.n_filters, rows, cols, tuple(t.shape)))

    @staticmethod
    def _stride(t):
        return 0 if t.dim() == 2 else t.shape[1] * t.shape[2]

    def _out(self, t):
        """bank mode: the device tensor; single mode: NumPy with the bank axis dropped."""
        if not self._single:
            return t
        return t[0].cpu().numpy()

    def _vec_out(self, t):
        """x-like vectors follow the shape of x in single mode."""
        if not self._single:
            return t
        v = t[0].cpu().numpy()
        return v.reshape(-1, 1) if self._x_col else v

    def _run(self, fn, *args):
        """``fn(*args)`` (a C-ABI call returning a status) with the bank's device current."""
        if torch.cuda.current_device() == self._device.index:
            _lib.check(fn(*args))
        else:
            with torch.cuda.device(self._device):
                _lib.check(fn(*args))

    # ------------------------------------------------------------------ state
    @property
    def x(self):
        self._flush()
        return self._x if not self._single else _Linked(self._vec_out(self._x), self, "x")

    @x.setter
    def x(self, v):
        self._flush()
        N, n = self.n_filters, self.dim_x
        t = to_dev(v, self._dtype, self._device)
        if self._single:
            if self._COLUMN_X and tuple(t.shape) == (n, 1):
                self._x_col = True
            elif tuple(t.shape) == (n,):
                self._x_col = False
            else:
                raise ValueError("x must have shape %s(%d,), got %s"
                                 % ("(%d,1) or " % n if self._COLUMN_X else "", n, tuple(t.shape)))
        else:
            if t.dim() == 3 and t.shape[-1] == 1:
                t = t[..., 0]
            if tuple(t.shape) == (n,):
                t = t.expand(N, n)
            if tuple(t.shape) != (N, n):
                raise ValueError("x must have shape (%d,) or (%d,%d), got %s" % (n, N, n, tuple(t.shape)))
        self._state_rebound()
        self._x = t.reshape(N, n).contiguous().clone()

    @property
    def P(self):
        self._flush()
        return self._P if not self._single else _Linked(self._P[0].cpu().numpy(), self, "P")

    @P.setter
    def P(self, v):
        self._flush()
        n = self.dim_x
        if np.isscalar(v):
            v = np.eye(n) * v
        t = to_dev(v, self._dtype, self._device)
        if tuple(t.shape) == (n, n):
            t = t.expand(self.n_filters, n, n)
        if tuple(t.shape) != (self.n_filters, n, n):
            raise ValueError("P must have shape (%d,%d) or (%d,%d,%d)" % (n, n, self.n_filters, n, n))
        self._state_rebound()
        self._P = t.contiguous().clone()

    # ------------------------------------------------------------------ models
    def _get_model(self, name):
        t = getattr(self, "_" + name)
        if t is None:
            return None
        if self._single:
            return _Linked(t.cpu().numpy(), self, name)
        # the caller may edit the live tensor in place: a deferred predict must run with the model it was issued with
        self._flush()
        self._model_hook(name, False)
        return t

    def _set_model(self, name, v, rows, cols):
        self._flush()
        setattr(self, "_" + name, None if v is None else self._model(v, rows, cols, name))
        self._model_hook(name, True)

    @property
    def B(self):
        """The control matrix, 0. (the reference's default) while there is none."""
        B = self._get_model("B")
        return 0. if B is None else B

    @B.setter
    def B(self, v):
        if np.isscalar(v) and v == 0:
            v = None                                        # dot(0, u) adds nothing
        elif np.isscalar(v):
            raise NotImplementedError("B must be a (dim_x, dim_u) matrix (or 0): a scalar B is not supported")
        self._set_model("B", v, self.dim_x, None if v is None else int(np.shape(v)[-1]))

    # ------------------------------------------------------------------ diagnostics
    def _diag(self, name):
        if not self.diagnostics:
            raise AttributeError("%s is only kept when the filter is built with diagnostics=True" % name)
        self._flush()
        return getattr(self, "_" + name)

    x_prior = property(lambda self: self._vec_out(self._diag("x_prior")))
    P_prior = property(lambda self: self._out(self._diag("P_prior")))
    x_post = property(lambda self: self._vec_out(self._diag("x_post")))
    P_post = property(lambda self: self._out(self._diag("P_post")))
    K = property(lambda self: self._out(self._diag("K")))
    y = property(lambda self: self._vec_out(self._diag("y")))
    S = property(lambda self: self._out(self._diag("S")))
    SI = property(lambda self: self._out(self._diag("SI")))

    @property
    def status(self):
        """int32[N]: 0 ok, nonzero where the reference raises ``LinAlgError`` (see the kernel's args struct)."""
        return self._diag("status")

    def check(self):
        """Raise ``np.linalg.LinAlgError`` if any filter's last step failed (see ``status``)."""
        bad = int((self.status != 0).sum().item())
        if bad:
            raise np.linalg.LinAlgError("%s in %d of %d filters" % (self._FAILURE, bad, self.n_filters))

    @property
    def log_likelihood(self):
        """log-likelihood of the last measurement (kalman_filter.py:1203-1210)."""
        ll = self._diag("ll")
        return float(ll[0].item()) if self._single else ll

    @property
    def likelihood(self):
        """kalman_filter.py:1213-1223 (exp of the log-likelihood, floored at float min)."""
        lk = torch.exp(self._diag("ll")).clamp_min(sys.float_info.min)
        return float(lk[0].item()) if self._single else lk

    @property
    def mahalanobis(self):
        """sqrt(y' SI y) (kalman_filter.py:1226-1239)."""
        y, SI = self._diag("y"), self._diag("SI")
        d = torch.sqrt(torch.einsum("ni,nij,nj->n", y, SI, y))
        return float(d[0].item()) if self._single else d

    @property
    def z(self):
        if self._z is None:
            return np.array([[None] * self.dim_z]).T
        return self._vec_out(self._z)

    # ------------------------------------------------------------------ inputs
    def _z_rows(self, z):
        """``z`` as a contiguous ``[N, m]`` device tensor.  Single mode flattens what the caller gives (the
        references form ``z - h(x)`` without checking its shape); bank mode takes ``(N, m)`` or ``(N, m, 1)``."""
        N, m = self.n_filters, self.dim_z
        if self._single:
            z = np.asarray(z, dtype=np.float64).reshape(1, -1)
        elif (isinstance(z, torch.Tensor) and z.device == self._device and z.dtype == self._dtype
                and z.dim() == 2 and z.shape[0] == N and z.shape[1] == m and z.is_contiguous()):
            return z                                        # already where the kernel wants it
        zt = to_dev(z, self._dtype, self._device)
        if zt.dim() == 3 and zt.shape[-1] == 1:
            zt = zt[..., 0]
        if tuple(zt.shape) != (N, m):
            raise ValueError("z must have shape (%d,%d), got %s" % (N, m, tuple(zt.shape)))
        return zt.contiguous()

    def _valid_mask(self, valid):
        """``valid`` (bool[N], 0 = no measurement) as a uint8 device tensor, or None."""
        if valid is None:
            return None
        vt = torch.as_tensor(valid, device=self._device).to(torch.uint8).contiguous()
        if tuple(vt.shape) != (self.n_filters,):
            raise ValueError("valid must have shape (%d,)" % self.n_filters)
        return vt

    def _history(self, Xs, Ps):
        """Smoother input: ``(T, N, n)`` / ``(T, N, n, n)`` device tensors, and whether single-mode ``Xs`` were
        columns ``(T, n, 1)``."""
        N, n = self.n_filters, self.dim_x
        Xt = to_dev(Xs, self._dtype, self._device)
        Pt = to_dev(Ps, self._dtype, self._device)
        T = Xt.shape[0]
        col = False
        if self._single:
            col = Xt.dim() == 3 and Xt.shape[-1] == 1
            Xt = Xt.reshape(T, 1, n)
            Pt = Pt.reshape(T, 1, n, n)
        if tuple(Xt.shape) != (T, N, n) or tuple(Pt.shape) != (T, N, n, n):
            raise ValueError("Xs / Ps must have shapes (T,%d,%d) / (T,%d,%d,%d), got %s / %s"
                             % (N, n, N, n, n, tuple(Xt.shape), tuple(Pt.shape)))
        return Xt.contiguous(), Pt.contiguous(), col
