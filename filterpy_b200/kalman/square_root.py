"""Host-side mirror of ``filterpy.kalman.SquareRootKalmanFilter`` for a BANK of filters on one H100
(filterpy/kalman/square_root.py: ``__init__`` :127-169, ``update`` :172-224, ``predict`` :226-248, properties
:274-340).

The filter carries the lower-triangular factor L = P1_2 of P = L L' and propagates it by Householder QR
factorisations, so the factor spans half the orders of magnitude of P: an fp32 bank whose covariances span
many decades stays accurate where the fp32 Joseph form of ``KalmanFilter`` does not (DESIGN.md §3.5c).
All arithmetic runs in ``csrc/srkf.cu`` behind ``bke_srkf_step`` and ``bke_cholesky_lower``.

The same two modes as ``KalmanFilter``: ``n_filters=None`` is a drop-in for one reference object (NumPy
attributes with the reference's shapes, ``x`` is ``(dim_x, 1)``; ``kf.x[0] = v`` and ``kf.F[0, 1] = dt``
write back), ``n_filters=N`` a bank of device tensors with a leading N axis, where a model given un-batched
is shared by the bank.  ``predict()`` is deferred and runs fused with the next ``update`` in one launch.
"""
import numpy as np
import torch

from .. import _lib
from .._dev import bke_dtype, ptr, require_cuda, resolve_dtype, stream_ptr, to_dev
from .kalman_filter import _Linked

__all__ = ["SquareRootKalmanFilter"]


def _is_zero_scalar(v):
    return np.isscalar(v) and v == 0


class SquareRootKalmanFilter(object):
    """``SquareRootKalmanFilter(dim_x, dim_z, dim_u=0)`` for ``n_filters`` filters at once.

    Attributes as in the reference: ``x``, ``P``, ``P1_2``, ``Q``, ``Q1_2``, ``R``, ``R1_2``, ``F``, ``H``,
    ``B``, ``K``, ``y``, ``S``, ``SI``, ``S1_2``, ``SI1_2``, ``z``, ``x_prior``, ``P_prior``, ``x_post``,
    ``P_post``.  Assigning ``P``, ``Q`` or ``R`` stores its lower Cholesky factor and raises
    ``np.linalg.LinAlgError`` when a matrix is not positive definite, as the reference's setters do;
    ``P1_2``, ``Q1_2`` and ``R1_2`` are read-only.  ``P``, ``Q``, ``R``, ``S``, ``SI`` and ``P_prior`` are
    formed from the factors on access.

    ``P_post`` returns the PRIOR factor's product, ``P1_2_prior P1_2_prior'``: the reference's property
    reads ``_P1_2_prior`` (square_root.py:300-303), and the mirror keeps that.  The posterior covariance is
    ``P``.

    Where a zero diagonal entry of ``S1_2`` makes the reference fall back on ``pinv``, the kernel sets
    ``status`` to 1, K = 0 and keeps the prior (include/bke.h, ``bke_srkf_args``); for ``S1_2 = 0`` that is the
    reference's result.  Like the reference, the mirror does not raise there.
    """

    def __init__(self, dim_x, dim_z, dim_u=0, n_filters=None, dtype=np.float64, device=None, diagnostics=True):
        if dim_x < 1:
            raise ValueError('dim_x must be 1 or greater')          # square_root.py:128-133
        if dim_z < 1:
            raise ValueError('dim_z must be 1 or greater')
        if dim_u < 0:
            raise ValueError('dim_u must be 0 or greater')
        self.dim_x, self.dim_z, self.dim_u = int(dim_x), int(dim_z), int(dim_u)
        self._single = n_filters is None
        self.n_filters = 1 if self._single else int(n_filters)
        if self.n_filters < 0:
            raise ValueError('n_filters must be 0 or greater')
        self._dtype = resolve_dtype(dtype)
        self._device = require_cuda(device)
        self._lib = _lib.load()
        self.diagnostics = bool(diagnostics)
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        kw = dict(dtype=self._dtype, device=self._device)
        self._x = torch.zeros(N, n, **kw)
        self._L = torch.eye(n, **kw).repeat(N, 1, 1)
        self._Lq = torch.eye(n, **kw)
        self._Lr = torch.eye(m, **kw)
        self._F = torch.eye(n, **kw)
        self._H = torch.zeros(m, n, **kw)
        self._B = None                    # the reference's B = 0.
        self._x_col = True
        self._pending = None              # the u of a deferred predict
        self._z = None
        if self.diagnostics:
            self._x_prior = self._x.clone(); self._L_prior = self._L.clone()
            self._x_post = self._x.clone()
            self._K = torch.zeros(N, n, m, **kw); self._y = torch.zeros(N, m, **kw)
            self._S1_2 = torch.zeros(N, m, m, **kw); self._SI1_2 = torch.zeros(N, m, m, **kw)
            self._status = torch.zeros(N, dtype=torch.int32, device=self._device)

    # ------------------------------------------------------------------ plumbing
    def _model(self, a, rows, cols, name):
        """(rows,cols) -> shared; (N,rows,cols) -> per filter; a scalar -> scalar * I."""
        if np.isscalar(a):
            if rows != cols:
                raise ValueError("%s: a scalar needs a square matrix" % name)
            return torch.eye(rows, dtype=self._dtype, device=self._device) * float(a)
        t = to_dev(a, self._dtype, self._device)
        if tuple(t.shape) == (rows, cols) or tuple(t.shape) == (self.n_filters, rows, cols):
            return t.contiguous()
        raise ValueError("%s must have shape (%d,%d) or (%d,%d,%d), got %s"
                         % (name, rows, cols, self.n_filters, rows, cols, tuple(t.shape)))

    @staticmethod
    def _stride(t):
        return 0 if t.dim() == 2 else t.shape[1] * t.shape[2]

    def _out(self, t):
        return t if not self._single else t[0].cpu().numpy()

    def _vec_out(self, t):
        if not self._single:
            return t
        v = t[0].cpu().numpy()
        return v.reshape(-1, 1) if self._x_col else v

    def _cholesky(self, v, k, name):
        """scipy.linalg.cholesky(v, lower=True) of a (k,k) or (N,k,k) value on the device (square_root.py:288,
        :314, :330); raises LinAlgError when a matrix is not positive definite."""
        t = self._model(v, k, k, name)
        cnt = 1 if t.dim() == 2 else t.shape[0]
        L = torch.empty_like(t)
        st = torch.zeros(cnt, dtype=torch.int32, device=self._device)
        with torch.cuda.device(self._device):
            _lib.check(self._lib.bke_cholesky_lower(cnt, k, bke_dtype(self._dtype), ptr(t), self._stride(t), ptr(L),
                                                    ptr(st), stream_ptr(self._device)))
        bad = int((st != 0).sum().item())
        if bad:
            raise np.linalg.LinAlgError("%s: %d of %d matrices are not positive definite" % (name, bad, cnt))
        return L

    @staticmethod
    def _product(L):
        return torch.matmul(L, L.transpose(-1, -2))

    # ------------------------------------------------------------------ state
    @property
    def x(self):
        self._flush()
        if not self._single:
            return self._x
        v = self._x[0].cpu().numpy()
        return _Linked(v.reshape(-1, 1) if self._x_col else v, self, "x")

    @x.setter
    def x(self, v):
        self._flush()
        n = self.dim_x
        t = to_dev(v, self._dtype, self._device)
        if self._single:
            if tuple(t.shape) not in ((n, 1), (n,)):
                raise ValueError("x must have shape (%d,1) or (%d,), got %s" % (n, n, tuple(t.shape)))
            self._x_col = t.dim() == 2
            self._x = t.reshape(1, n).clone()
            return
        if tuple(t.shape) == (n,):
            t = t.expand(self.n_filters, n)
        if tuple(t.shape) != (self.n_filters, n):
            raise ValueError("x must have shape (%d,) or (%d,%d), got %s" % (n, self.n_filters, n, tuple(t.shape)))
        self._x = t.contiguous().clone()

    @property
    def P(self):
        """covariance matrix L L' (square_root.py:290-293)"""
        self._flush()
        return self._out(self._product(self._L))

    @P.setter
    def P(self, v):
        self._flush()
        n = self.dim_x
        if np.isscalar(v):
            v = np.eye(n) * v
        L = self._cholesky(v, n, "P")
        self._L = (L.expand(self.n_filters, n, n) if L.dim() == 2 else L).contiguous().clone()

    @property
    def P1_2(self):
        """the lower Cholesky factor of P (read-only)"""
        self._flush()
        return self._out(self._L)

    # ------------------------------------------------------------------ models
    def _factor_prop(name, dim_attr):  # noqa: N805
        def get(self):
            self._flush()
            t = getattr(self, "_L" + name.lower())
            return self._product(t) if not self._single else self._product(t).cpu().numpy()

        def set_(self, v):
            self._flush()
            setattr(self, "_L" + name.lower(), self._cholesky(v, getattr(self, dim_attr), name))
        return property(get, set_)

    Q = _factor_prop("Q", "dim_x")
    R = _factor_prop("R", "dim_z")
    del _factor_prop

    Q1_2 = property(lambda self: self._Lq if not self._single else self._Lq.cpu().numpy(),
                    doc="the lower Cholesky factor of Q (read-only)")
    R1_2 = property(lambda self: self._Lr if not self._single else self._Lr.cpu().numpy(),
                    doc="the lower Cholesky factor of R (read-only)")

    def _matrix_prop(name, rows_attr, cols_attr):  # noqa: N805
        priv = "_" + name

        def get(self):
            t = getattr(self, priv)
            if self._single:
                return _Linked(t.cpu().numpy(), self, name)
            self._flush()          # the caller may edit the live tensor: a deferred predict runs with the old one
            return t

        def set_(self, v):
            self._flush()
            setattr(self, priv, self._model(v, getattr(self, rows_attr), getattr(self, cols_attr), name))
        return property(get, set_)

    F = _matrix_prop("F", "dim_x", "dim_x")
    H = _matrix_prop("H", "dim_z", "dim_x")
    del _matrix_prop

    @property
    def B(self):
        if self._B is None:
            return 0.
        return _Linked(self._B.cpu().numpy(), self, "B") if self._single else self._B

    @B.setter
    def B(self, v):
        self._flush()
        if v is None or _is_zero_scalar(v):
            self._B = None
            return
        if np.isscalar(v):
            raise NotImplementedError("B must be a (dim_x, dim_u) matrix (or 0): a scalar B is not supported")
        shp = np.shape(v) if not isinstance(v, torch.Tensor) else tuple(v.shape)
        self._B = self._model(v, self.dim_x, int(shp[-1]), "B")

    # ------------------------------------------------------------------ predict / update
    def predict(self, u=0):
        """square_root.py:226-248 (deferred and fused with the next ``update``).  ``u`` is ``(dim_u,)``, one
        row per filter ``(N, dim_u)``, or 0."""
        self._flush()
        self._pending = u

    def _flush(self):
        if self._pending is not None:
            u, self._pending = self._pending, None
            self._launch(_lib.BKE_DO_PREDICT, u, None, None, None)

    def update(self, z, R2=None, valid=None):
        """square_root.py:172-224.  ``z`` is ``(N, dim_z)`` in bank mode; ``z=None`` changes nothing
        (:189-193); ``valid[N]`` (0 = no measurement) does so per filter.  ``R2`` is a square root of the
        measurement noise for this call: a scalar means ``R2 * I`` (:195-198)."""
        u, self._pending = self._pending, None
        if z is None:
            if u is not None:
                self._launch(_lib.BKE_DO_PREDICT, u, None, None, None)
            self._z = None
            if self.diagnostics:
                self._x_post.copy_(self._x)
            return
        m = self.dim_z
        Lr = self._Lr if R2 is None else self._model(R2, m, m, "R2")
        zt = to_dev(np.asarray(z, dtype=np.float64).reshape(1, -1) if self._single else z, self._dtype, self._device)
        if tuple(zt.shape) != (self.n_filters, m):
            raise ValueError("z must have shape (%d,%d), got %s" % (self.n_filters, m, tuple(zt.shape)))
        vt = None
        if valid is not None:
            vt = torch.as_tensor(valid, device=self._device).to(torch.uint8).contiguous()
            if tuple(vt.shape) != (self.n_filters,):
                raise ValueError("valid must have shape (%d,)" % self.n_filters)
        flags = _lib.BKE_DO_UPDATE | (_lib.BKE_DO_PREDICT if u is not None else 0)
        self._launch(flags, u, zt.contiguous(), vt, Lr)
        self._z = zt
        if self.diagnostics:
            self._x_post.copy_(self._x)

    def _launch(self, flags, u, zt, vt, Lr):
        a = _lib.SrkfArgs()
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        a.n_filters, a.dim_x, a.dim_z = N, n, m
        a.dtype = bke_dtype(self._dtype)
        a.flags = flags
        a.x = a.x_out = ptr(self._x)
        a.L = a.L_out = ptr(self._L)
        a.F, a.F_stride = ptr(self._F), self._stride(self._F)
        a.Lq, a.Lq_stride = ptr(self._Lq), self._stride(self._Lq)
        a.H, a.H_stride = ptr(self._H), self._stride(self._H)
        if Lr is not None:
            a.Lr, a.Lr_stride = ptr(Lr), self._stride(Lr)
        ut = None                     # with B = 0 (None) dot(B, u) adds nothing (:240)
        if (flags & _lib.BKE_DO_PREDICT) and self._B is not None and u is not None and not _is_zero_scalar(u):
            du = self._B.shape[-1]
            ut = to_dev(u, self._dtype, self._device)
            if ut.dim() == 2 and ut.shape[-1] == 1 and ut.shape[0] == du:      # a (dim_u, 1) column
                ut = ut.reshape(du)
            if tuple(ut.shape) not in ((du,), (N, du)):
                raise ValueError("u must have shape (%d,) or (%d,%d), got %s" % (du, N, du, tuple(ut.shape)))
            ut = ut.contiguous()
            a.dim_u = du
            a.B, a.B_stride = ptr(self._B), self._stride(self._B)
            a.u, a.u_stride = ptr(ut), (0 if ut.dim() == 1 else du)
        a.z, a.z_valid = ptr(zt), ptr(vt)
        if self.diagnostics:
            if flags & _lib.BKE_DO_PREDICT:
                a.x_prior, a.L_prior = ptr(self._x_prior), ptr(self._L_prior)
            if flags & _lib.BKE_DO_UPDATE:
                a.K, a.y, a.S1_2, a.SI1_2 = ptr(self._K), ptr(self._y), ptr(self._S1_2), ptr(self._SI1_2)
                a.status = ptr(self._status)
        with torch.cuda.device(self._device):
            _lib.check(self._lib.bke_srkf_step(a, stream_ptr(self._device)))

    # ------------------------------------------------------------------ diagnostics
    def _diag(self, name):
        if not self.diagnostics:
            raise AttributeError("%s is only kept when the filter is built with diagnostics=True" % name)
        self._flush()
        return getattr(self, "_" + name)

    x_prior = property(lambda self: self._vec_out(self._diag("x_prior")))
    x_post = property(lambda self: self._vec_out(self._diag("x_post")))
    P_prior = property(lambda self: self._out(self._product(self._diag("L_prior"))))
    P_post = property(lambda self: self._out(self._product(self._diag("L_prior"))),
                      doc="the PRIOR factor's product, as the reference's property returns (square_root.py:300-303)")
    K = property(lambda self: self._out(self._diag("K")))
    S1_2 = property(lambda self: self._out(self._diag("S1_2")))
    SI1_2 = property(lambda self: self._out(self._diag("SI1_2")))
    S = property(lambda self: self._out(self._product(self._diag("S1_2"))))
    SI = property(lambda self: self._out(torch.matmul(self._diag("SI1_2").transpose(-1, -2), self._SI1_2)))
    status = property(lambda self: self._diag("status"))

    @property
    def y(self):
        t = self._diag("y")
        return t if not self._single else t[0].cpu().numpy().reshape(-1, 1)

    @property
    def z(self):
        if self._z is None:
            return np.array([[None] * self.dim_z]).T
        return self._z if not self._single else self._z[0].cpu().numpy().reshape(-1, 1)

    # ------------------------------------------------------------------ not offered
    @property
    def M(self):
        raise AttributeError("M (the reference's QR work matrix, square_root.py:163) is never formed: the kernel "
                             "builds it in registers or shared memory")

    def residual_of(self, z):
        raise NotImplementedError("residual_of is not offered by the GPU bank; compute z - H x from F, H and x")

    def measurement_of_state(self, x):
        raise NotImplementedError("measurement_of_state is not offered by the GPU bank; compute H x from H and x")
