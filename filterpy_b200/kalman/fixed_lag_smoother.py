"""Host-side mirror of ``filterpy.kalman.FixedLagSmoother`` for a BANK of filters on one H100
(filterpy/kalman/fixed_lag_smoother.py: ``__init__`` :85-131, ``smooth`` :133-215, ``smooth_batch`` :217-311,
``__repr__`` :313-330).

A fixed-lag smoother gives the smoothed estimate of epoch k once epoch k + N has been seen, while the bank keeps
stepping: the smoother a stream of tracks without an end needs (the RTS smoother waits for the last measurement).
All arithmetic runs in ``csrc/fls.cu`` behind ``bke_fls_smooth``.

The same two modes as ``KalmanFilter``: ``n_filters=None`` is a drop-in for one reference object (NumPy attributes
with the reference's shapes; ``xSmooth`` is a list of arrays shaped like ``x``), ``n_filters=N`` a bank of device
tensors with a leading N axis, where a model given un-batched is shared by the bank.  In bank mode the history is
a device tensor whose capacity doubles as it fills, and ``xSmooth`` is a ``[count, N, dim_x]`` view of it.
"""
import numpy as np
import torch

from .. import _lib
from .._dev import bke_dtype, ptr, stream_ptr, to_dev
from ._bank import _BankMirror, _model_prop

__all__ = ["FixedLagSmoother"]

_HISTORY_CAPACITY = 64          # rows of the first history buffer (bank mode); doubled when full


class FixedLagSmoother(_BankMirror):
    """``FixedLagSmoother(dim_x, dim_z, N=None)`` for ``n_filters`` filters at once.

    Attributes as in the reference: ``x``, ``P``, ``F``, ``Q``, ``H``, ``R``, ``B``, ``K``, ``y``, ``S``, ``x_s``,
    ``N``, ``count``, ``xSmooth``.  As in the reference, ``K`` and ``x_s`` keep their initial zeros (``smooth`` never
    writes them), and ``xSmooth`` only exists when ``N`` was given.

    A singular S makes the reference raise ``LinAlgError``.  Single mode raises it too (``y`` and ``S`` are set
    and nothing else changes, as in the reference).  In bank mode the kernel sets ``status`` to 1 for that filter,
    keeps it at its prior for the epoch and corrects no row (include/bke.h, ``bke_fls_args``); ``check()`` raises.
    ``batch_status`` is the status of the last bank-mode ``smooth_batch``.
    """

    def __init__(self, dim_x, dim_z, N=None, *, dim_u=0, n_filters=None, dtype=np.float64, device=None,
                 diagnostics=True):
        if dim_u < 0:
            raise ValueError('dim_u must be 0 or greater')
        if N is not None and int(N) < 0:
            raise ValueError('N must be 0 or greater')
        self._init_bank(dim_x, dim_z, n_filters, dtype, device, diagnostics)
        self.dim_u = int(dim_u)
        self.N = None if N is None else int(N)
        Nf, n, m = self.n_filters, self.dim_x, self.dim_z
        kw = dict(dtype=self._dtype, device=self._device)
        self._x = torch.zeros(Nf, n, **kw)                   # :113-123
        self._P = torch.eye(n, **kw).repeat(Nf, 1, 1)
        self._Q = torch.eye(n, **kw)
        self._F = torch.eye(n, **kw)
        self._H = torch.eye(m, n, **kw)
        self._R = torch.eye(m, **kw)
        self._B = None                                        # the reference's B = 0.
        self._y = torch.zeros(Nf, m, **kw)
        self._S = torch.zeros(Nf, m, m, **kw)
        self._y_set = False
        self._status = torch.zeros(Nf, dtype=torch.int32, device=self._device)
        self.batch_status = None
        self.count = 0
        self._hist = torch.empty(0 if self._single else _HISTORY_CAPACITY, Nf, n, **kw) if N is not None else None
        self._ws = None

    # ------------------------------------------------------------------ plumbing
    def _workspace(self, du, lag):
        nb = self._lib.bke_fls_workspace_bytes(self.n_filters, self.dim_x, self.dim_z, du, bke_dtype(self._dtype), lag)
        if nb == 0:
            return None, 0
        if self._ws is None or self._ws.numel() < nb:
            self._ws = torch.empty(nb, dtype=torch.uint8, device=self._device)    # the caching allocator aligns it
        return self._ws, nb

    def _zs(self, zs, T):
        """[T, N, m] device tensor from the caller's measurements (single mode: scalars, (m,) or (m,1) each)."""
        Nf, m = self.n_filters, self.dim_z
        if self._single:
            zs = np.asarray(zs, dtype=np.float64).reshape(T, 1, m)
        t = to_dev(zs, self._dtype, self._device)
        if t.dim() == 4 and t.shape[-1] == 1:
            t = t[..., 0]
        if t.dim() == 2 and m == 1 and tuple(t.shape) == (T, Nf):
            t = t.reshape(T, Nf, 1)
        if tuple(t.shape) != (T, Nf, m):
            raise ValueError("zs must have shape (%d,%d,%d), got %s" % (T, Nf, m, tuple(t.shape)))
        return t.contiguous()

    def _us(self, us, T):
        """[T, N, dim_u] device tensor, or None: with B = 0 the reference's dot(B, u) adds nothing (:175-176)."""
        if us is None or self._B is None:
            return None
        du = self._B.shape[-1]
        t = to_dev(np.asarray(us, dtype=np.float64) if not isinstance(us, torch.Tensor) else us, self._dtype, self._device)
        if t.dim() >= 1 and t.shape[-1] == 1 and du != 1:
            t = t[..., 0]
        if self._single:
            t = t.reshape(T, 1, du)
        elif t.dim() == 2 and tuple(t.shape) == (T, du):
            t = t.reshape(T, 1, du).expand(T, self.n_filters, du)
        if tuple(t.shape) != (T, self.n_filters, du):
            raise ValueError("us must have shape (%d,%d,%d), got %s" % (T, self.n_filters, du, tuple(t.shape)))
        return t.contiguous()

    def _launch(self, zt, ut, lag, count, xs, x_out, P_out, xhat, y, S, status):
        a = _lib.FlsArgs()
        k = a.step
        Nf, n, m = self.n_filters, self.dim_x, self.dim_z
        k.n_filters, k.dim_x, k.dim_z = Nf, n, m
        k.dtype = bke_dtype(self._dtype)
        k.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
        k.alpha_sq = 1.0
        k.x, k.P, k.x_out, k.P_out = ptr(self._x), ptr(self._P), ptr(x_out), ptr(P_out)
        k.F, k.F_stride = ptr(self._F), self._stride(self._F)
        k.H, k.H_stride = ptr(self._H), self._stride(self._H)
        k.Q, k.Q_stride = ptr(self._Q), self._stride(self._Q)
        k.R, k.R_stride = ptr(self._R), self._stride(self._R)
        du = 0
        if ut is not None:
            du = self._B.shape[-1]
            k.dim_u = du
            k.B, k.B_stride = ptr(self._B), self._stride(self._B)
            a.us = ptr(ut)
        k.y, k.S, k.status = ptr(y), ptr(S), ptr(status)
        a.n_steps, a.lag, a.count = zt.shape[0], lag, count
        a.zs, a.xs_smooth, a.xhat = ptr(zt), ptr(xs), ptr(xhat)
        ws, nb = self._workspace(du, lag)
        a.workspace, a.workspace_bytes = ptr(ws), nb
        self._run(self._lib.bke_fls_smooth, a, stream_ptr(self._device))

    # ------------------------------------------------------------------ state
    F = _model_prop("F", "dim_x", "dim_x")
    Q = _model_prop("Q", "dim_x", "dim_x")
    H = _model_prop("H", "dim_z", "dim_x")
    R = _model_prop("R", "dim_z", "dim_z")

    @property
    def K(self):
        """the reference's initial zeros((dim_x, 1)): smooth() never writes self.K (:186 binds a local)"""
        z = torch.zeros(self.n_filters, self.dim_x, 1, dtype=self._dtype, device=self._device)
        return self._out(z)

    @property
    def x_s(self):
        """the reference's initial zeros((dim_x, 1)): never written (:114)"""
        return self.K

    @property
    def y(self):
        t = self._diag("y")
        if not self._single:
            return t
        v = t[0].cpu().numpy()
        return v.reshape(-1, 1) if (self._x_col or not self._y_set) else v

    status = property(lambda self: self._status,
                      doc="int32[N]: 1 where the last smooth() call met a singular S (the reference raises LinAlgError)")

    @property
    def xSmooth(self):
        if self._hist is None:
            raise AttributeError("'FixedLagSmoother' object has no attribute 'xSmooth' (N was not given)")
        rows = self._hist[:self.count]
        if not self._single:
            return rows
        return [r.reshape(-1, 1) if self._x_col else r for r in rows[:, 0].cpu().numpy()]

    # ------------------------------------------------------------------ smoothing
    def _grow(self, need):
        cap = self._hist.shape[0]
        if need <= cap:
            return
        new = torch.empty(max(need, 2 * cap, _HISTORY_CAPACITY), self.n_filters, self.dim_x,
                          dtype=self._dtype, device=self._device)
        new[:self.count] = self._hist[:self.count]
        self._hist = new

    def smooth(self, z, u=None):
        """fixed_lag_smoother.py:133-215: one epoch for every filter.  ``z`` is ``(N, dim_z)`` in bank mode;
        ``u`` is ``(dim_u,)`` or ``(N, dim_u)`` and only counts when ``B`` is a matrix."""
        if self._hist is None:
            raise AttributeError("'FixedLagSmoother' object has no attribute 'xSmooth' (N was not given)")
        if z is None:
            raise TypeError("unsupported operand type(s) for -: 'NoneType' and 'float' (z is None: the reference "
                            "has no missing-measurement rule)")
        zt = self._zs([z] if self._single else to_dev(z, self._dtype, self._device).reshape(1, self.n_filters, -1), 1)
        ut = None
        if u is not None and self._B is not None:
            ut = self._us(np.asarray(u)[None] if not isinstance(u, torch.Tensor) else u[None], 1)
        self._grow(self.count + 1)
        if self._single:
            x_out, P_out = torch.empty_like(self._x), torch.empty_like(self._P)
        else:
            x_out, P_out = self._x, self._P
        y = self._y if self.diagnostics or self._single else None
        S = self._S if self.diagnostics or self._single else None
        self._launch(zt, ut, self.N, self.count, self._hist, x_out, P_out, None, y, S, self._status)
        self._y_set = True
        if self._single and int(self._status[0].item()) != 0:
            raise np.linalg.LinAlgError("Singular matrix")      # :184, after self.y and self.S were set
        self._x, self._P = x_out, P_out
        self.count += 1

    def smooth_batch(self, zs, N, us=None):
        """fixed_lag_smoother.py:217-311: ``(xSmooth, xhat)`` of T epochs from the current x and P, with lag ``N``
        (not ``self.N``).  Leaves x, P, count, y, S and the history alone.  Single mode returns NumPy shaped
        ``(T, dim_x)`` for a 1-D x and ``(T, dim_x, 1)`` for a column x; bank mode ``[T, N, dim_x]`` tensors."""
        if N is None:
            raise TypeError("'>=' not supported between instances of 'int' and 'NoneType' (smooth_batch needs N)")
        N = int(N)
        if N < 0:
            raise ValueError("N must be 0 or greater")
        T = len(zs)
        Nf, n = self.n_filters, self.dim_x
        kw = dict(dtype=self._dtype, device=self._device)
        xs, xhat = torch.empty(T, Nf, n, **kw), torch.empty(T, Nf, n, **kw)
        st = torch.zeros(Nf, dtype=torch.int32, device=self._device)
        if T and Nf:
            zt = self._zs(zs, T)
            ut = self._us(us, T)
            self._launch(zt, ut, N, 0, xs, torch.empty_like(self._x), torch.empty_like(self._P), xhat, None, None, st)
        if not self._single:
            self.batch_status = st
            return xs, xhat
        if T and int(st[0].item()) != 0:
            raise np.linalg.LinAlgError("Singular matrix")
        shape = (T, n, 1) if self._x_col else (T, n)
        return xs[:, 0].cpu().numpy().reshape(shape), xhat[:, 0].cpu().numpy().reshape(shape)

    def __repr__(self):
        rows = ['FixedLagSmoother object']
        for name in ("dim_x", "dim_z", "N", "x", "x_s", "P", "F", "Q", "R", "H", "K", "y", "S", "B"):
            try:
                v = getattr(self, name)
            except AttributeError:
                continue
            if isinstance(v, torch.Tensor):
                v = v.cpu().numpy()
            rows.append("%s = %s" % (name, np.array2string(np.asarray(v)) if not np.isscalar(v) and v is not None else v))
        return '\n'.join(rows)
