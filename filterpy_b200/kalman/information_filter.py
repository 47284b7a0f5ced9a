"""Host-side mirror of ``filterpy.kalman.InformationFilter`` for a BANK of filters on one H100
(filterpy/kalman/information_filter.py: ``__init__`` :130-175, ``update`` :178-243, ``predict`` :245-289,
``F`` / ``P`` :365-379).

The filter carries the information matrix ``P_inv`` = P^-1 instead of P, so a filter can start from no
information at all (``P_inv = 0``), as a bank of tracks being initiated does: the reference then runs its
no-information branch, per filter, until the information suffices to invert.  All arithmetic runs in
``csrc/information.cu`` behind ``bke_if_step`` and ``bke_inverse`` (DESIGN.md §3.5e).

The same two modes as ``KalmanFilter``: ``n_filters=None`` is a drop-in for one reference object (NumPy
attributes with the reference's shapes, and its exceptions), ``n_filters=N`` a bank of device tensors with a
leading N axis, where a model given un-batched is shared by the bank.  In bank mode ``predict()`` is deferred and
runs fused with the next ``update`` in one launch; single mode runs it at once, so that its ``LinAlgError`` comes
from ``predict()`` as the reference's does.
"""
import math
import sys

import numpy as np
import torch

from .. import _lib
from .._dev import bke_dtype, ptr, stream_ptr, to_dev
from ._bank import _BankMirror, _Linked, _model_prop

__all__ = ["InformationFilter"]


def _is_zero_scalar(v):
    return np.isscalar(v) and v == 0


class InformationFilter(_BankMirror):
    """``InformationFilter(dim_x, dim_z, dim_u=0, compute_log_likelihood=True)`` for ``n_filters`` filters at once.

    Attributes as in the reference: ``x``, ``P_inv``, ``P`` (= inv(P_inv)), ``F``, ``Q``, ``H``, ``R_inv``, ``B``,
    ``K``, ``y``, ``S`` (n x n: P_inv + H' R_inv H), ``z``, ``x_prior``, ``P_inv_prior``, ``x_post``, ``P_inv_post``,
    ``log_likelihood``, ``likelihood``, ``inv`` (np.linalg.inv only) and ``_no_information`` (bool, bool[N] in bank
    mode).  Assigning ``F`` stores it and then its inverse, which ``predict`` uses; an in-place edit of ``F``
    (``f.F[0, 1] = dt``, or the live tensor in bank mode) does not refresh the inverse, as in the reference.

    Deviations, both in bank mode only or documented:
      - a scalar ``P_inv`` is stored as ``s * I`` (the reference keeps the scalar, which its update would broadcast
        to every entry); a scalar ``Q`` or ``R_inv`` likewise;
      - bank mode reports the step's ``LinAlgError`` per filter in ``status`` / ``check()``, and ``P`` is NaN for
        the filters whose ``P_inv`` is singular.  A filter whose step failed keeps what the reference has set at
        its raise (a failed predict gets no update, whether or not a getter ran the predict on its own first).
    """

    _FAILURE = "Singular matrix"

    def __init__(self, dim_x, dim_z, dim_u=0, compute_log_likelihood=True, n_filters=None, dtype=np.float64,
                 device=None, diagnostics=True):
        if dim_u < 0:
            raise ValueError('dim_u must be 0 or greater')          # information_filter.py:136-137
        self._init_bank(dim_x, dim_z, n_filters, dtype, device, diagnostics)
        self.dim_u = int(dim_u)
        self.compute_log_likelihood = compute_log_likelihood
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        kw = dict(dtype=self._dtype, device=self._device)
        self._x = torch.zeros(N, n, **kw)
        self._P_inv = torch.eye(n, **kw).repeat(N, 1, 1)
        self._Q = torch.eye(n, **kw)
        self._F = None                    # the reference's _F = 0.: predict() raises until F is assigned
        self._F_inv = None
        self._H = torch.zeros(m, n, **kw)
        self._R_inv = torch.eye(m, **kw)
        self._B = None
        self._ni = torch.zeros(N, dtype=torch.uint8, device=self._device)
        self._pending = None              # the u of a deferred predict (bank mode)
        self._sticky = False              # a predict ran on its own: the next update keeps its status
        self._z = torch.zeros(N, m, **kw)
        # always kept: single mode raises from it whether or not the diagnostics are kept
        self._status = torch.zeros(N, dtype=torch.int32, device=self._device)
        if self.diagnostics:
            self._x_prior = self._x.clone(); self._P_inv_prior = self._P_inv.clone()
            self._x_post = self._x.clone(); self._P_inv_post = self._P_inv.clone()
            self._K = torch.zeros(N, n, m, **kw); self._y = torch.zeros(N, m, **kw)
            self._S = torch.zeros(N, n, n, **kw)
            self._ll = torch.full((N,), math.log(sys.float_info.min), **kw)

    # ------------------------------------------------------------------ plumbing
    def _inverse(self, t, k):
        """np.linalg.inv of a (k,k) or (N,k,k) device tensor: (inverse, number of singular matrices, status)."""
        cnt = 1 if t.dim() == 2 else t.shape[0]
        Ai = torch.empty_like(t)
        st = torch.zeros(cnt, dtype=torch.int32, device=self._device)
        self._run(self._lib.bke_inverse, cnt, k, bke_dtype(self._dtype), ptr(t), self._stride(t), ptr(Ai), ptr(st),
                  stream_ptr(self._device))
        return Ai, st

    # ------------------------------------------------------------------ state
    @property
    def P_inv(self):
        self._flush()
        return self._P_inv if not self._single else _Linked(self._P_inv[0].cpu().numpy(), self, "P_inv")

    @P_inv.setter
    def P_inv(self, v):
        self._flush()
        n = self.dim_x
        if np.isscalar(v):
            v = np.eye(n) * v
        t = to_dev(v, self._dtype, self._device)
        if tuple(t.shape) == (n, n):
            t = t.expand(self.n_filters, n, n)
        if tuple(t.shape) != (self.n_filters, n, n):
            raise ValueError("P_inv must have shape (%d,%d) or (%d,%d,%d)" % (n, n, self.n_filters, n, n))
        self._P_inv = t.contiguous().clone()

    @property
    def P(self):
        """inv(P_inv) (information_filter.py:376-379): raises LinAlgError when it is singular (single mode); NaN
        for those filters in bank mode."""
        self._flush()
        Pt, st = self._inverse(self._P_inv, self.dim_x)
        bad = st != 0
        if self._single:
            if bool(bad[0].item()):
                raise np.linalg.LinAlgError("Singular matrix")
            return Pt[0].cpu().numpy()
        return torch.where(bad[:, None, None], torch.full_like(Pt, float("nan")), Pt)

    @P.setter
    def P(self, v):
        raise AttributeError("P is read-only: it is inv(P_inv); assign P_inv")

    @property
    def _no_information(self):
        self._flush()
        return bool(self._ni[0].item()) if self._single else self._ni.bool()

    @_no_information.setter
    def _no_information(self, v):
        self._flush()
        t = torch.as_tensor(v, device=self._device).to(torch.uint8)
        self._ni = t.expand(self.n_filters).contiguous().clone()

    # ------------------------------------------------------------------ models
    @property
    def F(self):
        """The state transition matrix, 0. (the reference's default) until one is assigned."""
        if self._F is None:
            return 0.
        if self._single:
            return _Linked(self._F.cpu().numpy(), self, "_F_in_place")
        self._flush()
        return self._F

    @F.setter
    def F(self, v):
        """_F = F, then _F_inv = inv(F) (information_filter.py:370-374): a singular F raises LinAlgError after F is
        stored, and the previous inverse stays."""
        self._flush()
        self._F = self._model(v, self.dim_x, self.dim_x, "F")
        Fi, st = self._inverse(self._F, self.dim_x)
        bad = int((st != 0).sum().item())
        if bad:
            cnt = st.shape[0]
            raise np.linalg.LinAlgError("Singular matrix" if self._single else
                                        "F: %d of %d matrices are singular" % (bad, cnt))
        self._F_inv = Fi

    @property
    def _F_in_place(self):
        return self.F

    @_F_in_place.setter
    def _F_in_place(self, v):
        """where single mode's write-back F arrays land: the reference edits _F in place, without a new _F_inv"""
        self._flush()
        self._F = self._model(v, self.dim_x, self.dim_x, "F")

    Q = _model_prop("Q", "dim_x", "dim_x")
    H = _model_prop("H", "dim_z", "dim_x")
    R_inv = _model_prop("R_inv", "dim_z", "dim_z")

    @property
    def inv(self):
        return np.linalg.inv

    @inv.setter
    def inv(self, v):
        if v is not np.linalg.inv:
            raise NotImplementedError("the GPU bank inverts with np.linalg.inv's rule only (bke_inverse)")

    # ------------------------------------------------------------------ predict / update
    def predict(self, u=0):
        """information_filter.py:245-289.  ``u`` is ``(dim_u,)``, one row per filter ``(N, dim_u)``, or 0.  Bank
        mode defers it to the next ``update``; single mode runs it now and raises where the reference does."""
        if self._F_inv is None:
            raise AttributeError("'float' object has no attribute 'T'")       # dot(self._F_inv.T, ...) with _F_inv = 0.
        self._flush()
        if self._single:
            self._launch(_lib.BKE_DO_PREDICT, u, None, None, None)
            self._raise_on_status()
        else:
            self._pending = u
            self._sticky = False          # a new step: its first launch writes status afresh

    def _flush(self):
        """Run the deferred predict on its own (a getter or setter needs the predicted state).  Its status stays
        for the update that completes the step, which then skips the filters whose predict failed, as the fused
        launch does."""
        if self._pending is not None:
            u, self._pending = self._pending, None
            self._launch(_lib.BKE_DO_PREDICT, u, None, None, None)
            self._sticky = True

    def _raise_on_status(self):
        if bool((self._status[0] != 0).item()):
            raise np.linalg.LinAlgError("Singular matrix")

    def update(self, z, R_inv=None, valid=None):
        """information_filter.py:178-243.  ``z`` is ``(N, dim_z)`` in bank mode; ``z=None`` changes nothing
        (:194-198); ``valid[N]`` (0 = no measurement) does so per filter.  A scalar ``R_inv`` means ``R_inv * I``.
        With ``compute_log_likelihood`` and dim_z neither 1 nor dim_x, scipy cannot broadcast y against the mean
        of S: the update raises ValueError after x and P_inv are updated, as the reference does, wherever a filter
        took the informed branch."""
        u, self._pending = self._pending, None
        sticky, self._sticky = self._sticky, False
        if z is None:
            if u is not None:
                self._launch(_lib.BKE_DO_PREDICT, u, None, None, None)
            self._z = None
            if self.diagnostics:
                self._x_post.copy_(self._x); self._P_inv_post.copy_(self._P_inv)
            return
        m, n = self.dim_z, self.dim_x
        Ri = self._R_inv if R_inv is None else self._model(R_inv, m, m, "R_inv")
        zt = self._z_rows(z)
        vt = self._valid_mask(valid)
        if sticky and not self._single:
            # the step's predict ran on its own: a filter whose predict failed gets no update, as in the fused
            # launch (the reference raised before its update)
            ok = self._status == 0
            vt = (ok if vt is None else (vt != 0) & ok).to(torch.uint8)
        ll_mode = _lib.BKE_IF_LL_NONE
        if self.compute_log_likelihood and self.diagnostics:
            ll_mode = _lib.BKE_IF_LL_FULL if m == n else (_lib.BKE_IF_LL_BROADCAST if m == 1 else _lib.BKE_IF_LL_NONE)
        flags = _lib.BKE_DO_UPDATE | (_lib.BKE_DO_PREDICT if u is not None else 0)
        if sticky and not self._single:
            flags |= _lib.BKE_STATUS_STICKY
        self._launch(flags, u, zt, vt, Ri, ll_mode)
        if self._single:
            self._raise_on_status()                          # inv(S) raises before z is stored (:225)
        self._z = zt.clone() if self._single else zt         # the informed branch stores z before its logpdf (:232)
        if self.compute_log_likelihood and m not in (1, n):
            informed = (self._ni == 0) & (self._status == 0)
            if vt is not None:
                informed &= vt != 0
            if bool(informed.any().item()):
                raise ValueError("operands could not be broadcast together with shapes (1,%d) (%d,)" % (m, n))
        if self.diagnostics:
            self._x_post.copy_(self._x); self._P_inv_post.copy_(self._P_inv)

    def _launch(self, flags, u, zt, vt, Ri, ll_mode=_lib.BKE_IF_LL_NONE):
        if (flags & _lib.BKE_DO_PREDICT) and self._F_inv is None:
            raise AttributeError("'float' object has no attribute 'T'")
        a = _lib.IfArgs()
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        a.n_filters, a.dim_x, a.dim_z = N, n, m
        a.dtype = bke_dtype(self._dtype)
        a.flags = flags
        a.ll_mode = ll_mode
        a.x = a.x_out = ptr(self._x)
        a.P_inv = a.P_inv_out = ptr(self._P_inv)
        a.no_information = ptr(self._ni)
        if flags & _lib.BKE_DO_PREDICT:
            a.F, a.F_stride = ptr(self._F), self._stride(self._F)
            a.F_inv, a.F_inv_stride = ptr(self._F_inv), self._stride(self._F_inv)
            a.Q, a.Q_stride = ptr(self._Q), self._stride(self._Q)
        a.H, a.H_stride = ptr(self._H), self._stride(self._H)
        if Ri is not None:
            a.R_inv, a.R_inv_stride = ptr(Ri), self._stride(Ri)
        ut = None                     # with B = 0 (None) dot(B, u) adds nothing (:274)
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
                a.x_prior, a.P_inv_prior = ptr(self._x_prior), ptr(self._P_inv_prior)
            if flags & _lib.BKE_DO_UPDATE:
                a.K, a.y, a.S, a.log_likelihood = ptr(self._K), ptr(self._y), ptr(self._S), ptr(self._ll)
        a.status = ptr(self._status)
        self._run(self._lib.bke_if_step, a, stream_ptr(self._device))

    def batch_filter(self, zs, Rs=None, update_first=False, saver=None):
        raise NotImplementedError("this is not implemented yet")                # information_filter.py:326

    # ------------------------------------------------------------------ diagnostics
    P_inv_prior = property(lambda self: self._out(self._diag("P_inv_prior")))
    P_inv_post = property(lambda self: self._out(self._diag("P_inv_post")))

    def _absent(name):  # noqa: N805
        def get(self):
            raise AttributeError("'InformationFilter' object has no attribute '%s'" % name)
        return property(get)

    P_prior = _absent("P_prior")
    P_post = _absent("P_post")
    SI = _absent("SI")
    mahalanobis = _absent("mahalanobis")
    del _absent

    @property
    def z(self):
        if self._z is None:
            return None                                                      # update(None) stores None (:195)
        return self._z if not self._single else self._z[0].cpu().numpy().reshape(-1, 1)
