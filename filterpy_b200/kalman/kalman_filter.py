"""Host-side mirror of ``filterpy.kalman.KalmanFilter`` for a BANK of filters on one H100.

Same names, argument meaning and error behaviour as the reference
(``filterpy/kalman/kalman_filter.py``: ``__init__`` :387-434, ``predict`` :437-482, ``update``
:485-561, ``update_correlated`` :670-752, ``update_sequential`` :754-824, ``batch_filter`` :826-993, ``rts_smoother`` :995-1074,
``residual_of`` / ``measurement_of_state`` / ``log_likelihood_of`` :1175-1201, 1252-1260; procedural ``predict`` :1571,
``update`` :1401, ``batch_filter`` :1664, ``rts_smoother`` :1792), with one addition: a leading ``n_filters`` axis.  All arithmetic runs in
the hand-written CUDA kernels behind the C-ABI (``include/bke.h``); this file only validates
shapes, owns the device tensors and fills the argument structs.  There is no CPU fallback.

Two modes:

* ``KalmanFilter(dim_x, dim_z)``  — *single* mode, a drop-in for one reference object:
  attributes come back as NumPy arrays with the reference's shapes (``x`` is ``(dim_x, 1)``
  by default, kalman_filter.py:399), the bank has one filter.
* ``KalmanFilter(dim_x, dim_z, n_filters=N)`` — *bank* mode: attributes are device tensors with a
  leading N axis, ``x[N,n]  P[N,n,n]  z[N,m]``; a model matrix may be given un-batched
  (``(n,n)``) = shared by the bank.

``predict()`` followed by ``update(z)`` is fused into ONE kernel launch (the predict is deferred
until the next ``update`` or until somebody looks at the state).
"""
import ctypes
import math

import numpy as np
import torch

from .. import _lib
from .._dev import StepGraph, bke_dtype, ptr, require_cuda, resolve_dtype, stream_ptr, to_dev
from ..common.helpers import reshape_z
from ..stats.stats import LOG_DBL_MIN, _candidates, _valid, score as _score
from ._bank import _BankMirror, _model_prop

__all__ = ["KalmanFilter", "predict", "update", "batch_filter", "rts_smoother"]


class KalmanFilter(_BankMirror):
    def __init__(self, dim_x, dim_z, dim_u=0, n_filters=None, dtype=np.float64, device=None,
                 diagnostics=True):
        if dim_u < 0:
            raise ValueError('dim_u must be 0 or greater')
        self._init_bank(dim_x, dim_z, n_filters, dtype, device, diagnostics)
        self.dim_u = int(dim_u)
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        kw = dict(dtype=self._dtype, device=self._device)
        self._x = torch.zeros(N, n, **kw)
        self._P = torch.eye(n, **kw).repeat(N, 1, 1)
        self._Q = torch.eye(n, **kw)
        self._F = torch.eye(n, **kw)
        self._H = torch.zeros(m, n, **kw)
        self._R = torch.eye(m, **kw)
        self._M = torch.zeros(n, m, **kw)   # process-measurement cross-correlation (:407), read by update_correlated
        self._zrec = None                   # update_sequential's z record [N, m] (the blocks it has seen)
        self._B = None
        self._alpha_sq = 1.0
        self._pending = None          # deferred predict: dict(u,B,F,Q)
        self._z = None
        self.inv = np.linalg.inv      # kept for API parity; only the default is supported
        if self.diagnostics:
            self._alloc_diagnostics()
        self._host = {k: np.ascontiguousarray(getattr(self, "_" + k).cpu().numpy()) for k in "FQHR"}
        self._has_update = False
        self._post_alias = False      # True: x_post / P_post are the live x / P (nothing has moved them since the update)
        self._version = 0            # bumped whenever a tensor the kernels read is re-bound
        self._args_cache = {}
        # Every other launch that steps x, P walks the bank's tiles last to first (BKE_REVERSE_TILES): it
        # starts on the filters the previous launch finished, while their state and models are still in L2.
        self._reverse = False
        # Packed copy of the per-filter model words that differ between filters (bke_kf_scan_models,
        # bke_kf_pack_models): derived data, valid for one state of F, Q, H and R.  _model_version counts
        # re-bindings of F / Q / H / R and hand-outs of the live tensors; together with the tensors' own
        # version counters it names that state (the token of _sym_record).
        self._sym_ok = not self._single and N > 0 and (n, m) == (4, 2) and self._dtype == torch.float32
        self._sym_buf = None          # the current record, re-packed in place until a captured graph reads it
        self._sym_pinned = False      # True: a captured graph reads _sym_buf, so it is never written again
        self._sym_held = []           # earlier records captured graphs read (kept for the bank's lifetime)
        self._sym_map = None          # bke_kf_model_map on the device, filled by the scan
        self._sym_host_map = None     # the host copy of the map _sym_buf was packed with (launch parameters)
        self._sym_state = None        # (token, usable) of _sym_buf's pack
        self._model_version = 0
        self._model_last = None       # the token of the previous launch
        self._ring_notes = None       # capture(): what each launch of the capture pass was (see _fuse_ring)
        self._tile_order = None       # the fused rings' tile-order word {epoch, arrived} (device, see _fuse_ring)

    # ------------------------------------------------------------------ hooks of _BankMirror
    def _state_rebound(self):
        self._snapshot_post()
        self._version += 1

    def _model_hook(self, name, assigned):
        # a new or handed-out model invalidates the cached argument structs that carry its host copy, and
        # (F, Q, H, R) the packed model words.  M is in neither: update_correlated fills its struct every call.
        if name == "M":
            return
        if self._host.pop(name, None) is not None or assigned:
            self._version += 1
        if name in ("F", "Q", "H", "R"):
            self._model_version += 1
            t = getattr(self, "_" + name)
            if assigned and t is not None and t.dim() == 2:
                # host copy of a model shared by the bank: lets the kernels carry it in their launch
                # parameters (bke_kf_args.*_host)
                self._host[name] = np.ascontiguousarray(t.cpu().numpy())

    # ------------------------------------------------------------------ state attributes
    def _adopt_state(self, x_t, P_t):
        """Re-bind the state to caller-owned device tensors (no copy) and hand back a spare pair, so
        that a caller (IMMEstimator's mixing step) can double-buffer.  When x_post / P_post are
        still the live state, the outgoing buffers BECOME the stored posterior and the previous
        posterior buffers are the spare pair: a rotation instead of a copy."""
        self._flush()
        if self.diagnostics and self._post_alias:
            spare = (self._x_post, self._P_post)
            self._x_post, self._P_post = self._x, self._P
            self._post_alias = False
        else:
            spare = (self._x, self._P)
        self._x, self._P = x_t, P_t
        self._version += 1
        return spare

    F = _model_prop("F", "dim_x", "dim_x")
    Q = _model_prop("Q", "dim_x", "dim_x")
    H = _model_prop("H", "dim_z", "dim_x")
    R = _model_prop("R", "dim_z", "dim_z")
    M = _model_prop("M", "dim_x", "dim_z")

    @property
    def B(self):
        return self._get_model("B")

    @B.setter
    def B(self, v):
        cols = self.dim_u
        if cols == 0 and v is not None and not np.isscalar(v):
            cols = int(np.shape(v)[-1]) if np.ndim(v) >= 1 else 1     # the reference never checks B against dim_u
            if np.ndim(v) == 1:
                v = np.asarray(v).reshape(-1, 1); cols = 1
        self._set_model("B", v, self.dim_x, cols)

    @property
    def alpha(self):
        """Fading-memory setting (kalman_filter.py:1242-1266)."""
        return self._alpha_sq ** .5

    @alpha.setter
    def alpha(self, value):
        if not np.isscalar(value) or value < 1:
            raise ValueError('alpha must be a float greater than 1')
        self._flush()
        self._alpha_sq = float(value) ** 2
        self._version += 1

    # x_post / P_post (kalman_filter.py:560-561) equal x / P until the next predict runs: they are
    # the live tensors until then, and are snapshotted only when a predict is launched on its own
    x_post = property(lambda self: self._vec_out(self._diag("x" if self._post_alias_now() else "x_post")))
    P_post = property(lambda self: self._out(self._diag("P" if self._post_alias_now() else "P_post")))

    def _post_alias_now(self):
        if not self.diagnostics:
            raise AttributeError("x_post / P_post are only kept when the filter is built with diagnostics=True")
        self._flush()
        return self._post_alias

    def _snapshot_post(self):
        if self.diagnostics and self._post_alias:
            self._x_post.copy_(self._x); self._P_post.copy_(self._P)
        self._post_alias = False

    # ------------------------------------------------------------------ predict / update
    def predict(self, u=None, B=None, F=None, Q=None):
        """kalman_filter.py:437-482.  Deferred: fused with the next ``update``."""
        self._flush()
        self._pending = dict(u=u, B=B, F=F, Q=Q)

    def _flush(self):
        if self._pending is not None:
            pend, self._pending = self._pending, None
            self._launch(_lib.BKE_DO_PREDICT, pend, None, None, None, None)

    def update(self, z, R=None, H=None, valid=None):
        """kalman_filter.py:485-561.  ``z`` is ``(N, dim_z)`` in bank mode (``valid`` — bool[N] —
        marks the filters that have a measurement; the others behave as ``z=None``); in single
        mode anything the reference accepts.  ``z=None`` skips the update for the whole bank.

        A filter without a measurement keeps K, S and SI, and its log-likelihood becomes the
        reference's ``logpdf(y = 0, S)`` of the kept S (see ``_missed_log_likelihood``)."""
        pend, self._pending = self._pending, None
        if z is None:                                       # :515-520
            if pend is not None:
                self._launch(_lib.BKE_DO_PREDICT, pend, None, None, None, None)
            self._z = None
            if self.diagnostics:
                self._post_alias = True
                self._y.zero_()
                self._ll.copy_(_missed_log_likelihood(self._S))
            return
        if self._single and H is None:
            z = reshape_z(z, self.dim_z, 2 if self._x_col else 1)        # :527-529
        zt = self._z_rows(z)
        vt = self._valid_mask(valid)
        flags = _lib.BKE_DO_UPDATE | (_lib.BKE_DO_PREDICT if pend is not None else 0)
        self._launch(flags, pend, zt, vt, R, H)
        if vt is not None and self.diagnostics:
            # the kernels leave log_likelihood untouched where z_valid == 0
            self._ll.copy_(torch.where(vt.bool(), self._ll, _missed_log_likelihood(self._S)))
        self._z = zt

    def _step(self, a, rec):
        s = stream_ptr(self._device)
        if rec is not None:
            rc = self._lib.bke_kf_step_packed(a, ptr(rec) if rec.numel() else None, self._sym_host_map, s)
            if rc != _lib.BKE_ERR_UNSUPPORTED:
                return rc
            # arrays the packed kernel does not take (not 16-byte aligned): the dense models from now on
            self._sym_ok = False
            self._sym_drop()
        return self._lib.bke_kf_step(a, s)

    def _capturing(self):
        if torch.cuda.current_device() == self._device.index:
            return torch.cuda.is_current_stream_capturing()
        with torch.cuda.device(self._device):
            return torch.cuda.is_current_stream_capturing()

    def _sym_drop(self):
        """Stop using the current record.  One that a captured graph reads is kept, unchanged, for the
        bank's lifetime (_sym_held); any other is freed once no cached argument struct holds it."""
        if self._sym_buf is not None and self._sym_pinned:
            self._sym_held.append(self._sym_buf)
        self._sym_buf = self._sym_state = self._sym_host_map = None
        self._sym_pinned = False

    def _sym_record(self):
        """The packed copy of the per-filter model words for a launch with the bank's own models, or
        None (the kernels then read the dense F, Q, H and R).

        Most per-filter banks are a template plus a few per-filter parameters: the scan finds the words
        of F, the upper triangle of Q, H and the upper triangle of R that differ between filters, the
        record holds only those, and the words the whole bank shares ride in the launch parameters.
        The copy is derived data and must never go stale: it is used only while F, Q, H and R are in the
        state it was packed from, i.e. neither re-assigned, nor handed out by their getters, nor edited
        in place through torch (the tensors' version counters).  It is (re)packed only outside stream
        capture, and only when the models are the same as at the previous launch, so a loop that assigns
        a model every step never pays for a pack (two passes over the 176 B of models per filter, once);
        a bank with an asymmetric Q or R is scanned once per state of the models and then runs on the
        dense models.  A record that a CUDA graph was captured with is never written again: the graph
        keeps reading the models of its capture (see ``capture``), and a later pack goes to a new record."""
        if not self._sym_ok:
            return None
        F, Q, H, R = self._F, self._Q, self._H, self._R
        # the packed kernel takes per-filter models only, not a mixture with shared ones
        if any(t is None or t.dim() != 3 for t in (F, Q, H, R)):
            self._sym_drop()
            return None
        token = (self._model_version, F._version, Q._version, H._version, R._version)
        last, self._model_last = self._model_last, token
        if self._sym_state is not None and self._sym_state[0] == token:
            if not self._sym_state[1]:
                return None
            if not self._sym_pinned and self._capturing():
                self._sym_pinned = True
            return self._sym_buf
        if token != last or self._capturing():
            return None
        if self._sym_pinned:
            self._sym_drop()
        with torch.cuda.device(self._device):
            s = stream_ptr(self._device)
            if self._sym_map is None:
                self._sym_map = torch.empty(ctypes.sizeof(_lib.KfModelMap), dtype=torch.uint8, device=self._device)
            rc = self._lib.bke_kf_scan_models(self.n_filters, 4, 2, _lib.BKE_F32, ptr(F), ptr(Q), ptr(H), ptr(R),
                                              ptr(self._sym_map), s)
            if rc == _lib.BKE_ERR_UNSUPPORTED:
                self._sym_ok = False
                self._sym_drop()
                return None
            _lib.check(rc)
            hmap = _lib.KfModelMap.from_buffer_copy(self._sym_map.cpu().numpy().tobytes())     # the one host sync
            usable = hmap.asymmetric == 0
            if usable:
                nb = self._lib.bke_kf_packed_models_bytes(self.n_filters, hmap.varying)
                if self._sym_buf is None or self._sym_buf.numel() * 4 != nb:
                    self._sym_buf = torch.empty(nb // 4, dtype=torch.float32, device=self._device)
                    self._version += 1                      # the cached argument structs must keep the record alive
                rc = self._lib.bke_kf_pack_models(self.n_filters, 4, 2, _lib.BKE_F32, ptr(F), ptr(Q), ptr(H), ptr(R),
                                                  hmap.varying, ptr(self._sym_buf) if nb else None, s)
                if rc == _lib.BKE_ERR_UNSUPPORTED:
                    self._sym_ok = False
                    self._sym_drop()
                    return None
                _lib.check(rc)
                self._sym_host_map = hmap
        self._sym_state = (token, usable)
        return self._sym_buf if usable else None

    def _launch(self, flags, pend, zt, vt, R, H):
        if self._reverse:
            flags |= _lib.BKE_REVERSE_TILES
        self._reverse = not self._reverse
        # steady state of a filter loop: nothing but z changed since the last identical call ->
        # reuse the argument struct (the Python side of a launch drops to a few microseconds)
        plain = R is None and H is None and (pend is None or (pend.get("u") is None and pend.get("B") is None
                                                               and pend.get("F") is None and pend.get("Q") is None))
        rec = self._sym_record() if plain else None
        if self._ring_notes is not None and self._capturing():
            self._ring_notes.append((flags & ~_lib.BKE_REVERSE_TILES, plain and vt is None, rec, zt))
        if plain:
            hit = self._args_cache.get(flags)
            if hit is not None and hit[0] == self._version:
                a = hit[1]
                a.z = ptr(zt); a.z_valid = ptr(vt)
                if not (flags & _lib.BKE_DO_UPDATE):
                    self._snapshot_post()                   # a predict on its own is about to move x, P
                self._run(self._step, a, rec)
                if self.diagnostics and (flags & _lib.BKE_DO_UPDATE):
                    self._post_alias = True
                    if self._single:
                        self.check()
                return
        a, keep = self._args(flags, pend, zt, vt, R, H)
        if plain and len(self._host) == 4:                  # every model shared and known on the host
            hm = [self._host[k] for k in "FQHR"]
            a.F_host, a.Q_host, a.H_host, a.R_host = (h.ctypes.data for h in hm)
            keep += hm
        if self._sym_buf is not None:
            keep.append(self._sym_buf)
        if not (flags & _lib.BKE_DO_UPDATE):
            self._snapshot_post()                           # a predict on its own is about to move x, P
        self._run(self._step, a, rec)
        if plain:
            self._args_cache[flags] = (self._version, a, keep)      # keep: the tensors `a` points into
        if self.diagnostics and (flags & _lib.BKE_DO_UPDATE):
            self._post_alias = True
            if self._single:
                self.check()

    def _args(self, flags, pend, zt, vt, R, H):
        """A fresh argument struct of a step with the pending predict ``pend`` and the update's ``z`` / ``valid``
        tensors and per-call ``R`` / ``H``, and the tensors it points into."""
        a = _lib.KfArgs()
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        a.n_filters, a.dim_x, a.dim_z, a.dim_u = N, n, m, 0
        a.dtype = bke_dtype(self._dtype)
        a.flags = flags
        a.alpha_sq = self._alpha_sq
        a.x = a.x_out = ptr(self._x)
        a.P = a.P_out = ptr(self._P)
        keep = []
        if flags & _lib.BKE_DO_PREDICT:
            F = self._F if pend.get("F") is None else self._model(pend["F"], n, n, "F")
            Qo = pend.get("Q")
            Q = self._Q if Qo is None else self._model(Qo, n, n, "Q")      # scalar Q -> Q*I (:467-468)
            B = self._B if pend.get("B") is None else self._model(pend["B"], n, self.dim_u or np.shape(pend["B"])[-1], "B")
            u = pend.get("u")
            a.F, a.F_stride = ptr(F), self._stride(F)
            a.Q, a.Q_stride = ptr(Q), self._stride(Q)
            keep += [F, Q]
            if B is not None and u is not None:                             # :472-475
                du = B.shape[-1]
                ut = to_dev(u, self._dtype, self._device).reshape(-1, du) if not np.isscalar(u) else \
                    torch.full((1, 1), float(u), dtype=self._dtype, device=self._device)
                if ut.shape[0] not in (1, N):
                    raise ValueError("u must have shape (%d,) or (%d,%d)" % (du, N, du))
                a.dim_u = du
                a.B, a.B_stride = ptr(B), self._stride(B)
                a.u, a.u_stride = ptr(ut), (0 if ut.shape[0] == 1 else du)
                keep += [B, ut]
        if flags & _lib.BKE_DO_UPDATE:
            Rm = self._R if R is None else self._model(R, m, m, "R")        # scalar R -> R*I (:524-525)
            Hm = self._H if H is None else self._model(H, m, n, "H")
            a.H, a.H_stride = ptr(Hm), self._stride(Hm)
            a.R, a.R_stride = ptr(Rm), self._stride(Rm)
            a.z = ptr(zt)
            a.z_valid = ptr(vt)
            keep += [Rm, Hm, zt, vt]
        if self.diagnostics:
            if flags & _lib.BKE_DO_PREDICT:
                a.x_prior, a.P_prior = ptr(self._x_prior), ptr(self._P_prior)
            if flags & _lib.BKE_DO_UPDATE:
                a.K, a.y, a.S, a.SI = ptr(self._K), ptr(self._y), ptr(self._S), ptr(self._SI)
                a.log_likelihood = ptr(self._ll)
                a.status = ptr(self._status)
        return a, keep

    # ------------------------------------------------------------------ the other update forms
    def _form_launch(self, fn, *args):
        """Run ``update_correlated`` / ``update_sequential``'s C-ABI call.  Their argument structs are built
        per call and never cached, they leave the tile order and the packed model words alone, and a graph
        captured over them stays a graph of separate launches (the note below is never fusable)."""
        if self._ring_notes is not None and self._capturing():
            self._ring_notes.append((_lib.BKE_DO_UPDATE, False, None, None))
        self._run(fn, *args)
        if self.diagnostics:
            self._post_alias = True
            if self._single:
                self.check()

    def update_correlated(self, z, R=None, H=None, valid=None):
        """kalman_filter.py:670-752: ``update`` for process noise correlated with the measurement noise by
        ``M`` (``(dim_x, dim_z)`` shared or ``(N, dim_x, dim_z)`` per filter; zeros by default)::

            S = H P H' + H M + M' H' + R;  K = (P H' + M) S^-1;  x += K y;  P = P - K (H P + M')

        (not the Joseph form, and not symmetrised).  Arguments, ``valid``, the fused pending predict,
        ``z=None``, the diagnostics and the error behaviour are those of ``update``."""
        if z is None:                                       # :705-710 is update(None)
            return self.update(None)
        pend, self._pending = self._pending, None
        if self._single and H is None:
            z = reshape_z(z, self.dim_z, 2 if self._x_col else 1)        # :718-719
        zt = self._z_rows(z)
        vt = self._valid_mask(valid)
        flags = _lib.BKE_DO_UPDATE | (_lib.BKE_DO_PREDICT if pend is not None else 0)
        a, keep = self._args(flags, pend, zt, vt, R, H)
        Mt = self._M
        self._form_launch(self._lib.bke_kf_step_correlated, a, ptr(Mt), self._stride(Mt), stream_ptr(self._device))
        if vt is not None and self.diagnostics:
            self._ll.copy_(torch.where(vt.bool(), self._ll, _missed_log_likelihood(self._S)))
        self._z = zt

    def update_sequential(self, start, z_i, R_i=None, H_i=None, valid=None):
        """kalman_filter.py:754-824: the update with rows ``start .. start+L-1`` of the measurement alone.
        ``R_i`` defaults to that block of ``R`` (a scalar is ``R_i * I``), ``H_i`` to those rows of ``H``; both
        are read in place from the bank's ``R`` and ``H``.  ``K = P H_i' (1 / S_i)`` when ``L = 1`` (a zero
        ``S_i`` gives inf, never ``LinAlgError``), ``P H_i' inv(S_i)`` otherwise; x and P take the Joseph
        update with ``R_i``.

        Bank mode: ``z_i`` is ``(N, L)``, ``R_i`` ``(L, L)`` or ``(N, L, L)``, ``H_i`` ``(L, dim_x)`` or
        ``(N, L, dim_x)``, ``valid`` (bool[N]) as in ``update``.  Single mode: the reference's arguments.

        Rows ``start .. start+L-1`` of ``y`` and ``z`` and the columns of ``K`` receive the block's values;
        the others keep theirs (rows of ``z`` that no update has set read NaN, where the reference has None).
        ``S``, ``SI`` and ``log_likelihood`` are left as they were: the reference computes its log-likelihood
        lazily, so its value after this call depends on whether it was read before."""
        pend, self._pending = self._pending, None
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        if self._single:
            L = 1 if np.isscalar(z_i) else len(z_i)
            zt = to_dev(np.reshape(np.asarray(z_i, dtype=np.float64), (1, L)), self._dtype, self._device)   # :778-782
        else:
            zt = to_dev(z_i, self._dtype, self._device)
            if zt.dim() == 3 and zt.shape[-1] == 1:
                zt = zt[..., 0]
            if zt.dim() == 1:
                zt = zt.reshape(N, 1)
            if zt.dim() != 2 or zt.shape[0] != N:
                raise ValueError("z_i must have shape (%d, L), got %s" % (N, tuple(zt.shape)))
            zt = zt.contiguous()
            L = zt.shape[1]
        start = int(start)
        if start < 0 or L < 1 or start + L > m:
            raise ValueError("rows %d .. %d are not within the %d rows of z" % (start, start + L - 1, m))
        Rt = None if R_i is None else self._model(R_i, L, L, "R_i")           # scalar -> R_i * I (:787-788)
        if H_i is not None and self._single:
            H_i = np.reshape(np.asarray(H_i, dtype=np.float64), (L, n))       # :793
        Ht = None if H_i is None else self._model(H_i, L, n, "H_i")
        vt = self._valid_mask(valid)
        flags = _lib.BKE_DO_UPDATE | (_lib.BKE_DO_PREDICT if pend is not None else 0)
        a, keep = self._args(flags, pend, zt, vt, None, None)
        a.S = a.SI = a.log_likelihood = None
        if self._zrec is None:
            self._zrec = torch.full((N, m), math.nan, dtype=self._dtype, device=self._device)
        if self._z is not self._zrec:                       # the record starts from the last z
            if self._z is None or tuple(self._z.shape) != (N, m):
                self._zrec.fill_(math.nan)
            else:
                self._zrec.copy_(self._z)
        ra = _lib.KfRowsArgs()
        ra.step = a
        ra.start, ra.rows = start, L
        ra.H_i, ra.H_i_stride = (ptr(Ht), self._stride(Ht)) if Ht is not None else (None, 0)
        ra.R_i, ra.R_i_stride = (ptr(Rt), self._stride(Rt)) if Rt is not None else (None, 0)
        ra.z_record = ptr(self._zrec)
        self._form_launch(self._lib.bke_kf_update_rows, ra, stream_ptr(self._device))
        self._z = self._zrec

    # ------------------------------------------------------------------ scores without a step
    def _candidates(self, z):
        """Bank-mode ``z`` of the scoring methods -> (``z[N or 1, K, m]``, whether it was ``[N, m]``)."""
        return _candidates(z, self.n_filters, self.dim_z, self._dtype, self._device)

    def log_likelihood_of(self, z, valid=None):
        """kalman_filter.py:1252-1260: logpdf(z, H x, S) with the current x and the S stored by the last update,
        not one formed from P (after ``predict`` the result mixes the prior x with the old S, as the reference's
        docstring warns).  ``z=None`` is log(DBL_MIN).  Bank mode: ``z`` is ``[N, m]`` (results ``[N]``), ``[N, K, m]``
        or ``[1, K, m]`` (one scan for the whole bank; results ``[N, K]``); ``valid`` (bool, one per pair) marks
        missing candidates, which score log(DBL_MIN).  A singular S scores NaN (bank) or raises ``LinAlgError``
        (single mode), where scipy would return -inf or a pseudo-determinant value."""
        self._flush()
        S = self._diag("S")
        N = self.n_filters
        if z is None:
            return LOG_DBL_MIN if self._single else torch.full((N,), LOG_DBL_MIN, dtype=self._dtype, device=self._device)
        if self._single:
            zt, sq = to_dev(np.asarray(z, dtype=np.float64).reshape(1, 1, -1), self._dtype, self._device), True
            if zt.shape[-1] != self.dim_z:
                raise ValueError("z must hold %d values, got %d" % (self.dim_z, zt.shape[-1]))
        else:
            zt, sq = self._candidates(z)
        vt = _valid(valid, N, zt.shape[1], self._device)
        out = _score(zt, x=self._x, S=S, H=self._H, valid=vt, want=("log_likelihood", "status"))
        ll = out["log_likelihood"]
        if self._single:
            if int(out["status"][0].item()) != 0:
                raise np.linalg.LinAlgError("Singular matrix")
            return float(ll[0, 0].item())
        return ll[:, 0] if sq else ll

    def residual_of(self, z):
        """kalman_filter.py:1175-1181: z - H x_prior.  Bank mode: ``z`` as in ``log_likelihood_of``, the result
        ``[N, m]`` or ``[N, K, m]``."""
        self._flush()
        xp = self._diag("x_prior")
        m = self.dim_z
        if self._single:
            zr = reshape_z(z, m, 2 if self._x_col else 1)
            zt = to_dev(np.asarray(zr, dtype=np.float64).reshape(1, 1, m), self._dtype, self._device)
            y = _score(zt, x=xp, H=self._H, want=("y",))["y"][0, 0].cpu().numpy()
            return y.reshape(m, 1) if self._x_col else y
        zt, sq = self._candidates(z)
        y = _score(zt, x=xp, H=self._H, want=("y",))["y"]
        return y[:, 0] if sq else y

    def measurement_of_state(self, x):
        """kalman_filter.py:1183-1201: H x.  Bank mode: ``x[N, n]`` -> ``[N, m]``."""
        self._flush()
        n = self.dim_x
        if self._single:
            xa = np.asarray(x, dtype=np.float64)
            if xa.size != n:
                raise ValueError("x must hold %d values, got %d" % (n, xa.size))
            xt = to_dev(xa.reshape(1, n), self._dtype, self._device)
        else:
            xt = to_dev(x, self._dtype, self._device)
            if xt.dim() == 3 and xt.shape[-1] == 1:
                xt = xt[..., 0]
            if tuple(xt.shape) != (self.n_filters, n):
                raise ValueError("x must have shape (%d, %d), got %s" % (self.n_filters, n, tuple(xt.shape)))
        zh = _score(None, x=xt.contiguous(), H=self._H, want=("zhat",))["zhat"]
        if not self._single:
            return zh
        zh = zh[0].cpu().numpy()
        return zh.reshape(-1, 1) if xa.ndim == 2 else zh

    def capture(self, fn, warmup=2):
        """Capture ``fn`` — a fixed sequence of ``predict()/update(z_buffer)`` calls on this bank —
        into a CUDA graph; ``.replay()`` re-runs it with a single launch (see ``StepGraph``).  The
        state is NOT rolled back after the warm-up / capture runs: set ``x`` / ``P`` afterwards.

        A 4/2 float32 bank whose models are all per filter and whose Q and R are exactly symmetric
        steps from a packed copy of its model words (DESIGN.md §2): the graph reads the copy taken
        before the capture, and the words every filter shares are baked into its launch parameters,
        so F, Q, H and R are all frozen into it.  Re-capture after changing any of them, whether by
        assignment or in place; refilling z, x or P in place between replays works as for any
        graph.

        Consecutive launches walk the bank in alternating tile order (``BKE_REVERSE_TILES``, a
        scheduling hint: the results are the same either way).  In a graph of separate steps each
        captured launch keeps the order it was captured with: a graph with an even number of launches
        therefore alternates across replays too; with an odd number, the first launch of a replay runs
        in the same order as the last launch of the previous one, which costs that step the L2 reuse
        but nothing else.  The launches of a fused ring (below) instead take their order from a word
        the bank keeps on the device and each launch advances, so they alternate across replays
        whatever their number, a ring of one launch included.

        A ring of K plain ``predict(); update(z_i)`` pairs of such a bank (``diagnostics=False``, no
        ``valid``, no per-call model, and nothing else in ``fn``: no torch op, no other bank) is returned
        as a graph of ``ceil(K / 8)`` launches of ``bke_kf_steps_packed`` instead: each runs up to 8 of
        the steps back to back with x and P in registers, so the state crosses HBM once per launch and
        not once per step.  Inside a fused ring x and P exist in HBM only between replays; the results
        are bit for bit those of the separate steps.  The returned graph's ``launches`` and
        ``fused_steps`` say which of the two it is."""
        self._flush()
        self._ring_notes = []
        try:
            graph = StepGraph(fn, self._device, warmup)
        finally:
            notes, self._ring_notes = self._ring_notes, None
        graph.launches = len(notes)
        return self._fuse_ring(notes, graph) or graph

    def _fuse_ring(self, notes, graph):
        """The fused form of a captured ring, or None when the capture is anything but plain fused
        predict+update steps of this bank on one packed record: decided on the finished capture, from
        what ``_launch`` noted of each launch, and from the graph's node count, which tells whether
        ``fn`` recorded anything besides those launches."""
        step = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE
        rec = notes[0][2] if notes else None
        if (rec is None or self.diagnostics or graph.nodes != len(notes) or rec is not self._sym_buf
                or any(n[0] != step or not n[1] or n[2] is not rec for n in notes)):
            return None
        # (the argument structs are cached under the flags of their launch, tile order included)
        hit = self._args_cache.get(step) or self._args_cache[step | _lib.BKE_REVERSE_TILES]
        a = _lib.KfArgs.from_buffer_copy(hit[1])
        a.z_valid = None
        zs = [n[3] for n in notes]
        M = _lib.BKE_KF42_MAX_RING
        rings = [(ctypes.c_void_p * len(c))(*[ptr(z) for z in c]) for c in (zs[i:i + M] for i in range(0, len(zs), M))]
        # consecutive launches alternate the tile order, within a replay and across replays: each launch reads
        # the parity of the bank's launch count from this word and advances it on the device (a flag would be
        # frozen into the captured launch).  One word per bank, allocated here, outside any capture.
        if self._tile_order is None:
            self._tile_order = torch.zeros(2, dtype=torch.int32, device=self._device)
        order = self._tile_order
        a.flags = step
        a.tile_order = ptr(order)
        hmap, recp = self._sym_host_map, ptr(rec) if rec.numel() else None

        def call(ring):
            return self._lib.bke_kf_steps_packed(a, recp, hmap, ring, len(ring), stream_ptr(self._device))

        def fused():
            for ring in rings:
                self._run(call, ring)
        # once outside capture: the kernel's one-time function attribute must not be set under capture,
        # and a refusal (a z the ring does not take, such as one that overlaps x or P) leaves the graph of
        # separate steps
        with torch.cuda.device(self._device):
            rc = call(rings[0])
        if rc == _lib.BKE_ERR_UNSUPPORTED:
            return None
        _lib.check(rc)
        for ring in rings[1:]:
            self._run(call, ring)
        ring_graph = StepGraph(fused, self._device, warmup=0)
        ring_graph.launches, ring_graph.fused_steps = len(rings), len(zs)
        ring_graph._keep = (a, rec, hmap, rings, zs, order)     # what the captured launches point into
        return ring_graph

    # ------------------------------------------------------------------ batch_filter
    def batch_filter(self, zs, Fs=None, Qs=None, Hs=None, Rs=None, Bs=None, us=None,
                     update_first=False, saver=None, valid=None):
        """kalman_filter.py:826-993.  Bank mode: ``zs[T,N,dim_z]`` (``valid[T,N]`` optional) ->
        device tensors ``means[T,N,n] covariances[T,N,n,n] means_p covariances_p``.  Single mode:
        ``zs`` as in the reference (entries may be None), NumPy outputs with its shapes.

        With time-constant models the whole T-epoch loop is ONE kernel (bke_kf_batch_filter);
        per-epoch ``Fs/Qs/Hs/Rs/Bs/us`` or a ``saver`` run one fused launch per epoch.  Those launches
        step the bank like ``predict`` / ``update`` and alternate its tile order the same way (see
        ``capture``; the results do not depend on it)."""
        self._flush()
        N, n, m = self.n_filters, self.dim_x, self.dim_z
        # (the reference's np.size(zs, 0), kalman_filter.py:951; a list that mixes None with arrays is
        # ragged for NumPy >= 1.24, so lists are measured with len)
        T = zs.shape[0] if isinstance(zs, torch.Tensor) else (len(zs) if isinstance(zs, (list, tuple)) else np.size(zs, 0))
        if self._single:
            zarr = np.zeros((T, 1, m))
            vmask = np.ones((T, 1), dtype=bool)
            for i, z in enumerate(zs):
                if z is None:
                    vmask[i, 0] = False
                else:
                    zarr[i, 0] = np.asarray(z, dtype=np.float64).reshape(-1)[:m] if np.size(z) == m else \
                        reshape_z(z, m, 1)
            zt = to_dev(zarr, self._dtype, self._device)
            vt = None if vmask.all() else torch.from_numpy(vmask.astype(np.uint8)).to(self._device)
        else:
            zt = to_dev(zs, self._dtype, self._device)
            if tuple(zt.shape) != (T, N, m):
                raise ValueError("zs must have shape (T,%d,%d), got %s" % (N, m, tuple(zt.shape)))
            vt = None if valid is None else torch.as_tensor(valid, device=self._device).to(torch.uint8).contiguous()
        kw = dict(dtype=self._dtype, device=self._device)
        means = torch.empty(T, N, n, **kw); means_p = torch.empty(T, N, n, **kw)
        covs = torch.empty(T, N, n, n, **kw); covs_p = torch.empty(T, N, n, n, **kw)
        per_epoch = any(v is not None for v in (Fs, Qs, Hs, Rs, Bs, us)) or saver is not None
        if not per_epoch:
            b = _lib.KfBatchArgs()
            a = b.step
            a.n_filters, a.dim_x, a.dim_z, a.dim_u = N, n, m, 0
            a.dtype = bke_dtype(self._dtype)
            a.flags = _lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE | (_lib.BKE_UPDATE_FIRST if update_first else 0)
            a.alpha_sq = self._alpha_sq
            a.x = a.x_out = ptr(self._x); a.P = a.P_out = ptr(self._P)
            a.F, a.F_stride = ptr(self._F), self._stride(self._F)
            a.Q, a.Q_stride = ptr(self._Q), self._stride(self._Q)
            a.H, a.H_stride = ptr(self._H), self._stride(self._H)
            a.R, a.R_stride = ptr(self._R), self._stride(self._R)
            if self.diagnostics:
                a.status = ptr(self._status)
            b.n_steps = T
            b.zs, b.zs_valid = ptr(zt), ptr(vt)
            b.means, b.covariances, b.means_p, b.covariances_p = ptr(means), ptr(covs), ptr(means_p), ptr(covs_p)
            with torch.cuda.device(self._device):
                _lib.check(self._lib.bke_kf_batch_filter(b, stream_ptr(self._device)))
        else:
            def at(lst, i):
                return None if lst is None else lst[i]
            for i in range(T):
                v = None if vt is None else vt[i]
                zi = zt[i]
                if update_first:
                    self._launch(_lib.BKE_DO_UPDATE, None, zi, v, at(Rs, i), at(Hs, i))
                    means[i].copy_(self._x); covs[i].copy_(self._P)
                    self._launch(_lib.BKE_DO_PREDICT, dict(u=at(us, i), B=at(Bs, i), F=at(Fs, i), Q=at(Qs, i)),
                                 None, None, None, None)
                    means_p[i].copy_(self._x); covs_p[i].copy_(self._P)
                else:
                    pend = dict(u=at(us, i), B=at(Bs, i), F=at(Fs, i), Q=at(Qs, i))
                    if self.diagnostics:
                        self._launch(_lib.BKE_DO_PREDICT | _lib.BKE_DO_UPDATE, pend, zi, v, at(Rs, i), at(Hs, i))
                        means_p[i].copy_(self._x_prior); covs_p[i].copy_(self._P_prior)
                    else:
                        self._launch(_lib.BKE_DO_PREDICT, pend, None, None, None, None)
                        means_p[i].copy_(self._x); covs_p[i].copy_(self._P)
                        self._launch(_lib.BKE_DO_UPDATE, None, zi, v, at(Rs, i), at(Hs, i))
                    means[i].copy_(self._x); covs[i].copy_(self._P)
                if saver is not None:
                    saver.save()
        if self.diagnostics:
            self._post_alias = not update_first             # update_first ends on a predict (:980-985)
            if update_first and T > 0:
                self._x_post.copy_(means[T - 1]); self._P_post.copy_(covs[T - 1])
        if not self._single:
            return means, covs, means_p, covs_p
        self.check() if self.diagnostics else None
        shp = (T, n, 1) if self._x_col else (T, n)
        return (means[:, 0].cpu().numpy().reshape(shp), covs[:, 0].cpu().numpy(),
                means_p[:, 0].cpu().numpy().reshape(shp), covs_p[:, 0].cpu().numpy())

    def rts_smoother(self, Xs, Ps, Fs=None, Qs=None, inv=None):
        """Rauch-Tung-Striebel smoother over ``batch_filter``'s output (kalman_filter.py:995-1074).

        Bank mode: ``Xs[T,N,n]``, ``Ps[T,N,n,n]`` (the ``means`` / ``covariances`` tensors
        ``batch_filter`` returns) -> ``(x, P, K, Pp)`` tensors of the same layout.  Single mode:
        NumPy ``Xs (T,n)`` or ``(T,n,1)``, ``Ps (T,n,n)`` like the reference.  ``Fs`` / ``Qs`` are
        per-epoch lists (length T; step k uses entry k+1, :1068) or None = the filter's F / Q.
        Only the default ``inv`` (np.linalg.inv) is offered on the GPU."""
        if inv is not None and inv is not np.linalg.inv:
            raise NotImplementedError("rts_smoother: only the default inv (np.linalg.inv) runs on the GPU")
        if len(Xs) != len(Ps):
            raise ValueError('length of Xs and Ps must be the same')
        self._flush()
        return _rts(self, Xs, Ps, Fs, Qs, 1)

    def __repr__(self):
        return "KalmanFilter bank (H100): n_filters=%d dim_x=%d dim_z=%d dtype=%s device=%s" % (
            self.n_filters, self.dim_x, self.dim_z, self._dtype, self._device)


def _missed_log_likelihood(S):
    """log N(0; 0, S) for each filter: what the reference's ``log_likelihood`` returns after
    ``update(None)``, which clears the cached value and leaves y = 0 and the last S
    (kalman_filter.py:511-520, :1203-1210).  -inf where det S <= 0: a filter that has never had a
    measurement still has S = 0, where scipy's logpdf gives -inf (``likelihood`` then floors it at
    float min).  Evaluated in fp64 with torch ops that do not synchronise the host, so a CUDA graph
    can capture it."""
    sign, logdet = torch.linalg.slogdet(S.double())
    ll = -0.5 * (logdet + S.shape[-1] * math.log(2.0 * math.pi))
    return torch.where(sign > 0, ll, -math.inf).to(S.dtype)


def _rts(kf, Xs, Ps, Fs, Qs, shift):
    """Shared body of the two rts_smoother forms: fills bke_rts_args and launches."""
    dtype, device, single, N, n = kf._dtype, kf._device, kf._single, kf.n_filters, kf.dim_x
    is_np = not isinstance(Xs, torch.Tensor)
    Xt, Pt, col = kf._history(Xs, Ps)
    T = Xt.shape[0]

    def model(lst, default, name):
        """-> (tensor, per-filter stride, per-epoch stride)"""
        if lst is None:
            return default, KalmanFilter._stride(default), 0
        if len(lst) != T:
            raise ValueError("%s must have one entry per epoch (%d), got %d" % (name, T, len(lst)))
        mats = [to_dev(m, dtype, device) for m in lst]
        if any(m.shape[-2:] != (n, n) for m in mats):
            raise ValueError("%s entries must be (%d,%d)" % (name, n, n))
        batched = [m.dim() == 3 for m in mats]
        if any(batched) and not all(batched):
            mats = [m if m.dim() == 3 else m.expand(N, n, n) for m in mats]
        t = torch.stack(mats).contiguous()               # (T,n,n) or (T,N,n,n)
        if t.dim() == 4:
            return t, n * n, N * n * n
        return t, 0, n * n

    Ft, sF, tF = model(Fs, kf._F, "Fs")
    Qt, sQ, tQ = model(Qs, kf._Q, "Qs")
    kw = dict(dtype=dtype, device=device)
    x = torch.empty(T, N, n, **kw); P = torch.empty(T, N, n, n, **kw)
    K = torch.empty(T, N, n, n, **kw); Pp = torch.empty(T, N, n, n, **kw)
    status = torch.zeros(N, dtype=torch.int32, device=device)
    a = _lib.RtsArgs()
    a.n_filters, a.n_steps, a.dim_x, a.dtype, a.model_shift = N, T, n, bke_dtype(dtype), shift
    a.Xs, a.Ps = ptr(Xt), ptr(Pt)
    a.F, a.F_stride, a.F_step_stride = ptr(Ft), sF, tF
    a.Q, a.Q_stride, a.Q_step_stride = ptr(Qt), sQ, tQ
    a.x_out, a.P_out, a.K, a.Pp = ptr(x), ptr(P), ptr(K), ptr(Pp)
    a.status = ptr(status)
    kf._run(kf._lib.bke_kf_rts_smoother, a, stream_ptr(device))
    if not single:
        return x, P, K, Pp
    if int(status[0].item()) != 0:
        raise np.linalg.LinAlgError("Singular matrix")
    shp = (T, n, 1) if col else (T, n)
    out = (x[:, 0].reshape(shp), P[:, 0], K[:, 0], Pp[:, 0])
    return tuple(o.cpu().numpy() for o in out) if is_np else out


# ---------------------------------------------------------------------- procedural form
def _as_bank(a, tail, name, dtype, device):
    """Returns (tensor with a leading batch axis or shared, was_batched)."""
    t = to_dev(a, dtype, device)
    if t.dim() == len(tail):
        return t, False
    if t.dim() == len(tail) + 1:
        return t, True
    raise ValueError("%s has a bad number of dimensions: %s" % (name, tuple(t.shape)))


def _proc_filter(x, P, dtype, device):
    xa = np.asarray(x) if not isinstance(x, torch.Tensor) else x
    col = xa.ndim >= 2 and xa.shape[-1] == 1 and (np.ndim(P) == xa.ndim)
    xt = to_dev(x, resolve_dtype(dtype), require_cuda(device))
    if col:
        xt = xt[..., 0]
    batched = xt.dim() == 2
    N = xt.shape[0] if batched else None
    return xt, col, batched, N


def _run_proc(flags, x, P, F=None, Q=None, u=None, B=None, alpha=1., z=None, R=None, H=None,
              return_all=False, dtype=None, device=None):
    is_torch = isinstance(x, torch.Tensor)
    if dtype is None:
        dtype = x.dtype if is_torch else (np.asarray(x).dtype if np.asarray(x).dtype in (np.float32, np.float64) else np.float64)
    xt, col, batched, N = _proc_filter(x, P, dtype, device)
    n = xt.shape[-1]
    m = None
    if flags & _lib.BKE_DO_UPDATE:
        Hm = np.eye(n) if H is None else H
        m = (Hm.shape[-2] if hasattr(Hm, "shape") and np.ndim(Hm) >= 2 else 1)
    kf = KalmanFilter(n, m or 1, n_filters=N, dtype=dtype, device=device, diagnostics=return_all)
    if batched:
        kf.x = xt
    else:
        kf._x = xt.reshape(1, n).clone(); kf._x_col = col
    kf.P = P
    kf._alpha_sq = float(alpha) ** 2
    if flags & _lib.BKE_DO_PREDICT:
        kf.predict(u=None if (np.isscalar(u) and u == 0) else u, B=None if np.isscalar(B) else B,
                   F=np.eye(n) * F if np.isscalar(F) else F, Q=np.eye(n) * Q if np.isscalar(Q) else Q)
    if flags & _lib.BKE_DO_UPDATE:
        if z is None:
            kf._flush()
        else:
            kf.update(z, R=R, H=Hm if np.ndim(Hm) >= 2 else np.reshape(Hm, (1, -1)))
    kf._flush()

    def conv(t, vec=False):
        if batched:
            t2 = t[..., None] if (vec and col) else t
            return t2 if is_torch else t2.cpu().numpy()
        v = t[0]
        if vec and col:
            v = v[..., None]
        return v if is_torch else v.cpu().numpy()
    out = [conv(kf._x, True), conv(kf._P)]
    if return_all:
        if z is None:
            out += [None, None, None, None]
        else:
            ll = kf._ll if batched else kf._ll[0]
            out += [conv(kf._y, True), conv(kf._K), conv(kf._S), ll if is_torch else (ll.cpu().numpy() if batched else float(ll.item()))]
    return tuple(out)


def predict(x, P, F=1, Q=0, u=0, B=1, alpha=1., dtype=None, device=None):
    """Procedural predict (kalman_filter.py:1571-1621) on the GPU; x may carry a leading bank axis."""
    return _run_proc(_lib.BKE_DO_PREDICT, x, P, F=F, Q=Q, u=u, B=B, alpha=alpha, dtype=dtype, device=device)


def update(x, P, z, R, H=None, return_all=False, dtype=None, device=None):
    """Procedural update (kalman_filter.py:1401-1508) on the GPU."""
    if z is None:
        if return_all:
            return x, P, None, None, None, None
        return x, P
    return _run_proc(_lib.BKE_DO_UPDATE, x, P, z=z, R=R, H=H, return_all=return_all, dtype=dtype, device=device)


def batch_filter(x, P, zs, Fs, Qs, Hs, Rs, Bs=None, us=None, update_first=False, saver=None,
                 dtype=np.float64, device=None):
    """Procedural batch_filter (kalman_filter.py:1664-1788) for ONE filter with per-epoch model
    lists, run on the GPU (one fused launch per epoch)."""
    x = np.asarray(x, dtype=np.float64)
    n = x.shape[0]
    H0 = np.atleast_2d(Hs[0])
    kf = KalmanFilter(n, H0.shape[0], dtype=dtype, device=device, diagnostics=True)
    kf.x = x; kf.P = P
    T = len(zs) if isinstance(zs, (list, tuple)) else np.size(zs, 0)
    if us is None:
        us, Bs = None, None
    return kf.batch_filter(zs, Fs=list(Fs), Qs=list(Qs), Hs=[np.atleast_2d(h) for h in Hs], Rs=list(Rs),
                           Bs=Bs, us=us, update_first=update_first, saver=saver)


def rts_smoother(Xs, Ps, Fs, Qs, dtype=np.float64, device=None):
    """Procedural RTS smoother (kalman_filter.py:1792-1858) for ONE filter, run on the GPU.
    ``Fs`` / ``Qs``: one (n,n) matrix, or a per-epoch list (step k uses entry k, :1852)."""
    if len(Xs) != len(Ps):
        raise ValueError('length of Xs and Ps must be the same')
    Xa = np.asarray(Xs, dtype=np.float64)
    n = Xa.shape[1]
    T = Xa.shape[0]
    kf = KalmanFilter(n, 1, dtype=dtype, device=device, diagnostics=False)

    def per_epoch(m):
        a = np.asarray(m, dtype=np.float64)
        return [a] * T if a.ndim == 2 else list(m)
    return _rts(kf, Xa, np.asarray(Ps, dtype=np.float64), per_epoch(Fs), per_epoch(Qs), 0)
