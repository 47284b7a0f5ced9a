"""GPU mirrors of ``filterpy.discrete_bayes`` (filterpy/discrete_bayes/discrete_bayes.py): the discrete Bayes
(histogram) filter's ``normalize``, ``update`` and ``predict``.

The drop-ins keep the reference's signatures and semantics: ``normalize`` works in place and returns its
argument, ``update`` and ``predict`` return a new array.  They take a 1-D NumPy array (or, for ``update`` and
``predict``, anything ``np.asarray`` takes) or a CUDA tensor, run on the GPU and return the kind they were
given, bit for bit what the reference returns (csrc/discrete_bayes.cu).

The bank forms run one launch over ``pdf[B, M]``, one filter per row: ``normalize_bank``, ``update_bank``,
``predict_bank`` and the fused epoch ``predict_update_bank``.  They are separate names because the reference
already gives 2-D input a meaning of its own: its ``normalize`` divides a 2-D array by its column sums, and
``np.roll`` flattens it.  Offsets are one integer for the bank or one per row; the kernel is one ``[K]`` for
the bank or ``[B, K]``.

Differences from the reference:
  * offsets must be integral (an integral float such as ``2.0`` is taken as ``2``).  A fractional offset
    raises ``NotImplementedError``: the reference's wrap mode refuses one too, and its constant mode
    interpolates with an order-3 spline that is not reproduced here;
  * in constant mode the integer shift is exact, where the reference's spline shift carries roundoff
    (at most a few 1e-16 in fp64);
  * pdfs must be float32 or float64.
No CPU fallback.
"""
import numbers

import numpy as np
import torch

from .. import _lib
from .._dev import bke_dtype, require_cuda, stream_ptr

__all__ = ["normalize", "update", "predict", "normalize_bank", "update_bank", "predict_bank", "predict_update_bank"]

_FLOATS = (torch.float32, torch.float64)


def _on_device(a, dtype=None):
    """-> (was a CUDA tensor, contiguous CUDA tensor)."""
    if isinstance(a, torch.Tensor) and a.is_cuda:
        t = a if dtype is None else a.to(dtype)
        return True, t.contiguous()
    arr = np.asarray(a.cpu().numpy() if isinstance(a, torch.Tensor) else a)
    if dtype is not None:
        arr = arr.astype(np.float32 if dtype == torch.float32 else np.float64, copy=False)
    return False, torch.from_numpy(np.ascontiguousarray(arr)).to(require_cuda(None))


def _check_float(t, name):
    if t.dtype not in _FLOATS:
        raise TypeError("%s must be float32 or float64, not %s" % (name, t.dtype))


def _integral(v):
    if isinstance(v, numbers.Integral):
        return int(v)
    f = float(v)
    if not f.is_integer():
        raise NotImplementedError("offset %r is not an integer: fractional offsets (the reference's spline "
                                  "shift) are not supported" % (v,))
    return int(f)


def _offsets(offset, B, dev):
    """-> (scalar offset, per-row int64 tensor or None)."""
    if isinstance(offset, torch.Tensor) and offset.dim() == 0:
        offset = offset.item()
    if np.ndim(offset) == 0 and not isinstance(offset, torch.Tensor):
        return _integral(offset), None
    t = offset if isinstance(offset, torch.Tensor) else torch.from_numpy(np.asarray(offset))
    if t.dim() != 1 or t.shape[0] != B:
        raise ValueError("offset must be a scalar or have one entry per row (%d); got shape %s" % (B, tuple(t.shape)))
    if t.is_floating_point():
        if not bool(torch.all(t == torch.floor(t))) or not bool(torch.all(torch.isfinite(t))):
            raise NotImplementedError("offsets must be integers: fractional offsets (the reference's spline shift) "
                                      "are not supported")
    return 0, t.to(device=dev, dtype=torch.int64).contiguous()


def _kernel(kernel, B, dev):
    """-> fp64 kernel tensor [K] or [B, K], as scipy converts it, and its row stride."""
    k = (kernel.to(device=dev, dtype=torch.float64) if isinstance(kernel, torch.Tensor)
         else torch.from_numpy(np.ascontiguousarray(np.asarray(kernel, dtype=np.float64))).to(dev)).contiguous()
    if k.dim() == 0:
        k = k.reshape(1)
    if k.dim() == 1:
        stride = 0
    elif k.dim() == 2 and k.shape[0] == B:
        stride = k.shape[1]
    else:
        raise ValueError("kernel must be [K] or [n_rows, K]; got shape %s" % (tuple(k.shape),))
    if k.shape[-1] < 1:
        raise ValueError("kernel must have at least one weight")
    return k, stride


def _step(pdf, out, kernel=None, offset=0, likelihood=None, mode="wrap", cval=0.0, normalize=False, sums=None):
    """One bke_db_step over pdf[B, M] (contiguous CUDA tensors of one dtype) into out, which may be pdf."""
    B, M = pdf.shape
    dev = pdf.device
    a = _lib.DbArgs()
    a.n_rows, a.n_bins, a.dtype = B, M, bke_dtype(pdf.dtype)
    a.flags = (_lib.BKE_DB_NORMALIZE if normalize else 0) | (0 if mode == "wrap" else _lib.BKE_DB_CONSTANT)
    keep = []
    if kernel is not None:
        k, stride = _kernel(kernel, B, dev)
        off, offs = _offsets(offset, B, dev)
        keep += [k, offs]
        a.kernel, a.kernel_len, a.kernel_stride = k.data_ptr(), k.shape[-1], stride
        a.offsets = None if offs is None else offs.data_ptr()
        a.offset = off
        a.cval = float(cval)
    if likelihood is not None:
        if likelihood.shape != pdf.shape or likelihood.dtype != pdf.dtype or not likelihood.is_contiguous():
            raise ValueError("likelihood must be a contiguous tensor of the pdf's shape and dtype")
        a.likelihood = likelihood.data_ptr()
    a.pdf, a.out = pdf.data_ptr(), out.data_ptr()
    a.sums = None if sums is None else sums.data_ptr()
    lib = _lib.load()
    wsb = int(lib.bke_db_workspace_bytes(M, a.dtype))
    if wsb and B:
        ws = torch.empty(wsb + 256, dtype=torch.uint8, device=dev)
        keep.append(ws)
        a.workspace = ws.data_ptr() + (-ws.data_ptr()) % 256
        a.workspace_bytes = wsb
    with torch.cuda.device(dev):
        _lib.check(lib.bke_db_step(a, stream_ptr(dev)))
    return out


def _bank(pdf, name="pdf"):
    is_torch, t = _on_device(pdf)
    _check_float(t, name)
    if t.dim() != 2 or t.shape[1] < 1:
        raise ValueError("%s must be 2-D (n_rows, n_bins) with n_bins >= 1; got shape %s" % (name, tuple(t.shape)))
    return is_torch, t


def _back(t, is_torch):
    return t if is_torch else t.cpu().numpy()


def _common(likelihood, prior):
    """likelihood and prior on the device in NumPy's result dtype of prior * likelihood."""
    lt = likelihood if isinstance(likelihood, torch.Tensor) else torch.from_numpy(np.asarray(likelihood))
    pt = prior if isinstance(prior, torch.Tensor) else torch.from_numpy(np.asarray(prior))
    dtype = torch.result_type(pt, lt)
    is_torch, p = _on_device(prior, dtype)
    _, lk = _on_device(likelihood, dtype)
    _check_float(p, "prior")
    if lk.shape != p.shape:
        lk = torch.broadcast_to(lk, p.shape).contiguous()
    return is_torch, p, lk


def normalize_bank(pdf, sums=None):
    """``normalize`` of every row of ``pdf[B, M]``, in place: each row divided by the builtin ``sum`` of its
    fp64 values, as the reference divides one pdf.  Returns ``pdf``.  ``sums`` (optional, a float64 CUDA tensor
    of B elements) receives each row's sum."""
    is_torch, t = _bank(pdf)
    _step(t, t, normalize=True, sums=sums)
    if not is_torch or t.data_ptr() != pdf.data_ptr():
        _copy_back(pdf, t)
    return pdf


def update_bank(likelihood, prior):
    """``update(likelihood[b], prior[b])`` of every row: ``prior * likelihood`` in their dtype, normalised per row.
    Returns a new ``[B, M]`` array or tensor."""
    is_torch, p, lk = _common(likelihood, prior)
    if p.dim() != 2:
        raise ValueError("prior must be 2-D (n_rows, n_bins); got shape %s" % (tuple(p.shape),))
    out = torch.empty_like(p)
    return _back(_step(p, out, likelihood=lk, normalize=True), is_torch)


def predict_bank(pdf, offset, kernel, mode="wrap", cval=0.):
    """``predict(pdf[b], offset[b], kernel[b], mode, cval)`` of every row.  ``offset`` is one integer or one per
    row, ``kernel`` is ``[K]`` or ``[B, K]``.  Returns a new ``[B, M]`` array or tensor."""
    is_torch, t = _bank(pdf)
    out = torch.empty_like(t)
    return _back(_step(t, out, kernel=kernel, offset=offset, mode=mode, cval=cval), is_torch)


def predict_update_bank(pdf, offset, kernel, likelihood, mode="wrap", cval=0., out=None):
    """One epoch of every row's filter in one launch: ``update(likelihood, predict(pdf, offset, kernel, mode,
    cval))``, the prior rounded to the dtype before it is multiplied.  ``out`` (optional) receives the posterior
    and may be ``pdf`` itself; returns the posterior."""
    is_torch, t = _bank(pdf)
    _, lk = _on_device(likelihood, t.dtype)
    if lk.shape != t.shape:
        raise ValueError("likelihood must have the pdf's shape %s; got %s" % (tuple(t.shape), tuple(lk.shape)))
    if out is not None and tuple(out.shape) != tuple(t.shape):
        raise ValueError("out must have the pdf's shape %s; got %s" % (tuple(t.shape), tuple(out.shape)))
    if out is None:
        return _back(_step(t, torch.empty_like(t), kernel=kernel, offset=offset, likelihood=lk, mode=mode, cval=cval,
                           normalize=True), is_torch)
    if is_torch and isinstance(out, torch.Tensor) and out.is_cuda and out.is_contiguous() and out.dtype == t.dtype \
            and out.shape == t.shape:
        _step(t, out, kernel=kernel, offset=offset, likelihood=lk, mode=mode, cval=cval, normalize=True)
        return out
    o = torch.empty_like(t)
    _step(t, o, kernel=kernel, offset=offset, likelihood=lk, mode=mode, cval=cval, normalize=True)
    _copy_back(out, o)
    return out


def _copy_back(dst, t):
    if isinstance(dst, torch.Tensor):
        dst.copy_(t.reshape(dst.shape))
    else:
        dst[...] = t.cpu().numpy().reshape(dst.shape)


def _one(pdf, name):
    is_torch, t = _on_device(pdf)
    _check_float(t, name)
    if t.dim() != 1:
        raise ValueError("%s must be 1-D; the bank forms (normalize_bank, ...) take [n_rows, n_bins]" % name)
    if t.shape[0] < 1:
        raise ValueError("%s must not be empty" % name)
    return is_torch, t.reshape(1, -1)


def normalize(pdf):
    """Normalize ``pdf`` in place so that it sums to 1 and return it (discrete_bayes.py:26-48): ``pdf /=
    sum(np.asarray(pdf, dtype=float))``, the sum the builtin's sequential fp64 chain, the division in fp64."""
    if not isinstance(pdf, (np.ndarray, torch.Tensor)):
        raise TypeError("normalize works in place: pdf must be a NumPy array or a tensor")
    is_torch, t = _one(pdf, "pdf")
    _step(t, t, normalize=True)
    if not is_torch or t.data_ptr() != pdf.data_ptr():
        _copy_back(pdf, t)
    return pdf


def update(likelihood, prior):
    """The posterior ``normalize(prior * likelihood)`` as a new array (discrete_bayes.py:51-89)."""
    is_torch, p, lk = _common(likelihood, prior)
    if p.dim() != 1 or p.shape[0] < 1:
        raise ValueError("prior must be 1-D and not empty; update_bank takes [n_rows, n_bins]")
    p2 = p.reshape(1, -1)
    out = torch.empty_like(p2)
    return _back(_step(p2, out, likelihood=lk.reshape(1, -1), normalize=True).reshape(-1), is_torch)


def predict(pdf, offset, kernel, mode='wrap', cval=0.):
    """The prior: ``pdf`` moved by the integer ``offset`` and convolved with ``kernel``, wrapped around the array
    (``mode='wrap'``) or filled with ``cval`` (any other mode), as a new array (discrete_bayes.py:93-128)."""
    is_torch, t = _one(pdf, "pdf")
    if np.ndim(offset) != 0:
        raise ValueError("offset must be a scalar; predict_bank takes one per row")
    k = kernel if isinstance(kernel, torch.Tensor) else np.asarray(kernel, dtype=np.float64)
    if k.ndim != 1:
        raise ValueError("kernel must be 1-D")
    out = torch.empty_like(t)
    return _back(_step(t, out, kernel=k, offset=offset, mode=mode, cval=cval).reshape(-1), is_torch)
