"""The evaluators of ``filterpy.stats`` (filterpy/stats/stats.py) on the GPU, for one pair or a whole bank.

``mahalanobis`` :64-109, ``log_likelihood`` / ``likelihood`` :112-128, ``logpdf`` :131-154 and ``NEES``
:1138-1179 run on ``bke_score_measurements`` (include/bke.h): one launch scores N tracks against K candidates
each.  There is no CPU fallback.

*Single* calls take exactly what the reference takes and return what it returns (a Python float, or a list for
``NEES``); a length mismatch raises ``ValueError`` before any device is touched, and a singular covariance raises
``np.linalg.LinAlgError``, where the reference's ``inv`` does.

A covariance with a leading bank axis makes a *bank* call: ``cov`` / ``P`` of shape ``[N, ., .]`` (``ps`` of
shape ``[T, N, n, n]`` for ``NEES``), a shape that means nothing to the reference.  The candidates are then
``[N, m]`` (one per track, results ``[N]``), ``[N, K, m]`` (results ``[N, K]``) or ``[1, K, m]`` (one scan shared
by every track, results ``[N, K]``).  Results are device tensors when the covariance is a tensor, NumPy arrays
otherwise.  A track whose covariance is singular gets NaN scores (``status`` 1 of the C call) instead of a raise.

Deviations from scipy's ``multivariate_normal.logpdf(allow_singular=True)`` (INTEGRATION.md): a singular S raises
``LinAlgError`` (single) or scores NaN (bank) where scipy returns a pseudo-determinant value or ``-inf``; no
eigenvalue is dropped below scipy's cutoff; an indefinite S scores with log|det S| where scipy raises
``ValueError``.
"""
import math
import sys

import numpy as np
import torch

from .. import _lib
from .._dev import bke_dtype, ptr, require_cuda, stream_ptr

__all__ = ["mahalanobis", "log_likelihood", "likelihood", "logpdf", "NEES", "score_measurements"]

LOG_DBL_MIN = math.log(sys.float_info.min)


def score(z, *, x=None, mean=None, P=None, S=None, H=None, R=None, valid=None, want=("log_likelihood",)):
    """One ``bke_score_measurements`` launch on device tensors of one dtype (checked by the caller):
    ``x[N, n]`` or ``mean[N, m]``; ``P[N, n, n]`` (with ``R``) or ``S``; ``H``, ``R``, ``S`` ``[N, ., .]`` or shared
    ``[., .]``; ``z[N, K, m]`` or ``[1, K, m]`` (shared), or None when only ``zhat`` is wanted (K = 1);
    ``valid[N, K]`` (uint8) or None.  Returns ``{name: tensor}`` for the names in ``want``."""
    src = x if x is not None else mean
    N, dtype, device = src.shape[0], src.dtype, src.device
    m = mean.shape[-1] if mean is not None else (H.shape[-2] if H is not None else x.shape[-1])
    n = x.shape[-1] if x is not None else (P.shape[-1] if P is not None else m)
    K = 1 if z is None else z.shape[1]
    a = _lib.ScoreArgs()
    a.n_tracks, a.n_candidates, a.dim_x, a.dim_z, a.dtype = N, K, n, m, bke_dtype(dtype)
    a.x, a.mean, a.P = ptr(x), ptr(mean), ptr(P)

    def model(t, size):
        return ptr(t), (0 if t is None or t.dim() == 2 else size)
    a.S, a.S_stride = model(S, m * m)
    a.H, a.H_stride = model(H, m * n)
    a.R, a.R_stride = model(R, m * m)
    if z is not None:
        a.z, a.z_track_stride, a.z_cand_stride = ptr(z), (0 if z.shape[0] == 1 else K * m), m
    a.z_valid = ptr(valid)
    out = {}
    for name in want:
        if name == "zhat":
            out[name] = torch.empty(N, m, dtype=dtype, device=device)
        elif name == "y":
            out[name] = torch.empty(N, K, m, dtype=dtype, device=device)
        elif name == "status":
            out[name] = torch.empty(N, dtype=torch.int32, device=device)
        else:
            out[name] = torch.empty(N, K, dtype=dtype, device=device)
        setattr(a, name, ptr(out[name]))
    if N == 0 or K == 0:
        return out                  # nothing to score (the call would launch nothing)
    lib = _lib.load()
    with torch.cuda.device(device):
        _lib.check(lib.bke_score_measurements(a, stream_ptr(device)))
    return out


# ---------------------------------------------------------------------------------------------------- inputs
def _where(ref):
    """(dtype, device, as_tensor) of a call: a CUDA tensor sets both, anything else runs in fp64 on the current
    device and comes back as NumPy."""
    if isinstance(ref, torch.Tensor):
        dt = ref.dtype if ref.dtype in (torch.float32, torch.float64) else torch.float64
        return dt, require_cuda(ref.device if ref.is_cuda else None), True
    return torch.float64, require_cuda(None), False


def _dev(a, dtype, device):
    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=dtype).contiguous()
    return torch.as_tensor(np.array(a, dtype=np.float64), device=device).to(dtype).contiguous()


def _candidates(z, N, m, dtype, device):
    """Bank candidates -> (z[N or 1, K, m], squeeze): ``[N, m]`` is one per track (results ``[N]``)."""
    zt = _dev(z, dtype, device)
    if zt.dim() == 2 and tuple(zt.shape) == (N, m):
        return zt.reshape(N, 1, m), True
    if zt.dim() == 3 and zt.shape[0] in (1, N) and zt.shape[2] == m:
        return zt, False
    raise ValueError("candidates must have shape (%d, %d), (%d, K, %d) or (1, K, %d), got %s"
                     % (N, m, N, m, m, tuple(zt.shape)))


def _valid(valid, N, K, device):
    if valid is None:
        return None
    vt = torch.as_tensor(valid, device=device).to(torch.uint8).reshape(-1)
    if vt.numel() != N * K:
        raise ValueError("valid must have one entry per track and candidate (%d x %d)" % (N, K))
    return vt.contiguous()


def _back(t, squeeze, as_tensor):
    t = t[:, 0] if squeeze else t
    return t if as_tensor else t.cpu().numpy()


def _bank_model(t, N, r, c, name, dtype, device):
    mt = _dev(t, dtype, device)
    if tuple(mt.shape) == (r, c) or tuple(mt.shape) == (N, r, c):
        return mt
    raise ValueError("%s must have shape (%d, %d) or (%d, %d, %d), got %s" % (name, r, c, N, r, c, tuple(mt.shape)))


def _bank_mean(mean, N, m, dtype, device):
    mt = _dev(mean, dtype, device)
    if tuple(mt.shape) != (N, m):
        raise ValueError("mean must have shape (%d, %d), got %s" % (N, m, tuple(mt.shape)))
    return mt


def _single_scores(want, **kw):
    """One pair on the device; LinAlgError where the covariance is singular."""
    out = score(want=tuple(want) + ("status",), **kw)
    if int(out["status"][0].item()) != 0:
        raise np.linalg.LinAlgError("Singular matrix")
    return out


# ---------------------------------------------------------------------------------------------------- evaluators
def _validate_vector(u):
    # the reference's _validate_vector (stats.py:52-61)
    u = np.atleast_1d(np.asarray(u, dtype=np.float64).squeeze())
    if u.ndim > 1:
        raise ValueError("Input vector should be 1-D.")
    return u


def mahalanobis(x, mean, cov):
    """stats.py:64-109: sqrt((x - mean)' inv(cov) (x - mean)).  Bank: ``cov[N, m, m]``, ``mean[N, m]``, ``x`` the
    candidates."""
    if np.ndim(cov) == 3:
        dtype, device, as_t = _where(cov)
        S = _dev(cov, dtype, device)
        N, m = S.shape[0], S.shape[-1]
        mt = _bank_mean(mean, N, m, dtype, device)
        zt, sq = _candidates(x, N, m, dtype, device)
        return _back(score(zt, mean=mt, S=S, want=("mahalanobis",))["mahalanobis"], sq, as_t)
    x = _validate_vector(x)
    mean = _validate_vector(mean)
    if x.shape != mean.shape:
        raise ValueError("length of input vectors must be the same")
    S = np.atleast_2d(np.asarray(cov, dtype=np.float64))
    m = x.shape[0]
    if S.shape != (m, m):
        raise ValueError("cov must be (%d, %d) for vectors of length %d, got %s" % (m, m, m, S.shape))
    dev = require_cuda(None)
    d2 = float(_single_scores(("d2",), z=_dev(x.reshape(1, 1, m), torch.float64, dev),
                              mean=_dev(mean.reshape(1, m), torch.float64, dev), S=_dev(S, torch.float64, dev))["d2"][0, 0])
    return math.sqrt(d2)          # ValueError for a negative d2 (an indefinite cov), as the reference's math.sqrt


def _ll_inputs(z, x, P, H, R):
    """Bank arguments of log_likelihood / likelihood / score_measurements as device tensors."""
    dtype, device, as_t = _where(P)
    Pt = _dev(P, dtype, device)
    N, n = Pt.shape[0], Pt.shape[-1]
    Ht = _dev(H, dtype, device)
    if Ht.dim() not in (2, 3) or Ht.shape[-1] != n:
        raise ValueError("H must have shape (m, %d) or (%d, m, %d), got %s" % (n, N, n, tuple(Ht.shape)))
    m = Ht.shape[-2]
    Ht = _bank_model(Ht, N, m, n, "H", dtype, device)
    Rt = _bank_model(R, N, m, m, "R", dtype, device)
    xt = _dev(x, dtype, device)
    if xt.dim() == 3 and xt.shape[-1] == 1:
        xt = xt[..., 0]
    if tuple(xt.shape) != (N, n):
        raise ValueError("x must have shape (%d, %d), got %s" % (N, n, tuple(xt.shape)))
    zt, sq = _candidates(z, N, m, dtype, device)
    return dict(z=zt, x=xt.contiguous(), P=Pt, H=Ht, R=Rt), sq, as_t


def _ll_single(z, x, P, H, R, want):
    H = np.atleast_2d(np.asarray(H, dtype=np.float64))
    m, n = H.shape
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    P = np.atleast_2d(np.asarray(P, dtype=np.float64))
    zf = np.asarray(z, dtype=np.float64).reshape(-1)          # logpdf flattens z and the mean (stats.py:146-150)
    if x.shape != (n,) or P.shape != (n, n) or zf.shape != (m,):
        raise ValueError("shapes do not fit: z %s, x %s, P %s, H %s" % (zf.shape, x.shape, P.shape, H.shape))
    Rb = np.broadcast_to(np.asarray(R, dtype=np.float64), (m, m))   # np.dot(H, np.dot(P, H.T)) + R broadcasts R
    dev = require_cuda(None)
    d = lambda a: _dev(a, torch.float64, dev)                 # noqa: E731
    out = _single_scores((want,), z=d(zf.reshape(1, 1, m)), x=d(x.reshape(1, n)), P=d(P.reshape(1, n, n)), H=d(H),
                         R=d(np.ascontiguousarray(Rb)))
    return float(out[want][0, 0])


def log_likelihood(z, x, P, H, R):
    """stats.py:112-119: logpdf(z, H x, H P H' + R).  Bank: ``P[N, n, n]``, ``x[N, n]``, ``H`` / ``R`` shared or
    per track, ``z`` the candidates."""
    if np.ndim(P) == 3:
        kw, sq, as_t = _ll_inputs(z, x, P, H, R)
        return _back(score(want=("log_likelihood",), **kw)["log_likelihood"], sq, as_t)
    return _ll_single(z, x, P, H, R, "log_likelihood")


def likelihood(z, x, P, H, R):
    """stats.py:122-128: exp(log_likelihood(...)), with no floor."""
    if np.ndim(P) == 3:
        kw, sq, as_t = _ll_inputs(z, x, P, H, R)
        return _back(score(want=("likelihood",), **kw)["likelihood"], sq, as_t)
    return _ll_single(z, x, P, H, R, "likelihood")


def score_measurements(z, x, P, H, R, valid=None):
    """The gating step of a bank: ``(log_likelihood, mahalanobis)`` of every candidate against every track, both
    ``[N, K]`` (``[N]`` for ``z[N, m]``), from one launch that reads each track once.  ``P[N, n, n]``, ``x[N, n]``,
    ``H`` / ``R`` shared or per track; ``valid`` (bool, one per pair) marks missing candidates, which score
    ``log(DBL_MIN)`` and distance 0."""
    if np.ndim(P) != 3:
        raise ValueError("score_measurements scores a bank: P must be (N, n, n)")
    kw, sq, as_t = _ll_inputs(z, x, P, H, R)
    N, K = kw["x"].shape[0], kw["z"].shape[1]
    out = score(valid=_valid(valid, N, K, kw["x"].device), want=("log_likelihood", "mahalanobis"), **kw)
    return _back(out["log_likelihood"], sq, as_t), _back(out["mahalanobis"], sq, as_t)


def _scipy_cov(cov, dim):
    # scipy's _process_parameters: a scalar is cov * I, a vector the diagonal
    c = np.asarray(cov, dtype=np.float64)
    if c.ndim == 0:
        return c * np.eye(dim)
    if c.ndim == 1:
        return np.diag(c)
    return c


def logpdf(x, mean=None, cov=1, allow_singular=True):
    """stats.py:131-154: scipy's multivariate_normal.logpdf(x, mean, cov).  Bank: ``cov[N, m, m]``, ``mean[N, m]``
    (None: zeros), ``x`` the candidates.  ``allow_singular`` is accepted; a singular cov raises ``LinAlgError``
    (single) or scores NaN (bank) either way."""
    if np.ndim(cov) == 3:
        dtype, device, as_t = _where(cov)
        S = _dev(cov, dtype, device)
        N, m = S.shape[0], S.shape[-1]
        mt = torch.zeros(N, m, dtype=dtype, device=device) if mean is None else \
            _bank_mean(mean, N, m, dtype, device)
        zt, sq = _candidates(x, N, m, dtype, device)
        return _back(score(zt, mean=mt, S=S, want=("log_likelihood",))["log_likelihood"], sq, as_t)
    fx = np.asarray(x, dtype=np.float64).flatten()
    fm = np.zeros_like(fx) if mean is None else np.asarray(mean, dtype=np.float64).flatten()
    m = fm.shape[0]
    S = _scipy_cov(cov, m)
    if fx.shape != (m,) or S.shape != (m, m):
        raise ValueError("x, mean and cov do not fit: %s, %s, %s" % (fx.shape, fm.shape, S.shape))
    dev = require_cuda(None)
    d = lambda a: _dev(a, torch.float64, dev)                 # noqa: E731
    return float(_single_scores(("log_likelihood",), z=d(fx.reshape(1, 1, m)), mean=d(fm.reshape(1, m)),
                                S=d(S))["log_likelihood"][0, 0])


def NEES(xs, est_xs, ps):
    """stats.py:1138-1179: e' inv(p) e for e = xs - est_xs over the sequence, as a list.  Bank: ``ps[T, N, n, n]``,
    ``xs`` / ``est_xs`` ``[T, N, n]`` -> ``[T, N]`` (NaN where p is singular)."""
    if np.ndim(ps) == 4:
        dtype, device, as_t = _where(ps)
        Pt = _dev(ps, dtype, device)
        T, N, n = Pt.shape[0], Pt.shape[1], Pt.shape[-1]
        xt, et = _dev(xs, dtype, device), _dev(est_xs, dtype, device)
        if tuple(xt.shape) != (T, N, n) or tuple(et.shape) != (T, N, n):
            raise ValueError("xs and est_xs must have shape (%d, %d, %d)" % (T, N, n))
        d2 = score(xt.reshape(T * N, 1, n), mean=et.reshape(T * N, n), S=Pt.reshape(T * N, n, n), want=("d2",))["d2"]
        d2 = d2.reshape(T, N)
        return d2 if as_t else d2.cpu().numpy()
    est_err = np.asarray(xs, dtype=np.float64) - np.asarray(est_xs, dtype=np.float64)
    ps = np.asarray(ps, dtype=np.float64)
    T = min(len(est_err), len(ps))
    if T == 0:
        return []
    col = est_err.ndim == 3
    e = est_err[:T].reshape(T, -1)
    n = e.shape[1]
    if ps.shape[1:] != (n, n):
        raise ValueError("ps must be a sequence of (%d, %d) matrices, got %s" % (n, n, ps.shape[1:]))
    dev = require_cuda(None)
    d = lambda a: _dev(a, torch.float64, dev)                 # noqa: E731
    out = score(d(e.reshape(T, 1, n)), mean=torch.zeros(T, n, dtype=torch.float64, device=dev), S=d(ps[:T]),
                want=("d2", "status"))
    if bool((out["status"] != 0).any().item()):
        raise np.linalg.LinAlgError("singular matrix")
    d2 = out["d2"][:, 0].cpu().numpy()
    return [v.reshape(1, 1) if col else v for v in d2]
