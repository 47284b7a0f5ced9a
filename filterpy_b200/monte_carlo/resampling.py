"""GPU mirrors of ``filterpy.monte_carlo.systematic_resample`` / ``stratified_resample`` /
``multinomial_resample`` (filterpy/monte_carlo/resampling.py:117-150 / :80-114 / :153-176) and the
particle gather that follows them (docs/monte_carlo/resampling.rst:4-8).

Same call, same result: ``indexes`` is the ``int32`` array the reference returns for the same
weights and the same uniform draw(s) — bit for bit, because the CUDA path reproduces the strictly
sequential fp64 ``np.cumsum`` exactly (csrc/resample.cu).  The uniforms are drawn here from
``numpy.random.random`` exactly as the reference does (resampling.py:24,103,139), so seeding with
``np.random.seed`` reproduces the reference's stream.  No CPU fallback.
"""
import ctypes

import numpy as np
import torch
from numpy.random import random

from .. import _lib
from .._dev import require_cuda, stream_ptr

__all__ = ["systematic_resample", "stratified_resample", "multinomial_resample", "residual_resample",
           "gather_particles", "exact_cumsum", "ResamplePlan", "normalize_weights",
           "residual_resample_with_uniforms", "systematic_resample_bank", "stratified_resample_bank",
           "gather_particles_bank", "BankResamplePlan", "multinomial_resample_bank", "residual_resample_bank",
           "systematic_resample_bank_if_degenerate", "stratified_resample_bank_if_degenerate"]


class ResamplePlan(object):
    """Pre-allocated workspace + output for repeated resampling of ``n`` particles on one GPU
    (nothing is allocated and the host is not synchronised per call)."""

    def __init__(self, n, device=None):
        self.n = int(n)
        self.device = require_cuda(device)
        self._lib = _lib.load()
        self.ws_bytes = int(self._lib.bke_resample_workspace_bytes(self.n))
        self.workspace = torch.empty(self.ws_bytes + 256, dtype=torch.uint8, device=self.device)
        off = (-self.workspace.data_ptr()) % 256
        self._ws_ptr = self.workspace.data_ptr() + off
        self.indexes = torch.empty(self.n, dtype=torch.int32, device=self.device)
        self._info = torch.zeros(8, dtype=torch.int32, device=self.device)
        self.cumsum_last = torch.zeros(1, dtype=torch.float64, device=self.device)

    def _check_w(self, weights):
        if not (isinstance(weights, torch.Tensor) and weights.is_cuda and weights.dtype == torch.float64
                and weights.is_contiguous() and weights.numel() == self.n):
            raise ValueError("weights must be a contiguous float64 CUDA tensor of %d elements" % self.n)

    def systematic(self, weights, u, out=None):
        """indexes for the offset ``u`` (resampling.py:139: positions = (u + arange(N)) / N)."""
        self._check_w(weights)
        out = self.indexes if out is None else out
        with torch.cuda.device(self.device):
            _lib.check(self._lib.bke_systematic_resample(
                self.n, weights.data_ptr(), float(u), out.data_ptr(), self._ws_ptr, self.ws_bytes,
                self._info.data_ptr(), self.cumsum_last.data_ptr(), stream_ptr(self.device)))
        return out

    def stratified(self, weights, uniforms, out=None):
        """indexes for per-particle uniforms (resampling.py:103: positions = (U + range(N)) / N)."""
        self._check_w(weights)
        if not (isinstance(uniforms, torch.Tensor) and uniforms.is_cuda and uniforms.dtype == torch.float64
                and uniforms.is_contiguous() and uniforms.numel() == self.n):
            raise ValueError("uniforms must be a contiguous float64 CUDA tensor of %d elements" % self.n)
        out = self.indexes if out is None else out
        with torch.cuda.device(self.device):
            _lib.check(self._lib.bke_stratified_resample(
                self.n, weights.data_ptr(), uniforms.data_ptr(), out.data_ptr(), self._ws_ptr, self.ws_bytes,
                self._info.data_ptr(), self.cumsum_last.data_ptr(), stream_ptr(self.device)))
        return out

    def normalized(self, weights, u=None, uniforms=None, out=None, weights_out=None):
        """Fused normalise + resample: ``systematic_resample(weights / S)`` (``stratified_resample`` when
        ``uniforms`` is given) with ``S`` the engine's sum of the weights.  Returns (indexes, S tensor)."""
        self._check_w(weights)
        out = self.indexes if out is None else out
        total = torch.zeros(1, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._lib.bke_resample_normalized(
                self.n, weights.data_ptr(), float(u if u is not None else 0.0),
                uniforms.data_ptr() if uniforms is not None else None, out.data_ptr(),
                weights_out.data_ptr() if weights_out is not None else None, total.data_ptr(),
                self._ws_ptr, self.ws_bytes, self._info.data_ptr(), self.cumsum_last.data_ptr(),
                stream_ptr(self.device)))
        return out, total

    def cumsum(self, weights, out=None, last_one=False):
        """``np.cumsum(weights)`` bit for bit (sequential fp64 order), on the device."""
        self._check_w(weights)
        out = torch.empty(self.n, dtype=torch.float64, device=self.device) if out is None else out
        with torch.cuda.device(self.device):
            _lib.check(self._lib.bke_cumsum_exact(self.n, weights.data_ptr(), out.data_ptr(), int(bool(last_one)),
                                                  self._ws_ptr, self.ws_bytes, self._info.data_ptr(),
                                                  stream_ptr(self.device)))
        return out

    def multinomial(self, weights, uniforms, out=None, scratch=None, lut=True):
        """resampling.py:173-176 for the given uniforms: int64 indexes.  ``lut=False`` runs the plain
        bisection without the bracket table (same result)."""
        self._check_w(weights)
        if not (isinstance(uniforms, torch.Tensor) and uniforms.is_cuda and uniforms.dtype == torch.float64
                and uniforms.is_contiguous() and uniforms.numel() == self.n):
            raise ValueError("uniforms must be a contiguous float64 CUDA tensor of %d elements" % self.n)
        out = torch.empty(self.n, dtype=torch.int64, device=self.device) if out is None else out
        scratch = torch.empty(self.n, dtype=torch.float64, device=self.device) if scratch is None else scratch
        lut_ptr = self.indexes.data_ptr() if lut else None           # the plan's int32[n] doubles as the table
        with torch.cuda.device(self.device):
            _lib.check(self._lib.bke_multinomial_resample(
                self.n, weights.data_ptr(), uniforms.data_ptr(), out.data_ptr(), scratch.data_ptr(), lut_ptr,
                self._ws_ptr, self.ws_bytes, self._info.data_ptr(), stream_ptr(self.device)))
        return out

    def info(self):
        """int32[8] on the host: [0] positions >= cumsum[-1] (the reference raises IndexError),
        [1] sequential-fallback used, [2] tiles with raw elements, [3] long runs, [4] chain flag."""
        return self._info.cpu().numpy()

    def raise_if_overflow(self):
        inf = self.info()
        if inf[0] > 0:
            raise IndexError("index %d is out of bounds for axis 0 with size %d" % (self.n, self.n))


def normalize_weights(weights, plan=None):
    """weights / weights.sum() on the device (IEEE division by the engine's tree-ordered sum).
    Returns (normalised weights, sum tensor)."""
    plan = plan or ResamplePlan(weights.numel(), weights.device)
    lib = plan._lib
    total = torch.zeros(1, dtype=torch.float64, device=weights.device)
    out = torch.empty_like(weights)
    with torch.cuda.device(weights.device):
        _lib.check(lib.bke_weights_sum(plan.n, weights.data_ptr(), total.data_ptr(), plan._ws_ptr, plan.ws_bytes,
                                       stream_ptr(weights.device)))
        _lib.check(lib.bke_weights_scale(plan.n, weights.data_ptr(), total.data_ptr(), out.data_ptr(),
                                         stream_ptr(weights.device)))
    return out, total


def _weights_on_device(weights):
    is_torch = isinstance(weights, torch.Tensor)
    if is_torch and weights.is_cuda:
        w = weights.to(torch.float64).contiguous()
        dev = w.device
    else:
        dev = require_cuda(None)
        w = torch.from_numpy(np.ascontiguousarray(np.asarray(weights, dtype=np.float64))).to(dev)
    return is_torch, w, dev


def _run(weights, stratified):
    is_torch, w, dev = _weights_on_device(weights)
    n = w.numel()
    if n == 0:
        if stratified:
            random(0)
        else:
            random()
        return torch.zeros(0, dtype=torch.int32, device=dev) if is_torch else np.zeros(0, 'i')
    plan = ResamplePlan(n, dev)
    if stratified:
        U = torch.from_numpy(random(n)).to(dev)          # resampling.py:103
        idx = plan.stratified(w, U)
    else:
        idx = plan.systematic(w, random())               # resampling.py:139
    plan.raise_if_overflow()                             # resampling.py:145 (IndexError)
    return idx if is_torch else idx.cpu().numpy()


def systematic_resample(weights):
    """resampling.py:117-150 on the GPU; returns ``ndarray`` int32 (or a CUDA tensor when given one)."""
    return _run(weights, False)


def stratified_resample(weights):
    """resampling.py:80-114 on the GPU."""
    return _run(weights, True)


def multinomial_resample(weights):
    """resampling.py:153-176 on the GPU: ``searchsorted(cumsum(w) with [-1] = 1, random(N))``.
    Returns int64 indexes (what ``np.searchsorted`` returns), ndarray or CUDA tensor like the input."""
    is_torch, w, dev = _weights_on_device(weights)
    n = w.numel()
    if n == 0:
        np.cumsum(np.zeros(0))[-1:]                       # the reference fails on cumulative_sum[-1] (:174)
        raise IndexError("index -1 is out of bounds for axis 0 with size 0")
    plan = ResamplePlan(n, dev)
    U = torch.from_numpy(np.atleast_1d(random(n))).to(dev)   # resampling.py:176
    idx = plan.multinomial(w, U)
    return idx if is_torch else idx.cpu().numpy()


def residual_resample_with_uniforms(weights, uniforms_fn=random, max_sweeps=10000):
    """residual_resample for uniforms drawn by ``uniforms_fn(N - k)`` (the reference: ``random``);
    returns (indexes, info) with info = dict(k, sweeps, residual_sum)."""
    is_torch, w, dev = _weights_on_device(weights)
    n = w.numel()
    if n == 0:
        # resampling.py:70-72 on empty arrays: sum([]) = 0, cumulative_sum[-1] raises IndexError
        raise IndexError("index -1 is out of bounds for axis 0 with size 0")
    lib = _lib.load()
    ws_bytes = int(lib.bke_residual_workspace_bytes(n))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    idx = torch.zeros(n, dtype=torch.int32, device=dev)              # np.zeros(N, 'i') (:52)
    csum = torch.empty(n, dtype=torch.float64, device=dev)
    k_dev = torch.zeros(1, dtype=torch.int64, device=dev)
    rsum = torch.zeros(1, dtype=torch.float64, device=dev)
    st = stream_ptr(dev)
    with torch.cuda.device(dev):
        _lib.check(lib.bke_residual_prepare(n, w.data_ptr(), idx.data_ptr(), csum.data_ptr(), k_dev.data_ptr(),
                                            rsum.data_ptr(), ws.data_ptr(), ws_bytes, st))
        k = int(k_dev.item())
        if k > n:                                                     # indexes[k] = i runs off the end (:61)
            raise IndexError("index %d is out of bounds for axis 0 with size %d" % (n, n))
        m = n - k
        U = np.atleast_1d(uniforms_fn(m))                             # resampling.py:74: random(N - k)
        sweeps = 0
        if m > 0:
            keys = torch.from_numpy(np.ascontiguousarray(U, dtype=np.float64)).to(dev)
            r = [torch.empty(m, dtype=torch.int64, device=dev), torch.empty(m, dtype=torch.int64, device=dev)]
            changed = torch.zeros(1, dtype=torch.int32, device=dev)
            tail = idx[k:]
            # the int32 copies land directly in indexes[k:N] when that view is 4-byte aligned (always)
            _lib.check(lib.bke_searchsorted_bracket_sweep(n, csum.data_ptr(), m, keys.data_ptr(), None,
                                                          r[0].data_ptr(), tail.data_ptr(), changed.data_ptr(), st))
            cur = 0
            while True:
                sweeps += 1
                changed.zero_()
                _lib.check(lib.bke_searchsorted_bracket_sweep(n, csum.data_ptr(), m, keys.data_ptr(), r[cur].data_ptr(),
                                                              r[1 - cur].data_ptr(), tail.data_ptr(),
                                                              changed.data_ptr(), st))
                cur = 1 - cur
                if int(changed.item()) == 0:
                    break
                if sweeps >= max_sweeps:
                    raise RuntimeError("residual_resample: the bracket recurrence did not settle in %d sweeps"
                                       % max_sweeps)
    info = {"k": k, "sweeps": sweeps, "residual_sum": float(rsum.item())}
    return (idx if is_torch else idx.cpu().numpy()), info


def residual_resample(weights):
    """resampling.py:27-76 on the GPU, same call, same result for the same ``np.random`` state.

    The reference's ``residual = weights - num_copies`` (:69; not ``N*weights - num_copies``) is negative
    for every particle that got a copy, so the cumulative sum it bisects (:74) is not monotone and
    ``np.searchsorted``'s answer depends on the bracket NumPy carries from key to key.  The engine
    reproduces exactly that: the order-dependent sums in the reference's order, and NumPy's bracket
    recurrence as a parallel fixed-point iteration (csrc/residual.cu).  Returns ``ndarray`` int32 (or a
    CUDA tensor when given one)."""
    return residual_resample_with_uniforms(weights, random)[0]


def exact_cumsum(weights, last_one=False):
    """``np.cumsum(weights)`` (fp64, strictly sequential order) computed on the GPU, bit for bit."""
    is_torch, w, dev = _weights_on_device(weights)
    if w.numel() == 0:
        return w.clone() if is_torch else np.zeros(0)
    out = ResamplePlan(w.numel(), dev).cumsum(w, last_one=last_one)
    return out if is_torch else out.cpu().numpy()


def gather_particles(particles, indexes, out=None, check=True):
    """``particles[indexes]`` along axis 0 on the GPU — the step after every resample
    (docs/monte_carlo/resampling.rst:4-8: ``particles[:] = particles[indexes]``).

    ``particles`` is (N, ...) of any dtype, ``indexes`` int32 or int64 (what the resamplers return);
    NumPy in -> NumPy out, CUDA tensors in -> CUDA tensor out.  Raises IndexError for an index outside
    [0, N) like NumPy does (negative indexes are not wrapped); ``check=False`` skips that test and the
    host synchronisation it costs."""
    lib = _lib.load()
    is_torch = isinstance(particles, torch.Tensor)
    if is_torch and particles.is_cuda:
        dev = particles.device
        src = particles.contiguous()
    else:
        dev = require_cuda(None)
        src = torch.from_numpy(np.ascontiguousarray(np.asarray(particles))).to(dev)
    if isinstance(indexes, torch.Tensor):
        idx = indexes.to(dev)
    else:
        idx = torch.from_numpy(np.ascontiguousarray(np.asarray(indexes))).to(dev)
    if idx.dtype not in (torch.int32, torch.int64):
        raise IndexError("arrays used as indices must be of integer type")
    idx = idx.contiguous().reshape(-1)
    if src.dim() == 0:
        raise IndexError("too many indices for array")
    n_src = src.shape[0]
    n_out = idx.numel()
    row_bytes = (src.numel() // max(n_src, 1)) * src.element_size()
    shape = (n_out,) + tuple(src.shape[1:])
    if out is None:
        out = torch.empty(shape, dtype=src.dtype, device=dev)
    elif not (isinstance(out, torch.Tensor) and out.is_cuda and out.is_contiguous() and tuple(out.shape) == shape
              and out.dtype == src.dtype):
        raise ValueError("out must be a contiguous CUDA tensor of shape %s" % (shape,))
    if n_out and row_bytes:
        if n_src == 0:
            raise IndexError("index out of bounds for axis 0 with size 0")
        err = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.bke_gather_rows(n_out, n_src, row_bytes, src.data_ptr(), idx.data_ptr(),
                                           1 if idx.dtype == torch.int64 else 0, out.data_ptr(), err.data_ptr(),
                                           stream_ptr(dev)))
        if check and int(err.item()):
            raise IndexError("index out of bounds for axis 0 with size %d" % n_src)
    return out if (is_torch and particles.is_cuda) else out.cpu().numpy()


# ------------------------------------------------------------------------------------------- banks
def _bank_tensor_check(t, name, dtypes, shape, device):
    if not (isinstance(t, torch.Tensor) and t.device == device and t.dtype in dtypes and t.is_contiguous()
            and tuple(t.shape) == tuple(shape)):
        raise ValueError("%s must be a contiguous %s tensor of shape %s on %s"
                         % (name, " or ".join(str(d) for d in dtypes), tuple(shape), device))


class BankResamplePlan(object):
    """Output buffers for repeated resampling of a bank of ``n_sets`` particle sets of ``n_particles``
    each on one GPU (``csrc/resample_bank.cu``): row ``b`` of the weights is one set, resampled as the
    reference resamples one weight vector.  A call allocates nothing and does not synchronise the host,
    so it can be captured in a CUDA graph.

    ``status`` (int32 CUDA tensor [n_sets]) is 1 for a set whose positions ran past its cumulative sum
    (the reference's ``IndexError``, resampling.py:145; that row's indexes are unspecified), else 0.

    ``multinomial`` and ``residual`` run the reference's ``multinomial_resample`` / ``residual_resample``
    per row for caller-supplied uniforms.  Their first call allocates the plan's workspace (n_sets *
    n_particles doubles for the per-set cumulative sums), so make one call before capturing a graph.
    After them ``status`` has bit 0 set where the reference raises (residual: k > M) and bit 1 (value 2)
    where the set took NumPy's carried-bracket search because its cumulative sum is not sorted."""

    def __init__(self, n_sets, n_particles, device=None):
        self.n_sets = int(n_sets)
        self.n_particles = int(n_particles)
        if self.n_sets < 0 or self.n_particles < 0:
            raise ValueError("n_sets and n_particles must be >= 0")
        self.device = require_cuda(device)
        self._lib = _lib.load()
        self.indexes = torch.empty((self.n_sets, self.n_particles), dtype=torch.int32, device=self.device)
        self.status = torch.zeros(self.n_sets, dtype=torch.int32, device=self.device)
        self._err = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.n_copies = torch.zeros(self.n_sets, dtype=torch.int64, device=self.device)
        self._ws = None
        self._idx64 = None
        self._neff = None                                 # resample_if_degenerate's buffers, made on first use

    def _workspace(self):
        if self._ws is None:
            nbytes = int(self._lib.bke_residual_resample_bank_workspace_bytes(self.n_sets, self.n_particles))
            self._ws = torch.empty(max(nbytes // 8, 1), dtype=torch.float64, device=self.device)
        return self._ws

    def multinomial(self, weights, uniforms, out=None):
        """indexes[b] = ``searchsorted(cumsum(weights[b]) with [-1] = 1, uniforms[b])`` (resampling.py:173-176),
        int64 (B, M) like ``np.searchsorted``; ``uniforms`` float64 CUDA tensor [n_sets, M]."""
        shape = (self.n_sets, self.n_particles)
        _bank_tensor_check(weights, "weights", (torch.float64,), shape, self.device)
        _bank_tensor_check(uniforms, "uniforms", (torch.float64,), shape, self.device)
        if out is None:
            if self._idx64 is None:
                self._idx64 = torch.empty(shape, dtype=torch.int64, device=self.device)
            out = self._idx64
        _bank_tensor_check(out, "out", (torch.int64,), shape, self.device)
        ws = self._workspace()
        a = _lib.MultinomialResampleBankArgs()
        a.n_sets, a.n_particles = self.n_sets, self.n_particles
        a.weights, a.uniforms, a.indexes, a.status = (weights.data_ptr(), uniforms.data_ptr(), out.data_ptr(),
                                                      self.status.data_ptr())
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel() * 8
        with torch.cuda.device(self.device):
            _lib.check(self._lib.bke_multinomial_resample_bank(ctypes.byref(a), stream_ptr(self.device)))
        return out

    def _residual_args(self, weights, uniforms, out):
        out = self.indexes if out is None else out
        _bank_tensor_check(out, "out", (torch.int32,), (self.n_sets, self.n_particles), self.device)
        ws = self._workspace()
        a = _lib.ResidualResampleBankArgs()
        a.n_sets, a.n_particles = self.n_sets, self.n_particles
        a.weights = weights.data_ptr() if weights is not None else None
        a.uniforms = uniforms.data_ptr() if uniforms is not None else None
        a.indexes, a.n_copies, a.status = out.data_ptr(), self.n_copies.data_ptr(), self.status.data_ptr()
        a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel() * 8
        return a, out

    def residual_prepare(self, weights, out=None):
        """The deterministic part of residual_resample (resampling.py:52-72) for every row: ``out[b, :k_b]``
        (default: ``indexes``), ``n_copies[b] = k_b`` and the per-set cumulative sums in the workspace."""
        _bank_tensor_check(weights, "weights", (torch.float64,), (self.n_sets, self.n_particles), self.device)
        a, out = self._residual_args(weights, None, out)
        with torch.cuda.device(self.device):
            _lib.check(self._lib.bke_residual_resample_bank_prepare(ctypes.byref(a), stream_ptr(self.device)))
        return out

    def residual_search(self, uniforms, out=None):
        """``out[b, k_b:] = searchsorted(cumulative_sum_b, uniforms[b, :M - k_b])`` (resampling.py:74) after
        ``residual_prepare`` on the same plan and ``out``; the rest of each row of ``uniforms`` is not read."""
        _bank_tensor_check(uniforms, "uniforms", (torch.float64,), (self.n_sets, self.n_particles), self.device)
        a, out = self._residual_args(None, uniforms, out)
        with torch.cuda.device(self.device):
            _lib.check(self._lib.bke_residual_resample_bank_search(ctypes.byref(a), stream_ptr(self.device)))
        return out

    def residual(self, weights, uniforms, out=None):
        """residual_resample (resampling.py:27-76) of every row for caller-supplied uniforms: row b uses
        ``uniforms[b, :M - k_b]``.  int32 (B, M); ``raise_if_overflow`` reports a row with k > M."""
        out = self.residual_prepare(weights, out)
        return self.residual_search(uniforms, out)

    def _run(self, weights, u, uniforms, out):
        shape = (self.n_sets, self.n_particles)
        _bank_tensor_check(weights, "weights", (torch.float64,), shape, self.device)
        out = self.indexes if out is None else out
        _bank_tensor_check(out, "out", (torch.int32,), shape, self.device)
        a = _lib.ResampleBankArgs()
        a.n_sets, a.n_particles = self.n_sets, self.n_particles
        a.weights, a.indexes, a.status = weights.data_ptr(), out.data_ptr(), self.status.data_ptr()
        a.u = u.data_ptr() if u is not None else None
        a.uniforms = uniforms.data_ptr() if uniforms is not None else None
        with torch.cuda.device(self.device):
            _lib.check(self._lib.bke_resample_bank(ctypes.byref(a), stream_ptr(self.device)))
        return out

    def systematic(self, weights, u, out=None):
        """indexes[b] for the offsets ``u[b]`` (float64 CUDA tensor [n_sets]; resampling.py:139:
        positions = (u[b] + arange(M)) / M)."""
        _bank_tensor_check(u, "u", (torch.float64,), (self.n_sets,), self.device)
        return self._run(weights, u, None, out)

    def stratified(self, weights, uniforms, out=None):
        """indexes[b] for the per-particle uniforms ``uniforms[b]`` (float64 CUDA tensor [n_sets, M];
        resampling.py:103: positions = (U[b] + arange(M)) / M)."""
        _bank_tensor_check(uniforms, "uniforms", (torch.float64,), (self.n_sets, self.n_particles), self.device)
        return self._run(weights, None, uniforms, out)

    def gather(self, particles, indexes=None, out=None):
        """``out[b] = particles[b][indexes[b]]`` (indexes default: the plan's last result).  No host
        synchronisation: an index outside [0, n_particles) is reported by ``raise_if_bad_index``."""
        indexes = self.indexes if indexes is None else indexes
        if not (isinstance(particles, torch.Tensor) and particles.device == self.device
                and tuple(particles.shape[:2]) == (self.n_sets, self.n_particles)):
            raise ValueError("particles must be a CUDA tensor of shape (%d, %d, ...) on %s"
                             % (self.n_sets, self.n_particles, self.device))
        return _gather_bank(particles, indexes, out, self._err)

    def _gated(self, entry, weights, particles, u, uniforms, threshold):
        shape = (self.n_sets, self.n_particles)
        _bank_tensor_check(weights, "weights", (torch.float64,), shape, self.device)
        if not (isinstance(particles, torch.Tensor) and particles.device == self.device and particles.is_contiguous()
                and particles.dim() >= 2 and tuple(particles.shape[:2]) == shape):
            raise ValueError("particles must be a contiguous tensor of shape (%d, %d, ...) on %s"
                             % (self.n_sets, self.n_particles, self.device))
        if self._neff is None:
            nbytes = int(self._lib.bke_resample_bank_gated_workspace_bytes(self.n_sets))
            self._gated_ws = torch.empty(max((nbytes + 3) // 4, 1), dtype=torch.int32, device=self.device)
            self._neff = torch.empty(self.n_sets, dtype=torch.float64, device=self.device)
            self._resampled = torch.zeros(self.n_sets, dtype=torch.bool, device=self.device)
            if self.n_particles == 0:                     # 1. / np.sum(np.square([])) is inf: nothing resamples
                self._neff.fill_(float("inf"))
        a = _lib.ResampleBankGatedArgs()
        a.n_sets, a.n_particles = self.n_sets, self.n_particles
        a.weights = weights.data_ptr()
        a.u = u.data_ptr() if u is not None else None
        a.uniforms = uniforms.data_ptr() if uniforms is not None else None
        a.threshold = float(self.n_particles / 2 if threshold is None else threshold)
        a.particles = particles.data_ptr()
        a.particle_bytes = (particles.numel() // max(self.n_sets * self.n_particles, 1)) * particles.element_size()
        a.indexes, a.status = self.indexes.data_ptr(), self.status.data_ptr()
        a.neff, a.resampled = self._neff.data_ptr(), self._resampled.data_ptr()
        a.workspace, a.workspace_bytes = self._gated_ws.data_ptr(), self._gated_ws.numel() * 4
        try:
            with torch.cuda.device(self.device):
                _lib.check(entry(ctypes.byref(a), stream_ptr(self.device)))
        except ValueError as e:
            if "shared memory" in str(e):
                raise ValueError("%s; resample larger sets with systematic / stratified and gather_particles_bank"
                                 % e) from None
            raise
        return self._resampled, self._neff

    def resample_if_degenerate(self, weights, particles, u=None, uniforms=None, threshold=None):
        """One particle-filter epoch of every set, resampling only the degenerate ones, in place:

        ``w = w / np.sum(w)``; ``neff = 1. / np.sum(np.square(w))``; where ``neff < threshold`` (default
        ``n_particles / 2``), ``particles[b] = particles[b][systematic_resample(w)]`` for the offset ``u[b]``
        (``stratified_resample`` for ``uniforms[b]``) and ``w = 1 / n_particles``.  The sums are NumPy's
        pairwise sums, so the weights, ``neff`` and the decisions are those of NumPy bit for bit.

        ``weights`` float64 [n_sets, n_particles] and ``particles`` (n_sets, n_particles, ...) of any dtype
        are updated in place; give exactly one of ``u`` float64 [n_sets] and ``uniforms`` float64
        [n_sets, n_particles] (only the rows of resampled sets are read).  Returns the plan's
        ``(resampled bool [n_sets], neff float64 [n_sets])``; ``indexes`` holds the resampled rows' indexes
        and ``status`` is 1 where a resampled set's positions ran past its cumulative sum (the reference's
        IndexError): that set keeps its particles and its normalised weights.

        One set's particle row must fit in one CTA's shared memory (227 KB on the H100).  The first call
        allocates the plan's buffers; later calls allocate nothing and do not synchronise the host, so they
        can be captured in a CUDA graph."""
        if u is not None:
            _bank_tensor_check(u, "u", (torch.float64,), (self.n_sets,), self.device)
        if uniforms is not None:
            _bank_tensor_check(uniforms, "uniforms", (torch.float64,), (self.n_sets, self.n_particles), self.device)
        if (u is None) == (uniforms is None):
            raise ValueError("give exactly one of u (systematic) and uniforms (stratified)")
        return self._gated(self._lib.bke_resample_bank_gated, weights, particles, u, uniforms, threshold)

    def raise_if_overflow(self):
        """IndexError naming the first set whose positions ran past its cumulative sum (host sync)."""
        _raise_first_overflow(self.status, self.n_particles)

    def raise_if_bad_index(self):
        """IndexError if a ``gather`` since the last check met an index outside [0, n_particles) (host sync)."""
        if int(self._err.item()):
            self._err.zero_()
            raise IndexError("index out of bounds for axis 1 with size %d" % self.n_particles)


def _raise_first_overflow(status, n_particles):
    bad = torch.nonzero(status & 1).flatten()
    if bad.numel():
        raise IndexError("set %d: index %d is out of bounds for axis 0 with size %d"
                         % (int(bad[0]), n_particles, n_particles))


def _run_bank(weights, stratified):
    is_torch, w, dev = _weights_on_device(weights)
    if w.dim() != 2:
        raise ValueError("weights must be 2-D (n_sets, n_particles); got shape %s" % (tuple(w.shape),))
    B, M = w.shape
    # the reference's loop draws random() (random(M) stratified) once per row; random(B) and random((B, M))
    # take the same values from the global stream in the same order
    draw = random((B, M)) if stratified else random(B)
    plan = BankResamplePlan(B, M, dev)
    if B and M:
        U = torch.from_numpy(np.ascontiguousarray(draw)).to(dev)
        idx = plan.stratified(w, U) if stratified else plan.systematic(w, U)
        plan.raise_if_overflow()                          # resampling.py:145 (IndexError), first failing row
    else:
        idx = plan.indexes
    return idx if is_torch else idx.cpu().numpy()


def systematic_resample_bank(weights):
    """``systematic_resample`` (resampling.py:117-150) of every row of ``weights[B, M]`` in one launch:
    returns int32 ``(B, M)``, an ndarray for array input, a CUDA tensor for a CUDA tensor.  Seeded with
    ``np.random.seed``, the result and the stream position afterwards equal a Python loop of the
    reference over the rows.  A failing row raises ``IndexError`` naming the first such row, where that
    loop would have stopped; unlike the loop, the bank has by then drawn the uniforms of all B rows."""
    return _run_bank(weights, False)


def stratified_resample_bank(weights):
    """``stratified_resample`` (resampling.py:80-114) of every row of ``weights[B, M]`` in one launch
    (uniforms drawn as ``random((B, M))``); otherwise as ``systematic_resample_bank``."""
    return _run_bank(weights, True)


def _bank_2d(weights):
    is_torch, w, dev = _weights_on_device(weights)
    if w.dim() != 2:
        raise ValueError("weights must be 2-D (n_sets, n_particles); got shape %s" % (tuple(w.shape),))
    B, M = w.shape
    if B and not M:                                       # cumulative_sum[-1] = 1. of row 0, before any draw
        raise IndexError("set 0: index -1 is out of bounds for axis 0 with size 0")
    return is_torch, w, dev, B, M


def multinomial_resample_bank(weights):
    """``multinomial_resample`` (resampling.py:153-176) of every row of ``weights[B, M]``: int64 ``(B, M)``,
    an ndarray for array input, a CUDA tensor for a CUDA tensor.  Draws ``random((B, M))``, the values and
    stream position of a Python loop of the reference over the rows, and returns that loop's result bit
    for bit, NumPy's bracket-carrying ``searchsorted`` included (csrc/resample_bank.cu)."""
    is_torch, w, dev, B, M = _bank_2d(weights)
    draw = random((B, M))
    plan = BankResamplePlan(B, M, dev)
    if B:
        idx = plan.multinomial(w, torch.from_numpy(np.ascontiguousarray(draw)).to(dev))
    else:
        idx = torch.zeros((0, M), dtype=torch.int64, device=dev)
    return idx if is_torch else idx.cpu().numpy()


def residual_resample_bank(weights):
    """``residual_resample`` (resampling.py:27-76) of every row of ``weights[B, M]``: int32 ``(B, M)``, ndarray
    or CUDA tensor like the input.  The deterministic copies and cumulative sums run first on the GPU; the
    copy counts k_b are then read back (one host synchronisation) to draw ``random(M - k_b)`` for every row
    in row order as one draw, which are the values and the stream position of the reference's loop.  A row
    with k_b > M raises ``IndexError`` naming it, after drawing only for the rows before it, as the loop
    does."""
    is_torch, w, dev, B, M = _bank_2d(weights)
    if not B:
        idx = torch.zeros((0, M), dtype=torch.int32, device=dev)
        return idx if is_torch else idx.cpu().numpy()
    plan = BankResamplePlan(B, M, dev)
    plan.residual_prepare(w)
    k = plan.n_copies.cpu().numpy()
    bad = np.flatnonzero(k > M)
    first = int(bad[0]) if bad.size else B
    draw = random(int((M - k[:first]).sum()))
    if first < B:                                         # indexes[k] = i runs off the end (:61)
        raise IndexError("set %d: index %d is out of bounds for axis 0 with size %d" % (first, M, M))
    U = torch.zeros((B, M), dtype=torch.float64, device=dev)
    keep = torch.arange(M, device=dev)[None, :] < torch.from_numpy(M - k).to(dev)[:, None]
    U[keep] = torch.from_numpy(np.ascontiguousarray(draw)).to(dev)     # row b's M - k_b draws, in row order
    idx = plan.residual_search(U)
    return idx if is_torch else idx.cpu().numpy()


def _run_bank_if_degenerate(weights, particles, threshold, stratified):
    w_dev = isinstance(weights, torch.Tensor) and weights.is_cuda
    p_dev = isinstance(particles, torch.Tensor) and particles.is_cuda
    if w_dev != p_dev:
        raise ValueError("weights and particles must both be CUDA tensors or both be arrays")
    if w_dev:
        w, p, dev = weights, particles, weights.device
        if not (w.dtype == torch.float64 and w.is_contiguous() and p.is_contiguous() and p.device == dev):
            raise ValueError("weights must be a contiguous float64 CUDA tensor and particles a contiguous tensor on "
                             "its device (both are updated in place)")
    else:
        if not (isinstance(weights, np.ndarray) and weights.dtype == np.float64 and isinstance(particles, np.ndarray)):
            raise ValueError("weights must be a float64 ndarray and particles an ndarray (both are updated in place)")
        dev = require_cuda(None)
        w = torch.from_numpy(np.ascontiguousarray(weights)).to(dev)
        p = torch.from_numpy(np.ascontiguousarray(particles)).to(dev)
    if w.dim() != 2 or p.dim() < 2 or tuple(p.shape[:2]) != tuple(w.shape):
        raise ValueError("weights must be (n_sets, n_particles) and particles (n_sets, n_particles, ...)")
    B, M = w.shape
    plan = BankResamplePlan(B, M, dev)
    resampled, neff = plan._gated(plan._lib.bke_resample_bank_gated_stats, w, p, None, None, threshold)
    mask = resampled.cpu().numpy()
    n_res = int(mask.sum())
    # the loop draws random() (stratified: random(M)) for each set it resamples, in row order; one draw of
    # random(n_res) (random((n_res, M))) takes the same values and leaves the stream in the same place
    draw = random((n_res, M)) if stratified else random(n_res)
    if n_res:
        rows = torch.from_numpy(np.flatnonzero(mask)).to(dev)
        U = torch.zeros((B, M) if stratified else (B,), dtype=torch.float64, device=dev)
        U[rows] = torch.from_numpy(np.ascontiguousarray(draw)).to(dev)
        plan._gated(plan._lib.bke_resample_bank_gated_apply, w, p, None if stratified else U,
                    U if stratified else None, threshold)
    if not w_dev:
        np.copyto(weights, w.cpu().numpy())
        np.copyto(particles, p.cpu().numpy())
        resampled, neff = mask, neff.cpu().numpy()
    if n_res:
        _raise_first_overflow(plan.status, M)
    return resampled, neff


def systematic_resample_bank_if_degenerate(weights, particles, threshold=None):
    """A particle filter's resampling step on every set of a bank, where it is due, in place::

        w = w / np.sum(w); neff = 1. / np.sum(np.square(w))
        if neff < threshold:                 # default n_particles / 2
            particles[:] = particles[systematic_resample(w)]; w = np.full(M, 1. / M)

    for each row of ``weights[B, M]`` (float64) and ``particles[B, M, ...]`` (any dtype): ndarrays, updated in
    place, or CUDA tensors, updated in place.  Returns ``(resampled bool[B], neff[B])`` of the same kind.
    The sums are NumPy's pairwise sums, so every result is that loop's bit for bit.  Seeded with
    ``np.random.seed``, ``random()`` is drawn for the resampled sets in row order, the values and stream
    position of the loop: the statistics run first and the mask is read back (one host synchronisation).

    A set whose positions run past its cumulative sum keeps its particles and normalised weights, and
    ``IndexError`` names the first such set.  By then every row has been processed and drawn for, where the
    loop would have stopped at that set.  One set's particle row must fit in one CTA's shared memory
    (227 KB on the H100); ``gather_particles_bank`` serves larger sets."""
    return _run_bank_if_degenerate(weights, particles, threshold, False)


def stratified_resample_bank_if_degenerate(weights, particles, threshold=None):
    """As ``systematic_resample_bank_if_degenerate`` with ``stratified_resample``: each resampled set draws
    ``random(M)``, taken for all of them as ``random((n_res, M))``."""
    return _run_bank_if_degenerate(weights, particles, threshold, True)


def _gather_bank(particles, indexes, out, err):
    """particles (B, M, ...) and indexes (B, M) contiguous on one CUDA device; the kernel reads raw rows."""
    if not (isinstance(particles, torch.Tensor) and particles.is_cuda and particles.is_contiguous()
            and particles.dim() >= 2):
        raise ValueError("particles must be a contiguous CUDA tensor of shape (n_sets, n_particles, ...)")
    dev = particles.device
    _bank_tensor_check(indexes, "indexes", (torch.int32, torch.int64), particles.shape[:2], dev)
    B, M = indexes.shape
    row_bytes = (particles.numel() // max(B * M, 1)) * particles.element_size()
    if out is None:
        out = torch.empty_like(particles)
    else:
        _bank_tensor_check(out, "out", (particles.dtype,), particles.shape, dev)
    if B * M and row_bytes:
        with torch.cuda.device(dev):
            _lib.check(_lib.load().bke_gather_rows_bank(B, M, row_bytes, particles.data_ptr(), indexes.data_ptr(),
                                                        1 if indexes.dtype == torch.int64 else 0, out.data_ptr(),
                                                        err.data_ptr(), stream_ptr(dev)))
    return out


def gather_particles_bank(particles, indexes, out=None, check=True):
    """``particles[b][indexes[b]]`` for every set b of a bank, on the GPU: ``particles`` is (B, M, ...) of
    any dtype, ``indexes`` (B, M) int32 or int64 (what the bank resamplers return).  NumPy in -> NumPy out,
    CUDA tensors in -> CUDA tensor out.  Raises IndexError for an index outside [0, M) like NumPy does
    (negative indexes are not wrapped); ``check=False`` skips that test and the host synchronisation it
    costs."""
    is_torch = isinstance(particles, torch.Tensor) and particles.is_cuda
    if is_torch:
        dev = particles.device
        src = particles.contiguous()
    else:
        dev = require_cuda(None)
        src = torch.from_numpy(np.ascontiguousarray(np.asarray(particles))).to(dev)
    if isinstance(indexes, torch.Tensor):
        idx = indexes.to(dev)
    else:
        idx = torch.from_numpy(np.ascontiguousarray(np.asarray(indexes))).to(dev)
    if idx.dtype not in (torch.int32, torch.int64):
        raise IndexError("arrays used as indices must be of integer type")
    if idx.dim() != 2 or src.dim() < 2:
        raise ValueError("particles must be (n_sets, n_particles, ...) and indexes (n_sets, n_particles)")
    idx = idx.contiguous()
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    out = _gather_bank(src, idx, out, err)
    if check and int(err.item()):
        raise IndexError("index out of bounds for axis 1 with size %d" % idx.shape[1])
    return out if is_torch else out.cpu().numpy()
