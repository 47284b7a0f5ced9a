"""Device-memory plumbing shared by the host-side mirrors (torch is used for allocation, streams
and host<->device copies only; all arithmetic happens in libbke.so)."""
import ctypes

import numpy as np
import torch

from . import _lib

_TORCH = {np.dtype(np.float32): torch.float32, np.dtype(np.float64): torch.float64}


def resolve_dtype(dtype):
    if isinstance(dtype, torch.dtype):
        if dtype not in (torch.float32, torch.float64):
            raise ValueError("dtype must be float32 or float64")
        return dtype
    return _TORCH[np.dtype(dtype)]


def bke_dtype(tdtype):
    return _lib.BKE_F32 if tdtype == torch.float32 else _lib.BKE_F64


def require_cuda(device):
    """Resolve the device; fail loudly when no GPU is present (no CPU fallback)."""
    if not torch.cuda.is_available():
        raise _lib.BkeError("filterpy_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    dev = torch.device(device if device is not None else "cuda")
    if dev.type != "cuda":
        raise ValueError("device must be a CUDA device")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def to_dev(a, dtype, device):
    """numpy / list / scalar / torch tensor -> contiguous device tensor of `dtype`."""
    if isinstance(a, torch.Tensor):
        # a pinned host tensor is copied asynchronously on the current stream (stream-ordered with the
        # kernels that consume it); the caller must not overwrite it before that stream has moved on
        nb = (not a.is_cuda) and a.is_pinned()
        return a.to(device=device, dtype=dtype, non_blocking=nb).contiguous()
    arr = np.ascontiguousarray(np.asarray(a, dtype=np.float64 if dtype == torch.float64 else np.float32))
    return torch.from_numpy(arr).to(device)


def ptr(t):
    return None if t is None else t.data_ptr()


def stream_ptr(device):
    return torch.cuda.current_stream(device).cuda_stream


def _capture_nodes(stream):
    n = ctypes.c_int64()
    _lib.check(_lib.load().bke_capture_node_count(stream.cuda_stream, ctypes.byref(n)))
    return n.value


class StepGraph(object):
    """A CUDA graph of a fixed sequence of engine calls (e.g. ``kf.predict(); kf.update(z_buf)`` for a
    ring of measurement buffers).  Replaying it re-runs exactly those kernels on the same device
    buffers with one launch: the inner loop of a tracker that refills ``z_buf`` every epoch pays no
    per-kernel launch latency.  Capture needs calls that neither allocate nor synchronise, i.e. banks
    built with ``diagnostics=False`` and device-resident inputs.  One exception to "the same device
    buffers": a 4/2 float32 bank with symmetric per-filter Q and R is captured reading a packed copy
    of them, so its Q and R are frozen at capture (``KalmanFilter.capture``); re-capture after
    changing them.

    ``nodes`` is the number of graph nodes ``fn`` recorded.  ``launches`` and ``fused_steps`` are set by
    ``KalmanFilter.capture``: the bank's kernel launches per replay, and how many predict+update steps
    those launches run as fused rings (0: one launch per step)."""

    launches = None
    fused_steps = 0

    def __init__(self, fn, device, warmup=2):
        side = torch.cuda.Stream(device)
        side.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(side):
            for _ in range(warmup):           # lazy one-time work (function attributes, tensor maps) happens here
                fn()
        torch.cuda.current_stream(device).wait_stream(side)
        torch.cuda.synchronize(device)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=side):
            before = _capture_nodes(side)
            fn()
            self.nodes = _capture_nodes(side) - before

    def replay(self):
        self.graph.replay()
