"""``torch.ops.bke.*`` — the engine's C-ABI (include/bke.h) as PyTorch operators on CUDA tensors.

The same symbols exposed as torch.ops.* via a C++ extension for zero-copy CUDA tensors.
``load()`` builds (first use, g++ against the installed PyTorch) and loads
``filterpy_b200/_C/libbke_torch_ops.so``, which links ``libbke.so``; afterwards

    x, P = torch.ops.bke.kf_step(x, P, F, H, Q, R, z)              # kalman_filter.py:437-561 for a bank
    x, P = torch.ops.bke.kf_predict(x, P, F, Q)                    # :437-482
    x, P = torch.ops.bke.ukf_step(x, P, Q, R, z, dt, alpha, beta, kappa, fx_model, hx_model)   # UKF.py:364-491
    x, P = torch.ops.bke.ckf_step(x, P, Q, R, z, dt, fx_model, hx_model)   # CubatureKalmanFilter.py:292-389
    x, L = torch.ops.bke.srkf_step(x, L, F, H, Lq, Lr, z)          # square_root.py:172-248 (L = P1_2)
    idx  = torch.ops.bke.systematic_resample(weights, u)           # resampling.py:117-150 (int32, bit-exact)
    idx  = torch.ops.bke.stratified_resample(weights, uniforms)    # resampling.py:80-114

Models are shared by the bank when 2-D (stride 0) and per filter when 3-D.  Only the CUDA backend is
registered: CPU tensors raise ``NotImplementedError`` (no CPU fallback).  The operators run on the
current CUDA stream and allocate their outputs (and the resampling workspace) through PyTorch's allocator.
"""
import torch

from .. import _build

_loaded = False


def load():
    global _loaded
    if not _loaded:
        torch.ops.load_library(_build.build_torch_ops())
        _loaded = True
    return torch.ops.bke
