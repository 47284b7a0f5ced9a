"""``torch.ops.bke.*`` — the engine's C-ABI (include/bke.h) as PyTorch operators on CUDA tensors.

The same symbols exposed as torch.ops.* via a C++ extension for zero-copy CUDA tensors.
``load()`` builds (first use, g++ against the installed PyTorch) and loads
``filterpy_b200/_C/libbke_torch_ops.so``, which links ``libbke.so``; afterwards

    x, P = torch.ops.bke.kf_step(x, P, F, H, Q, R, z)              # kalman_filter.py:437-561 for a bank
    x, P = torch.ops.bke.kf_predict(x, P, F, Q)                    # :437-482
    x, P = torch.ops.bke.kf_step_correlated(x, P, F, H, Q, R, M, z)   # predict + update_correlated, :670-752
    x, P = torch.ops.bke.kf_update_rows(x, P, F, H, Q, R, z_i, start)  # predict + update_sequential, :754-824
    x, P = torch.ops.bke.ukf_step(x, P, Q, R, z, dt, alpha, beta, kappa, fx_model, hx_model)   # UKF.py:364-491
    x, P = torch.ops.bke.ukf_step(..., simplex=True)               # the same on SimplexSigmaPoints(n)
    x, P = torch.ops.bke.ckf_step(x, P, Q, R, z, dt, fx_model, hx_model)   # CubatureKalmanFilter.py:292-389
    x, P, s = torch.ops.bke.enkf_step(x, P, sigmas, Q, R, z, dt, fx_model, hx_model, seed, counter)   # ensemble_kalman_filter.py:218-290
    x, L = torch.ops.bke.srkf_step(x, L, F, H, Lq, Lr, z)          # square_root.py:172-248 (L = P1_2)
    x, P_inv, ni, status = torch.ops.bke.if_step(x, P_inv, ni, F, F_inv, Q, H, R_inv, z)   # information_filter.py:178-289
    x, dx, ddx, n, res, pred = torch.ops.bke.poly_filter(x, dx, ddx, n, z, g, h, k, dt, dt2, hdt2, family, order, batch)
                                                                   # gh_filter.py, least_squares.py, fading_memory.py
    ll, d = torch.ops.bke.score_measurements(z, x, None, P, None, H, R, None, ["log_likelihood", "mahalanobis"])
                                                                   # stats.py:64-154, N tracks x K candidates z[N|1, K, m]
    ll, d, status = torch.ops.bke.ukf_score_measurements(x, P, R, z, alpha, beta, kappa, hx_model)
                                                                   # UKF update(z) log_likelihood / mahalanobis per candidate
    means, covs, means_p, covs_p, mus = torch.ops.bke.imm_batch_filter(xs, Ps, Fs, Qs, Hs, Rs, alpha_sqs, Ss, lls, mu, cbar,
                                                                       trans, zs, valid)   # IMMEstimator.batch_filter
    xs, xhat = torch.ops.bke.fls_smooth_batch(x, P, F, H, Q, R, zs, N)   # fixed_lag_smoother.py:217-311
    idx  = torch.ops.bke.systematic_resample(weights, u)           # resampling.py:117-150 (int32, bit-exact)
    idx  = torch.ops.bke.stratified_resample(weights, uniforms)    # resampling.py:80-114
    idx  = torch.ops.bke.systematic_resample_bank(weights, u)      # every row of weights[B, M], u[B]
    idx  = torch.ops.bke.stratified_resample_bank(weights, uniforms)   # uniforms[B, M]
    idx  = torch.ops.bke.multinomial_resample_bank(weights, uniforms)  # int64, resampling.py:153-176 per row
    idx  = torch.ops.bke.residual_resample_bank(weights, uniforms)     # row b uses uniforms[b, :M - k_b]
    res, neff = torch.ops.bke.systematic_resample_bank_if_degenerate(weights, particles, u, threshold)
    res, neff = torch.ops.bke.stratified_resample_bank_if_degenerate(weights, particles, uniforms, threshold)
                                     # normalise, neff, resample + gather the sets with neff < threshold, in place

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
