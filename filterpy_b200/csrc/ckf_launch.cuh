// ckf_launch.cuh — host helpers shared by the pre-built (ckf.cu) and the run-time compiled (ukf_rtc.cu)
// instances of the CKF kernel: parameter block and dynamic shared-memory size.
#pragma once
#include <math.h>
#include "ckf_kernel.cuh"

namespace bke {

// resident CTAs per SM an instance is compiled for (its registers are capped accordingly).  For n >= 6 the
// fused step keeps the drawing posterior (x, U) live through the update, which the UKF does not: 2 in
// fp64 and 3 in fp32 are the highest occupancies at which those instances do not spill (the UKF's 3 / 5
// spill 0.7-1.0 KB / 0.3 KB per thread); smaller states need no cap
constexpr int ckf_occupancy(int n, bool f64)
{
    return n >= 6 ? (f64 ? 2 : 3) : 1;
}

template <typename T>
inline void ckf_fill_params(const bke_ckf_args &a, ckfk::CkfP<T> &p)
{
    p.N = a.n_filters; p.flags = a.flags; p.dt = (T)a.dt;
    p.root_n = (T)sqrt((double)a.dim_x);
    p.x = (const T *)a.x; p.P = (const T *)a.P; p.Q = (const T *)a.Q; p.R = (const T *)a.R;
    p.F = (const T *)a.F; p.H = (const T *)a.H; p.z = (const T *)a.z;
    p.sQ = a.Q_stride; p.sR = a.R_stride; p.sF = a.F_stride; p.sH = a.H_stride;
    p.valid = a.z_valid;
    p.x_out = (T *)a.x_out; p.P_out = (T *)a.P_out; p.x_prior = (T *)a.x_prior; p.P_prior = (T *)a.P_prior;
    p.K = (T *)a.K; p.y = (T *)a.y; p.S = (T *)a.S; p.SI = (T *)a.SI; p.ll = (T *)a.log_likelihood;
    p.status = a.status;
    p.sigmas_f = (T *)a.sigmas_f;
    p.fx_args = nullptr; p.hx_args = nullptr; p.s_fx_args = 0; p.s_hx_args = 0;
}

// the slab (measurement-space points + parked prior, or one P / Q tile) and the staged F / H
template <typename T>
inline size_t ckf_smem_bytes(int N, int M, bool fx_linear, bool F_shared, bool hx_linear, bool H_shared)
{
    const int PADP = (N * N) | 1;
    const int zpark = 2 * N * M + N * (N + 1) / 2;
    size_t smem = sizeof(T) * (size_t)(zpark > PADP ? zpark : PADP) * ukfk::UB;
    if (fx_linear) smem += sizeof(T) * (F_shared ? N * N : N * N * ukfk::UB);
    if (hx_linear) smem += sizeof(T) * (H_shared ? M * N : M * N * ukfk::UB);
    return smem;
}

inline bool ckf_has_extras(const bke_ckf_args &a)
{
    return a.x_prior || a.P_prior || a.K || a.y || a.S || a.SI || a.log_likelihood;
}

}  // namespace bke
