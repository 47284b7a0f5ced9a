// enkf_launch.cuh — host helpers shared by the pre-built (enkf.cu) and the run-time compiled (ukf_rtc.cu)
// instances of the EnKF kernel: parameter block, grid and dynamic shared-memory size.
#pragma once
#include "enkf_kernel.cuh"

namespace bke {

// A CTA stages its EW ensembles in shared memory when they fit in this many bytes; larger ensembles run
// their passes over the output array (enkf_kernel.cuh).
constexpr size_t ENKF_SMEM_MAX = 64 * 1024;

inline size_t enkf_smem_bytes(int n, int n_members, size_t elem)
{
    const size_t b = (size_t)enkfk::EW * (size_t)n_members * (size_t)(n | 1) * elem;
    return b <= ENKF_SMEM_MAX ? b : 0;
}

template <typename T>
inline void enkf_fill_params(const bke_enkf_args &a, enkfk::EnkfP<T> &p)
{
    p.N = a.n_filters; p.Nm = a.n_members; p.flags = a.flags;
    p.seed = a.seed; p.counter = a.counter;
    p.onchip = enkf_smem_bytes(a.dim_x, a.n_members, sizeof(T)) != 0;
    p.dt = (T)a.dt;
    p.x = (const T *)a.x; p.P = (const T *)a.P; p.Q = (const T *)a.Q; p.R = (const T *)a.R;
    p.F = (const T *)a.F; p.H = (const T *)a.H; p.z = (const T *)a.z;
    p.sQ = a.Q_stride; p.sR = a.R_stride; p.sF = a.F_stride; p.sH = a.H_stride;
    p.valid = a.z_valid;
    p.sig_in = (const T *)a.sigmas; p.sig_out = (T *)a.sigmas_out;
    p.x_out = (T *)a.x_out; p.P_out = (T *)a.P_out; p.x_prior = (T *)a.x_prior; p.P_prior = (T *)a.P_prior;
    p.K = (T *)a.K; p.S = (T *)a.S; p.SI = (T *)a.SI;
    p.status = a.status;
    p.fx_args = nullptr; p.hx_args = nullptr; p.s_fx_args = 0; p.s_hx_args = 0;
}

inline bool enkf_has_extras(const bke_enkf_args &a)
{
    return a.x_prior || a.P_prior || a.K || a.S || a.SI;
}

inline unsigned enkf_grid(int64_t n_filters)
{
    return (unsigned)((n_filters + enkfk::EW - 1) / enkfk::EW);
}

}  // namespace bke
