// ukf_launch.cuh — host helpers shared by the pre-built (ukf.cu) and the run-time compiled (ukf_rtc.cu)
// instances of the UKF kernel: parameter block and dynamic shared-memory size.
#pragma once
#include "ukf_kernel.cuh"

namespace bke {

// resident CTAs per SM an instance is compiled for (its registers are capped accordingly): for n >= 6,
// 3 in fp64 and 5 in fp32; smaller states need no cap.  A simplex instance (n + 1 dense offset rows live
// through the update) whose hx is not a range model takes 2 / 4: at 3 / 5 ptxas spilled 136-200 B in the
// 6/3 linear-hx ones, at 2 / 4 none; the range models fit 3 / 5 without a spill
constexpr int ukf_occupancy(int n, bool f64, bool simplex = false, bool range_hx = false)
{
    return n >= 6 ? ((simplex && !range_hx) ? (f64 ? 2 : 4) : (f64 ? 3 : 5)) : 1;
}

template <typename T>
inline void ukf_fill_params(const bke_ukf_args &a, int N, ukfk::UkfP<T> &p)
{
    p.N = a.n_filters; p.flags = a.flags; p.dt = (T)a.dt;
    if (a.flags & BKE_UKF_SIMPLEX) {                                        // sigma_points.py:516-522
        p.scale = T(1);
        p.wm0 = p.wc0 = p.wi = (T)(1. / (N + 1));
    } else {
        const double lambda_ = a.alpha * a.alpha * (N + a.kappa) - N;     // sigma_points.py:167
        const double c = .5 / (N + lambda_);
        p.scale = (T)(lambda_ + N);
        p.wm0 = (T)(lambda_ / (N + lambda_));
        p.wc0 = (T)(lambda_ / (N + lambda_) + (1 - a.alpha * a.alpha + a.beta));
        p.wi = (T)c;
    }
    p.x = (const T *)a.x; p.P = (const T *)a.P; p.Q = (const T *)a.Q; p.R = (const T *)a.R;
    p.F = (const T *)a.F; p.H = (const T *)a.H; p.z = (const T *)a.z;
    p.sQ = a.Q_stride; p.sR = a.R_stride; p.sF = a.F_stride; p.sH = a.H_stride;
    p.valid = a.z_valid;
    p.x_out = (T *)a.x_out; p.P_out = (T *)a.P_out; p.x_prior = (T *)a.x_prior; p.P_prior = (T *)a.P_prior;
    p.K = (T *)a.K; p.y = (T *)a.y; p.S = (T *)a.S; p.SI = (T *)a.SI; p.ll = (T *)a.log_likelihood;
    p.status = a.status;
    p.fx_args = nullptr; p.hx_args = nullptr; p.s_fx_args = 0; p.s_hx_args = 0;
}

// the slab (measurement-space sigma points + parked prior, or one P / Q tile) and the staged F / H;
// n_sigmas: 2N + 1 (Merwe) or N + 1 (simplex)
template <typename T>
inline size_t ukf_smem_bytes(int N, int M, int n_sigmas, bool fx_linear, bool F_shared, bool hx_linear, bool H_shared)
{
    const int PADP = (N * N) | 1;
    const int zpark = n_sigmas * M + N * (N + 1) / 2;
    size_t smem = sizeof(T) * (size_t)(zpark > PADP ? zpark : PADP) * ukfk::UB;
    if (fx_linear) smem += sizeof(T) * (F_shared ? N * N : N * N * ukfk::UB);
    if (hx_linear) smem += sizeof(T) * (H_shared ? M * N : M * N * ukfk::UB);
    return smem;
}

}  // namespace bke
