// sigma_launch.cuh — host side shared by the sigma-point families (UKF, CKF, EnKF), pre-built (ukf.cu,
// ukf_simplex.cu, ukf_score.cu, ckf.cu, enkf.cu) and run-time compiled (ukf_rtc.cu): the instance table, parameter
// blocks, dynamic shared-memory sizes, grids and occupancy caps.  (The launch, launch_kernel, and the
// argument checks, validate_*, live in api.cu.)
#pragma once
#include <math.h>
#include "ckf_kernel.cuh"
#include "enkf_kernel.cuh"
#include "ukf_score_kernel.cuh"

// The pre-built (dim_x, dim_z, fx, hx) instances of every family, in dispatch order.  X(n, m, fx, hx) per row.
#define BKE_SIGMA_INSTANCES(X)                     \
    X(6, 3, BKE_FX_CONST_VEL, BKE_HX_RANGE_AZ_EL)   \
    X(6, 3, BKE_FX_CONST_VEL, BKE_HX_LINEAR)        \
    X(6, 3, BKE_FX_LINEAR, BKE_HX_LINEAR)           \
    X(6, 3, BKE_FX_LINEAR, BKE_HX_RANGE_AZ_EL)      \
    X(4, 2, BKE_FX_CONST_VEL, BKE_HX_RANGE_BEARING) \
    X(4, 2, BKE_FX_LINEAR, BKE_HX_RANGE_BEARING)    \
    X(4, 2, BKE_FX_CONST_VEL, BKE_HX_LINEAR)        \
    X(4, 2, BKE_FX_LINEAR, BKE_HX_LINEAR)           \
    X(1, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)           \
    X(2, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)           \
    X(2, 1, BKE_FX_CONST_VEL, BKE_HX_LINEAR)        \
    X(2, 2, BKE_FX_LINEAR, BKE_HX_LINEAR)           \
    X(3, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)           \
    X(3, 3, BKE_FX_LINEAR, BKE_HX_LINEAR)           \
    X(4, 4, BKE_FX_LINEAR, BKE_HX_LINEAR)

namespace bke {

// a dispatch row: launch_inst<T, n, m, fx, hx>(a, s) when the args `a` ask for that instance
#define BKE_SIGMA_DISPATCH_ROW(NN, MM, FXX, HXX) \
    if (a.dim_x == NN && a.dim_z == MM && a.fx_model == FXX && a.hx_model == HXX) return launch_inst<T, NN, MM, FXX, HXX>(a, s);

// resident CTAs per SM an instance is compiled for (its registers are capped accordingly): for n >= 6,
// 3 in fp64 and 5 in fp32; smaller states need no cap.  A simplex instance (n + 1 dense offset rows live
// through the update) whose hx is not a range model takes 2 / 4: at 3 / 5 ptxas spilled 136-200 B in the
// 6/3 linear-hx ones, at 2 / 4 none; the range models fit 3 / 5 without a spill
constexpr int ukf_occupancy(int n, bool f64, bool simplex = false, bool range_hx = false)
{
    return n >= 6 ? ((simplex && !range_hx) ? (f64 ? 2 : 4) : (f64 ? 3 : 5)) : 1;
}

// The CKF: for n >= 6 the fused step keeps the drawing posterior (x, U) live through the update, which the
// UKF does not: 2 in fp64 and 3 in fp32 are the highest occupancies at which those instances do not spill
// (the UKF's 3 / 5 spill 0.7-1.0 KB / 0.3 KB per thread); smaller states need no cap
constexpr int ckf_occupancy(int n, bool f64)
{
    return n >= 6 ? (f64 ? 2 : 3) : 1;
}

// the fields the UKF, CKF and EnKF parameter blocks share (no user-model arguments: set_user_args)
template <typename T, typename Args, typename Prm>
inline void fill_common(const Args &a, Prm &p)
{
    p.N = a.n_filters; p.flags = a.flags; p.dt = (T)a.dt;
    p.x = (const T *)a.x; p.P = (const T *)a.P; p.Q = (const T *)a.Q; p.R = (const T *)a.R;
    p.F = (const T *)a.F; p.H = (const T *)a.H; p.z = (const T *)a.z;
    p.sQ = a.Q_stride; p.sR = a.R_stride; p.sF = a.F_stride; p.sH = a.H_stride;
    p.valid = a.z_valid;
    p.x_out = (T *)a.x_out; p.P_out = (T *)a.P_out; p.x_prior = (T *)a.x_prior; p.P_prior = (T *)a.P_prior;
    p.K = (T *)a.K; p.S = (T *)a.S; p.SI = (T *)a.SI;
    p.status = a.status;
    p.fx_args = nullptr; p.hx_args = nullptr; p.s_fx_args = 0; p.s_hx_args = 0;
}

// the parameter vectors of BKE_FX_USER / BKE_HX_USER (run-time compiled instances)
template <typename T, typename Prm>
inline void set_user_args(Prm &p, const void *fx_args, int64_t s_fx, const void *hx_args, int64_t s_hx)
{
    p.fx_args = (const T *)fx_args; p.s_fx_args = s_fx;
    p.hx_args = (const T *)hx_args; p.s_hx_args = s_hx;
}

// the point set's scale and weights: Merwe's (alpha, beta, kappa) or the simplex set's (BKE_UKF_SIMPLEX in a.flags)
template <typename T, typename Args, typename Prm>
inline void ukf_set_weights(const Args &a, int N, Prm &p)
{
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
}

template <typename T>
inline void ukf_fill_params(const bke_ukf_args &a, int N, ukfk::UkfP<T> &p)
{
    fill_common<T>(a, p);
    p.y = (T *)a.y; p.ll = (T *)a.log_likelihood;
    ukf_set_weights<T>(a, N, p);
}

// the UKF score's parameter block (no user-model arguments: set_user_args)
template <typename T>
inline void ukf_score_fill_params(const bke_ukf_score_args &a, ukfk::UkfScoreP<T> &p)
{
    p.N = a.n_filters; p.K = a.n_candidates;
    p.di = ukfk::UB / p.K; p.dk = ukfk::UB - p.di * p.K;
    ukf_set_weights<T>(a, a.dim_x, p);
    p.x = (const T *)a.x; p.P = (const T *)a.P; p.R = (const T *)a.R; p.H = (const T *)a.H; p.z = (const T *)a.z;
    p.sR = a.R_stride; p.sH = a.H_stride; p.zt = a.z_track_stride; p.zc = a.z_cand_stride;
    p.valid = a.z_valid;
    p.zhat = (T *)a.zhat; p.y = (T *)a.y; p.d2 = (T *)a.d2; p.maha = (T *)a.mahalanobis;
    p.ll = (T *)a.log_likelihood; p.lk = (T *)a.likelihood; p.status = a.status;
    p.hx_args = nullptr; p.s_hx_args = 0;
}

// the UKF score's dynamic shared memory: the hx slab (or one P tile), the tile's slots and the staged H
template <typename T>
inline size_t ukf_score_smem_bytes(int N, int M, bool simplex, bool hx_linear, bool H_shared)
{
    const int PADP = (N * N) | 1, zs = (simplex ? N + 1 : 2 * N + 1) * M;
    size_t smem = sizeof(T) * ((size_t)(zs > PADP ? zs : PADP) + (size_t)(M + M * M + 1)) * ukfk::UB;
    if (hx_linear) smem += sizeof(T) * (H_shared ? M * N : M * N * ukfk::UB);
    return smem;
}

template <typename T>
inline void ckf_fill_params(const bke_ckf_args &a, ckfk::CkfP<T> &p)
{
    fill_common<T>(a, p);
    p.y = (T *)a.y; p.ll = (T *)a.log_likelihood;
    p.root_n = (T)sqrt((double)a.dim_x);
    p.sigmas_f = (T *)a.sigmas_f;
}

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
    fill_common<T>(a, p);
    p.Nm = a.n_members;
    p.seed = a.seed; p.counter = a.counter;
    p.onchip = enkf_smem_bytes(a.dim_x, a.n_members, sizeof(T)) != 0;
    p.sig_in = (const T *)a.sigmas; p.sig_out = (T *)a.sigmas_out;
}

// the slab (measurement-space sigma points + parked prior, or one P / Q tile) and the staged F / H;
// n_sigmas: 2N + 1 (Merwe), N + 1 (simplex) or 2N (cubature)
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

inline unsigned ukf_grid(int64_t n_filters) { return (unsigned)((n_filters + ukfk::UB - 1) / ukfk::UB); }

inline unsigned enkf_grid(int64_t n_filters) { return (unsigned)((n_filters + enkfk::EW - 1) / enkfk::EW); }

// whether a UKF / CKF step writes any optional output (selects the instance that has them compiled in)
template <typename Args>
inline bool has_extras(const Args &a)
{
    return a.x_prior || a.P_prior || a.K || a.y || a.S || a.SI || a.log_likelihood;
}

// the EnKF has no y and no log-likelihood
inline bool enkf_has_extras(const bke_enkf_args &a)
{
    return a.x_prior || a.P_prior || a.K || a.S || a.SI;
}

}  // namespace bke
