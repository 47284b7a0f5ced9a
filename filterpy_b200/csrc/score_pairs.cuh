// score_pairs.cuh — phase B of the measurement scores: the work on one track x candidate pair, shared by
// bke_score_measurements (score.cu) and bke_ukf_score (ukf_score_kernel.cuh).  Free of host headers: NVRTC compiles
// it into the run-time UKF models too.
//
// A tile's phase A leaves each track's slot in shared memory: zhat[m], SI[m*m] (S^-1, or NaN) and log|det S|.  Each
// kernel walks its tile's nt * K outputs in pair order (one contiguous range: coalesced stores for any K) and calls
// pair_reg / pair_any per pair:
//   y = residual(z_ik, zhat);  d2 = y' SI y;  ll = -0.5 (d2 + log|det S| + m log 2pi)
// The parameter block PP names its fields K, z, zt, zc (z_ik = z + i zt + k zc), valid, and the outputs y, d2, maha,
// ll, lk (NULL = not wanted).
#pragma once
#include "bke_internal.cuh"

namespace bke {
namespace scorek {

template <typename T>
__device__ __forceinline__ T qnan() { return T(__int_as_float(0x7fc00000)); }

// the track's slot in the tile: zhat[m], SI[m*m], log|det S|
__host__ __device__ __forceinline__ int slot_words(int m) { return m + m * m + 1; }

template <typename T>
__device__ __forceinline__ T log_dbl_min() { return T(-708.39641853226408); }      // log(sys.float_info.min)

// The residual of pair_reg: SubResidual is y = z - zhat (the linear scores, and a UKF without residual_z), written out
// in pair_reg itself (called through an apply function it changed score.cu's 1/1 fp32 code); any other type R forms
// it with R::apply(z_ik, zhat, y)
struct SubResidual {};
template <typename R> struct is_sub_residual { static constexpr bool value = false; };
template <> struct is_sub_residual<SubResidual> { static constexpr bool value = true; };

// the scores of one pair from d2 = y' SI y (valid) and write-out
template <typename T, typename PP>
__device__ __forceinline__ void put_scores(const PP &p, int64_t pr, bool valid, T q, T logdet, int m)
{
    const T ll = valid ? T(-0.5) * (q + logdet + T(m) * T(LOG_2PI)) : log_dbl_min<T>();
    if (!valid) q = T(0);
    if (p.d2) p.d2[pr] = q;
    if (p.maha) p.maha[pr] = sqrt(q);
    if (p.ll) p.ll[pr] = ll;
    if (p.lk) p.lk[pr] = exp(ll);
}

// one pair, m = M in registers, with the residual Res
template <typename T, int M, typename Res, typename PP>
__device__ __forceinline__ void pair_reg(const PP &p, int64_t f, int64_t k, const T *slot, bool cov)
{
    const int64_t pr = f * p.K + k;
    const bool valid = !p.valid || p.valid[pr];
    T y[M];
    if (valid) {
        const T *z = p.z + f * p.zt + k * p.zc;
        if constexpr (is_sub_residual<Res>::value) {
#pragma unroll
            for (int a = 0; a < M; a++) y[a] = z[a] - slot[a];
        } else {
            Res::apply(z, slot, y);
        }
    } else {
#pragma unroll
        for (int a = 0; a < M; a++) y[a] = T(0);
    }
    if (p.y) {
#pragma unroll
        for (int a = 0; a < M; a++) p.y[pr * M + a] = y[a];
    }
    if (!cov) return;
    const T *SI = slot + M;
    T q = T(0);
#pragma unroll
    for (int a = 0; a < M; a++) {
        T s = T(0);
#pragma unroll
        for (int b = 0; b < M; b++) s += SI[a * M + b] * y[b];
        q += y[a] * s;
    }
    put_scores<T>(p, pr, valid, q, slot[M + M * M], M);
}

// one pair, any m: y_a is formed again where it is needed (z_ik stays in L1)
template <typename T, typename PP>
__device__ __forceinline__ void pair_any(const PP &p, int64_t f, int64_t k, const T *slot, bool cov, int m)
{
    const int64_t pr = f * p.K + k;
    const bool valid = !p.valid || p.valid[pr];
    const T *z = p.z + f * p.zt + k * p.zc;
    if (p.y)
        for (int a = 0; a < m; a++) p.y[pr * m + a] = valid ? z[a] - slot[a] : T(0);
    if (!cov) return;
    const T *SI = slot + m;
    T q = T(0);
    if (valid)
        for (int a = 0; a < m; a++) {
            T s = T(0);
            for (int b = 0; b < m; b++) s += SI[a * m + b] * (z[b] - slot[b]);
            q += (z[a] - slot[a]) * s;
        }
    put_scores<T>(p, pr, valid, q, slot[m + m * m], m);
}

}  // namespace scorek
}  // namespace bke
