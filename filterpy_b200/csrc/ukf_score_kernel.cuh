// ukf_score_kernel.cuh — measurement scores of N UKF tracks against K candidates each (bke_ukf_score, host side in
// ukf_score.cu).  Free of host headers: nvcc compiles the pre-built instances and NVRTC the run-time UKF models
// (ukf_rtc.cu) around user hx / hooks.
//
// For track i and candidate z_ik: what the reference's UnscentedKalmanFilter reports as log_likelihood and
// mahalanobis right after update(z_ik) from the track's current (x, P) (UKF.py:459-477, 742-777), without touching
// the track:
//   sigma points of (x, P) (UKF.py:407);  Zs = hx(Xs);  (zhat, S) = UT(Zs, Wm, Wc, R, z_mean_fn, residual_z)
//   y = residual_z(z_ik, zhat);  d2 = y' S^-1 y;  ll = -0.5 (d2 + log|det S| + m log 2pi)
// One CTA of UB threads per tile of UB tracks:
//   phase A  one thread per track: the step's measurement half (meas_ut, ukf_kernel.cuh) leaves zhat, S^-1 and
//            log|det S| in the track's slot of the tile (score_pairs.cuh); a failed Cholesky (BKE_STATUS_NOT_PD) or a
//            singular S (BKE_STATUS_SINGULAR_S) stores NaN instead, which makes every valid score of the track NaN.
//   phase B  score.cu's coalesced walk over the tile's nt * K pairs with score_pairs.cuh's per-pair work, y in
//            registers, with residual_z where the model has the hook.
#pragma once
#include "ukf_kernel.cuh"
#include "score_pairs.cuh"

namespace bke {
namespace ukfk {

template <typename T>
struct UkfScoreP {
    int64_t N, K;
    int64_t di, dk;                  // the pair walk's step: UB = di * K + dk pairs
    T scale;                         // n + lambda (1 for the simplex set)
    T wm0, wc0, wi;
    const T *x, *P, *R, *H, *z;
    int64_t sR, sH, zt, zc;
    const uint8_t *valid;
    T *zhat, *y, *d2, *maha, *ll, *lk;
    int32_t *status;
    const T *hx_args;                // BKE_HX_USER: the parameter vectors handed to hx
    int64_t s_hx_args;
};

// y = residual_z(z_ik, zhat) (UKF.py:477)
struct HookResidualZ {
    template <typename T, int M>
    static __device__ __forceinline__ void apply(const T *z, const T *zhat, T (&y)[M])
    {
        T zv[M], zh[M];
#pragma unroll
        for (int a = 0; a < M; a++) { zv[a] = z[a]; zh[a] = zhat[a]; }
        bke_hook_residual_z<T>(zv, zh, y);
    }
};

template <bool HOOK> struct ZResidual { using type = scorek::SubResidual; };
template <> struct ZResidual<true> { using type = HookResidualZ; };

// SPX: the simplex point set instead of Merwe's (as ukf_kernel)
template <typename T, int N, int M, int HX, int OCC, bool SPX>
__global__ void __launch_bounds__(UB, OCC) ukf_score_kernel(const UkfScoreP<T> p)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int NS = SPX ? N + 1 : 2 * N + 1;
    constexpr int PADP = (N * N) | 1;                        // odd per-filter stride of the P slab
    constexpr int PER = M + M * M + 1;                       // a track's slot: zhat, S^-1, log|det S|
    constexpr int SLAB = (NS * M > PADP ? NS * M : PADP) * UB;
    T *zs = reinterpret_cast<T *>(smem_raw);                 // [NS*M][UB]: hx of the points; first the P staging slab
    T *tile = zs + SLAB;                                     // [UB][PER]
    T *Hs = tile + UB * PER;                                 // [M*N] or [M*N][UB]
    const int tid = threadIdx.x;
    const int64_t tile0 = (int64_t)blockIdx.x * UB, f = tile0 + tid;
    const bool live = f < p.N;
    const int64_t fc = live ? f : p.N - 1;                   // clamp: dead threads redo the last track
    const int cnt = (int)((p.N - tile0) < UB ? (p.N - tile0) : UB);
    const int tl = live ? tid : cnt - 1;

    int hstride = 1, hoff = 0;
    if (HX == BKE_HX_LINEAR) {
        if (p.sH == 0) { for (int e = tid; e < M * N; e += UB) Hs[e] = p.H[e]; }
        else {
            for (int e = 0; e < M * N; e++) Hs[e * UB + tid] = p.H[fc * p.sH + e];
            hstride = UB; hoff = tid;
        }
    }
    const T *Hp = Hs + hoff;
    const T *hxa = (HX == BKE_HX_USER && p.hx_args) ? p.hx_args + fc * p.s_hx_args : nullptr;
    T x[N], P[N][N];
#pragma unroll
    for (int i = 0; i < N; i++) x[i] = p.x[fc * N + i];
    slab_load<T, N * N, PADP>(zs, p.P + tile0 * N * N, cnt);
    __syncthreads();
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) P[i][j] = zs[tl * PADP + i * N + j];
    __syncthreads();                                         // the slab now holds hx(sigma points)

    int st = BKE_STATUS_OK;
    T U[SPX ? N + 1 : N][N], zm[M], S[M][M], SI[M][M], logdet;
    const bool ok = meas_ut<T, N, M, HX, SPX>(p, x, P, U, zs, tid, Hp, hstride, hxa, st, zm, S, SI, logdet,
        [] {},
        [&](T (&Rv)[M][M]) {
            const T *Rf = p.R + fc * p.sR;
#pragma unroll
            for (int a = 0; a < M; a++)
#pragma unroll
                for (int b = 0; b < M; b++) Rv[a][b] = Rf[a * M + b];
        },
        [](auto, T, const T (&)[M]) {});
    if (!ok && st == BKE_STATUS_OK) st = BKE_STATUS_SINGULAR_S;
    if (live) {
        T *slot = tile + tid * PER;
        const bool good = st == BKE_STATUS_OK;
#pragma unroll
        for (int a = 0; a < M; a++) {
            slot[a] = zm[a];
            if (p.zhat) p.zhat[f * M + a] = zm[a];
        }
#pragma unroll
        for (int a = 0; a < M; a++)
#pragma unroll
            for (int b = 0; b < M; b++) slot[M + a * M + b] = good ? SI[a][b] : scorek::qnan<T>();
        slot[M + M * M] = good ? logdet : scorek::qnan<T>();
        if (p.status) p.status[f] = st;
    }
    __syncthreads();
    const bool cov = p.d2 || p.maha || p.ll || p.lk;
    if (!(p.y || cov)) return;
    // score.cu's pair walk: thread t starts at pair t of the tile and steps by UB = di * K + dk pairs
    const int64_t K = p.K, di = p.di, dk = p.dk;
    int64_t i = tid < K ? 0 : tid / (int)K, k = tid - i * K;
    while (i < cnt) {
        scorek::pair_reg<T, M, typename ZResidual<(HOOKS & BKE_HOOK_RESIDUAL_Z) != 0>::type>(p, tile0 + i, k, tile + i * PER, cov);
        k += dk; i += di;
        if (k >= K) { k -= K; i++; }
    }
}

}  // namespace ukfk
}  // namespace bke
