// score.cu — measurement scoring of N tracks against K candidates each (bke_score_measurements).
//
// Per track: zhat = H x (x when H is NULL) or the given mean;  S = H P H' + R (P + R when H is NULL) or the given S;
// SI = S^-1 and log|det S| by reg_inverse (kf_regtile.cuh) or warp_inverse (kf_warp.cuh), the inverse of the step
// kernels.  Per pair: y = z - zhat;  d2 = y' SI y;  ll = -0.5 (d2 + log|det S| + m log 2pi), the step kernels'
// log_likelihood (kf_direct.cu, kf_generic.cu) in the same order of operations.
//
// One CTA of 128 threads per tile of tracks (a grid-stride loop over tiles):
//   phase A  each track's zhat, SI and log|det S| go to the tile's slot in shared memory (m + m^2 + 1 words),
//            zhat and status to HBM.  A register tile per thread for the shapes dispatch_m lists, a warp per track
//            (warp_inverse on a scratch copy of S) for every other.  A singular S stores NaN in SI and log|det S|,
//            which makes every score of the track NaN without a branch in phase B.
//   phase B  the tile's outputs out[t0 : t0 + nt, 0 : K] are one contiguous range of nt * K words: the threads walk
//            it in pair order, so stores (and the loads of per-track candidates [N, K, m]) are coalesced for any K.
//            The per-pair work is score_pairs.cuh's (shared with bke_ukf_score): m <= 4 keeps y in registers; a
//            larger m re-reads z_ik (L1) instead.
#include "bke_internal.cuh"
#include "kf_regtile.cuh"
#include "kf_warp.cuh"
#include "score_pairs.cuh"

namespace bke {
namespace {
using namespace scorek;

constexpr int THREADS = 128;

template <typename T>
struct ScP {
    int64_t N, K;
    int64_t di, dk;                  // the pair walk's step, THREADS = di * K + dk pairs
    int n, m, tile, scratch;         // tile: tracks per tile;  scratch: words per warp (warp phase A)
    const T *x, *mean, *P, *S, *H, *R, *z;
    int64_t sS, sH, sR, zt, zc;
    const uint8_t *valid;
    T *zhat, *y, *d2, *maha, *ll, *lk;
    int32_t *status;
};

// ---- phase A, one thread per track: compile-time n = N, m = M
template <typename T, int N, int M>
__device__ __forceinline__ void track_reg(const ScP<T> &p, int64_t f, T *slot)
{
    T zh[M], Hm[M][N];
    if (p.H) {
        const T *h = p.H + f * p.sH;
#pragma unroll
        for (int a = 0; a < M; a++)
#pragma unroll
            for (int k = 0; k < N; k++) Hm[a][k] = h[a * N + k];
    }
    if (p.x) {
        T x[N];
#pragma unroll
        for (int k = 0; k < N; k++) x[k] = p.x[f * N + k];
        if (p.H) {
#pragma unroll
            for (int a = 0; a < M; a++) {
                T s = Hm[a][0] * x[0];
#pragma unroll
                for (int k = 1; k < N; k++) s += Hm[a][k] * x[k];
                zh[a] = s;
            }
        } else {
#pragma unroll
            for (int a = 0; a < M; a++) zh[a] = x[a];      // H is NULL only where n == m
        }
    } else {
#pragma unroll
        for (int a = 0; a < M; a++) zh[a] = p.mean[f * M + a];
    }
#pragma unroll
    for (int a = 0; a < M; a++) slot[a] = zh[a];
    if (p.zhat) {
#pragma unroll
        for (int a = 0; a < M; a++) p.zhat[f * M + a] = zh[a];
    }
    if (!p.P && !p.S) return;
    T S[M][M];
    if (p.S) {
        const T *s = p.S + f * p.sS;
#pragma unroll
        for (int a = 0; a < M; a++)
#pragma unroll
            for (int b = 0; b < M; b++) S[a][b] = s[a * M + b];
    } else {
        const T *Pf = p.P + f * (N * N), *R = p.R + f * p.sR;
        if (p.H) {
            // reg_update's S = H (P H') + R, kf_regtile.cuh
            T PHT[N][M];
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int a = 0; a < M; a++) {
                    T s = Pf[i * N] * Hm[a][0];
#pragma unroll
                    for (int k = 1; k < N; k++) s += Pf[i * N + k] * Hm[a][k];
                    PHT[i][a] = s;
                }
#pragma unroll
            for (int a = 0; a < M; a++)
#pragma unroll
                for (int b = 0; b < M; b++) {
                    T s = Hm[a][0] * PHT[0][b];
#pragma unroll
                    for (int k = 1; k < N; k++) s += Hm[a][k] * PHT[k][b];
                    S[a][b] = s + R[a * M + b];
                }
        } else {
#pragma unroll
            for (int a = 0; a < M; a++)
#pragma unroll
                for (int b = 0; b < M; b++) S[a][b] = Pf[a * N + b] + R[a * M + b];
        }
    }
    T SI[M][M], logdet;
    const bool ok = reg_inverse<T, M>(S, SI, logdet);
#pragma unroll
    for (int a = 0; a < M; a++)
#pragma unroll
        for (int b = 0; b < M; b++) slot[M + a * M + b] = ok ? SI[a][b] : qnan<T>();
    slot[M + M * M] = ok ? logdet : qnan<T>();
    if (p.status) p.status[f] = ok ? BKE_STATUS_OK : BKE_STATUS_SINGULAR_S;
}

// ---- phase A, one warp per track: any n, m.  scr: the warp's scratch, m*m (S) + m (pivot column) + n*m (P H')
template <typename T>
__device__ void track_warp(const ScP<T> &p, int64_t f, T *slot, T *scr, int lane)
{
    const int n = p.n, m = p.m, mm = m * m;
    const T *Hf = p.H ? p.H + f * p.sH : nullptr;
    for (int a = lane; a < m; a += 32) {
        T z;
        if (p.x) {
            if (Hf) {
                z = T(0);
                for (int k = 0; k < n; k++) z += Hf[a * n + k] * p.x[f * n + k];
            } else {
                z = p.x[f * n + a];
            }
        } else {
            z = p.mean[f * m + a];
        }
        slot[a] = z;
        if (p.zhat) p.zhat[f * m + a] = z;
    }
    if (!p.P && !p.S) return;
    T *A = scr, *col = scr + mm, *PHT = col + m;
    if (p.S) {
        warp_copy_in(A, p.S + f * p.sS, mm, lane);
    } else {
        const T *Pf = p.P + f * ((int64_t)n * n), *R = p.R + f * p.sR;
        if (Hf) {
            // kf_generic.cu's S = H (P H') + R
            warp_mm<true>(Pf, Hf, n, n, m, lane, [&](int e, int, int, T s) { PHT[e] = s; });
            __syncwarp();
            for (int e = lane; e < mm; e += 32) {
                const int a = e / m, b = e - a * m;
                T s = T(0);
                for (int q = 0; q < n; q++) s += Hf[a * n + q] * PHT[q * m + b];
                A[e] = s + R[e];
            }
        } else {
            for (int e = lane; e < mm; e += 32) A[e] = Pf[e] + R[e];
        }
    }
    __syncwarp();
    T logdet = T(0);
    const bool ok = warp_inverse(A, slot + m, col, m, lane, logdet);
    __syncwarp();           // a failed warp_inverse returns with no barrier
    if (!ok)
        for (int e = lane; e < mm; e += 32) slot[m + e] = qnan<T>();
    if (lane == 0) {
        slot[m + mm] = ok ? logdet : qnan<T>();
        if (p.status) p.status[f] = ok ? BKE_STATUS_OK : BKE_STATUS_SINGULAR_S;
    }
    __syncwarp();
}

// N > 0: phase A in registers at n = N (M > 0);  N == 0: phase A by warps.  M > 0: phase B at m = M;  M == 0: any m.
template <typename T, int N, int M>
__global__ void __launch_bounds__(THREADS) score_kernel(const ScP<T> p)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    T *tile = reinterpret_cast<T *>(smem_raw);
    const int m = M > 0 ? M : p.m, per = slot_words(m);
    T *scratch = tile + (int64_t)p.tile * per;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool cov = (p.P || p.S) && (p.d2 || p.maha || p.ll || p.lk);
    const bool sweep = p.y || cov;
    const int64_t K = p.K, di = p.di, dk = p.dk;
    for (int64_t t0 = (int64_t)blockIdx.x * p.tile; t0 < p.N; t0 += (int64_t)gridDim.x * p.tile) {
        const int nt = (int)min((int64_t)p.tile, p.N - t0);
        if constexpr (N > 0) {
            for (int i = threadIdx.x; i < nt; i += THREADS) track_reg<T, N, M>(p, t0 + i, tile + i * per);
        } else {
            for (int i = warp; i < nt; i += THREADS / 32)
                track_warp<T>(p, t0 + i, tile + i * per, scratch + (int64_t)warp * p.scratch, lane);
        }
        __syncthreads();
        if (sweep) {
            // thread t starts at pair t of the tile (the walk stays written out here: routed through a shared
            // function it changed every instance's code)
            int64_t i = threadIdx.x < K ? 0 : (int)threadIdx.x / (int)K, k = threadIdx.x - i * K;
            while (i < nt) {
                if constexpr (M > 0) pair_reg<T, M, SubResidual>(p, t0 + i, k, tile + i * per, cov);
                else pair_any<T>(p, t0 + i, k, tile + i * per, cov, p.m);
                k += dk; i += di;
                if (k >= K) { k -= K; i++; }
            }
        }
        __syncthreads();
    }
}

template <typename T>
ScP<T> params(const bke_score_args &a)
{
    ScP<T> p;
    p.N = a.n_tracks; p.K = a.n_candidates;
    p.di = THREADS / p.K; p.dk = THREADS - p.di * p.K;
    p.n = (a.x || a.P) ? a.dim_x : a.dim_z; p.m = a.dim_z;
    p.tile = THREADS; p.scratch = 0;
    p.x = (const T *)a.x; p.mean = (const T *)a.mean; p.P = (const T *)a.P; p.S = (const T *)a.S;
    p.H = (const T *)a.H; p.R = (const T *)a.R; p.z = (const T *)a.z;
    p.sS = a.S_stride; p.sH = a.H_stride; p.sR = a.R_stride; p.zt = a.z_track_stride; p.zc = a.z_cand_stride;
    p.valid = a.z_valid;
    p.zhat = (T *)a.zhat; p.y = (T *)a.y; p.d2 = (T *)a.d2; p.maha = (T *)a.mahalanobis;
    p.ll = (T *)a.log_likelihood; p.lk = (T *)a.likelihood; p.status = a.status;
    return p;
}

template <typename T, int N, int M>
int launch(ScP<T> p, cudaStream_t s)
{
    const int per = slot_words(M > 0 ? M : p.m);
    size_t smem = 0;
    if (N > 0) {
        smem = (size_t)p.tile * per * sizeof(T);
    } else {
        p.scratch = (p.m * p.m + p.m + p.n * p.m + 1) & ~1;
        const size_t scr = (size_t)(THREADS / 32) * p.scratch * sizeof(T), budget = 200 * 1024;
        // a tile small enough to leave room for several CTAs per SM, at least one track per warp
        while (p.tile > THREADS / 32 && (size_t)p.tile * per * sizeof(T) + scr > 64 * 1024) p.tile >>= 1;
        smem = (size_t)p.tile * per * sizeof(T) + scr;
        if (smem > budget) {
            set_error("bke_score_measurements: dim_x=%d dim_z=%d needs %zu B of shared memory per CTA (> %zu)", p.n, p.m,
                      smem, budget);
            return BKE_ERR_UNSUPPORTED;
        }
    }
    if (smem > 48 * 1024 &&
        check_cuda(cudaFuncSetAttribute(score_kernel<T, N, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                   "cudaFuncSetAttribute"))
        return BKE_ERR_CUDA;
    const int64_t tiles = (p.N + p.tile - 1) / p.tile, cap = (int64_t)sm_count() * 16;
    const unsigned grid = (unsigned)(tiles < cap ? tiles : cap);
    score_kernel<T, N, M><<<grid, THREADS, smem, s>>>(p);
    return check_cuda(cudaGetLastError(), "score_kernel launch");
}

// phase B at m = M; phase A in registers where (n, M) is one of the register shapes
template <typename T, int M>
int dispatch_m(const ScP<T> &p, cudaStream_t s)
{
    const int n = p.n;
    if (n == M) return launch<T, M, M>(p, s);
    if constexpr (M == 1) {
        if (n == 2) return launch<T, 2, 1>(p, s);
        if (n == 3) return launch<T, 3, 1>(p, s);
        if (n == 4) return launch<T, 4, 1>(p, s);
    } else if constexpr (M == 2) {
        if (n == 4) return launch<T, 4, 2>(p, s);
    } else if constexpr (M == 3) {
        if (n == 6) return launch<T, 6, 3>(p, s);
    }
    return launch<T, 0, M>(p, s);
}

template <typename T>
int dispatch(const bke_score_args &a, cudaStream_t s)
{
    const ScP<T> p = params<T>(a);
    switch (p.m) {
    case 1: return dispatch_m<T, 1>(p, s);
    case 2: return dispatch_m<T, 2>(p, s);
    case 3: return dispatch_m<T, 3>(p, s);
    case 4: return dispatch_m<T, 4>(p, s);
    default: return launch<T, 0, 0>(p, s);
    }
}

}  // namespace

int launch_score(const bke_score_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

}  // namespace bke
