// ckf_kernel.cuh — device code of the cubature Kalman filter bank (see ckf.cu for the host side).
// Free of host headers: compiled by nvcc into libbke.so (closed set of fx / hx models) and by NVRTC around
// user-supplied fx / hx device functions (ukf_rtc.cu, bke_ckf_model_compile).
//
// Per filter, m = 2n cubature points (filterpy/kalman/CubatureKalmanFilter.py:52-61 points, :317-327
// predict, :362-379 update, ckf_transform :87-98; reference @ 3b51149):
//   U  = chol_upper(P) * sqrt(n)              scipy's upper factor, then scaled (not chol(nP))
//   Xs = {x + U[k,:], x - U[k,:]}, k < n      no centre point
//   f_k = fx(Xs_k);  x- = sum f_k / m;  P- = sum (f_k - x-)(f_k - x-)' / m + Q
//   Z_k = hx(f_k)                              the propagated points of the last predict, NOT redrawn
//   z^ = sum Z_k / m;  S = sum (Z_k - z^)(..)' / m + R;  Pxz = sum (f_k - x-)(Z_k - z^)' / m
//   K = Pxz S^-1;  x = x- + K (z - z^);  P = P- - K S K'
// The covariance sums are CENTRED.  The reference forms them as raw second moments
// (sum f f' - m x x') / m, which loses |x|^2 / P digits to cancellation: about 1e-2 relative in fp32 on
// tracking banks with positions of ~500 and unit covariances.  The mathematics is the same.
//
// Register plan (as ukf_kernel.cuh): x, U and the accumulators live in registers; the 2n propagated
// points are NOT stored — the cheap process models are evaluated again for each pass over them (mean,
// P-, measurement points, cross covariance) from (x, U) — while the measurement-space points are parked
// in the conflict-free [point][component][thread] slab and the prior covariance in the park slab.
// An update-only launch has no (x, U) to regenerate from: it reads the points of the last predict from
// sigmas_f[N][2n][n], which a launch with BKE_DO_PREDICT writes when the pointer is non-NULL.
#pragma once
#include "ukf_kernel.cuh"

namespace bke {
namespace ckfk {

using ukfk::UB;

template <typename T>
struct CkfP {
    int64_t N;
    unsigned flags;
    T dt;
    T root_n;                // sqrt(n): the scale of the Cholesky factor (CubatureKalmanFilter.py:56)
    const T *x, *P, *Q, *R, *F, *H, *z;
    int64_t sQ, sR, sF, sH;
    const uint8_t *valid;
    T *x_out, *P_out, *x_prior, *P_prior, *K, *y, *S, *SI, *ll;
    int32_t *status;
    T *sigmas_f;             // [N][2n][n] or NULL
    const T *fx_args, *hx_args;     // BKE_FX_USER / BKE_HX_USER: parameter vectors handed to the user's functions
    int64_t s_fx_args, s_hx_args;   // 0 = one vector for the bank, else elements per filter
};

// The update half of ukf_kernel, as functions.  (Calling them from ukf_kernel as well changed the code
// the compiler emits for two of the UKF's sixty instances, so the UKF keeps its inline copy.)
//
// Parks the prior covariance's upper triangle in the [NT][UB] slab `park` while the update works.  A
// (never expected) non-symmetric P keeps its lower triangle in filter f's P_out.  Returns whether it did.
using ukfk::tri_index;

template <typename T, int N>
__device__ __forceinline__ bool park_prior(T *park, int tid, const T (&P)[N][N], bool live, T *P_out, int64_t f)
{
    bool asym = false;
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = i; j < N; j++) {
            park[tri_index<N>(i, j) * UB + tid] = P[i][j];
            if (j > i) asym = asym || (P[j][i] != P[i][j]);
        }
    if (asym && live) {
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < i; j++) P_out[f * N * N + i * N + j] = P[i][j];
    }
    return asym;
}

// K = Pxz S^-1, y = z - z^, x += K y, the optional outputs (they leave while S, SI, y are still in
// registers) and S K' for the covariance update P -= K (S K')
template <bool EXTRAS, typename T, int N, int M, typename Prm>
__device__ __forceinline__ void gain_update(const Prm &p, int64_t f, bool live, KfUpdateOut<T, N, M> &o, const T (&Pxz)[N][M],
                                            const T (&zv)[M], const T (&zm)[M], T (&x)[N], T (&SK)[M][N])
{
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int a = 0; a < M; a++) {
            T s = Pxz[i][0] * o.SI[0][a];
#pragma unroll
            for (int b = 1; b < M; b++) s += Pxz[i][b] * o.SI[b][a];
            o.K[i][a] = s;
        }
    if constexpr (ukfk::HOOKS & BKE_HOOK_RESIDUAL_Z) {
        ukfk::bke_hook_residual_z<T>(zv, zm, o.y);                // the only hook the CKF calls (:376)
    } else {
#pragma unroll
        for (int a = 0; a < M; a++) o.y[a] = zv[a] - zm[a];
    }
#pragma unroll
    for (int i = 0; i < N; i++) {
        T s = x[i];
#pragma unroll
        for (int a = 0; a < M; a++) s += o.K[i][a] * o.y[a];
        x[i] = s;
    }
    if (EXTRAS && live) {
        if (p.K) for (int i = 0; i < N; i++) for (int a = 0; a < M; a++) p.K[f * N * M + i * M + a] = o.K[i][a];
        if (p.y) for (int a = 0; a < M; a++) p.y[f * M + a] = o.y[a];
        if (p.S) for (int a = 0; a < M; a++) for (int b = 0; b < M; b++) p.S[f * M * M + a * M + b] = o.S[a][b];
        if (p.SI) for (int a = 0; a < M; a++) for (int b = 0; b < M; b++) p.SI[f * M * M + a * M + b] = o.SI[a][b];
        if (p.ll) {
            T q = T(0);
#pragma unroll
            for (int a = 0; a < M; a++) {
                T s = T(0);
#pragma unroll
                for (int b = 0; b < M; b++) s += o.SI[a][b] * o.y[b];
                q += o.y[a] * s;
            }
            p.ll[f] = T(-0.5) * (q + o.logdet + T(M) * T(LOG_2PI));
        }
    }
#pragma unroll
    for (int a = 0; a < M; a++)
#pragma unroll
        for (int j = 0; j < N; j++) {
            T s = o.S[a][0] * o.K[j][0];
#pragma unroll
            for (int b = 1; b < M; b++) s += o.S[a][b] * o.K[j][b];
            SK[a][j] = s;
        }
}

// the prior covariance back from its parking place (park_prior), then P -= K (S K') when `good`
template <typename T, int N, int M>
__device__ __forceinline__ void posterior_cov(const T *park, int tid, T (&P)[N][N], bool asym, bool live, const T *P_out, int64_t f,
                                              bool good, const T (&K)[N][M], const T (&SK)[M][N])
{
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = i; j < N; j++) { P[i][j] = park[tri_index<N>(i, j) * UB + tid]; P[j][i] = P[i][j]; }
    if (asym && live) {
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < i; j++) P[i][j] = P_out[f * N * N + i * N + j];
    }
    if (good) {
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = i; j < N; j++) {
                T s = K[i][0] * SK[0][j];
#pragma unroll
                for (int a = 1; a < M; a++) s += K[i][a] * SK[a][j];
                P[i][j] -= s;
                if (j > i) P[j][i] -= s;
            }
    }
}

// EXTRAS: the optional outputs (priors, K, y, S, SI, log-likelihood) are compiled in
template <typename T, int N, int M, int FX, int HX, int OCC, bool EXTRAS>
__global__ void __launch_bounds__(UB, OCC) ckf_kernel(CkfP<T> p)
{
    using namespace ukfk;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int NP = 2 * N;                                // cubature points
    constexpr int PADP = (N * N) | 1;                        // odd per-filter stride of the P / Q slab
    constexpr int NT = N * (N + 1) / 2;
    constexpr int SLAB = (NP * M + NT > PADP ? NP * M + NT : PADP) * UB;
    T *zs = reinterpret_cast<T *>(smem_raw);                 // [NP*M][UB]; doubles as the staging slab for P, Q, P_out
    T *park = zs + NP * M * UB;                              // [NT][UB]: the prior covariance while the update works
    T *Fs = zs + SLAB;                                       // [N*N] or [N*N][UB]
    const bool do_p = p.flags & BKE_DO_PREDICT, do_u = p.flags & BKE_DO_UPDATE;
    const int tid = threadIdx.x;
    const int64_t f = (int64_t)blockIdx.x * UB + tid;
    const bool live = f < p.N;
    const int64_t fc = live ? f : p.N - 1;                   // clamp: dead threads redo the last filter

    // stage F / H (linear models) in shared memory
    int fstride = 1, foff = 0;
    T *Hs = Fs;
    if (FX == BKE_FX_LINEAR && do_p) {
        if (p.sF == 0) { for (int e = tid; e < N * N; e += UB) Fs[e] = p.F[e]; Hs = Fs + N * N; }
        else {
            for (int e = 0; e < N * N; e++) Fs[e * UB + tid] = p.F[fc * p.sF + e];
            fstride = UB; foff = tid; Hs = Fs + N * N * UB;
        }
    }
    int hstride = 1, hoff = 0;
    if (HX == BKE_HX_LINEAR && do_u) {
        if (p.sH == 0) { for (int e = tid; e < M * N; e += UB) Hs[e] = p.H[e]; }
        else {
            for (int e = 0; e < M * N; e++) Hs[e * UB + tid] = p.H[fc * p.sH + e];
            hstride = UB; hoff = tid;
        }
    }
    __syncthreads();
    const T *Fp = Fs + foff, *Hp = Hs + hoff;
    const T *fxa = (FX == BKE_FX_USER && p.fx_args) ? p.fx_args + fc * p.s_fx_args : nullptr;
    const T *hxa = (HX == BKE_HX_USER && p.hx_args) ? p.hx_args + fc * p.s_hx_args : nullptr;

    const int64_t tile0 = (int64_t)blockIdx.x * UB;
    const int cnt = (int)((p.N - tile0) < UB ? (p.N - tile0) : UB);
    const int tl = live ? tid : cnt - 1;                     // slab row of this thread's filter
    T x[N], P[N][N];
#pragma unroll
    for (int i = 0; i < N; i++) x[i] = p.x[fc * N + i];
    slab_load<T, N * N, PADP>(zs, p.P + tile0 * N * N, cnt);
    __syncthreads();
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) P[i][j] = zs[tl * PADP + i * N + j];
    __syncthreads();
    const bool q_dense = do_p && p.sQ != 0;
    if (q_dense) slab_load<T, N * N, PADP>(zs, p.Q + tile0 * N * N, cnt);     // parked until the end of predict
    __syncthreads();
    int st = BKE_STATUS_OK;
    T xs[N], U[N][N];                                        // the posterior the points are drawn from
    T *sf = (p.sigmas_f && live) ? p.sigmas_f + f * NP * N : nullptr;

    // propagated point k: regenerated from (xs, U) after a predict, else the stored points of the last one
    auto point = [&](auto kc, T (&fs)[N]) {
        constexpr int K = decltype(kc)::value;
        if (do_p) {
            T sp[N];
            sigma_point<T, N, K + 1>(xs, U, sp);              // UKF point K+1 is x + U[K] (K < n), x - U[K-n]
            apply_fx<T, N, FX>(sp, fs, p.dt, Fp, fstride, fxa);
        } else {
            const T *g = p.sigmas_f + (fc * NP + K) * N;
#pragma unroll
            for (int i = 0; i < N; i++) fs[i] = g[i];
        }
    };

    if (do_p) {
        if (!chol_upper<T, N>(P, U)) st = BKE_STATUS_NOT_PD;
#pragma unroll
        for (int i = 0; i < N; i++) {
            xs[i] = x[i];
#pragma unroll
            for (int j = i; j < N; j++) U[i][j] *= p.root_n;
        }
        // pass 1: mean of the propagated points
        T xm[N];
#pragma unroll
        for (int i = 0; i < N; i++) xm[i] = T(0);
        for_sigma<0, NP>([&](auto kc) {
            T fs[N];
            point(kc, fs);
#pragma unroll
            for (int i = 0; i < N; i++) xm[i] += fs[i];
        });
#pragma unroll
        for (int i = 0; i < N; i++) xm[i] = xm[i] / T(NP);
        // pass 2: centred covariance (upper triangle); the points leave for sigmas_f here
        T Pm[N][N];
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = i; j < N; j++) Pm[i][j] = T(0);
        for_sigma<0, NP>([&](auto kc) {
            constexpr int K = decltype(kc)::value;
            T fs[N], d[N];
            point(kc, fs);
            if (sf) {
#pragma unroll
                for (int i = 0; i < N; i++) sf[K * N + i] = fs[i];
            }
#pragma unroll
            for (int i = 0; i < N; i++) d[i] = fs[i] - xm[i];
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = i; j < N; j++) Pm[i][j] += d[i] * d[j];
        });
        const T inv_m = T(1) / T(NP);                        // P *= 1 / m (CubatureKalmanFilter.py:95)
#pragma unroll
        for (int i = 0; i < N; i++) {
            x[i] = xm[i];
#pragma unroll
            for (int j = i; j < N; j++) {
                const T c = Pm[i][j] * inv_m;
                P[i][j] = c + (q_dense ? zs[tl * PADP + i * N + j] : p.Q[i * N + j]);
                if (j > i) P[j][i] = c + (q_dense ? zs[tl * PADP + j * N + i] : p.Q[j * N + i]);
            }
        }
        if (EXTRAS && live) {
            if (p.x_prior) for (int i = 0; i < N; i++) p.x_prior[f * N + i] = x[i];
            if (p.P_prior) for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) p.P_prior[f * N * N + i * N + j] = P[i][j];
        }
    }

    __syncthreads();                                         // Q has been consumed: the slab now holds hx(points)
    if (do_u) {
        const bool has_z = (p.valid == nullptr) || (p.valid[fc] != 0);
        if (has_z && st == BKE_STATUS_OK) {
            // P is not needed again until the posterior: park it in shared memory and free the registers
            const bool asym = park_prior<T, N>(park, tid, P, live, p.P_out, f);
            T zm[M];
#pragma unroll
            for (int a = 0; a < M; a++) zm[a] = T(0);
            if constexpr (HX == BKE_HX_LINEAR || HX == BKE_HX_USER) {
                for_sigma<0, NP>([&](auto kc) {
                    constexpr int K = decltype(kc)::value;
                    T fs[N], h[M];
                    point(kc, fs);
                    apply_hx<T, N, M, HX>(fs, h, Hp, hstride, hxa);
#pragma unroll
                    for (int a = 0; a < M; a++) { zm[a] += h[a]; zs[(K * M + a) * UB + tid] = h[a]; }
                });
            } else {
                // Transcendental measurement models: the position components of each point are parked in
                // the slab, then a run-time loop evaluates hx in place (2n unrolled sqrt / atan2 bodies
                // would bloat the fp64 kernel the way DESIGN §3.5 records for the UKF).  The points are fx
                // outputs with no centre point among them, so hx is the plain library evaluation.
                for_sigma<0, NP>([&](auto kc) {
                    constexpr int K = decltype(kc)::value;
                    T fs[N];
                    point(kc, fs);
#pragma unroll
                    for (int a = 0; a < M; a++) zs[(K * M + a) * UB + tid] = fs[2 * a];   // positions sit at 0, 2, 4
                });
#pragma unroll 1
                for (int k = 0; k < NP; k++) {
                    T pos[M], h[M];
#pragma unroll
                    for (int a = 0; a < M; a++) pos[a] = zs[(k * M + a) * UB + tid];
                    hx_positions<T, M, HX>(pos, h);
#pragma unroll
                    for (int a = 0; a < M; a++) { zm[a] += h[a]; zs[(k * M + a) * UB + tid] = h[a]; }
                }
            }
#pragma unroll
            for (int a = 0; a < M; a++) zm[a] = zm[a] / T(NP);
            KfUpdateOut<T, N, M> o;
            T Pxz[N][M];
#pragma unroll
            for (int a = 0; a < M; a++)
#pragma unroll
                for (int b = a; b < M; b++) o.S[a][b] = T(0);
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int a = 0; a < M; a++) Pxz[i][a] = T(0);
            // pass over the points again: S and the cross covariance with dx = f_k - x
            // (x is the prior mean; after an update-only launch, the state the reference's update sees)
            for_sigma<0, NP>([&](auto kc) {
                constexpr int K = decltype(kc)::value;
                T fs[N], dz[M];
                point(kc, fs);
#pragma unroll
                for (int a = 0; a < M; a++) dz[a] = zs[(K * M + a) * UB + tid] - zm[a];
#pragma unroll
                for (int a = 0; a < M; a++)
#pragma unroll
                    for (int b = a; b < M; b++) o.S[a][b] += dz[a] * dz[b];
#pragma unroll
                for (int i = 0; i < N; i++) {
                    const T dx = fs[i] - x[i];
#pragma unroll
                    for (int a = 0; a < M; a++) Pxz[i][a] += dx * dz[a];
                }
            });
            T zv[M];
            {
                const T *Rf = p.R + fc * p.sR;
                const T inv_m = T(1) / T(NP);
#pragma unroll
                for (int a = 0; a < M; a++) {
                    zv[a] = p.z[fc * M + a];
#pragma unroll
                    for (int b = a; b < M; b++) {
                        const T c = o.S[a][b] * inv_m;
                        o.S[a][b] = c + Rf[a * M + b];
                        if (b > a) o.S[b][a] = c + Rf[b * M + a];
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int a = 0; a < M; a++) Pxz[i][a] = Pxz[i][a] / T(NP);
            o.ok = reg_inverse<T, M>(o.S, o.SI, o.logdet);
            if (!o.ok) st = BKE_STATUS_SINGULAR_S;
            const bool good = o.ok && st == BKE_STATUS_OK;
            T SK[M][N];
            if (good) gain_update<EXTRAS>(p, f, live, o, Pxz, zv, zm, x, SK);
            posterior_cov<T, N, M>(park, tid, P, asym, live, p.P_out, f, good, o.K, SK);
        }
    }
    __syncthreads();                                         // the slab is free again: stage the posterior covariance
    if (live) {
#pragma unroll
        for (int i = 0; i < N; i++) p.x_out[f * N + i] = x[i];
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < N; j++) zs[tid * PADP + i * N + j] = P[i][j];
        if (p.status) p.status[f] = st;
    }
    __syncthreads();
    slab_store<T, N * N, PADP>(p.P_out + tile0 * N * N, zs, cnt);
}

}  // namespace ckfk
}  // namespace bke
