// imm.cu — IMMEstimator.batch_filter for a bank of tracks (filterpy/kalman/IMM.py:160-247): T epochs of
// predict(); update(z) in ONE launch, the time loop inside the kernel.
//
// Layout: one thread per (track, model).  A track's models sit in an aligned group of G = 2, 4 or 8 lanes
// (G >= M, the next power of two); lane j of the group owns model j's x, P and the diagnostics it carries from
// epoch to epoch (the kept S, K, y, SI, log-likelihood), its mode probability mu_j and cbar_j.  Lanes j >= M
// hold no model: they run model 0's arithmetic and never publish it, but take their share of the output
// stores.  Everything that needs another model's state goes through __shfl_sync within the group:
//   mixing (IMM.py:201-213)         lane i forms x0_i, P0_i from every model's x_j, P_j and omega[j][i]
//   combined estimate (:228-237)    every lane forms the mean; row r of the covariance is stored by lane r % G
//   mode probabilities (:178-184, :239-247)   mu, cbar and omega's column i from the models' likelihoods
// with the formulas and the order of summation of csrc/mix.cu (the row-parallel and element-parallel forms
// sum alike) and the step arithmetic of kf_regtile.cuh.  omega is not carried: lane i recomputes its column
// from mu and cbar with mix.cu's expression, so it has the bits of the stored one.
//
// Traffic per track-epoch: z (m) and zs_valid in, the five outputs out (2 n + 2 n^2 scalars and M fp64);
// 192 B at 4/2 fp32 with M = 3.  State, diagnostics, models and probabilities are read once and written once
// per call: every thread holds its model's F, Q, H, R, x, P and the kept S, K, y, SI in registers.
// Instances: 2/1 and 3/1 in fp32 and fp64, 4/2 in fp32, for G = 2, 4, 8, none with local-memory spills.  4/2
// fp64 (56-104 B of spills per thread at 255 registers, even with H and R read every epoch) and 6/3 (both
// dtypes) do not fit; they return BKE_ERR_UNSUPPORTED and the mirror runs the separate launches.
#include <float.h>
#include <math.h>
#include <type_traits>
#include "bke_internal.cuh"
#include "kf_regtile.cuh"

namespace bke {
namespace {

constexpr int kImmBlock = 128;

// log N(0; 0, S) of the kept S (KalmanFilter.update(None) then log_likelihood, kalman_filter.py:515-520,
// :1203-1210; the mirror's _missed_log_likelihood): -inf where det S <= 0
template <int MZ>
__device__ __forceinline__ double missed_ll(const double (&S)[MZ][MZ])
{
    static_assert(MZ >= 1 && MZ <= 3, "closed-form determinant");
    double det;
    if constexpr (MZ == 1) det = S[0][0];
    else if constexpr (MZ == 2) det = S[0][0] * S[1][1] - S[0][1] * S[1][0];
    else det = S[0][0] * (S[1][1] * S[2][2] - S[1][2] * S[2][1]) - S[0][1] * (S[1][0] * S[2][2] - S[1][2] * S[2][0]) +
               S[0][2] * (S[1][0] * S[2][1] - S[1][1] * S[2][0]);
    return det > 0.0 ? -0.5 * (log(det) + MZ * LOG_2PI) : -INFINITY;
}

// one row of N scalars, with the widest store the row's size allows (the array base is 16-byte aligned)
template <typename T, int N>
__device__ __forceinline__ void store_row(T *dst, const T (&v)[N])
{
    constexpr int B = N * (int)sizeof(T);
    if constexpr (B % 16 == 0) {
        using V = typename std::conditional<sizeof(T) == 4, float4, double2>::type;
        constexpr int E = 16 / sizeof(T);
#pragma unroll
        for (int i = 0; i < N / E; i++) {
            V w;
            if constexpr (sizeof(T) == 4) w = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
            else w = make_double2(v[2 * i], v[2 * i + 1]);
            reinterpret_cast<V *>(dst)[i] = w;
        }
    } else if constexpr (sizeof(T) == 4 && B % 8 == 0) {
#pragma unroll
        for (int i = 0; i < N / 2; i++) reinterpret_cast<float2 *>(dst)[i] = make_float2(v[2 * i], v[2 * i + 1]);
    } else {
#pragma unroll
        for (int i = 0; i < N; i++) dst[i] = v[i];
    }
}

// arr[i] of an array in the parameter block, read with constant indices
template <typename V>
__device__ __forceinline__ V pick(const V (&arr)[BKE_MM_MAX_MODELS], int i)
{
    V v = arr[0];
#pragma unroll
    for (int q = 1; q < BKE_MM_MAX_MODELS; q++) v = q == i ? arr[q] : v;
    return v;
}

template <typename T>
struct ImmModelPtrs { const T *F, *Q, *H, *R; };

template <typename T, int N, int MZ>
struct ImmModels {
    T F[N][N], Q[N][N], H[MZ][N], R[MZ][MZ];
    __device__ __forceinline__ void load(const ImmModelPtrs<T> &p)
    {
#pragma unroll
        for (int i = 0; i < N * N; i++) { (&F[0][0])[i] = p.F[i]; (&Q[0][0])[i] = p.Q[i]; }
#pragma unroll
        for (int i = 0; i < MZ * N; i++) (&H[0][0])[i] = p.H[i];
#pragma unroll
        for (int i = 0; i < MZ * MZ; i++) (&R[0][0])[i] = p.R[i];
    }
};

template <typename T, int N, int MZ, int G>
__global__ void __launch_bounds__(kImmBlock) imm_batch_kernel(const bke_imm_batch_args a)
{
    const int64_t t = ((int64_t)blockIdx.x * kImmBlock + threadIdx.x) / G;      // the track
    if (t >= a.n_tracks) return;                                                // whole groups leave together
    const int j = threadIdx.x & (G - 1);
    const unsigned gmask = ((1u << G) - 1u) << ((threadIdx.x & 31) & ~(G - 1));
    const int M = a.n_models;
    const bool live = j < M;
    const int64_t NT = a.n_tracks, Tn = a.n_steps;
    auto shfl = [&](auto v, int src) { return __shfl_sync(gmask, v, src, G); };

    // this lane's model arrays are picked from the parameter block with constant indices where they are used (a
    // dynamic index would copy the block to local memory; pointers held across the time loop cost registers)
    const int jm = live ? j : 0;
    const T alpha_sq = (T)pick(a.alpha_sq, jm);
    const double *trans = a.trans;
    const T *zs = (const T *)a.zs;
    const uint8_t *valid = a.zs_valid;
    auto models = [&]() { return ImmModelPtrs<T>{(const T *)pick(a.F, jm) + t * pick(a.F_stride, jm),
                                                 (const T *)pick(a.Q, jm) + t * pick(a.Q_stride, jm),
                                                 (const T *)pick(a.H, jm) + t * pick(a.H_stride, jm),
                                                 (const T *)pick(a.R, jm) + t * pick(a.R_stride, jm)}; };

    T x[N], P[N][N], S[MZ][MZ], SI[MZ][MZ], K[N][MZ], y[MZ], ll;
    {
        const T *xg = (const T *)pick(a.x, jm), *Pg = (const T *)pick(a.P, jm), *Sg = (const T *)pick(a.S, jm);
        const T *SIg = (const T *)pick(a.SI, jm), *Kg = (const T *)pick(a.K, jm), *yg = (const T *)pick(a.y, jm);
#pragma unroll
        for (int i = 0; i < N; i++) x[i] = xg[t * N + i];
#pragma unroll
        for (int i = 0; i < N * N; i++) (&P[0][0])[i] = Pg[t * N * N + i];
#pragma unroll
        for (int i = 0; i < MZ * MZ; i++) { (&S[0][0])[i] = Sg[t * MZ * MZ + i]; (&SI[0][0])[i] = SIg[t * MZ * MZ + i]; }
#pragma unroll
        for (int i = 0; i < N * MZ; i++) (&K[0][0])[i] = Kg[t * N * MZ + i];
#pragma unroll
        for (int i = 0; i < MZ; i++) y[i] = yg[t * MZ + i];
        ll = ((const T *)pick(a.log_likelihood, jm))[t];
    }
    double mu_j = live ? a.mu[t * M + j] : 0.0, cb_j = live ? a.cbar[t * M + j] : 1.0;
    int st_last = BKE_STATUS_OK, st_any = BKE_STATUS_OK;

    ImmModels<T, N, MZ> md;
    md.load(models());

    // combined estimate (IMM.py:228-237) of the group's models with the weights mu -> xo[n], Po[n][n] of the track
    auto estimate = [&](T *xo, T *Po) {
        T w[G], m[N];
#pragma unroll
        for (int q = 0; q < G; q++) w[q] = (T)shfl(mu_j, q);
#pragma unroll
        for (int c = 0; c < N; c++) m[c] = T(0);
#pragma unroll
        for (int q = 0; q < G; q++) {
            if (q < M) {
#pragma unroll
                for (int c = 0; c < N; c++) m[c] += shfl(x[c], q) * w[q];
            }
        }
#pragma unroll
        for (int r = 0; r < N; r++) {
            T acc[N];
#pragma unroll
            for (int c = 0; c < N; c++) acc[c] = T(0);
#pragma unroll
            for (int q = 0; q < G; q++) {
                if (q < M) {
                    const T xr = shfl(x[r], q) - m[r];
#pragma unroll
                    for (int c = 0; c < N; c++) {
                        const T xc = shfl(x[c], q), pv = shfl(P[r][c], q);
                        acc[c] += w[q] * (xr * (xc - m[c]) + pv);
                    }
                }
            }
            if (r % G == j) store_row<T, N>(Po + r * N, acc);
        }
#pragma unroll
        for (int c = 0; c < N; c++) if (c % G == j) xo[c] = m[c];
    };

    for (int64_t k = 0; k < Tn; k++) {
        const int64_t e = k * NT + t;                       // (epoch, track)
        T z[MZ];
#pragma unroll
        for (int i = 0; i < MZ; i++) z[i] = zs[e * MZ + i];
        const bool has_z = valid == nullptr || valid[e] != 0;

        // ---- predict (IMM.py:186-226): mixed initial conditions of model j, omega[q][j] = M[q][j] mu_q / cbar_j
        {
            const double rc = 1.0 / cb_j;
            T w[G], x0[N], P0[N][N];
#pragma unroll
            for (int q = 0; q < G; q++) {
                const double mq = shfl(mu_j, q);
                w[q] = q < M ? (T)((trans[q * M + jm] * mq) * rc) : T(0);
            }
#pragma unroll
            for (int c = 0; c < N; c++) x0[c] = T(0);
#pragma unroll
            for (int q = 0; q < G; q++) {
                if (q < M) {
#pragma unroll
                    for (int c = 0; c < N; c++) x0[c] += shfl(x[c], q) * w[q];
                }
            }
#pragma unroll
            for (int i = 0; i < N * N; i++) (&P0[0][0])[i] = T(0);
#pragma unroll
            for (int q = 0; q < G; q++) {
                if (q < M) {
                    T xq[N];
#pragma unroll
                    for (int c = 0; c < N; c++) xq[c] = shfl(x[c], q);
#pragma unroll
                    for (int r = 0; r < N; r++) {
                        const T xr = xq[r] - x0[r];
#pragma unroll
                        for (int c = 0; c < N; c++) P0[r][c] += w[q] * (xr * (xq[c] - x0[c]) + shfl(P[r][c], q));
                    }
                }
            }
#pragma unroll
            for (int c = 0; c < N; c++) x[c] = x0[c];
#pragma unroll
            for (int i = 0; i < N * N; i++) (&P[0][0])[i] = (&P0[0][0])[i];
        }
        reg_predict<T, N>(x, P, md.F, md.Q, alpha_sq);
        if (k == Tn - 1 && live) {
            T *xpg = (T *)pick(a.x_prior, jm), *Ppg = (T *)pick(a.P_prior, jm);
#pragma unroll
            for (int i = 0; i < N; i++) xpg[t * N + i] = x[i];
#pragma unroll
            for (int i = 0; i < N * N; i++) Ppg[t * N * N + i] = (&P[0][0])[i];
        }
        estimate((T *)a.means_p + e * N, (T *)a.covariances_p + e * N * N);

        // ---- update (IMM.py:160-184)
        int st = BKE_STATUS_OK;
        if (has_z) {
            KfUpdateOut<T, N, MZ> o;
            reg_update<T, N, MZ>(x, P, md.H, md.R, z, o);
#pragma unroll
            for (int i = 0; i < MZ * MZ; i++) (&S[0][0])[i] = (&o.S[0][0])[i];        // stored even when singular
            if (o.ok) {
#pragma unroll
                for (int i = 0; i < MZ * MZ; i++) (&SI[0][0])[i] = (&o.SI[0][0])[i];
#pragma unroll
                for (int i = 0; i < N * MZ; i++) (&K[0][0])[i] = (&o.K[0][0])[i];
                T q = T(0);
#pragma unroll
                for (int u = 0; u < MZ; u++) {
                    T s = T(0);
#pragma unroll
                    for (int b = 0; b < MZ; b++) s += o.SI[u][b] * o.y[b];
                    q += o.y[u] * s;
                }
                ll = T(-0.5) * (q + o.logdet + T(MZ) * T(LOG_2PI));
#pragma unroll
                for (int i = 0; i < MZ; i++) y[i] = o.y[i];
            } else {
                st = BKE_STATUS_SINGULAR_S;                 // the prior and the previous log-likelihood stay
            }
        } else {
            double Sd[MZ][MZ];
#pragma unroll
            for (int i = 0; i < MZ * MZ; i++) (&Sd[0][0])[i] = (double)(&S[0][0])[i];
            ll = (T)missed_ll<MZ>(Sd);
#pragma unroll
            for (int i = 0; i < MZ; i++) y[i] = T(0);
        }
        st_last = st;
        st_any = st_any ? st_any : st;

        // mode probabilities: mu = cbar L / sum(cbar L); cbar = mu . M
        double L = exp((double)ll);
        if (L == 0.0) L = DBL_MIN;                          // kalman_filter.py:1221-1222
        const double pj = cb_j * L;
        double sum = 0.0;
#pragma unroll
        for (int q = 0; q < G; q++) {
            const double v = shfl(pj, q);
            if (q < M) sum += v;
        }
        const double rs = 1.0 / sum;
        mu_j = pj * rs;
        double cs = 0.0;
#pragma unroll
        for (int q = 0; q < G; q++) {
            const double v = shfl(mu_j, q);
            if (q < M) cs += v * trans[q * M + jm];
        }
        cb_j = cs;
        if (live) a.mus[e * M + j] = mu_j;
        estimate((T *)a.means + e * N, (T *)a.covariances + e * N * N);
    }

    // omega's column j from the final mu and cbar (mix.cu's expression)
    const double rc = 1.0 / cb_j;
#pragma unroll
    for (int q = 0; q < G; q++) {
        const double mq = shfl(mu_j, q);
        if (live && q < M) a.omega[(t * M + q) * M + j] = (trans[q * M + j] * mq) * rc;
    }
    if (!live) return;
    a.mu[t * M + j] = mu_j;
    a.cbar[t * M + j] = cb_j;
    T *xg = (T *)pick(a.x, j), *Pg = (T *)pick(a.P, j), *Sg = (T *)pick(a.S, j), *SIg = (T *)pick(a.SI, j);
    T *Kg = (T *)pick(a.K, j), *yg = (T *)pick(a.y, j);
#pragma unroll
    for (int i = 0; i < N; i++) xg[t * N + i] = x[i];
#pragma unroll
    for (int i = 0; i < N * N; i++) Pg[t * N * N + i] = (&P[0][0])[i];
#pragma unroll
    for (int i = 0; i < MZ * MZ; i++) { Sg[t * MZ * MZ + i] = (&S[0][0])[i]; SIg[t * MZ * MZ + i] = (&SI[0][0])[i]; }
#pragma unroll
    for (int i = 0; i < N * MZ; i++) Kg[t * N * MZ + i] = (&K[0][0])[i];
#pragma unroll
    for (int i = 0; i < MZ; i++) yg[t * MZ + i] = y[i];
    ((T *)pick(a.log_likelihood, j))[t] = ll;
    pick(a.status, j)[t] = (a.flags & BKE_STATUS_STICKY) ? st_any : st_last;
}

template <typename T, int N, int MZ, int G>
int launch_g(const bke_imm_batch_args &a, cudaStream_t s)
{
    const int64_t threads = a.n_tracks * G;
    const unsigned grid = (unsigned)((threads + kImmBlock - 1) / kImmBlock);
    bke_imm_batch_args p = a;
    return launch_kernel((const void *)imm_batch_kernel<T, N, MZ, G>, grid, kImmBlock, 0, &p, s, "imm_batch_kernel");
}

template <typename T, int N, int MZ>
int launch_shape(const bke_imm_batch_args &a, cudaStream_t s)
{
    if (a.n_models <= 2) return launch_g<T, N, MZ, 2>(a, s);
    if (a.n_models <= 4) return launch_g<T, N, MZ, 4>(a, s);
    return launch_g<T, N, MZ, 8>(a, s);
}

}  // namespace

bool imm_batch_has_instance(int dim_x, int dim_z, int dtype)
{
    return (dim_x == 2 && dim_z == 1) || (dim_x == 3 && dim_z == 1) || (dim_x == 4 && dim_z == 2 && dtype == BKE_F32);
}

int launch_imm_batch(const bke_imm_batch_args &a, cudaStream_t s)
{
    const int n = a.dim_x, m = a.dim_z;
    if (a.dtype == BKE_F32) {
        if (n == 2 && m == 1) return launch_shape<float, 2, 1>(a, s);
        if (n == 3 && m == 1) return launch_shape<float, 3, 1>(a, s);
        if (n == 4 && m == 2) return launch_shape<float, 4, 2>(a, s);
    } else {
        if (n == 2 && m == 1) return launch_shape<double, 2, 1>(a, s);
        if (n == 3 && m == 1) return launch_shape<double, 3, 1>(a, s);
    }
    set_error("bke_imm_batch_filter: no fused instance for dim_x=%d, dim_z=%d in this dtype", n, m);
    return BKE_ERR_UNSUPPORTED;
}

}  // namespace bke
