// enkf_kernel.cuh — device code of the ensemble Kalman filter bank (see enkf.cu for the host side).
// Free of host headers: compiled by nvcc into libbke.so (closed set of fx / hx models) and by NVRTC around
// user-supplied fx / hx device functions (ukf_rtc.cu, bke_enkf_model_compile).
//
// Per filter, with Nm members s_i (filterpy/kalman/ensemble_kalman_filter.py: initialize :187-215,
// update :218-273, predict :275-290; reference @ 3b51149):
//   initialize:  s_i = x + L_P xi_i                         (x and P themselves are kept as given)
//   predict:     s_i = fx(s_i, dt) + L_Q xi_i;  x = mean(s);  P = sum (s_i - x)(s_i - x)' / (Nm - 1)
//   update:      h_i = hx(s_i);  z^ = mean(h);  S = sum (h_i - z^)(..)' / (Nm - 1) + R
//                Pxz = sum (s_i - x)(h_i - z^)' / (Nm - 1)   with the STORED x, not a fresh mean
//                SI = S^-1;  K = Pxz SI;  s_i += K (z + L_R xi_i - h_i);  x = mean(s);  P = P - K S K'
// (P after an update is NOT the ensemble covariance: the reference subtracts K S K' from the stored P.)
//
// Noise stream: xi are standard normals from Philox4x32-10 (Salmon et al., SC'11) written out below, keyed
// with (seed, filter index) and counted with (component pair, member, draw call, filter index >> 32), turned
// into normals by Box-Muller on uniforms in (0, 1].  A filter's numbers depend on nothing but its index, the
// seed and the draw-call counter, so they do not change with the size of the bank or the launch geometry.
// oracle/enkf.py replicates the stream in NumPy.  L is the lower factor of a symmetric positive SEMI-definite
// matrix (psd_factor), so rank-deficient noise covariances (and Q = 0) are drawn from exactly.
//
// Work split: one warp per filter, members across its lanes (member i on lane i % 32).  The ensemble of a
// filter sits in shared memory when it fits (Ew warps of a CTA each hold Nm x (n|1) elements, the odd stride
// keeps the lane-strided rows conflict-free); otherwise the passes run over the output array in global
// memory, where the re-reads of the filter's rows hit L2.  Means and centred sums are butterfly shuffles:
// every lane ends with the same bits.  The small linear algebra (factors, S^-1, K, P - K S K') is evaluated
// by every lane of the warp on the same values.
#pragma once
#include "ukf_kernel.cuh"

namespace bke {
namespace enkfk {

constexpr int EW = 4;                 // warps (= filters) per CTA
constexpr int EB = 32 * EW;

template <typename T>
struct EnkfP {
    int64_t N;                        // filters
    int32_t Nm;                       // members per filter
    unsigned flags;
    uint32_t seed, counter;           // noise key; draw call of the first draw of the launch
    int32_t onchip;                   // the ensemble is staged in shared memory
    T dt;
    const T *x, *P, *Q, *R, *F, *H, *z;
    int64_t sQ, sR, sF, sH;
    const uint8_t *valid;
    const T *sig_in;                  // [N][Nm][n]
    T *sig_out;                       // [N][Nm][n]; may alias sig_in
    T *x_out, *P_out, *x_prior, *P_prior, *K, *S, *SI;
    int32_t *status;
    const T *fx_args, *hx_args;
    int64_t s_fx_args, s_hx_args;
};

template <typename T>
struct EnkfInitP {
    int64_t N;
    int32_t Nm;
    uint32_t seed, counter;
    const T *x, *P;
    T *sig_out;
    int32_t *status;
};

// ------------------------------------------------------------------------------------------ noise
// Philox4x32-10: ten rounds of the 4x32 S-box, the key bumped by the Weyl constants between rounds
__device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1)
{
#pragma unroll
    for (int r = 0; r < 10; r++) {
        const uint32_t lo0 = 0xD2511F53u * c[0], hi0 = __umulhi(0xD2511F53u, c[0]);
        const uint32_t lo1 = 0xCD9E8D57u * c[2], hi1 = __umulhi(0xCD9E8D57u, c[2]);
        const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
        c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
}

// Box-Muller on one Philox output.  fp64: u1 = (c0:c1 top 53 bits + 1) 2^-53 in (0, 1], u2 = (c2:c3 top 53
// bits) 2^-53.  fp32: u1 = (float(c0) + 1) 2^-32 in (0, 1] and u2 = float(c2) 2^-32 (u2 may round up to 1),
// 24-bit uniforms from one word each.  They are not the fp64 uniforms rounded: the fp32 normals differ from
// the fp64 stream by up to about 1e-3 sigma in the tails (small c0, c0 near 2^32), and oracle/enkf.py draws
// the fp32 stream from these uniforms.  z0 = sqrt(-2 ln u1) cos(2 pi u2), z1 = sqrt(-2 ln u1) sin(2 pi u2).
template <typename T>
__device__ __forceinline__ void box_muller(const uint32_t (&c)[4], T &z0, T &z1)
{
    if constexpr (sizeof(T) == 8) {
        const double u1 = (double)((((uint64_t)c[0] << 21) | (c[1] >> 11)) + 1ull) * 0x1p-53;
        const double u2 = (double)(((uint64_t)c[2] << 21) | (c[3] >> 11)) * 0x1p-53;
        const double r = sqrt(-2.0 * log(u1));
        double s, co;
        sincospi(2.0 * u2, &s, &co);
        z0 = r * co; z1 = r * s;
    } else {
        const float u1 = ((float)c[0] + 1.0f) * 0x1p-32f;
        const float u2 = (float)c[2] * 0x1p-32f;
        const float r = sqrtf(-2.0f * logf(u1));
        float s, co;
        sincospif(2.0f * u2, &s, &co);
        z0 = r * co; z1 = r * s;
    }
}

// the K standard normals of (filter f, draw call, member); components 2q and 2q+1 come from counter q
template <typename T, int K>
__device__ __forceinline__ void std_normals(uint32_t seed, int64_t f, uint32_t call, uint32_t member, T (&xi)[K])
{
#pragma unroll
    for (int q = 0; q < (K + 1) / 2; q++) {
        uint32_t c[4] = {(uint32_t)q, member, call, (uint32_t)((uint64_t)f >> 32)};
        philox4x32_10(c, seed, (uint32_t)f);
        T z0, z1;
        box_muller<T>(c, z0, z1);
        xi[2 * q] = z0;
        if (2 * q + 1 < K) xi[2 * q + 1] = z1;
    }
}

// Lower factor L (L L' = C) of a symmetric positive semi-definite K x K matrix, reading C's lower triangle.
// Cholesky, except that a pivot d <= tol max(diag C), tol = 16 K eps, zeroes its column: the rank-deficient
// directions of C get no noise.  Returns false (C clearly indefinite) when such a pivot is below -tol
// max(diag C) or the column it zeroes has an entry above sqrt(tol) max(diag C) (a PSD matrix with a zero
// pivot has a zero column below it).
template <typename T, int K>
__device__ __forceinline__ bool psd_factor(const T *C, T (&L)[K][K])
{
    constexpr T eps = sizeof(T) == 8 ? T(2.220446049250313e-16) : T(1.1920929e-07);
    T mx = T(0);
#pragma unroll
    for (int i = 0; i < K; i++) mx = fmax(mx, C[i * K + i]);
    const T tol = T(16 * K) * eps * mx, tol_off = sqrt(T(16 * K) * eps) * mx;
    bool ok = true;
#pragma unroll
    for (int j = 0; j < K; j++) {
#pragma unroll
        for (int i = 0; i < j; i++) L[i][j] = T(0);
        T d = C[j * K + j];
#pragma unroll
        for (int k = 0; k < j; k++) d -= L[j][k] * L[j][k];
        const bool piv = d > tol;
        ok = ok && (d >= -tol);
        const T r = piv ? sqrt(d) : T(0);
        L[j][j] = r;
        const T inv = piv ? T(1) / r : T(0);
#pragma unroll
        for (int i = j + 1; i < K; i++) {
            T s = C[i * K + j];
#pragma unroll
            for (int k = 0; k < j; k++) s -= L[i][k] * L[j][k];
            ok = ok && (piv || !(fabs(s) > tol_off));
            L[i][j] = s * inv;
        }
    }
    return ok;
}

// e = L xi (L lower)
template <typename T, int K>
__device__ __forceinline__ void lower_mul(const T (&L)[K][K], const T (&xi)[K], T (&e)[K])
{
#pragma unroll
    for (int i = 0; i < K; i++) {
        T s = L[i][0] * xi[0];
#pragma unroll
        for (int j = 1; j <= i; j++) s += L[i][j] * xi[j];
        e[i] = s;
    }
}

template <typename T, int K>
__device__ __forceinline__ void warp_sum(T (&v)[K])
{
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
        for (int k = 0; k < K; k++) v[k] += __shfl_xor_sync(FULL, v[k], off);
}

// ------------------------------------------------------------------------------------------ kernels
// initialize (:206): s_i = x + L_P xi_i.  An indefinite P sets status and leaves every member at x.
template <typename T, int N>
__global__ void __launch_bounds__(EB) enkf_init_kernel(EnkfInitP<T> p)
{
    const int lane = threadIdx.x & 31;
    const int64_t f = (int64_t)blockIdx.x * EW + (threadIdx.x >> 5);
    if (f >= p.N) return;
    T L[N][N], x[N];
    const bool ok = psd_factor<T, N>(p.P + f * N * N, L);
#pragma unroll
    for (int i = 0; i < N; i++) x[i] = p.x[f * N + i];
    T *out = p.sig_out + f * (int64_t)p.Nm * N;
    for (int i = lane; i < p.Nm; i += 32) {
        T xi[N], e[N];
        std_normals<T, N>(p.seed, f, p.counter, (uint32_t)i, xi);
        lower_mul<T, N>(L, xi, e);
#pragma unroll
        for (int k = 0; k < N; k++) out[(int64_t)i * N + k] = ok ? x[k] + e[k] : x[k];
    }
    if (p.status && lane == 0) p.status[f] = ok ? BKE_STATUS_OK : BKE_STATUS_NOT_PD;
}

// One launch: predict (BKE_DO_PREDICT, draw call `counter`), update (BKE_DO_UPDATE, draw call counter + 1
// after a predict, else `counter`), or both.  A filter whose noise covariance is indefinite (status NOT_PD)
// or whose S is singular (SINGULAR_S) keeps the state it had before the failing half.
// EXTRAS: the optional outputs (x_prior, P_prior, K, S, SI) are compiled in.
template <typename T, int N, int M, int FX, int HX, bool EXTRAS>
__global__ void __launch_bounds__(EB) enkf_kernel(EnkfP<T> p)
{
    using namespace ukfk;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    constexpr int PADN = N | 1;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t f = (int64_t)blockIdx.x * EW + w;
    if (f >= p.N) return;                                    // whole warps leave; no CTA-wide barrier follows
    const bool do_p = p.flags & BKE_DO_PREDICT, do_u = p.flags & BKE_DO_UPDATE;
    const int Nm = p.Nm;
    const T inv_n = T(1) / T(Nm), inv_n1 = T(1) / T(Nm - 1);
    const T *src = p.sig_in + f * (int64_t)Nm * N;
    T *gout = p.sig_out + f * (int64_t)Nm * N;
    T *ens = p.onchip ? reinterpret_cast<T *>(smem_raw) + (size_t)w * Nm * PADN : gout;
    const int es = p.onchip ? PADN : N;                      // element distance between members in `ens`
    if (ens != src)
        for (int e = lane; e < Nm * N; e += 32) ens[(e / N) * es + e % N] = src[e];
    __syncwarp();

    const T *Fp = (FX == BKE_FX_LINEAR && do_p) ? p.F + f * p.sF : nullptr;
    const T *Hp = (HX == BKE_HX_LINEAR && do_u) ? p.H + f * p.sH : nullptr;
    const T *fxa = (FX == BKE_FX_USER && p.fx_args) ? p.fx_args + f * p.s_fx_args : nullptr;
    const T *hxa = (HX == BKE_HX_USER && p.hx_args) ? p.hx_args + f * p.s_hx_args : nullptr;

    T x[N], P[N][N];
#pragma unroll
    for (int i = 0; i < N; i++) x[i] = p.x[f * N + i];
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int j = 0; j < N; j++) P[i][j] = p.P[f * N * N + i * N + j];
    int st = BKE_STATUS_OK;

    if (do_p) {
        T L[N][N];
        if (!psd_factor<T, N>(p.Q + f * p.sQ, L)) st = BKE_STATUS_NOT_PD;
        if (st == BKE_STATUS_OK) {
            // s_i = fx(s_i) + L_Q xi_i, and their sum
            T acc[N];
#pragma unroll
            for (int k = 0; k < N; k++) acc[k] = T(0);
            for (int i = lane; i < Nm; i += 32) {
                T s[N], fs[N], xi[N], e[N];
#pragma unroll
                for (int k = 0; k < N; k++) s[k] = ens[i * es + k];
                apply_fx<T, N, FX>(s, fs, p.dt, Fp, 1, fxa);
                std_normals<T, N>(p.seed, f, p.counter, (uint32_t)i, xi);
                lower_mul<T, N>(L, xi, e);
#pragma unroll
                for (int k = 0; k < N; k++) { fs[k] += e[k]; ens[i * es + k] = fs[k]; acc[k] += fs[k]; }
            }
            warp_sum<T, N>(acc);
#pragma unroll
            for (int k = 0; k < N; k++) x[k] = acc[k] * inv_n;
            // centred sum about the mean (upper triangle)
            constexpr int NT = N * (N + 1) / 2;
            T pa[NT];
#pragma unroll
            for (int k = 0; k < NT; k++) pa[k] = T(0);
            for (int i = lane; i < Nm; i += 32) {
                T d[N];
#pragma unroll
                for (int k = 0; k < N; k++) d[k] = ens[i * es + k] - x[k];
#pragma unroll
                for (int a = 0; a < N; a++)
#pragma unroll
                    for (int b = a; b < N; b++) pa[tri_index<N>(a, b)] += d[a] * d[b];
            }
            warp_sum<T, NT>(pa);
#pragma unroll
            for (int a = 0; a < N; a++)
#pragma unroll
                for (int b = a; b < N; b++) { P[a][b] = pa[tri_index<N>(a, b)] * inv_n1; P[b][a] = P[a][b]; }
            if (EXTRAS && lane == 0) {
                if (p.x_prior) for (int i = 0; i < N; i++) p.x_prior[f * N + i] = x[i];
                if (p.P_prior) for (int i = 0; i < N; i++) for (int j = 0; j < N; j++) p.P_prior[f * N * N + i * N + j] = P[i][j];
            }
        }
    }

    const bool has_z = p.valid == nullptr || p.valid[f] != 0;
    if (do_u && has_z && st == BKE_STATUS_OK) {
        // z^ = mean hx(s_i)
        T zm[M];
#pragma unroll
        for (int a = 0; a < M; a++) zm[a] = T(0);
        for (int i = lane; i < Nm; i += 32) {
            T s[N], h[M];
#pragma unroll
            for (int k = 0; k < N; k++) s[k] = ens[i * es + k];
            apply_hx<T, N, M, HX>(s, h, Hp, 1, hxa);
#pragma unroll
            for (int a = 0; a < M; a++) zm[a] += h[a];
        }
        warp_sum<T, M>(zm);
#pragma unroll
        for (int a = 0; a < M; a++) zm[a] *= inv_n;
        // S and Pxz as centred sums (S upper triangle first, then N x M cross terms)
        constexpr int MT = M * (M + 1) / 2;
        T acc[MT + N * M];
#pragma unroll
        for (int k = 0; k < MT + N * M; k++) acc[k] = T(0);
        for (int i = lane; i < Nm; i += 32) {
            T s[N], h[M];
#pragma unroll
            for (int k = 0; k < N; k++) s[k] = ens[i * es + k];
            apply_hx<T, N, M, HX>(s, h, Hp, 1, hxa);
#pragma unroll
            for (int a = 0; a < M; a++) h[a] -= zm[a];
#pragma unroll
            for (int a = 0; a < M; a++)
#pragma unroll
                for (int b = a; b < M; b++) acc[tri_index<M>(a, b)] += h[a] * h[b];
#pragma unroll
            for (int k = 0; k < N; k++) {
                const T dx = s[k] - x[k];
#pragma unroll
                for (int a = 0; a < M; a++) acc[MT + k * M + a] += dx * h[a];
            }
        }
        warp_sum<T, MT + N * M>(acc);
        const T *Rf = p.R + f * p.sR;
        T S[M][M], SI[M][M], Kg[N][M];
#pragma unroll
        for (int a = 0; a < M; a++)
#pragma unroll
            for (int b = a; b < M; b++) {
                const T c = acc[tri_index<M>(a, b)] * inv_n1;
                S[a][b] = c + Rf[a * M + b];
                S[b][a] = c + Rf[b * M + a];
            }
        T logdet;
        if (!reg_inverse<T, M>(S, SI, logdet)) st = BKE_STATUS_SINGULAR_S;
        T LR[M][M];
        if (st == BKE_STATUS_OK && !psd_factor<T, M>(Rf, LR)) st = BKE_STATUS_NOT_PD;
        if (st == BKE_STATUS_OK) {
#pragma unroll
            for (int k = 0; k < N; k++)
#pragma unroll
                for (int a = 0; a < M; a++) {
                    T s = T(0);
#pragma unroll
                    for (int b = 0; b < M; b++) s += acc[MT + k * M + b] * inv_n1 * SI[b][a];
                    Kg[k][a] = s;
                }
            T zv[M];
#pragma unroll
            for (int a = 0; a < M; a++) zv[a] = p.z[f * M + a];
            const uint32_t call = p.counter + (do_p ? 1u : 0u);
            // s_i += K (z + L_R xi_i - hx(s_i)), and their sum
            T xs[N];
#pragma unroll
            for (int k = 0; k < N; k++) xs[k] = T(0);
            for (int i = lane; i < Nm; i += 32) {
                T s[N], h[M], xi[M], r[M];
#pragma unroll
                for (int k = 0; k < N; k++) s[k] = ens[i * es + k];
                apply_hx<T, N, M, HX>(s, h, Hp, 1, hxa);
                std_normals<T, M>(p.seed, f, call, (uint32_t)i, xi);
                lower_mul<T, M>(LR, xi, r);
#pragma unroll
                for (int a = 0; a < M; a++) h[a] = zv[a] + r[a] - h[a];
#pragma unroll
                for (int k = 0; k < N; k++) {
                    T v = s[k];
#pragma unroll
                    for (int a = 0; a < M; a++) v += Kg[k][a] * h[a];
                    ens[i * es + k] = v;
                    xs[k] += v;
                }
            }
            warp_sum<T, N>(xs);
#pragma unroll
            for (int k = 0; k < N; k++) x[k] = xs[k] * inv_n;
            // P -= K (S K')
            T SK[M][N];
#pragma unroll
            for (int a = 0; a < M; a++)
#pragma unroll
                for (int j = 0; j < N; j++) {
                    T s = S[a][0] * Kg[j][0];
#pragma unroll
                    for (int b = 1; b < M; b++) s += S[a][b] * Kg[j][b];
                    SK[a][j] = s;
                }
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = 0; j < N; j++) {
                    T s = Kg[i][0] * SK[0][j];
#pragma unroll
                    for (int a = 1; a < M; a++) s += Kg[i][a] * SK[a][j];
                    P[i][j] -= s;
                }
            if (EXTRAS && lane == 0) {
                if (p.K) for (int i = 0; i < N; i++) for (int a = 0; a < M; a++) p.K[f * N * M + i * M + a] = Kg[i][a];
                if (p.S) for (int a = 0; a < M; a++) for (int b = 0; b < M; b++) p.S[f * M * M + a * M + b] = S[a][b];
                if (p.SI) for (int a = 0; a < M; a++) for (int b = 0; b < M; b++) p.SI[f * M * M + a * M + b] = SI[a][b];
            }
        }
    }

    __syncwarp();
    if (p.onchip)
        for (int e = lane; e < Nm * N; e += 32) gout[e] = ens[(e / N) * es + e % N];
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < N; i++) p.x_out[f * N + i] = x[i];
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < N; j++) p.P_out[f * N * N + i * N + j] = P[i][j];
        if (p.status) p.status[f] = st;
    }
}

}  // namespace enkfk
}  // namespace bke
