// information.cu — information filter bank (bke_if_step) and the batched inverse of the F setter and the P
// property (bke_inverse).
//
// Arithmetic follows filterpy/kalman/information_filter.py (reference @ 3b51149); "inv" is np.linalg.inv:
//   predict :258-289   A = F_inv' P_inv F_inv
//                      inv(A) succeeds:  if no_information: x = inv(P_inv) x (0 x if that inv fails), flag cleared;
//                                        x = F x + B u;  P_inv = inv(inv(A) + Q);  priors = (x, P_inv)
//                      inv(A) fails:     flag set;  I_PF = I - P_inv F_inv;  FTI = inv(F');  AQI = inv(A + Q);
//                                        x = FTI ((I_PF AQI) (FTI x));  priors = (x, AQI);  P_inv unchanged
//   update  :194-243   no_information:   x = P_inv x + (H' R_inv) z;  P_inv = P_inv + (H' R_inv) H;  ll = log(DBL_MIN)
//                      otherwise:        y = z - H x;  S = P_inv + (H' R_inv) H;  K = (inv(S) H') R_inv;  x = x + K y;
//                                        P_inv = S;  ll = logpdf(y, cov=S) (scipy broadcasts y over n when m == 1)
// "inv fails" is the rule of reg_inverse (kf_regtile.cuh) and warp_inverse (kf_warp.cuh): a zero pivot of the
// partially pivoted elimination (for n = 2 in the register tile, LAPACK's dgetrf2 decision: see if_inverse).
// The inverses of AI + Q, F', A + Q and S are not caught by the reference: where one fails the filter gets
// BKE_STATUS_SINGULAR_S and stops with what the reference has set by then.  inv(A) and inv(P_inv) are caught: they pick a branch, per filter, inside the one launch.
//
// Two paths, picked by shape: a register tile per thread (16-byte row loads as in kf_direct.cu) for kf_direct's
// shapes without control input, and a warp per filter with the matrices in the warp's slice of shared memory for
// every other shape and for a control input.
#include "bke_internal.cuh"
#include "kf_regtile.cuh"
#include "kf_rowio.cuh"
#include "kf_warp.cuh"

namespace bke {
namespace {

template <typename T>
struct IfP {
    int64_t N;
    int n, m, du, ll_mode;
    unsigned flags;
    const T *x, *Pi;
    T *x_out, *Pi_out;
    uint8_t *ni;
    const T *F, *Fi, *Q, *H, *Ri, *B, *u, *z;
    int64_t sF, sFi, sQ, sH, sRi, sB, su;
    const uint8_t *valid;
    T *x_prior, *Pi_prior, *K, *y, *S, *ll;
    int32_t *status;
};

template <typename T>
__device__ __forceinline__ T log_float_min() { return T(-708.39641853226408); }   // log(DBL_MIN), information_filter.py:214

// -0.5 (n log 2pi + log|det S| + q), q = y' SI y (m == n) or y0^2 sum(SI) (m == 1: y repeated n times)
template <typename T>
__device__ __forceinline__ T if_logpdf(int n, T logdet, T q)
{
    return T(-0.5) * (T(n) * T(LOG_2PI) + logdet + q);
}

// The inverse of the register tile.  For n = 2 it is not reg_inverse, whose closed-form determinant contracts to an
// FMA and so misses a zero pivot that LAPACK finds (A = [[a, -a], [-a, a]]): the 2 x 2 inverse comes from
// dgetrf2's LU, pivot, reciprocal, u11 = d - l b rounded term by term, so that the singular / non-singular
// decision, SI and logdet all come from the same factors.  Every other n is reg_inverse.
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }

template <typename T, int N>
__device__ __forceinline__ bool if_inverse(const T (&S)[N][N], T (&SI)[N][N], T &logdet)
{
    if constexpr (N == 2) {
        const bool sw = fabs(S[1][0]) > fabs(S[0][0]);      // the rows of P S
        const T a = sw ? S[1][0] : S[0][0], b = sw ? S[1][1] : S[0][1], c = sw ? S[0][0] : S[1][0], d = sw ? S[0][1] : S[1][1];
        const T ra = T(1) / a, l = mul_rn(c, ra), u = sub_rn(d, mul_rn(l, b));
        const T ru = T(1) / u, t = b * ra * ru;
        // (P S)^-1 = U^-1 L^-1 = [[1/a + t l, -t], [-l / u, 1/u]];  S^-1 = (P S)^-1 P swaps its columns back
        const T x00 = ra + t * l, x01 = -t, x10 = -l * ru, x11 = ru;
        SI[0][0] = sw ? x01 : x00; SI[0][1] = sw ? x00 : x01;
        SI[1][0] = sw ? x11 : x10; SI[1][1] = sw ? x10 : x11;
        logdet = log(fabs(a)) + log(fabs(u));
        return a != T(0) && u != T(0);
    } else {
        return reg_inverse<T, N>(S, SI, logdet);
    }
}

template <typename T, int N, int M, bool EX>
__global__ void __launch_bounds__(128) if_reg_kernel(IfP<T> p)
{
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.N) return;
    T x[N], Pi[N][N];
    ldv_rw<T, N>(x, p.x + f * N);
    ldv_rw<T, N * N>(&Pi[0][0], p.Pi + f * N * N);
    bool ni = p.ni[f] != 0;
    int st = BKE_STATUS_OK;
    if (p.flags & BKE_DO_PREDICT) {
        T Fi[N][N], A[N][N], AI[N][N], Q[N][N], F[N][N], ld;
        ldv<T, N * N>(&Fi[0][0], p.Fi + f * p.sFi);
        {
            T PF[N][N];
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = 0; j < N; j++) {
                    T s = T(0);
#pragma unroll
                    for (int k = 0; k < N; k++) s += Pi[i][k] * Fi[k][j];
                    PF[i][j] = s;
                }
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = 0; j < N; j++) {
                    T s = T(0);
#pragma unroll
                    for (int k = 0; k < N; k++) s += Fi[k][i] * PF[k][j];
                    A[i][j] = s;                                       // F_inv' (P_inv F_inv)
                }
        }
        const bool invertible = if_inverse<T, N>(A, AI, ld);
        ldv<T, N * N>(&Q[0][0], p.Q + f * p.sQ);
        ldv<T, N * N>(&F[0][0], p.F + f * p.sF);
        if (invertible) {
            if (ni) {
                T PiI[N][N], xn[N];
                const bool ok = if_inverse<T, N>(Pi, PiI, ld);
#pragma unroll
                for (int i = 0; i < N; i++) {
                    T s = T(0);
#pragma unroll
                    for (int k = 0; k < N; k++) s += PiI[i][k] * x[k];
                    xn[i] = ok ? s : T(0) * x[i];                      // dot(0, x)
                }
#pragma unroll
                for (int i = 0; i < N; i++) x[i] = xn[i];
                ni = false;
            }
            T xn[N];
#pragma unroll
            for (int i = 0; i < N; i++) {
                T s = T(0);
#pragma unroll
                for (int k = 0; k < N; k++) s += F[i][k] * x[k];
                xn[i] = s;
            }
#pragma unroll
            for (int i = 0; i < N; i++) {
                x[i] = xn[i];
#pragma unroll
                for (int j = 0; j < N; j++) AI[i][j] += Q[i][j];
            }
            T Pn[N][N];
            if (if_inverse<T, N>(AI, Pn, ld)) {
#pragma unroll
                for (int i = 0; i < N; i++)
#pragma unroll
                    for (int j = 0; j < N; j++) Pi[i][j] = Pn[i][j];
                if (EX && p.x_prior) stv<T, N>(p.x_prior + f * N, x);
                if (EX && p.Pi_prior) stv<T, N * N>(p.Pi_prior + f * N * N, &Pi[0][0]);
            } else {
                st = BKE_STATUS_SINGULAR_S;                            // inv(AI + Q) raises (:275)
            }
        } else {
            ni = true;
            T IPF[N][N], FT[N][N], FTI[N][N], AQI[N][N];
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = 0; j < N; j++) {
                    T s = T(0);
#pragma unroll
                    for (int k = 0; k < N; k++) s += Pi[i][k] * Fi[k][j];
                    IPF[i][j] = (i == j ? T(1) : T(0)) - s;
                    FT[i][j] = F[j][i];
                    A[i][j] += Q[i][j];
                }
            const bool ok_f = if_inverse<T, N>(FT, FTI, ld);
            const bool ok_a = if_inverse<T, N>(A, AQI, ld);
            if (ok_f && ok_a) {
                T u[N], v[N];
#pragma unroll
                for (int i = 0; i < N; i++) {
                    T s = T(0);
#pragma unroll
                    for (int k = 0; k < N; k++) s += FTI[i][k] * x[k];
                    u[i] = s;                                          // FTIX
                }
#pragma unroll
                for (int i = 0; i < N; i++) {
                    T s = T(0);
#pragma unroll
                    for (int j = 0; j < N; j++) {
                        T w = T(0);
#pragma unroll
                        for (int k = 0; k < N; k++) w += IPF[i][k] * AQI[k][j];
                        s += w * u[j];
                    }
                    v[i] = s;                                          // (I_PF AQI) FTIX
                }
#pragma unroll
                for (int i = 0; i < N; i++) {
                    T s = T(0);
#pragma unroll
                    for (int k = 0; k < N; k++) s += FTI[i][k] * v[k];
                    x[i] = s;
                }
                if (EX && p.x_prior) stv<T, N>(p.x_prior + f * N, x);
                if (EX && p.Pi_prior) stv<T, N * N>(p.Pi_prior + f * N * N, &AQI[0][0]);
            } else {
                st = BKE_STATUS_SINGULAR_S;                            // inv(F') or inv(A + Q) raises (:282, :284)
            }
        }
    }
    if (st == BKE_STATUS_OK && (p.flags & BKE_DO_UPDATE) && (p.valid == nullptr || p.valid[f] != 0)) {
        T H[M][N], Ri[M][M], z[M], HR[N][M];
        ldv<T, M * N>(&H[0][0], p.H + f * p.sH);
        ldv<T, M * M>(&Ri[0][0], p.Ri + f * p.sRi);
        ldv<T, M>(z, p.z + f * M);
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int b = 0; b < M; b++) {
                T s = T(0);
#pragma unroll
                for (int a = 0; a < M; a++) s += H[a][i] * Ri[a][b];
                HR[i][b] = s;                                          // dot(H_T, R_inv)
            }
        if (ni) {
            T xn[N];
#pragma unroll
            for (int i = 0; i < N; i++) {
                T s = T(0), t = T(0);
#pragma unroll
                for (int k = 0; k < N; k++) s += Pi[i][k] * x[k];
#pragma unroll
                for (int b = 0; b < M; b++) t += HR[i][b] * z[b];
                xn[i] = s + t;
            }
#pragma unroll
            for (int i = 0; i < N; i++) {
                x[i] = xn[i];
#pragma unroll
                for (int j = 0; j < N; j++) {
                    T s = T(0);
#pragma unroll
                    for (int b = 0; b < M; b++) s += HR[i][b] * H[b][j];
                    Pi[i][j] += s;
                }
            }
            if (p.ll) p.ll[f] = log_float_min<T>();
        } else {
            T y[M], S[N][N], SI[N][N], logdet;
#pragma unroll
            for (int a = 0; a < M; a++) {
                T s = T(0);
#pragma unroll
                for (int k = 0; k < N; k++) s += H[a][k] * x[k];
                y[a] = z[a] - s;
            }
#pragma unroll
            for (int i = 0; i < N; i++)
#pragma unroll
                for (int j = 0; j < N; j++) {
                    T s = T(0);
#pragma unroll
                    for (int b = 0; b < M; b++) s += HR[i][b] * H[b][j];
                    S[i][j] = Pi[i][j] + s;
                }
            if (EX && p.y) stv<T, M>(p.y + f * M, y);
            if (EX && p.S) stv<T, N * N>(p.S + f * N * N, &S[0][0]);
            if (if_inverse<T, N>(S, SI, logdet)) {
                T K[N][M];
#pragma unroll
                for (int i = 0; i < N; i++) {
                    T SH[M];
#pragma unroll
                    for (int a = 0; a < M; a++) {
                        T s = T(0);
#pragma unroll
                        for (int k = 0; k < N; k++) s += SI[i][k] * H[a][k];
                        SH[a] = s;                                     // dot(inv(S), H_T)
                    }
#pragma unroll
                    for (int b = 0; b < M; b++) {
                        T s = T(0);
#pragma unroll
                        for (int a = 0; a < M; a++) s += SH[a] * Ri[a][b];
                        K[i][b] = s;
                    }
                }
#pragma unroll
                for (int i = 0; i < N; i++) {
                    T s = T(0);
#pragma unroll
                    for (int b = 0; b < M; b++) s += K[i][b] * y[b];
                    x[i] += s;
#pragma unroll
                    for (int j = 0; j < N; j++) Pi[i][j] = S[i][j];
                }
                if (EX && p.K) stv<T, N * M>(p.K + f * N * M, &K[0][0]);
                if (p.ll_mode != BKE_IF_LL_NONE) {
                    T q = T(0);
#pragma unroll
                    for (int i = 0; i < N; i++)
#pragma unroll
                        for (int j = 0; j < N; j++)
                            q += p.ll_mode == BKE_IF_LL_FULL ? y[i % M] * SI[i][j] * y[j % M] : SI[i][j];
                    if (p.ll_mode == BKE_IF_LL_BROADCAST) q *= y[0] * y[0];
                    p.ll[f] = if_logpdf<T>(N, logdet, q);
                }
            } else {
                st = BKE_STATUS_SINGULAR_S;                            // inv(S) raises (:225)
            }
        }
    }
    stv<T, N>(p.x_out + f * N, x);
    stv<T, N * N>(p.Pi_out + f * N * N, &Pi[0][0]);
    p.ni[f] = ni ? 1 : 0;
    if (p.status && (st != BKE_STATUS_OK || !(p.flags & BKE_STATUS_STICKY))) p.status[f] = st;
}

// per-warp slice: x, xp, v, col (n each), y, zc (m each) | Pi, Fi, A, B1, B2, B3 (n*n each) | H, HR, SH, K (m*n
// each) | Ri (m*m)
inline int if_per_warp(int n, int m)
{
    return 4 * n + 2 * m + 6 * n * n + 4 * m * n + m * m;
}

template <typename T>
__global__ void __launch_bounds__(128) if_warp_kernel(IfP<T> p, int per_warp)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const int n = p.n, m = p.m, nn = n * n, nm = n * m, mm = m * m;
    T *x = reinterpret_cast<T *>(smem_raw) + (size_t)wib * per_warp;
    T *xp = x + n, *v = xp + n, *col = v + n, *y = col + n, *zc = y + m;
    T *Pi = zc + m, *Fi = Pi + nn, *A = Fi + nn, *B1 = A + nn, *B2 = B1 + nn, *B3 = B2 + nn;
    T *H = B3 + nn, *HR = H + nm, *SH = HR + nm, *K = SH + nm, *Ri = K + nm;

    for (int64_t f = (int64_t)blockIdx.x * wpb + wib; f < p.N; f += (int64_t)gridDim.x * wpb) {
        warp_copy_in(x, p.x + f * n, n, lane);
        warp_copy_in(Pi, p.Pi + f * nn, nn, lane);
        bool ni = p.ni[f] != 0;
        int st = BKE_STATUS_OK;
        T ld;
        __syncwarp();
        if (p.flags & BKE_DO_PREDICT) {
            const T *F = p.F + f * p.sF, *Q = p.Q + f * p.sQ;
            warp_copy_in(Fi, p.Fi + f * p.sFi, nn, lane);
            __syncwarp();
            warp_mm<false>(Pi, Fi, n, n, n, lane, [&](int e, int, int, T s) { B1[e] = s; });        // P_inv F_inv
            __syncwarp();
            for (int e = lane; e < nn; e += 32) {
                int i = e / n, j = e - i * n;
                T s = T(0);
                for (int k = 0; k < n; k++) s += Fi[k * n + i] * B1[k * n + j];
                A[e] = s;                                              // F_inv' (P_inv F_inv)
                B2[e] = s;
            }
            __syncwarp();
            if (warp_inverse(B2, B3, col, n, lane, ld)) {              // B3 = inv(A)
                if (ni) {
                    for (int e = lane; e < nn; e += 32) B2[e] = Pi[e];
                    __syncwarp();
                    const bool ok = warp_inverse(B2, B1, col, n, lane, ld);
                    for (int i = lane; i < n; i += 32) {
                        T s = T(0);
                        for (int k = 0; k < n; k++) s += B1[i * n + k] * x[k];
                        xp[i] = ok ? s : T(0) * x[i];                  // dot(0, x)
                    }
                    __syncwarp();
                    for (int i = lane; i < n; i += 32) x[i] = xp[i];
                    ni = false;
                    __syncwarp();
                }
                for (int i = lane; i < n; i += 32) {
                    T s = T(0);
                    for (int k = 0; k < n; k++) s += F[i * n + k] * x[k];
                    if (p.B != nullptr && p.u != nullptr) {
                        const T *Bf = p.B + f * p.sB, *uf = p.u + f * p.su;
                        T b = T(0);
                        for (int q = 0; q < p.du; q++) b += Bf[i * p.du + q] * uf[q];
                        s += b;
                    }
                    xp[i] = s;
                }
                for (int e = lane; e < nn; e += 32) B3[e] += Q[e];
                __syncwarp();
                for (int i = lane; i < n; i += 32) x[i] = xp[i];
                if (warp_inverse(B3, B1, col, n, lane, ld)) {
                    for (int e = lane; e < nn; e += 32) Pi[e] = B1[e];
                    __syncwarp();
                    if (p.x_prior) for (int i = lane; i < n; i += 32) p.x_prior[f * n + i] = x[i];
                    if (p.Pi_prior) for (int e = lane; e < nn; e += 32) p.Pi_prior[f * nn + e] = Pi[e];
                } else {
                    st = BKE_STATUS_SINGULAR_S;                        // inv(AI + Q) raises (:275)
                }
            } else {
                // a failed warp_inverse returns from its pivot search with no barrier: the lanes may still be
                // reading B2 there
                __syncwarp();
                ni = true;
                warp_mm<false>(Pi, Fi, n, n, n, lane, [&](int e, int i, int j, T s) { B1[e] = (i == j ? T(1) : T(0)) - s; });
                for (int e = lane; e < nn; e += 32) {
                    int i = e / n, j = e - i * n;
                    B2[e] = F[j * n + i];                              // F'
                }
                __syncwarp();
                for (int e = lane; e < nn; e += 32) Fi[e] = A[e] + Q[e];
                const bool ok_f = warp_inverse(B2, B3, col, n, lane, ld);      // B3 = FTI
                __syncwarp();
                const bool ok_a = ok_f && warp_inverse(Fi, A, col, n, lane, ld);  // A = AQI
                __syncwarp();
                if (ok_a) {
                    for (int i = lane; i < n; i += 32) {
                        T s = T(0);
                        for (int k = 0; k < n; k++) s += B3[i * n + k] * x[k];
                        xp[i] = s;                                     // FTIX
                    }
                    warp_mm<false>(B1, A, n, n, n, lane, [&](int e, int, int, T s) { B2[e] = s; });  // I_PF AQI
                    __syncwarp();
                    for (int i = lane; i < n; i += 32) {
                        T s = T(0);
                        for (int k = 0; k < n; k++) s += B2[i * n + k] * xp[k];
                        v[i] = s;
                    }
                    __syncwarp();
                    for (int i = lane; i < n; i += 32) {
                        T s = T(0);
                        for (int k = 0; k < n; k++) s += B3[i * n + k] * v[k];
                        x[i] = s;
                    }
                    __syncwarp();
                    if (p.x_prior) for (int i = lane; i < n; i += 32) p.x_prior[f * n + i] = x[i];
                    if (p.Pi_prior) for (int e = lane; e < nn; e += 32) p.Pi_prior[f * nn + e] = A[e];
                } else {
                    st = BKE_STATUS_SINGULAR_S;                        // inv(F') or inv(A + Q) raises (:282, :284)
                }
            }
            __syncwarp();
        }
        if (st == BKE_STATUS_OK && (p.flags & BKE_DO_UPDATE) && (p.valid == nullptr || p.valid[f] != 0)) {
            warp_copy_in(H, p.H + f * p.sH, nm, lane);
            warp_copy_in(Ri, p.Ri + f * p.sRi, mm, lane);
            warp_copy_in(zc, p.z + f * m, m, lane);
            __syncwarp();
            for (int e = lane; e < nm; e += 32) {
                int i = e / m, b = e - i * m;
                T s = T(0);
                for (int a = 0; a < m; a++) s += H[a * n + i] * Ri[a * m + b];
                HR[e] = s;                                             // dot(H_T, R_inv)
            }
            __syncwarp();
            warp_mm<false>(HR, H, n, m, n, lane, [&](int e, int, int, T s) { B1[e] = Pi[e] + s; });
            if (ni) {
                for (int i = lane; i < n; i += 32) {
                    T s = T(0), t = T(0);
                    for (int k = 0; k < n; k++) s += Pi[i * n + k] * x[k];
                    for (int b = 0; b < m; b++) t += HR[i * m + b] * zc[b];
                    xp[i] = s + t;
                }
                __syncwarp();
                for (int i = lane; i < n; i += 32) x[i] = xp[i];
                for (int e = lane; e < nn; e += 32) Pi[e] = B1[e];
                if (p.ll && lane == 0) p.ll[f] = log_float_min<T>();
            } else {
                for (int a = lane; a < m; a += 32) {
                    T s = T(0);
                    for (int k = 0; k < n; k++) s += H[a * n + k] * x[k];
                    y[a] = zc[a] - s;
                }
                __syncwarp();
                for (int e = lane; e < nn; e += 32) B2[e] = B1[e];
                if (p.y) for (int a = lane; a < m; a += 32) p.y[f * m + a] = y[a];
                if (p.S) for (int e = lane; e < nn; e += 32) p.S[f * nn + e] = B1[e];
                __syncwarp();
                T logdet = T(0);
                if (warp_inverse(B2, B3, col, n, lane, logdet)) {     // B3 = inv(S)
                    warp_mm<true>(B3, H, n, n, m, lane, [&](int e, int, int, T s) { SH[e] = s; });   // inv(S) H'
                    __syncwarp();
                    warp_mm<false>(SH, Ri, n, m, m, lane, [&](int e, int, int, T s) { K[e] = s; });
                    __syncwarp();
                    for (int i = lane; i < n; i += 32) {
                        T s = T(0);
                        for (int b = 0; b < m; b++) s += K[i * m + b] * y[b];
                        x[i] += s;
                    }
                    for (int e = lane; e < nn; e += 32) Pi[e] = B1[e];
                    if (p.K) for (int e = lane; e < nm; e += 32) p.K[f * nm + e] = K[e];
                    if (p.ll_mode != BKE_IF_LL_NONE && lane == 0) {
                        T q = T(0);
                        for (int i = 0; i < n; i++)
                            for (int j = 0; j < n; j++)
                                q += p.ll_mode == BKE_IF_LL_FULL ? y[i % m] * B3[i * n + j] * y[j % m] : B3[i * n + j];
                        if (p.ll_mode == BKE_IF_LL_BROADCAST) q *= y[0] * y[0];
                        p.ll[f] = if_logpdf<T>(n, logdet, q);
                    }
                } else {
                    st = BKE_STATUS_SINGULAR_S;                        // inv(S) raises (:225)
                }
            }
        }
        __syncwarp();
        for (int i = lane; i < n; i += 32) p.x_out[f * n + i] = x[i];
        for (int e = lane; e < nn; e += 32) p.Pi_out[f * nn + e] = Pi[e];
        if (lane == 0) {
            p.ni[f] = ni ? 1 : 0;
            if (p.status && (st != BKE_STATUS_OK || !(p.flags & BKE_STATUS_STICKY))) p.status[f] = st;
        }
        __syncwarp();
    }
}

template <typename T>
IfP<T> params(const bke_if_args &a)
{
    IfP<T> p;
    p.N = a.n_filters; p.n = a.dim_x; p.m = a.dim_z; p.du = a.dim_u; p.ll_mode = a.ll_mode; p.flags = a.flags;
    p.x = (const T *)a.x; p.Pi = (const T *)a.P_inv; p.x_out = (T *)a.x_out; p.Pi_out = (T *)a.P_inv_out;
    p.ni = a.no_information;
    p.F = (const T *)a.F; p.Fi = (const T *)a.F_inv; p.Q = (const T *)a.Q; p.H = (const T *)a.H;
    p.Ri = (const T *)a.R_inv; p.B = (const T *)a.B; p.u = (const T *)a.u; p.z = (const T *)a.z;
    p.sF = a.F_stride; p.sFi = a.F_inv_stride; p.sQ = a.Q_stride; p.sH = a.H_stride; p.sRi = a.R_inv_stride;
    p.sB = a.B_stride; p.su = a.u_stride;
    p.valid = a.z_valid;
    p.x_prior = (T *)a.x_prior; p.Pi_prior = (T *)a.P_inv_prior; p.K = (T *)a.K; p.y = (T *)a.y; p.S = (T *)a.S;
    p.ll = (T *)a.log_likelihood; p.status = a.status;
    return p;
}

template <typename T, int N, int M>
int launch_reg(const bke_if_args &a, cudaStream_t s)
{
    if (!(vec_ok<T, N>(a.x) && vec_ok<T, N * N>(a.P_inv) && vec_ok<T, N * N>(a.F, a.F_stride) &&
          vec_ok<T, N * N>(a.F_inv, a.F_inv_stride) && vec_ok<T, N * N>(a.Q, a.Q_stride) &&
          vec_ok<T, M * N>(a.H, a.H_stride) && vec_ok<T, M * M>(a.R_inv, a.R_inv_stride) && vec_ok<T, M>(a.z) &&
          vec_ok<T, N>(a.x_out) && vec_ok<T, N * N>(a.P_inv_out) && vec_ok<T, N>(a.x_prior) &&
          vec_ok<T, N * N>(a.P_inv_prior) && vec_ok<T, N * M>(a.K) && vec_ok<T, M>(a.y) && vec_ok<T, N * N>(a.S)))
        return BKE_ERR_UNSUPPORTED;
    IfP<T> p = params<T>(a);
    const unsigned grid = (unsigned)((p.N + 127) / 128);
    if (a.x_prior || a.P_inv_prior || a.K || a.y || a.S) if_reg_kernel<T, N, M, true><<<grid, 128, 0, s>>>(p);
    else if_reg_kernel<T, N, M, false><<<grid, 128, 0, s>>>(p);
    return check_cuda(cudaGetLastError(), "if_reg_kernel launch");
}

template <typename T>
int launch_warp(const bke_if_args &a, cudaStream_t s)
{
    IfP<T> p = params<T>(a);
    const int per_warp = (if_per_warp(a.dim_x, a.dim_z) + 3) & ~3;
    const size_t bytes_per_warp = (size_t)per_warp * sizeof(T), budget = 200 * 1024;
    WarpShape w;
    if (int rc = warp_shape((const void *)if_warp_kernel<T>, bytes_per_warp, budget, p.N, w)) {
        if (rc == BKE_ERR_UNSUPPORTED)
            set_error("bke_if_step: dim_x=%d dim_z=%d needs %zu B of shared memory per filter (> %zu)", a.dim_x, a.dim_z,
                      bytes_per_warp, budget);
        return rc;
    }
    if_warp_kernel<T><<<w.grid, w.wpb * 32, w.smem, s>>>(p, per_warp);
    return check_cuda(cudaGetLastError(), "if_warp_kernel launch");
}

// the register instances: kf_direct.cu's shapes; 6/3 in fp32 only (DESIGN.md §3.5e)
template <typename T>
int dispatch(const bke_if_args &a, cudaStream_t s)
{
    int rc = BKE_ERR_UNSUPPORTED;
    if (a.B == nullptr || a.u == nullptr) {
        const int n = a.dim_x, m = a.dim_z;
        if (n == 4 && m == 2) rc = launch_reg<T, 4, 2>(a, s);
        else if (n == 1 && m == 1) rc = launch_reg<T, 1, 1>(a, s);
        else if (n == 2 && m == 1) rc = launch_reg<T, 2, 1>(a, s);
        else if (n == 2 && m == 2) rc = launch_reg<T, 2, 2>(a, s);
        else if (n == 3 && m == 1) rc = launch_reg<T, 3, 1>(a, s);
        else if (n == 4 && m == 1) rc = launch_reg<T, 4, 1>(a, s);
        else if (n == 4 && m == 4) rc = launch_reg<T, 4, 4>(a, s);
        else if constexpr (sizeof(T) == 4) {
            if (n == 6 && m == 3) rc = launch_reg<T, 6, 3>(a, s);
        }
    }
    return rc == BKE_ERR_UNSUPPORTED ? launch_warp<T>(a, s) : rc;
}

// ---- bke_inverse: one warp per matrix, warp_inverse on a copy in shared memory
template <typename T>
__global__ void __launch_bounds__(128) inverse_kernel(int64_t N, int k, const T *A, int64_t stride, T *Ai, int32_t *status,
                                                      int per_warp)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const int kk = k * k;
    T *W = reinterpret_cast<T *>(smem_raw) + (size_t)wib * per_warp, *X = W + kk, *col = X + kk;
    for (int64_t f = (int64_t)blockIdx.x * wpb + wib; f < N; f += (int64_t)gridDim.x * wpb) {
        warp_copy_in(W, A + f * stride, kk, lane);
        __syncwarp();
        T ld;
        const bool ok = warp_inverse(W, X, col, k, lane, ld);
        __syncwarp();
        for (int e = lane; e < kk; e += 32) Ai[f * kk + e] = X[e];
        if (status && lane == 0) status[f] = ok ? BKE_STATUS_OK : BKE_STATUS_SINGULAR_S;
        __syncwarp();
    }
}

template <typename T>
int launch_inv(int64_t N, int k, const void *A, int64_t stride, void *Ai, int32_t *status, cudaStream_t s)
{
    const int per_warp = (2 * k * k + k + 3) & ~3;
    const size_t bytes_per_warp = (size_t)per_warp * sizeof(T), budget = 200 * 1024;
    WarpShape w;
    if (int rc = warp_shape((const void *)inverse_kernel<T>, bytes_per_warp, budget, N, w)) {
        if (rc == BKE_ERR_UNSUPPORTED)
            set_error("bke_inverse: k=%d needs %zu B of shared memory per matrix (> %zu)", k, bytes_per_warp, budget);
        return rc;
    }
    inverse_kernel<T><<<w.grid, w.wpb * 32, w.smem, s>>>(N, k, (const T *)A, stride, (T *)Ai, status, per_warp);
    return check_cuda(cudaGetLastError(), "inverse_kernel launch");
}

}  // namespace

int launch_if(const bke_if_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

int launch_inverse(int64_t n_filters, int32_t k, int32_t dtype, const void *A, int64_t stride, void *Ai, int32_t *status,
                   cudaStream_t s)
{
    return dtype == BKE_F32 ? launch_inv<float>(n_filters, k, A, stride, Ai, status, s)
                            : launch_inv<double>(n_filters, k, A, stride, Ai, status, s);
}

}  // namespace bke
