// srkf.cu — square-root Kalman filter bank (bke_srkf_step) and the Cholesky factor of the setters
// (bke_cholesky_lower).
//
// Arithmetic follows filterpy/kalman/square_root.py (reference @ 3b51149), with L = P1_2 lower triangular:
//   predict  :239-248   x = F x (+ B u);  R~ = qr([F L | Lq]')[1] (2n x n);  L = R~[:n,:n]'
//   update   :195-224   M = [[Lr', 0], [(H L)', L']] ((m+n) x (m+n));  r = qr(M)[1];
//                       S1_2 = r[:m,:m]';  SI1_2 = S1_2^-1;  K = r[:m,m:]' SI1_2;
//                       y = z - H x;  x += K y;  L = r[m:,m:]'
//   z is None:189-193   nothing changes (z_valid[f] == 0)
// The QR restates LAPACK's dgeqr2 / dlarfg (what scipy.linalg.qr calls at these sizes) and forms R only:
// column j has alpha = A[j,j] and the sub-column below it; when the sub-column is exactly zero, tau = 0 and
// A[j,j] keeps its sign, otherwise beta = -copysign(|(alpha, sub)|, alpha), the sub-column becomes
// v = sub / (alpha - beta) (v_j = 1), A[j,j] = beta, and the columns to the right get A -= tau v (v' A)
// with tau = (beta - alpha) / beta.  So R, and hence L, has dgeqr2's signs: L itself, not only L L', matches.
// A zero diagonal entry of S1_2 (where the reference's pinv takes over) sets status BKE_STATUS_SINGULAR_S,
// K = 0, SI1_2 = 0 and keeps the prior: for S1_2 = 0 that is the reference's result exactly.
//
// Two paths, picked by shape: a register tile per thread (one thread per filter, 16-byte row loads as in
// kf_direct.cu) for the small shapes listed in dispatch(), and a warp per filter with the matrices in the
// warp's slice of shared memory (as in kf_generic.cu) for every other shape and for a control input.
#include "bke_internal.cuh"
#include "kf_rowio.cuh"
#include "kf_warp.cuh"
#include "ukf_kernel.cuh"

namespace bke {
namespace {

template <typename T>
struct SrP {
    int64_t N;
    int n, m, du;
    unsigned flags;
    const T *x, *L;
    T *x_out, *L_out;
    const T *F, *H, *Lq, *Lr, *B, *u, *z;
    int64_t sF, sH, sLq, sLr, sB, su;
    const uint8_t *valid;
    T *x_prior, *L_prior, *K, *y, *S1_2, *SI1_2;
    int32_t *status;
};

template <typename T>
__device__ __forceinline__ void householder(T alpha, T ss, T &beta, T &tau, T &scale)
{
    beta = -copysign(sqrt(alpha * alpha + ss), alpha);
    tau = (beta - alpha) / beta;
    scale = T(1) / (alpha - beta);
}

// dgeqr2 on A[R][C] in registers: on return the upper triangle of A[:C] is R; the entries below the
// diagonal hold the Householder vectors and are not part of the result
template <typename T, int R, int C>
__device__ __forceinline__ void reg_qr(T (&A)[R][C])
{
#pragma unroll
    for (int j = 0; j < C && j + 1 < R; j++) {
        T ss = T(0);
#pragma unroll
        for (int i = j + 1; i < R; i++) ss += A[i][j] * A[i][j];
        if (ss == T(0)) continue;                         // tau = 0: no reflection
        T beta, tau, sc;
        householder(A[j][j], ss, beta, tau, sc);
#pragma unroll
        for (int i = j + 1; i < R; i++) A[i][j] *= sc;
        A[j][j] = beta;
#pragma unroll
        for (int k = j + 1; k < C; k++) {
            T w = A[j][k];
#pragma unroll
            for (int i = j + 1; i < R; i++) w += A[i][j] * A[i][k];
            w *= tau;
            A[j][k] -= w;
#pragma unroll
            for (int i = j + 1; i < R; i++) A[i][k] -= A[i][j] * w;
        }
    }
}

// X = S^-1 for lower-triangular S (forward substitution, column by column); false when a diagonal entry is 0
template <typename T, int M>
__device__ __forceinline__ bool reg_tri_inv(const T (&S)[M][M], T (&X)[M][M])
{
    bool ok = true;
#pragma unroll
    for (int a = 0; a < M; a++) ok = ok && S[a][a] != T(0);
#pragma unroll
    for (int c = 0; c < M; c++) {
#pragma unroll
        for (int i = 0; i < M; i++) {
            if (i < c) { X[i][c] = T(0); continue; }
            T s = (i == c) ? T(1) : T(0);
#pragma unroll
            for (int k = c; k < i; k++) s -= S[i][k] * X[k][c];
            X[i][c] = s / S[i][i];
        }
    }
    return ok;
}

template <typename T, int N, int M, bool EX>
__global__ void __launch_bounds__(128) srkf_reg_kernel(SrP<T> p)
{
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.N) return;
    T x[N], L[N][N];
    ldv_rw<T, N>(x, p.x + f * N);
    ldv_rw<T, N * N>(&L[0][0], p.L + f * N * N);
    int st = BKE_STATUS_OK;
    if (p.flags & BKE_DO_PREDICT) {
        T F[N][N], A[2 * N][N];
        ldv<T, N * N>(&F[0][0], p.F + f * p.sF);
        ldv<T, N * N>(&A[N][0], p.Lq + f * p.sLq);
        T xp[N];
#pragma unroll
        for (int i = 0; i < N; i++) {
            T s = T(0);
#pragma unroll
            for (int q = 0; q < N; q++) s += F[i][q] * x[q];
            xp[i] = s;
        }
#pragma unroll
        for (int i = 0; i < N; i++) {
            x[i] = xp[i];
#pragma unroll
            for (int k = 0; k < N; k++) {
                T s = T(0);
#pragma unroll
                for (int q = 0; q < N; q++) s += F[k][q] * L[q][i];
                A[i][k] = s;                                           // (F L)'
            }
        }
#pragma unroll
        for (int i = 0; i < N; i++)                                    // Lq' in place: A[N + i][k] = Lq[k][i]
#pragma unroll
            for (int k = i + 1; k < N; k++) { T t = A[N + i][k]; A[N + i][k] = A[N + k][i]; A[N + k][i] = t; }
        reg_qr<T, 2 * N, N>(A);
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int k = 0; k < N; k++) L[i][k] = k <= i ? A[k][i] : T(0);
        if (EX && p.x_prior) stv<T, N>(p.x_prior + f * N, x);
        if (EX && p.L_prior) stv<T, N * N>(p.L_prior + f * N * N, &L[0][0]);
    }
    if ((p.flags & BKE_DO_UPDATE) && (p.valid == nullptr || p.valid[f] != 0)) {
        constexpr int D = M + N;
        T H[M][N], Lr[M][M], z[M], Mx[D][D];
        ldv<T, M * N>(&H[0][0], p.H + f * p.sH);
        ldv<T, M * M>(&Lr[0][0], p.Lr + f * p.sLr);
        ldv<T, M>(z, p.z + f * M);
#pragma unroll
        for (int a = 0; a < M; a++) {
#pragma unroll
            for (int b = 0; b < M; b++) Mx[a][b] = Lr[b][a];
#pragma unroll
            for (int k = 0; k < N; k++) Mx[a][M + k] = T(0);
        }
#pragma unroll
        for (int i = 0; i < N; i++) {
#pragma unroll
            for (int b = 0; b < M; b++) {
                T s = T(0);
#pragma unroll
                for (int q = 0; q < N; q++) s += H[b][q] * L[q][i];
                Mx[M + i][b] = s;                                      // (H L)'
            }
#pragma unroll
            for (int k = 0; k < N; k++) Mx[M + i][M + k] = L[k][i];
        }
        reg_qr<T, D, D>(Mx);
        T S[M][M], SI[M][M], y[M];
#pragma unroll
        for (int a = 0; a < M; a++)
#pragma unroll
            for (int b = 0; b < M; b++) S[a][b] = b <= a ? Mx[b][a] : T(0);
        const bool ok = reg_tri_inv<T, M>(S, SI);
#pragma unroll
        for (int a = 0; a < M; a++) {
            T s = T(0);
#pragma unroll
            for (int q = 0; q < N; q++) s += H[a][q] * x[q];
            y[a] = z[a] - s;
        }
        T K[N][M];
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int b = 0; b < M; b++) {
                T s = T(0);
#pragma unroll
                for (int a = 0; a < M; a++) s += Mx[a][M + i] * SI[a][b];
                K[i][b] = ok ? s : T(0);
            }
        if (ok) {
#pragma unroll
            for (int i = 0; i < N; i++) {
                T s = T(0);
#pragma unroll
                for (int b = 0; b < M; b++) s += K[i][b] * y[b];
                x[i] += s;
#pragma unroll
                for (int k = 0; k < N; k++) L[i][k] = k <= i ? Mx[M + k][M + i] : T(0);
            }
        } else {
            st = BKE_STATUS_SINGULAR_S;
#pragma unroll
            for (int a = 0; a < M; a++)
#pragma unroll
                for (int b = 0; b < M; b++) SI[a][b] = T(0);
        }
        if (EX && p.K) stv<T, N * M>(p.K + f * N * M, &K[0][0]);
        if (EX && p.y) stv<T, M>(p.y + f * M, y);
        if (EX && p.S1_2) stv<T, M * M>(p.S1_2 + f * M * M, &S[0][0]);
        if (EX && p.SI1_2) stv<T, M * M>(p.SI1_2 + f * M * M, &SI[0][0]);
    }
    stv<T, N>(p.x_out + f * N, x);
    stv<T, N * N>(p.L_out + f * N * N, &L[0][0]);
    if (p.status) p.status[f] = st;
}

// dgeqr2 on the R x C row-major matrix A in shared memory, by one warp: a warp reduction for the
// sub-column's norm, lanes over the columns to the right for the reflection
template <typename T>
__device__ void warp_qr(T *A, int R, int C, int lane)
{
    for (int j = 0; j < C && j + 1 < R; j++) {
        T ss = T(0);
        for (int i = j + 1 + lane; i < R; i += 32) ss += A[i * C + j] * A[i * C + j];
        ss = warp_sum(ss);
        if (ss == T(0)) continue;
        T beta, tau, sc;
        householder(A[j * C + j], ss, beta, tau, sc);
        for (int i = j + 1 + lane; i < R; i += 32) A[i * C + j] *= sc;
        __syncwarp();
        if (lane == 0) A[j * C + j] = beta;
        for (int k = j + 1 + lane; k < C; k += 32) {
            T w = A[j * C + k];
            for (int i = j + 1; i < R; i++) w += A[i * C + j] * A[i * C + k];
            w *= tau;
            A[j * C + k] -= w;
            for (int i = j + 1; i < R; i++) A[i * C + k] -= A[i * C + j] * w;
        }
        __syncwarp();
    }
}

// per-warp slice: x, xp, y (n, n, m) | L, T1 (n*n, max(n*n, m*n)) | H, K (m*n each) | S, SI (m*m each) | W
template <typename T>
__global__ void __launch_bounds__(128) srkf_warp_kernel(SrP<T> p, int per_warp)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    const int n = p.n, m = p.m, nn = n * n, nm = n * m, mm = m * m, D = n + m;
    T *x = reinterpret_cast<T *>(smem_raw) + (size_t)wib * per_warp;
    T *xp = x + n, *y = xp + n, *L = y + m, *T1 = L + nn;
    T *H = T1 + (nn > nm ? nn : nm), *K = H + nm, *S = K + nm, *SI = S + mm, *W = SI + mm;

    for (int64_t f = (int64_t)blockIdx.x * wpb + wib; f < p.N; f += (int64_t)gridDim.x * wpb) {
        warp_copy_in(x, p.x + f * n, n, lane);
        warp_copy_in(L, p.L + f * nn, nn, lane);
        int st = BKE_STATUS_OK;
        __syncwarp();
        if (p.flags & BKE_DO_PREDICT) {
            warp_copy_in(T1, p.F + f * p.sF, nn, lane);
            __syncwarp();
            for (int i = lane; i < n; i += 32) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += T1[i * n + q] * x[q];
                if (p.B != nullptr && p.u != nullptr) {
                    const T *Bf = p.B + f * p.sB, *uf = p.u + f * p.su;
                    T b = T(0);
                    for (int q = 0; q < p.du; q++) b += Bf[i * p.du + q] * uf[q];
                    s += b;
                }
                xp[i] = s;
            }
            // W = [F L | Lq]' (2n x n): W[i][k] = (F L)[k][i], W[n + i][k] = Lq[k][i]
            warp_mm<false>(T1, L, n, n, n, lane, [&](int, int k, int i, T s) { W[i * n + k] = s; });
            const T *Lq = p.Lq + f * p.sLq;
            for (int e = lane; e < nn; e += 32) { int k = e / n, i = e - k * n; W[(n + i) * n + k] = Lq[e]; }
            __syncwarp();
            warp_qr(W, 2 * n, n, lane);
            for (int e = lane; e < nn; e += 32) { int i = e / n, k = e - i * n; L[e] = k <= i ? W[k * n + i] : T(0); }
            for (int i = lane; i < n; i += 32) x[i] = xp[i];
            __syncwarp();
            if (p.x_prior) for (int i = lane; i < n; i += 32) p.x_prior[f * n + i] = x[i];
            if (p.L_prior) for (int e = lane; e < nn; e += 32) p.L_prior[f * nn + e] = L[e];
        }
        if ((p.flags & BKE_DO_UPDATE) && (p.valid == nullptr || p.valid[f] != 0)) {
            warp_copy_in(H, p.H + f * p.sH, nm, lane);
            __syncwarp();
            // W = M = [[Lr', 0], [(H L)', L']]
            const T *Lr = p.Lr + f * p.sLr;
            for (int e = lane; e < D * D; e += 32) {
                int r = e / D, c = e - r * D;
                T v;
                if (r < m) v = c < m ? Lr[c * m + r] : T(0);
                else if (c >= m) v = L[(c - m) * n + (r - m)];
                else { v = T(0); for (int q = 0; q < n; q++) v += H[c * n + q] * L[q * n + (r - m)]; }
                W[e] = v;
            }
            for (int a = lane; a < m; a += 32) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += H[a * n + q] * x[q];
                y[a] = p.z[f * m + a] - s;
            }
            __syncwarp();
            warp_qr(W, D, D, lane);
            bool ok = true;
            for (int a = 0; a < m; a++) ok = ok && W[a * D + a] != T(0);
            for (int e = lane; e < mm; e += 32) { int a = e / m, b = e - a * m; S[e] = b <= a ? W[b * D + a] : T(0); }
            __syncwarp();
            for (int c = lane; c < m; c += 32)                     // column c of S^-1 by forward substitution
                for (int i = 0; i < m; i++) {
                    if (i < c || !ok) { SI[i * m + c] = T(0); continue; }
                    T s = (i == c) ? T(1) : T(0);
                    for (int k = c; k < i; k++) s -= S[i * m + k] * SI[k * m + c];
                    SI[i * m + c] = s / S[i * m + i];
                }
            __syncwarp();
            for (int e = lane; e < nm; e += 32) {
                int i = e / m, b = e - i * m;
                T s = T(0);
                for (int a = 0; a < m; a++) s += W[a * D + m + i] * SI[a * m + b];
                K[e] = s;                                          // 0 when singular: SI = 0
            }
            __syncwarp();
            if (ok) {
                for (int i = lane; i < n; i += 32) {
                    T s = T(0);
                    for (int b = 0; b < m; b++) s += K[i * m + b] * y[b];
                    x[i] += s;
                }
                for (int e = lane; e < nn; e += 32) { int i = e / n, k = e - i * n; L[e] = k <= i ? W[(m + k) * D + m + i] : T(0); }
            } else {
                st = BKE_STATUS_SINGULAR_S;
            }
            __syncwarp();
            if (p.K) for (int e = lane; e < nm; e += 32) p.K[f * nm + e] = K[e];
            if (p.y) for (int a = lane; a < m; a += 32) p.y[f * m + a] = y[a];
            if (p.S1_2) for (int e = lane; e < mm; e += 32) p.S1_2[f * mm + e] = S[e];
            if (p.SI1_2) for (int e = lane; e < mm; e += 32) p.SI1_2[f * mm + e] = SI[e];
        }
        __syncwarp();
        for (int i = lane; i < n; i += 32) p.x_out[f * n + i] = x[i];
        for (int e = lane; e < nn; e += 32) p.L_out[f * nn + e] = L[e];
        if (p.status && lane == 0) p.status[f] = st;
        __syncwarp();
    }
}

template <typename T>
SrP<T> params(const bke_srkf_args &a)
{
    SrP<T> p;
    p.N = a.n_filters; p.n = a.dim_x; p.m = a.dim_z; p.du = a.dim_u; p.flags = a.flags;
    p.x = (const T *)a.x; p.L = (const T *)a.L; p.x_out = (T *)a.x_out; p.L_out = (T *)a.L_out;
    p.F = (const T *)a.F; p.H = (const T *)a.H; p.Lq = (const T *)a.Lq; p.Lr = (const T *)a.Lr;
    p.B = (const T *)a.B; p.u = (const T *)a.u; p.z = (const T *)a.z;
    p.sF = a.F_stride; p.sH = a.H_stride; p.sLq = a.Lq_stride; p.sLr = a.Lr_stride; p.sB = a.B_stride; p.su = a.u_stride;
    p.valid = a.z_valid;
    p.x_prior = (T *)a.x_prior; p.L_prior = (T *)a.L_prior; p.K = (T *)a.K; p.y = (T *)a.y;
    p.S1_2 = (T *)a.S1_2; p.SI1_2 = (T *)a.SI1_2; p.status = a.status;
    return p;
}

template <typename T, int N, int M>
int launch_reg(const bke_srkf_args &a, cudaStream_t s)
{
    if (!(vec_ok<T, N>(a.x) && vec_ok<T, N * N>(a.L) && vec_ok<T, N * N>(a.F, a.F_stride) &&
          vec_ok<T, N * N>(a.Lq, a.Lq_stride) && vec_ok<T, M * N>(a.H, a.H_stride) && vec_ok<T, M * M>(a.Lr, a.Lr_stride) &&
          vec_ok<T, M>(a.z) && vec_ok<T, N>(a.x_out) && vec_ok<T, N * N>(a.L_out) && vec_ok<T, N>(a.x_prior) &&
          vec_ok<T, N * N>(a.L_prior) && vec_ok<T, N * M>(a.K) && vec_ok<T, M>(a.y) && vec_ok<T, M * M>(a.S1_2) &&
          vec_ok<T, M * M>(a.SI1_2)))
        return BKE_ERR_UNSUPPORTED;
    SrP<T> p = params<T>(a);
    const unsigned grid = (unsigned)((p.N + 127) / 128);
    if (a.x_prior || a.L_prior || a.K || a.y || a.S1_2 || a.SI1_2) srkf_reg_kernel<T, N, M, true><<<grid, 128, 0, s>>>(p);
    else srkf_reg_kernel<T, N, M, false><<<grid, 128, 0, s>>>(p);
    return check_cuda(cudaGetLastError(), "srkf_reg_kernel launch");
}

template <typename T>
int launch_warp(const bke_srkf_args &a, cudaStream_t s)
{
    SrP<T> p = params<T>(a);
    const int n = a.dim_x, m = a.dim_z, nn = n * n, nm = n * m, D = n + m;
    // layout must match the kernel: x, xp, y, L, T1, H, K, S, SI, W
    int per_warp = 2 * n + m + nn + (nn > nm ? nn : nm) + 2 * nm + 2 * m * m + (2 * nn > D * D ? 2 * nn : D * D);
    per_warp = (per_warp + 3) & ~3;
    const size_t bytes_per_warp = (size_t)per_warp * sizeof(T), budget = 200 * 1024;
    WarpShape w;
    if (int rc = warp_shape((const void *)srkf_warp_kernel<T>, bytes_per_warp, budget, p.N, w)) {
        if (rc == BKE_ERR_UNSUPPORTED)
            set_error("bke_srkf_step: dim_x=%d dim_z=%d needs %zu B of shared memory per filter (> %zu)", n, m, bytes_per_warp, budget);
        return rc;
    }
    srkf_warp_kernel<T><<<w.grid, w.wpb * 32, w.smem, s>>>(p, per_warp);
    return check_cuda(cudaGetLastError(), "srkf_warp_kernel launch");
}

// the register instances: every one compiles without spills (`_build.py --ptxas-v`)
template <typename T>
int dispatch(const bke_srkf_args &a, cudaStream_t s)
{
    int rc = BKE_ERR_UNSUPPORTED;
    if (a.B == nullptr || a.u == nullptr) {
        const int n = a.dim_x, m = a.dim_z;
        if (n == 4 && m == 2) rc = launch_reg<T, 4, 2>(a, s);
        else if (n == 1 && m == 1) rc = launch_reg<T, 1, 1>(a, s);
        else if (n == 2 && m == 2) rc = launch_reg<T, 2, 2>(a, s);
        else if (n == 3 && m == 1) rc = launch_reg<T, 3, 1>(a, s);
        else if (n == 4 && m == 1) rc = launch_reg<T, 4, 1>(a, s);
    }
    return rc == BKE_ERR_UNSUPPORTED ? launch_warp<T>(a, s) : rc;
}

// ---- bke_cholesky_lower: L = cholesky(A, lower=True), the lower triangle of A read.  chol_upper of A'
// reads A's lower triangle and gives U = L'.
template <typename T, int K>
__global__ void __launch_bounds__(128) chol_lower_kernel(int64_t N, const T *A, int64_t stride, T *L, int32_t *status)
{
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= N) return;
    T At[K][K], U[K][K];
    const T *Af = A + f * stride;
#pragma unroll
    for (int i = 0; i < K; i++)
#pragma unroll
        for (int j = 0; j < K; j++) At[i][j] = Af[j * K + i];
    const bool ok = ukfk::chol_upper<T, K>(At, U);
#pragma unroll
    for (int i = 0; i < K; i++)
#pragma unroll
        for (int j = 0; j < K; j++) L[f * K * K + i * K + j] = j <= i ? U[j][i] : T(0);
    if (status) status[f] = ok ? BKE_STATUS_OK : BKE_STATUS_NOT_PD;
}

template <typename T, int K>
int launch_chol(int64_t N, int32_t k, const void *A, int64_t stride, void *L, int32_t *status, cudaStream_t s)
{
    if (k != K) {
        if constexpr (K < BKE_CHOLESKY_MAX_DIM) return launch_chol<T, K + 1>(N, k, A, stride, L, status, s);
        return BKE_ERR_UNSUPPORTED;
    }
    chol_lower_kernel<T, K><<<(unsigned)((N + 127) / 128), 128, 0, s>>>(N, (const T *)A, stride, (T *)L, status);
    return check_cuda(cudaGetLastError(), "chol_lower_kernel launch");
}

}  // namespace

int launch_srkf(const bke_srkf_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

int launch_cholesky_lower(int64_t n_filters, int32_t k, int32_t dtype, const void *A, int64_t stride, void *L,
                          int32_t *status, cudaStream_t s)
{
    return dtype == BKE_F32 ? launch_chol<float, 1>(n_filters, k, A, stride, L, status, s)
                            : launch_chol<double, 1>(n_filters, k, A, stride, L, status, s);
}

}  // namespace bke
