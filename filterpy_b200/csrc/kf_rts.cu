// kf_rts.cu — Rauch-Tung-Striebel smoother over the outputs of batch_filter for a bank of filters
// (filterpy/kalman/kalman_filter.py:995-1074 KalmanFilter.rts_smoother, procedural twin :1792-1858).
//
// Per filter, backwards over the epochs k = T-2 .. 0 (:1067-1072):
//     Pp[k] = F P[k] F' + Q
//     K[k]  = P[k] F' inv(Pp[k])
//     x[k] += K[k] (x[k+1] - F x[k])
//     P[k] += K[k] (P[k+1] - Pp[k]) K[k]'
// with x[k+1], P[k+1] the already smoothed values; the last epoch is copied (K = 0, Pp = P).
//
// Data layout is the one batch_filter writes: means[T,N,n], covariances[T,N,n,n] (epoch-major, so
// consecutive threads = consecutive filters read consecutive rows).  One thread owns one filter and
// carries the smoothed (x, P) of epoch k+1 in registers; per filter-step it reads x[k], P[k] and
// writes x, P, K, Pp: (2n + 4n^2) scalars = 288 B at n = 4 fp32.
#include "bke_internal.cuh"
#include "kf_regtile.cuh"
#include "kf_rowio.cuh"

namespace bke {
namespace {

template <typename T>
struct RtsP {
    int64_t N, Tn;
    int n;                       // dim_x (generic kernel)
    int shift;                   // model of recursion step k is epoch k + shift (1: method, 0: procedural)
    const T *Xs, *Ps, *F, *Q;
    int64_t sF, sQ, tF, tQ;      // per-filter and per-epoch strides (elements); 0 = shared / constant
    T *x_out, *P_out, *K, *Pp;
    int32_t *status;
};

// time-constant models, everything in registers
template <typename T, int N>
__global__ void __launch_bounds__(128) rts_reg_kernel(RtsP<T> p)
{
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.N) return;
    // fp32: F, Q and the prefetched epoch k-1 all live in registers (168); fp64 at n = 4 would need
    // ~290, so Q is re-read every epoch (an L1 hit) and nothing is prefetched
    constexpr bool LEAN = sizeof(T) == 8 && N >= 4;
    T F[N][N], Q[N][N];
    ldv_rw<T, N * N>(&F[0][0], p.F + f * p.sF);
    if constexpr (!LEAN) ldv_rw<T, N * N>(&Q[0][0], p.Q + f * p.sQ);
    T xs[N], Ps[N][N];                                  // smoothed state of epoch k+1
    int64_t tf = (p.Tn - 1) * p.N + f;
    ldv_rw<T, N>(xs, p.Xs + tf * N);
    ldv_rw<T, N * N>(&Ps[0][0], p.Ps + tf * N * N);
    stv<T, N>(p.x_out + tf * N, xs);
    stv<T, N * N>(p.P_out + tf * N * N, &Ps[0][0]);
    if (p.Pp) stv<T, N * N>(p.Pp + tf * N * N, &Ps[0][0]);      // Pp = Ps.copy() (:1065)
    if (p.K) {
        T Z[N * N];
#pragma unroll
        for (int i = 0; i < N * N; i++) Z[i] = T(0);
        stv<T, N * N>(p.K + tf * N * N, Z);
    }
    int stt = BKE_STATUS_OK;
    T xk[N], Pk[N][N];
    if (p.Tn > 1) {
        tf -= p.N;
        ldv_rw<T, N>(xk, p.Xs + tf * N);
        ldv_rw<T, N * N>(&Pk[0][0], p.Ps + tf * N * N);
    }
    for (int64_t k = p.Tn - 2; k >= 0; k--) {
        // prefetch epoch k-1 while epoch k computes
        T xn[N], Pn[N][N];
        if constexpr (!LEAN) {
            if (k > 0) {
                ldv_rw<T, N>(xn, p.Xs + (tf - p.N) * N);
                ldv_rw<T, N * N>(&Pn[0][0], p.Ps + (tf - p.N) * N * N);
            }
        } else {
            ldv_rw<T, N * N>(&Q[0][0], p.Q + f * p.sQ);
        }
        T FP[N][N], Pp[N][N], PFt[N][N];
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < N; j++) {
                T s = F[i][0] * Pk[0][j];
#pragma unroll
                for (int q = 1; q < N; q++) s += F[i][q] * Pk[q][j];
                FP[i][j] = s;
            }
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < N; j++) {
                T s = FP[i][0] * F[j][0];
                T r = Pk[i][0] * F[j][0];
#pragma unroll
                for (int q = 1; q < N; q++) { s += FP[i][q] * F[j][q]; r += Pk[i][q] * F[j][q]; }
                Pp[i][j] = s + Q[i][j];
                PFt[i][j] = r;
            }
        T PpI[N][N], logdet;
        const bool ok = reg_inverse<T, N>(Pp, PpI, logdet);
        if (!ok) stt = BKE_STATUS_SINGULAR_S;
        T K[N][N];
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < N; j++) {
                T s = PFt[i][0] * PpI[0][j];
#pragma unroll
                for (int q = 1; q < N; q++) s += PFt[i][q] * PpI[q][j];
                K[i][j] = s;
            }
        T d[N];
#pragma unroll
        for (int i = 0; i < N; i++) {
            T s = F[i][0] * xk[0];
#pragma unroll
            for (int q = 1; q < N; q++) s += F[i][q] * xk[q];
            d[i] = xs[i] - s;
        }
#pragma unroll
        for (int i = 0; i < N; i++) {
            T s = K[i][0] * d[0];
#pragma unroll
            for (int q = 1; q < N; q++) s += K[i][q] * d[q];
            xk[i] += s;
        }
        T KD[N][N];                                     // K (P[k+1] - Pp)
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < N; j++) {
                T s = K[i][0] * (Ps[0][j] - Pp[0][j]);
#pragma unroll
                for (int q = 1; q < N; q++) s += K[i][q] * (Ps[q][j] - Pp[q][j]);
                KD[i][j] = s;
            }
#pragma unroll
        for (int i = 0; i < N; i++)
#pragma unroll
            for (int j = 0; j < N; j++) {
                T s = KD[i][0] * K[j][0];
#pragma unroll
                for (int q = 1; q < N; q++) s += KD[i][q] * K[j][q];
                Pk[i][j] += s;
            }
        stv<T, N>(p.x_out + tf * N, xk);
        stv<T, N * N>(p.P_out + tf * N * N, &Pk[0][0]);
        if (p.K) stv<T, N * N>(p.K + tf * N * N, &K[0][0]);
        if (p.Pp) stv<T, N * N>(p.Pp + tf * N * N, &Pp[0][0]);
#pragma unroll
        for (int i = 0; i < N; i++) {
            xs[i] = xk[i];
#pragma unroll
            for (int j = 0; j < N; j++) Ps[i][j] = Pk[i][j];
        }
        tf -= p.N;
        if constexpr (!LEAN) {
#pragma unroll
            for (int i = 0; i < N; i++) {
                xk[i] = xn[i];
#pragma unroll
                for (int j = 0; j < N; j++) Pk[i][j] = Pn[i][j];
            }
        } else if (k > 0) {
            ldv_rw<T, N>(xk, p.Xs + tf * N);
            ldv_rw<T, N * N>(&Pk[0][0], p.Ps + tf * N * N);
        }
    }
    if (p.status) p.status[f] = stt;
}

// any n <= RTS_MAXN, per-epoch models allowed; thread-private arrays (local memory) — the
// correctness path, not a tuned one
constexpr int RTS_MAXN = 12;

template <typename T>
__global__ void __launch_bounds__(64) rts_generic_kernel(RtsP<T> p)
{
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.N) return;
    const int n = p.n;
    T xs[RTS_MAXN], Ps[RTS_MAXN * RTS_MAXN], xk[RTS_MAXN], Pk[RTS_MAXN * RTS_MAXN];
    T A[RTS_MAXN * RTS_MAXN], B[RTS_MAXN * RTS_MAXN], C[RTS_MAXN * RTS_MAXN], Kk[RTS_MAXN * RTS_MAXN];
    int64_t tf = (p.Tn - 1) * p.N + f;
    for (int i = 0; i < n; i++) { xs[i] = p.Xs[tf * n + i]; p.x_out[tf * n + i] = xs[i]; }
    for (int i = 0; i < n * n; i++) {
        Ps[i] = p.Ps[tf * n * n + i];
        p.P_out[tf * n * n + i] = Ps[i];
        if (p.Pp) p.Pp[tf * n * n + i] = Ps[i];
        if (p.K) p.K[tf * n * n + i] = T(0);
    }
    int stt = BKE_STATUS_OK;
    for (int64_t k = p.Tn - 2; k >= 0; k--) {
        tf -= p.N;
        const T *F = p.F + f * p.sF + (k + p.shift) * p.tF;
        const T *Q = p.Q + f * p.sQ + (k + p.shift) * p.tQ;
        for (int i = 0; i < n; i++) xk[i] = p.Xs[tf * n + i];
        for (int i = 0; i < n * n; i++) Pk[i] = p.Ps[tf * n * n + i];
        // A = F Pk ; B = Pp = A F' + Q ; C = Pk F'
        for (int i = 0; i < n; i++)
            for (int j = 0; j < n; j++) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += F[i * n + q] * Pk[q * n + j];
                A[i * n + j] = s;
            }
        for (int i = 0; i < n; i++)
            for (int j = 0; j < n; j++) {
                T s = T(0), r = T(0);
                for (int q = 0; q < n; q++) { s += A[i * n + q] * F[j * n + q]; r += Pk[i * n + q] * F[j * n + q]; }
                B[i * n + j] = s + Q[i * n + j];
                C[i * n + j] = r;
            }
        if (p.Pp) for (int i = 0; i < n * n; i++) p.Pp[tf * n * n + i] = B[i];
        // A = inv(B) by Gauss-Jordan with partial pivoting (B is overwritten: keep D = Ps - Pp first)
        for (int i = 0; i < n * n; i++) Ps[i] -= B[i];                          // Ps := P[k+1] - Pp
        for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) A[i * n + j] = (i == j) ? T(1) : T(0);
        for (int c = 0; c < n; c++) {
            int pr = c;
            T best = fabs(B[c * n + c]);
            for (int r = c + 1; r < n; r++) { const T v = fabs(B[r * n + c]); if (v > best) { best = v; pr = r; } }
            if (best == T(0)) { stt = BKE_STATUS_SINGULAR_S; break; }
            if (pr != c)
                for (int j = 0; j < n; j++) {
                    T t0 = B[c * n + j]; B[c * n + j] = B[pr * n + j]; B[pr * n + j] = t0;
                    T t1 = A[c * n + j]; A[c * n + j] = A[pr * n + j]; A[pr * n + j] = t1;
                }
            const T d = T(1) / B[c * n + c];
            for (int j = 0; j < n; j++) { B[c * n + j] *= d; A[c * n + j] *= d; }
            for (int r = 0; r < n; r++) {
                if (r == c) continue;
                const T fm = B[r * n + c];
                for (int j = 0; j < n; j++) { B[r * n + j] -= fm * B[c * n + j]; A[r * n + j] -= fm * A[c * n + j]; }
            }
        }
        // K = C inv(Pp)
        for (int i = 0; i < n; i++)
            for (int j = 0; j < n; j++) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += C[i * n + q] * A[q * n + j];
                Kk[i * n + j] = s;
            }
        // x[k] += K (x[k+1] - F x[k])
        for (int i = 0; i < n; i++) {
            T s = T(0);
            for (int q = 0; q < n; q++) s += F[i * n + q] * xk[q];
            B[i] = xs[i] - s;
        }
        for (int i = 0; i < n; i++) {
            T s = T(0);
            for (int q = 0; q < n; q++) s += Kk[i * n + q] * B[q];
            xs[i] = xk[i] + s;
        }
        // P[k] += K D K'
        for (int i = 0; i < n; i++)
            for (int j = 0; j < n; j++) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += Kk[i * n + q] * Ps[q * n + j];
                C[i * n + j] = s;
            }
        for (int i = 0; i < n; i++)
            for (int j = 0; j < n; j++) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += C[i * n + q] * Kk[j * n + q];
                Pk[i * n + j] += s;
            }
        for (int i = 0; i < n; i++) p.x_out[tf * n + i] = xs[i];
        for (int i = 0; i < n * n; i++) {
            Ps[i] = Pk[i];
            p.P_out[tf * n * n + i] = Pk[i];
            if (p.K) p.K[tf * n * n + i] = Kk[i];
        }
    }
    if (p.status) p.status[f] = stt;
}

template <typename T>
int launch_t(const bke_rts_args &a, cudaStream_t s)
{
    RtsP<T> p;
    p.N = a.n_filters; p.Tn = a.n_steps; p.n = a.dim_x; p.shift = a.model_shift;
    p.Xs = (const T *)a.Xs; p.Ps = (const T *)a.Ps; p.F = (const T *)a.F; p.Q = (const T *)a.Q;
    p.sF = a.F_stride; p.sQ = a.Q_stride; p.tF = a.F_step_stride; p.tQ = a.Q_step_stride;
    p.x_out = (T *)a.x_out; p.P_out = (T *)a.P_out; p.K = (T *)a.K; p.Pp = (T *)a.Pp;
    p.status = a.status;
    const bool constant = a.F_step_stride == 0 && a.Q_step_stride == 0;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(a.Xs) | reinterpret_cast<uintptr_t>(a.Ps) | reinterpret_cast<uintptr_t>(a.F) |
                          reinterpret_cast<uintptr_t>(a.Q) | reinterpret_cast<uintptr_t>(a.x_out) | reinterpret_cast<uintptr_t>(a.P_out) |
                          reinterpret_cast<uintptr_t>(a.K) | reinterpret_cast<uintptr_t>(a.Pp)) & 15) == 0 &&
                        (a.F_stride * (int64_t)sizeof(T)) % 16 == 0 && (a.Q_stride * (int64_t)sizeof(T)) % 16 == 0;
    const unsigned grid128 = (unsigned)((p.N + 127) / 128);
    if (constant && vec_ok && a.dim_x == 4) { rts_reg_kernel<T, 4><<<grid128, 128, 0, s>>>(p); }
    else if (constant && vec_ok && a.dim_x == 2) { rts_reg_kernel<T, 2><<<grid128, 128, 0, s>>>(p); }
    else rts_generic_kernel<T><<<(unsigned)((p.N + 63) / 64), 64, 0, s>>>(p);
    return check_cuda(cudaGetLastError(), "rts launch");
}

}  // namespace

int launch_rts(const bke_rts_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? launch_t<float>(a, s) : launch_t<double>(a, s);
}

}  // namespace bke

using namespace bke;

extern "C" int bke_kf_rts_smoother(const bke_rts_args *args, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    const bke_rts_args &a = *args;
    if (a.n_filters < 0 || a.n_steps < 0) { set_error("negative sizes"); return BKE_ERR_BAD_ARG; }
    if (a.dim_x < 1 || a.dim_x > RTS_MAXN) { set_error("bke_kf_rts_smoother: dim_x must be in [1, %d]", RTS_MAXN); return BKE_ERR_UNSUPPORTED; }
    if (int rc = check_dtype(a.dtype)) return rc;
    if (a.model_shift != 0 && a.model_shift != 1) { set_error("model_shift must be 0 or 1"); return BKE_ERR_BAD_ARG; }
    if (a.n_filters == 0 || a.n_steps == 0) return BKE_OK;
    if (!a.Xs || !a.Ps || !a.F || !a.Q || !a.x_out || !a.P_out) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    if (a.F_stride < 0 || a.Q_stride < 0 || a.F_step_stride < 0 || a.Q_step_stride < 0) { set_error("negative stride"); return BKE_ERR_BAD_ARG; }
    if (int rc = require_device()) return rc;
    return launch_rts(a, (cudaStream_t)stream);
}
