// fls.cu — FixedLagSmoother.smooth / smooth_batch for a bank (filterpy/kalman/fixed_lag_smoother.py:133-215,
// :217-311).  Two paths behind bke_fls_smooth:
//
//   * fused (1/1, 2/1, 4/2, fp32 / fp64, no control input, lag <= BKE_FLS_FUSED_MAX_LAG): one thread owns one
//     filter and runs the T-epoch loop inside the kernel, like kf_batch.cu.  x, P and the time-constant models
//     stay in registers and the KF half is kf_regtile.cuh's reg_predict / reg_update.  The lag window (the
//     N history rows that can still change) stays on chip in a shared-memory ring [slot][component][thread]:
//     it is seeded from the history at the start, so that smooth() (T = 1) runs the same code as
//     smooth_batch, and each row is stored to HBM exactly once, when it leaves the window or when the call
//     ends.  Traffic per filter-step is m + 2n scalars (z in, the finished row and xhat out) plus the window's
//     seed and drain once per call.
//   * per-epoch (every other call): launch_kf_any (bke_kf_step's dispatch) with its x_prior, K, y and SI
//     outputs in the workspace, then fls_correct_kernel on the history rows in HBM.
//
// The correction of row k-i is the reference's PS_i HTSI y with PS_i = P (F - K H)'^i (:199-206), reassociated
// as P (A^i g) with A = (F - K H)' and g = H' (SI y): 2n^2 FMAs per lag row instead of n^2 m + n^3.
#include "bke_internal.cuh"
#include "kf_regtile.cuh"
#include "kf_rowio.cuh"

namespace bke {
namespace {

constexpr int FLS_THREADS = 128;

template <typename T>
struct FlsP {
    int64_t Nf, Tn, lag, count;
    const T *x, *P, *F, *Q, *H, *R, *zs;
    int64_t sF, sQ, sH, sR;
    T *x_out, *P_out, *xs, *xhat, *y, *S;
    int32_t *status;
};

template <typename T, int N, int M>
__global__ void __launch_bounds__(FLS_THREADS) fls_fused_kernel(FlsP<T> p)
{
    extern __shared__ __align__(16) unsigned char fsm[];
    T *win = reinterpret_cast<T *>(fsm);                     // [slot][component][thread]
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.Nf) return;                                   // no block-wide barrier below: a thread only touches its own column
    const int tid = threadIdx.x, bd = blockDim.x;
    const int64_t L = p.lag, c0 = p.count, Nf = p.Nf;
    auto row_ptr = [&](int64_t r) { return p.xs + (r * Nf + f) * N; };
    auto slot = [&](int64_t s, int c) -> T & { return win[((int)s * N + c) * bd + tid]; };

    T x[N], P[N][N], F[N][N], Q[N][N], H[M][N], R[M][M];
    ld_scalar<T, N>(x, p.x + f * N);
    ld_scalar<T, N * N>(&P[0][0], p.P + f * N * N);
    ld_scalar<T, N * N>(&F[0][0], p.F + f * p.sF);
    ld_scalar<T, N * N>(&Q[0][0], p.Q + f * p.sQ);
    ld_scalar<T, M * N>(&H[0][0], p.H + f * p.sH);
    ld_scalar<T, M * M>(&R[0][0], p.R + f * p.sR);
    // the live rows count-N+1 .. count-1 (fixed_lag_smoother.py: rows a later epoch still corrects)
    for (int64_t r = (c0 - L + 1 > 0 ? c0 - L + 1 : 0); r < c0; r++) {
        const T *src = row_ptr(r);
        const int64_t s = r % L;
#pragma unroll
        for (int c = 0; c < N; c++) slot(s, c) = src[c];
    }
    int st = BKE_STATUS_OK;
    T zn[M];
    ld_scalar<T, M>(zn, p.zs + f * M);
    for (int64_t t = 0; t < p.Tn; t++) {
        const int64_t k = c0 + t;
        T z[M];
#pragma unroll
        for (int a = 0; a < M; a++) z[a] = zn[a];
        if (t + 1 < p.Tn) ld_scalar<T, M>(zn, p.zs + ((t + 1) * Nf + f) * M);   // fetched while epoch t computes
        reg_predict<T, N>(x, P, F, Q, T(1));                 // :174-178, no fading factor
        T xp[N];
#pragma unroll
        for (int i = 0; i < N; i++) xp[i] = x[i];
        KfUpdateOut<T, N, M> o;
        reg_update<T, N, M>(x, P, H, R, z, o);               // :181-191; a singular S keeps the prior
        if (!o.ok) st = BKE_STATUS_SINGULAR_S;
        if (p.xhat) st_scalar<T, N>(p.xhat + (t * Nf + f) * N, x);
        if (t + 1 == p.Tn) {
            if (p.y) st_scalar<T, M>(p.y + f * M, o.y);
            if (p.S) st_scalar<T, M * M>(p.S + f * M * M, &o.S[0][0]);
        }
        if (L == 0) {                                        // every row is x_pre and nothing is corrected
            st_scalar<T, N>(row_ptr(k), xp);
            continue;
        }
        const int64_t sk = k % L;
        if (k < L) {                                         // :207-211 (x is the prior when S was singular)
#pragma unroll
            for (int c = 0; c < N; c++) slot(sk, c) = x[c];
        } else {
#pragma unroll
            for (int c = 0; c < N; c++) slot(sk, c) = xp[c];  // :193
            if (o.ok) {
                // g = H' (SI y);  A = (F - K H)'  (:196-197)
                T w[M], v[N], A[N][N];
#pragma unroll
                for (int a = 0; a < M; a++) {
                    T s = o.SI[a][0] * o.y[0];
#pragma unroll
                    for (int b = 1; b < M; b++) s += o.SI[a][b] * o.y[b];
                    w[a] = s;
                }
#pragma unroll
                for (int j = 0; j < N; j++) {
                    T s = H[0][j] * w[0];
#pragma unroll
                    for (int a = 1; a < M; a++) s += H[a][j] * w[a];
                    v[j] = s;
                }
#pragma unroll
                for (int i = 0; i < N; i++)
#pragma unroll
                    for (int j = 0; j < N; j++) {
                        T s = F[i][j];
#pragma unroll
                        for (int a = 0; a < M; a++) s -= o.K[i][a] * H[a][j];
                        A[j][i] = s;
                    }
                int64_t s = sk;
                for (int64_t i = 0; i < L; i++) {            // :199-206: row k-i += P A^i g
#pragma unroll
                    for (int r = 0; r < N; r++) {
                        T c = P[r][0] * v[0];
#pragma unroll
                        for (int q = 1; q < N; q++) c += P[r][q] * v[q];
                        slot(s, r) += c;
                    }
                    if (i + 1 < L) {
                        T vn[N];
#pragma unroll
                        for (int r = 0; r < N; r++) {
                            T c = A[r][0] * v[0];
#pragma unroll
                            for (int q = 1; q < N; q++) c += A[r][q] * v[q];
                            vn[r] = c;
                        }
#pragma unroll
                        for (int r = 0; r < N; r++) v[r] = vn[r];
                    }
                    s = (s == 0) ? L - 1 : s - 1;
                }
            }
        }
        const int64_t fin = k - L + 1;                       // final from now on: leaves the window
        if (fin >= 0) {
            T *dst = row_ptr(fin);
            const int64_t s = fin % L;
#pragma unroll
            for (int c = 0; c < N; c++) dst[c] = slot(s, c);
        }
    }
    if (L > 0) {
        const int64_t end = c0 + p.Tn;
        for (int64_t r = (end - L + 1 > 0 ? end - L + 1 : 0); r < end; r++) {
            T *dst = row_ptr(r);
            const int64_t s = r % L;
#pragma unroll
            for (int c = 0; c < N; c++) dst[c] = slot(s, c);
        }
    }
    st_scalar<T, N>(p.x_out + f * N, x);
    st_scalar<T, N * N>(p.P_out + f * N * N, &P[0][0]);
    if (p.status) p.status[f] = st;
}

template <typename T, int N, int M>
int launch_fused(const bke_fls_args &a, cudaStream_t s)
{
    const bke_kf_args &k = a.step;
    FlsP<T> p;
    p.Nf = k.n_filters; p.Tn = a.n_steps; p.lag = a.lag; p.count = a.count;
    p.x = (const T *)k.x; p.P = (const T *)k.P; p.F = (const T *)k.F; p.Q = (const T *)k.Q;
    p.H = (const T *)k.H; p.R = (const T *)k.R; p.zs = (const T *)a.zs;
    p.sF = k.F_stride; p.sQ = k.Q_stride; p.sH = k.H_stride; p.sR = k.R_stride;
    p.x_out = (T *)k.x_out; p.P_out = (T *)k.P_out; p.xs = (T *)a.xs_smooth; p.xhat = (T *)a.xhat;
    p.y = (T *)k.y; p.S = (T *)k.S; p.status = k.status;
    const size_t smem = (size_t)a.lag * N * FLS_THREADS * sizeof(T);
    auto kern = fls_fused_kernel<T, N, M>;
    if (smem > 48 * 1024 &&
        check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute"))
        return BKE_ERR_CUDA;
    const int64_t grid = (p.Nf + FLS_THREADS - 1) / FLS_THREADS;
    kern<<<(unsigned)grid, FLS_THREADS, smem, s>>>(p);
    return check_cuda(cudaGetLastError(), "fls_fused_kernel launch");
}

// ---- per-epoch path ----------------------------------------------------------------------------------------
template <typename T>
struct FlsCorrP {
    int64_t Nf, lag, k, t;
    int n, m;
    const T *F, *H;
    int64_t sF, sH;
    const T *x_post, *P_post, *x_pre, *K, *y, *SI;
    const T *z;                                              // the epoch's measurements [Nf,m]
    T *y_last;                                               // the last epoch's y in the workspace, else NULL
    const int32_t *st_epoch;
    T *v, *vn, *w;                                           // per-filter scratch [Nf,n], [Nf,n], [Nf,m]
    T *xs, *xhat;
    int32_t *status;
};

// epoch k's history work for one filter: row k, then the lag correction of rows k .. k-N+1 in HBM
template <typename T>
__global__ void __launch_bounds__(128) fls_correct_kernel(FlsCorrP<T> p)
{
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.Nf) return;
    const int n = p.n, m = p.m;
    const int64_t L = p.lag, k = p.k, Nf = p.Nf;
    const int32_t st = p.st_epoch[f];
    if (st != BKE_STATUS_OK && p.status) p.status[f] = st;
    const T *xpost = p.x_post + f * n, *xpre = p.x_pre + f * n;
    if (st != BKE_STATUS_OK && p.y_last) {
        // the step leaves y alone where S is singular; the call's y is still z - H x_pre (the reference sets
        // self.y before inv(S) raises, and the fused kernel stores it too)
        const T *H = p.H + f * p.sH, *z = p.z + f * m;
        for (int a = 0; a < m; a++) {
            T s = z[a];
            for (int j = 0; j < n; j++) s -= H[a * n + j] * xpre[j];
            p.y_last[f * m + a] = s;
        }
    }
    if (p.xhat)
        for (int i = 0; i < n; i++) p.xhat[(p.t * Nf + f) * n + i] = xpost[i];
    T *rk = p.xs + (k * Nf + f) * n;
    if (k < L) {
        for (int i = 0; i < n; i++) rk[i] = xpost[i];
        return;
    }
    for (int i = 0; i < n; i++) rk[i] = xpre[i];
    if (st != BKE_STATUS_OK) return;
    const T *P = p.P_post + f * n * n, *F = p.F + f * p.sF, *H = p.H + f * p.sH;
    const T *K = p.K + f * n * m, *y = p.y + f * m, *SI = p.SI + f * m * m;
    T *v = p.v + f * n, *vn = p.vn + f * n, *w = p.w + f * m;
    for (int a = 0; a < m; a++) {
        T s = T(0);
        for (int b = 0; b < m; b++) s += SI[a * m + b] * y[b];
        w[a] = s;
    }
    for (int j = 0; j < n; j++) {
        T s = T(0);
        for (int a = 0; a < m; a++) s += H[a * n + j] * w[a];
        v[j] = s;
    }
    for (int64_t i = 0; i < L; i++) {
        T *row = p.xs + ((k - i) * Nf + f) * n;
        for (int r = 0; r < n; r++) {
            T c = T(0);
            for (int q = 0; q < n; q++) c += P[r * n + q] * v[q];
            row[r] += c;
        }
        if (i + 1 < L) {
            // (F - K H)' v = F' v - H' (K' v)
            for (int a = 0; a < m; a++) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += K[q * m + a] * v[q];
                w[a] = s;
            }
            for (int j = 0; j < n; j++) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += F[q * n + j] * v[q];
                for (int a = 0; a < m; a++) s -= H[a * n + j] * w[a];
                vn[j] = s;
            }
            T *tmp = v; v = vn; vn = tmp;
        }
    }
}

size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

// the workspace of the per-epoch path: x_pre, K, y, SI, v, vn, w (dtype) and the epoch's status (int32)
struct WsLayout {
    size_t xpre, K, y, SI, v, vn, w, st, total;
    WsLayout(int64_t Nf, int n, int m, size_t es)
    {
        size_t o = 0;
        auto take = [&](size_t bytes) { size_t at = o; o += align16(bytes); return at; };
        xpre = take(Nf * n * es); K = take(Nf * n * m * es); y = take(Nf * m * es); SI = take(Nf * m * m * es);
        v = take(Nf * n * es); vn = take(Nf * n * es); w = take(Nf * m * es); st = take(Nf * sizeof(int32_t));
        total = o;
    }
};

bool fused_shape(int n, int m, int du_used, int dtype, int64_t lag)
{
    (void)dtype;
    return du_used == 0 && lag <= BKE_FLS_FUSED_MAX_LAG && ((n == 1 && m == 1) || (n == 2 && m == 1) || (n == 4 && m == 2));
}

template <typename T>
int launch_per_epoch(const bke_fls_args &a, cudaStream_t s)
{
    const bke_kf_args &k0 = a.step;
    const int64_t Nf = k0.n_filters;
    const int n = k0.dim_x, m = k0.dim_z, du = a.us ? k0.dim_u : 0;
    const WsLayout ws(Nf, n, m, sizeof(T));
    char *wb = (char *)a.workspace;
    if (k0.status && check_cuda(cudaMemsetAsync(k0.status, 0, sizeof(int32_t) * (size_t)Nf, s), "memset status")) return BKE_ERR_CUDA;
    FlsCorrP<T> c;
    c.Nf = Nf; c.lag = a.lag; c.n = n; c.m = m;
    c.F = (const T *)k0.F; c.H = (const T *)k0.H; c.sF = k0.F_stride; c.sH = k0.H_stride;
    c.x_post = (const T *)k0.x_out; c.P_post = (const T *)k0.P_out;
    c.x_pre = (const T *)(wb + ws.xpre); c.K = (const T *)(wb + ws.K); c.y = (const T *)(wb + ws.y);
    c.SI = (const T *)(wb + ws.SI); c.st_epoch = (const int32_t *)(wb + ws.st);
    c.v = (T *)(wb + ws.v); c.vn = (T *)(wb + ws.vn); c.w = (T *)(wb + ws.w);
    c.xs = (T *)a.xs_smooth; c.xhat = (T *)a.xhat; c.status = k0.status;
    const unsigned grid = (unsigned)((Nf + 127) / 128);
    for (int64_t t = 0; t < a.n_steps; t++) {
        bke_kf_args k = k0;
        k.flags = BKE_DO_PREDICT | BKE_DO_UPDATE;            // the epoch's own status: every filter written
        k.alpha_sq = 1.0;
        if (t > 0) { k.x = k0.x_out; k.P = k0.P_out; }
        k.z = (const char *)a.zs + (size_t)t * Nf * m * sizeof(T);
        k.z_valid = nullptr;
        if (du) { k.u = (const char *)a.us + (size_t)t * Nf * du * sizeof(T); k.u_stride = du; }
        else { k.B = nullptr; k.u = nullptr; k.dim_u = 0; }
        k.x_prior = wb + ws.xpre; k.P_prior = nullptr;
        k.K = wb + ws.K; k.y = wb + ws.y; k.SI = wb + ws.SI; k.log_likelihood = nullptr;
        k.S = (t + 1 == a.n_steps) ? k0.S : nullptr;
        k.status = (int32_t *)(wb + ws.st);
        int rc = launch_kf_any(k, s);
        if (rc) return rc;
        c.k = a.count + t; c.t = t;
        c.z = (const T *)k.z; c.y_last = (t + 1 == a.n_steps && k0.y) ? (T *)(wb + ws.y) : nullptr;
        fls_correct_kernel<T><<<grid, 128, 0, s>>>(c);
        if ((rc = check_cuda(cudaGetLastError(), "fls_correct_kernel launch"))) return rc;
    }
    if (k0.y && check_cuda(cudaMemcpyAsync(k0.y, wb + ws.y, (size_t)Nf * m * sizeof(T), cudaMemcpyDeviceToDevice, s), "copy y"))
        return BKE_ERR_CUDA;
    return BKE_OK;
}

}  // namespace

size_t fls_workspace_bytes(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dim_u, int32_t dtype, int64_t lag)
{
    if (n_filters <= 0 || dim_x < 1 || dim_z < 1 || (dtype != BKE_F32 && dtype != BKE_F64)) return 0;
    if (fused_shape(dim_x, dim_z, dim_u, dtype, lag)) return 0;
    return WsLayout(n_filters, dim_x, dim_z, dtype == BKE_F32 ? 4 : 8).total;
}

int launch_fls(const bke_fls_args &a, cudaStream_t s)
{
    const bke_kf_args &k = a.step;
    if (fused_shape(k.dim_x, k.dim_z, a.us ? k.dim_u : 0, k.dtype, a.lag)) {
        const bool f32 = k.dtype == BKE_F32;
        if (k.dim_x == 4) return f32 ? launch_fused<float, 4, 2>(a, s) : launch_fused<double, 4, 2>(a, s);
        if (k.dim_x == 2) return f32 ? launch_fused<float, 2, 1>(a, s) : launch_fused<double, 2, 1>(a, s);
        return f32 ? launch_fused<float, 1, 1>(a, s) : launch_fused<double, 1, 1>(a, s);
    }
    const size_t need = WsLayout(k.n_filters, k.dim_x, k.dim_z, k.dtype == BKE_F32 ? 4 : 8).total;
    if (!a.workspace || a.workspace_bytes < need) {
        set_error("bke_fls_smooth: this call runs the per-epoch path and needs a workspace of %zu bytes "
                  "(bke_fls_workspace_bytes), got %zu", need, a.workspace ? a.workspace_bytes : (size_t)0);
        return BKE_ERR_BAD_ARG;
    }
    if ((reinterpret_cast<uintptr_t>(a.workspace) & 15u) != 0) { set_error("bke_fls_smooth: workspace must be 16-byte aligned"); return BKE_ERR_BAD_ARG; }
    return k.dtype == BKE_F32 ? launch_per_epoch<float>(a, s) : launch_per_epoch<double>(a, s);
}

}  // namespace bke
