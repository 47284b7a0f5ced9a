// ut.cu — stand-alone sigma-point generation and unscented transform for a bank (the fused UKF step
// in ukf.cu does both on chip; these entry points serve callers of
// MerweScaledSigmaPoints.sigma_points (filterpy/kalman/sigma_points.py:124-177),
// SimplexSigmaPoints.sigma_points (:454-513) and
// unscented_transform (filterpy/kalman/unscented_transform.py:22-128) themselves).
// One warp per filter, matrices in the warp's slice of shared memory: sigma points for any n <= 32, the
// transform for any k <= 256 points of n <= 64 (up to 4 warps per block, fewer when their slices do not fit).
#include "bke_internal.cuh"
#include "ukf_kernel.cuh"

namespace bke {
namespace {

// SPX: SimplexSigmaPoints (sigma_points.py:499-513, scale = 1): lane i forms column i of the offsets
// D_n .. D_0 with the running suffix sum of ukf_kernel.cuh's simplex_offsets
template <typename T, bool SPX = false>
__global__ void __launch_bounds__(128) k_sigma_points(int64_t N, int n, T scale, const T *x, const T *P, T *sig, int32_t *status)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    T *U = reinterpret_cast<T *>(smem_raw) + (size_t)wib * (n * n + n);
    T *xs = U + n * n;
    const int ns = SPX ? n + 1 : 2 * n + 1;
    for (int64_t f = (int64_t)blockIdx.x * wpb + wib; f < N; f += (int64_t)gridDim.x * wpb) {
        for (int e = lane; e < n * n; e += 32) U[e] = scale * P[f * n * n + e];
        for (int e = lane; e < n; e += 32) xs[e] = x[f * n + e];
        __syncwarp();
        int st = BKE_STATUS_OK;
        // upper Cholesky (reads the upper triangle only, like scipy.linalg.cholesky): U'U = A, in place
        for (int j = 0; j < n; j++) {
            T d = U[j * n + j];
            for (int k = 0; k < j; k++) d -= U[k * n + j] * U[k * n + j];
            if (!(d > T(0))) st = BKE_STATUS_NOT_PD;
            const T r = sqrt(d);
            __syncwarp();
            if (lane == 0) U[j * n + j] = r;
            for (int i = j + 1 + lane; i < n; i += 32) {
                T s = U[j * n + i];
                for (int k = 0; k < j; k++) s -= U[k * n + j] * U[k * n + i];
                U[j * n + i] = s / r;
            }
            __syncwarp();
        }
        T *o = sig + f * (int64_t)ns * n;
        if constexpr (SPX) {
            for (int i = lane; i < n; i += 32) {
                T S = T(0);
                for (int j = n; j >= 2; j--) {
                    T v = xs[i];
                    if (i >= j - 1) {
                        const T c = ukfk::simplex_coef<T>(n, j), u = U[(j - 1) * n + i];
                        v = xs[i] + (T(-j) * c * u + S);
                        S += c * u;
                    }
                    o[j * n + i] = v;
                }
                const T c1 = ukfk::simplex_coef<T>(n, 1), u = U[i];
                o[i] = xs[i] + (S - c1 * u);
                o[n + i] = xs[i] + (S + c1 * u);
            }
            if (status && lane == 0) status[f] = st;
            __syncwarp();
            continue;
        }
        for (int e = lane; e < ns * n; e += 32) {
            const int s = e / n, i = e - s * n;
            T v = xs[i];
            if (s >= 1 && s <= n) { const int k = s - 1; if (i >= k) v = xs[i] + U[k * n + i]; }      // x - (-U[k]) (sigma_points.py:174)
            else if (s > n) { const int k = s - 1 - n; if (i >= k) v = xs[i] - U[k * n + i]; }
            o[e] = v;
        }
        if (status && lane == 0) status[f] = st;
        __syncwarp();
    }
}

template <typename T>
__global__ void __launch_bounds__(128) k_unscented_transform(int64_t N, int ns, int n, const T *sig, const T *Wm, const T *Wc,
                                                            const T *noise, int64_t noise_stride, T *x_out, T *P_out)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    T *S = reinterpret_cast<T *>(smem_raw) + (size_t)wib * (ns * n + n);
    T *xm = S + ns * n;
    for (int64_t f = (int64_t)blockIdx.x * wpb + wib; f < N; f += (int64_t)gridDim.x * wpb) {
        for (int e = lane; e < ns * n; e += 32) S[e] = sig[f * (int64_t)ns * n + e];
        __syncwarp();
        for (int i = lane; i < n; i += 32) {            // x = dot(Wm, sigmas)   (unscented_transform.py:104)
            T s = T(0);
            for (int k = 0; k < ns; k++) s += Wm[k] * S[k * n + i];
            xm[i] = s;
            x_out[f * n + i] = s;
        }
        __syncwarp();
        for (int e = lane; e < n * n; e += 32) {         // P = y' diag(Wc) y (+ noise)   (:117-126)
            const int a = e / n, b = e - a * n;
            T s = T(0);
            for (int k = 0; k < ns; k++) s += Wc[k] * (S[k * n + a] - xm[a]) * (S[k * n + b] - xm[b]);
            if (noise) s += noise[f * noise_stride + e];
            P_out[f * n * n + e] = s;
        }
        __syncwarp();
    }
}

template <typename T>
int sigma_t(int64_t N, int n, double alpha, double kappa, const void *x, const void *P, void *sig, int32_t *status, cudaStream_t s)
{
    const double lambda_ = alpha * alpha * (n + kappa) - n;
    const size_t smem = 4 * sizeof(T) * (size_t)(n * n + n);
    int64_t grid = (N + 3) / 4, cap = (int64_t)sm_count() * 16;
    k_sigma_points<T><<<(unsigned)(grid < cap ? grid : cap), 128, smem, s>>>(N, n, (T)(lambda_ + n), (const T *)x, (const T *)P, (T *)sig, status);
    return check_cuda(cudaGetLastError(), "k_sigma_points launch");
}

template <typename T>
int simplex_t(int64_t N, int n, const void *x, const void *P, void *sig, int32_t *status, cudaStream_t s)
{
    const size_t smem = 4 * sizeof(T) * (size_t)(n * n + n);
    int64_t grid = (N + 3) / 4, cap = (int64_t)sm_count() * 16;
    k_sigma_points<T, true><<<(unsigned)(grid < cap ? grid : cap), 128, smem, s>>>(N, n, T(1), (const T *)x, (const T *)P, (T *)sig, status);
    return check_cuda(cudaGetLastError(), "k_sigma_points launch");
}

template <typename T>
int ut_t(int64_t N, int ns, int n, const void *sig, const void *Wm, const void *Wc, const void *noise, int64_t nstride,
         void *x_out, void *P_out, cudaStream_t s)
{
    // the budget is the device's opt-in shared memory per block: one warp's slice (at most
    // 8 * (256 * 64 + 64) B = 131,584 B) always fits an H100's 227 KB
    const size_t per_warp = sizeof(T) * (size_t)(ns * n + n);
    int dev = 0, optin = 0;
    if (check_cuda(cudaGetDevice(&dev), "cudaGetDevice") ||
        check_cuda(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev), "cudaDeviceGetAttribute"))
        return BKE_ERR_CUDA;
    WarpShape w;
    if (int rc = warp_shape((const void *)k_unscented_transform<T>, per_warp, (size_t)optin, N, w)) {
        if (rc == BKE_ERR_UNSUPPORTED)
            set_error("bke_unscented_transform: n_sigmas=%d dim=%d needs %zu B of shared memory per filter (> %d)", ns, n, per_warp, optin);
        return rc;
    }
    k_unscented_transform<T><<<w.grid, 32 * w.wpb, w.smem, s>>>(N, ns, n, (const T *)sig, (const T *)Wm, (const T *)Wc,
                                                              (const T *)noise, nstride, (T *)x_out, (T *)P_out);
    return check_cuda(cudaGetLastError(), "k_unscented_transform launch");
}

}  // namespace
}  // namespace bke

using namespace bke;

extern "C" {

int bke_merwe_sigma_points(int64_t n_filters, int32_t dim_x, int32_t dtype, double alpha, double beta, double kappa,
                           const void *x, const void *P, void *sigmas, int32_t *status, void *stream)
{
    (void)beta;
    if (n_filters < 0 || dim_x < 1 || dim_x > 32) { set_error("bad dimensions (1 <= dim_x <= 32)"); return BKE_ERR_BAD_ARG; }
    if (int rc = check_dtype(dtype)) return rc;
    if (n_filters == 0) return BKE_OK;
    if (!x || !P || !sigmas) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    if (int rc = require_device()) return rc;
    return dtype == BKE_F32 ? sigma_t<float>(n_filters, dim_x, alpha, kappa, x, P, sigmas, status, (cudaStream_t)stream)
                            : sigma_t<double>(n_filters, dim_x, alpha, kappa, x, P, sigmas, status, (cudaStream_t)stream);
}

int bke_simplex_sigma_points(int64_t n_filters, int32_t dim_x, int32_t dtype, const void *x, const void *P, void *sigmas,
                             int32_t *status, void *stream)
{
    if (n_filters < 0 || dim_x < 1 || dim_x > 32) { set_error("bad dimensions (1 <= dim_x <= 32)"); return BKE_ERR_BAD_ARG; }
    if (int rc = check_dtype(dtype)) return rc;
    if (n_filters == 0) return BKE_OK;
    if (!x || !P || !sigmas) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    if (int rc = require_device()) return rc;
    return dtype == BKE_F32 ? simplex_t<float>(n_filters, dim_x, x, P, sigmas, status, (cudaStream_t)stream)
                            : simplex_t<double>(n_filters, dim_x, x, P, sigmas, status, (cudaStream_t)stream);
}

int bke_unscented_transform(int64_t n_filters, int32_t n_sigmas, int32_t dim, int32_t dtype, const void *sigmas,
                            const void *Wm, const void *Wc, const void *noise_cov, int64_t noise_stride,
                            void *x_out, void *P_out, void *stream)
{
    if (n_filters < 0 || n_sigmas < 1 || dim < 1 || dim > 64 || n_sigmas > 256) { set_error("bad dimensions"); return BKE_ERR_BAD_ARG; }
    if (int rc = check_dtype(dtype)) return rc;
    if (n_filters == 0) return BKE_OK;
    if (!sigmas || !Wm || !Wc || !x_out || !P_out) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    if (int rc = require_device()) return rc;
    return dtype == BKE_F32 ? ut_t<float>(n_filters, n_sigmas, dim, sigmas, Wm, Wc, noise_cov, noise_stride, x_out, P_out, (cudaStream_t)stream)
                            : ut_t<double>(n_filters, n_sigmas, dim, sigmas, Wm, Wc, noise_cov, noise_stride, x_out, P_out, (cudaStream_t)stream);
}

}  // extern "C"
