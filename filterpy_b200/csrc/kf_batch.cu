// kf_batch.cu — KalmanFilter.batch_filter for a bank (filterpy/kalman/kalman_filter.py:826-993,
// procedural twin :1664-1788): the T-epoch loop runs INSIDE the kernel.  One thread owns one
// filter; x, P and the (time-constant) models F, Q, H, R stay in registers for all T epochs, each
// epoch streams z[t] in (coalesced: consecutive threads read consecutive filters) and the four
// outputs means/covariances/means_p/covariances_p out.  Algorithmic traffic per filter-step is
// (m + 2n + 2n^2) scalars (168 B for 4/2 fp32) instead of the 344 B of a stand-alone step.
// The outputs are 95 % of that traffic: a full warp stages its 32 filters' four output blocks of an
// epoch in shared memory (they are dense [32][n] / [32][n][n] pieces of the output arrays) and one
// lane sends them off with four bulk copies (cp.async.bulk.global.shared::cta), double-buffered so
// that epoch t+1 computes while epoch t's copies drain.  (Per-thread 16-byte stores put 32 half-filled
// sectors on the wire per instruction.)
//
// Shapes without a register-tiled instantiation fall back to looping bke_kf_step on the host
// (still on the GPU, one launch per epoch).
#include <stdlib.h>
#include "bke_internal.cuh"
#include "kf_regtile.cuh"
#include "kf_rowio.cuh"
#include "ptx.cuh"

namespace bke {
namespace {

template <typename T>
struct BatchP {
    int64_t N, Tn;
    bool update_first;
    T alpha_sq;
    const T *x, *P, *F, *Q, *H, *R, *zs;
    int64_t sF, sQ, sH, sR;
    const uint8_t *valid;
    T *x_out, *P_out, *means, *covs, *means_p, *covs_p;
    int32_t *status;
};

// per-warp staging of one epoch's outputs: [means_p | covs_p | means | covs], each 32 filters deep
template <typename T, int N>
struct BatchStage {
    static constexpr int XB = 32 * N * (int)sizeof(T), PB = 32 * N * N * (int)sizeof(T);
    static constexpr int O_XP = 0, O_PP = XB, O_X = XB + PB, O_P = 2 * XB + PB;
    static constexpr int BYTES = 2 * (XB + PB);
    static_assert(XB % 16 == 0 && PB % 16 == 0, "bulk copies move multiples of 16 bytes");
};

template <typename T, int N, int M, bool STAGED>
__global__ void __launch_bounds__(128) kf_batch_kernel(BatchP<T> p)
{
    using St = BatchStage<T, N>;
    extern __shared__ __align__(128) unsigned char bsm[];
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const int64_t f0 = f - lane;                              // the warp's first filter
    // a full warp sends its outputs through shared memory and bulk copies; a ragged last warp stores directly
    const bool staged = STAGED && (f0 + 32 <= p.N);
    unsigned char *wst = bsm + (size_t)(threadIdx.x >> 5) * 2 * St::BYTES;
    if (f >= p.N) return;
    T x[N], P[N][N], F[N][N], Q[N][N], H[M][N], R[M][M];
    ld_scalar<T, N>(x, p.x + f * N);
    ld_scalar<T, N * N>(&P[0][0], p.P + f * N * N);
    ld_scalar<T, N * N>(&F[0][0], p.F + f * p.sF);
    ld_scalar<T, N * N>(&Q[0][0], p.Q + f * p.sQ);
    ld_scalar<T, M * N>(&H[0][0], p.H + f * p.sH);
    ld_scalar<T, M * M>(&R[0][0], p.R + f * p.sR);
    int st = BKE_STATUS_OK;
    // the measurement of epoch t+1 is fetched while epoch t computes: one exposed DRAM latency per
    // epoch was the dominant stall of the first version (long_scoreboard 7 per issue)
    T zn[M];
    bool has_zn = true;
    if (p.Tn > 0) {
        ld_scalar<T, M>(zn, p.zs + f * M);
        has_zn = p.valid == nullptr || p.valid[f] != 0;
    }
    for (int64_t t = 0; t < p.Tn; t++) {
        const int64_t tf = t * p.N + f;
        unsigned char *buf = wst + (t & 1) * St::BYTES;
        if (staged) {
            if (lane == 0) bulk_wait_read<1>();               // the copies of epoch t-2 have read this buffer
            __syncwarp();
        }
        T z[M];
#pragma unroll
        for (int a = 0; a < M; a++) z[a] = zn[a];
        const bool has_z = has_zn;
        if (t + 1 < p.Tn) {
            ld_scalar<T, M>(zn, p.zs + (tf + p.N) * M);
            has_zn = p.valid == nullptr || p.valid[tf + p.N] != 0;
        }
        auto upd = [&]() {
            if (has_z) {
                KfUpdateOut<T, N, M> o;
                reg_update<T, N, M>(x, P, H, R, z, o);
                if (!o.ok) st = BKE_STATUS_SINGULAR_S;
            }
            if (staged) {
                stv<T, N>(reinterpret_cast<T *>(buf + St::O_X) + lane * N, x);
                stv<T, N * N>(reinterpret_cast<T *>(buf + St::O_P) + lane * N * N, &P[0][0]);
            } else {
                if (p.means) stv<T, N>(p.means + tf * N, x);
                if (p.covs) stv<T, N * N>(p.covs + tf * N * N, &P[0][0]);
            }
        };
        auto pred = [&]() {
            reg_predict<T, N>(x, P, F, Q, p.alpha_sq);
            if (staged) {
                stv<T, N>(reinterpret_cast<T *>(buf + St::O_XP) + lane * N, x);
                stv<T, N * N>(reinterpret_cast<T *>(buf + St::O_PP) + lane * N * N, &P[0][0]);
            } else {
                if (p.means_p) stv<T, N>(p.means_p + tf * N, x);
                if (p.covs_p) stv<T, N * N>(p.covs_p + tf * N * N, &P[0][0]);
            }
        };
        if (p.update_first) { upd(); pred(); } else { pred(); upd(); }
        if (staged) {
            fence_proxy_async();                              // the staged rows become visible to the copy engine
            __syncwarp();
            if (lane == 0) {
                const int64_t e0 = t * p.N + f0;
                if (p.means_p) bulk_store(p.means_p + e0 * N, buf + St::O_XP, St::XB);
                if (p.covs_p) bulk_store(p.covs_p + e0 * N * N, buf + St::O_PP, St::PB);
                if (p.means) bulk_store(p.means + e0 * N, buf + St::O_X, St::XB);
                if (p.covs) bulk_store(p.covs + e0 * N * N, buf + St::O_P, St::PB);
                bulk_commit();
            }
        }
    }
    if (staged && lane == 0) bulk_wait_all();
    stv<T, N>(p.x_out + f * N, x);
    stv<T, N * N>(p.P_out + f * N * N, &P[0][0]);
    if (p.status) p.status[f] = st;
}

template <typename T, int N, int M>
int launch_reg(const bke_kf_batch_args &a, cudaStream_t s)
{
    const bke_kf_args &k = a.step;
    BatchP<T> p;
    p.N = k.n_filters; p.Tn = a.n_steps; p.update_first = k.flags & BKE_UPDATE_FIRST;
    p.alpha_sq = (T)k.alpha_sq;
    p.x = (const T *)k.x; p.P = (const T *)k.P; p.F = (const T *)k.F; p.Q = (const T *)k.Q;
    p.H = (const T *)k.H; p.R = (const T *)k.R; p.zs = (const T *)a.zs;
    p.sF = k.F_stride; p.sQ = k.Q_stride; p.sH = k.H_stride; p.sR = k.R_stride;
    p.valid = a.zs_valid;
    p.x_out = (T *)k.x_out; p.P_out = (T *)k.P_out;
    p.means = (T *)a.means; p.covs = (T *)a.covariances; p.means_p = (T *)a.means_p; p.covs_p = (T *)a.covariances_p;
    p.status = k.status;
    int64_t grid = (p.N + 127) / 128;
    // an epoch's slice of every output array must start on a 16-byte boundary for the bulk copies (the arrays
    // themselves are checked by the caller); otherwise every thread stores its own outputs
    const bool staged = ((size_t)p.N * N * sizeof(T)) % 16 == 0 && p.N >= 32;
    if (staged) {
        constexpr int smem = 4 * 2 * BatchStage<T, N>::BYTES;
        auto kern = kf_batch_kernel<T, N, M, true>;
        if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
        kern<<<(unsigned)grid, 128, smem, s>>>(p);
    } else {
        kf_batch_kernel<T, N, M, false><<<(unsigned)grid, 128, 0, s>>>(p);
    }
    return check_cuda(cudaGetLastError(), "kf_batch_kernel launch");
}

bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int launch_host_loop(const bke_kf_batch_args &a, cudaStream_t s)
{
    // One bke_kf_step per epoch.  The posterior of epoch t is written straight into means[t] /
    // covariances[t] and read from there by epoch t+1 (no copies); without those outputs the
    // state ping-pongs in place in x_out / P_out.
    const bke_kf_args &k0 = a.step;
    const size_t es = k0.dtype == BKE_F32 ? 4 : 8;
    const int64_t N = k0.n_filters, n = k0.dim_x, m = k0.dim_z;
    const bool uf = k0.flags & BKE_UPDATE_FIRST;
    const char *xin = (const char *)k0.x, *Pin = (const char *)k0.P;
    // status is sticky over the epochs (like the in-kernel time loop): zeroed once, then every
    // per-epoch launch writes it only where the epoch failed
    if (k0.status && check_cuda(cudaMemsetAsync(k0.status, 0, sizeof(int32_t) * (size_t)N, s), "memset status")) return BKE_ERR_CUDA;
    for (int64_t t = 0; t < a.n_steps; t++) {
        bke_kf_args k = k0;
        k.flags = BKE_DO_PREDICT | BKE_DO_UPDATE | (uf ? BKE_UPDATE_FIRST : 0) | BKE_STATUS_STICKY;
        k.x = xin; k.P = Pin;
        k.z = (const char *)a.zs + (size_t)t * N * m * es;
        k.z_valid = a.zs_valid ? a.zs_valid + t * N : nullptr;
        k.K = k.y = k.S = k.SI = k.log_likelihood = nullptr;
        char *post_x = a.means ? (char *)a.means + (size_t)t * N * n * es : (char *)k0.x_out;
        char *post_P = a.covariances ? (char *)a.covariances + (size_t)t * N * n * n * es : (char *)k0.P_out;
        char *prior_x = a.means_p ? (char *)a.means_p + (size_t)t * N * n * es : nullptr;
        char *prior_P = a.covariances_p ? (char *)a.covariances_p + (size_t)t * N * n * n * es : nullptr;
        int rc;
        if (!uf) {
            k.x_out = post_x; k.P_out = post_P; k.x_prior = prior_x; k.P_prior = prior_P;
            rc = launch_kf_any(k, s);
            if (rc) return rc;
            xin = post_x; Pin = post_P;
        } else {
            // update -> means[t]; predict -> means_p[t] which also feeds epoch t+1
            bke_kf_args ku = k; ku.flags = BKE_DO_UPDATE | BKE_STATUS_STICKY; ku.x_out = post_x; ku.P_out = post_P; ku.x_prior = ku.P_prior = nullptr;
            rc = launch_kf_any(ku, s);
            if (rc) return rc;
            bke_kf_args kp = k; kp.flags = BKE_DO_PREDICT; kp.x = post_x; kp.P = post_P;
            kp.x_out = prior_x ? prior_x : (char *)k0.x_out; kp.P_out = prior_P ? prior_P : (char *)k0.P_out;
            kp.x_prior = kp.P_prior = nullptr; kp.status = nullptr;
            rc = launch_kf_any(kp, s);
            if (rc) return rc;
            xin = (const char *)kp.x_out; Pin = (const char *)kp.P_out;
        }
    }
    if (a.n_steps > 0) {
        if (xin != (const char *)k0.x_out &&
            check_cuda(cudaMemcpyAsync(k0.x_out, xin, (size_t)N * n * es, cudaMemcpyDeviceToDevice, s), "copy final x")) return BKE_ERR_CUDA;
        if (Pin != (const char *)k0.P_out &&
            check_cuda(cudaMemcpyAsync(k0.P_out, Pin, (size_t)N * n * n * es, cudaMemcpyDeviceToDevice, s), "copy final P")) return BKE_ERR_CUDA;
    } else {
        if (k0.x_out != k0.x && check_cuda(cudaMemcpyAsync(k0.x_out, k0.x, (size_t)N * n * es, cudaMemcpyDeviceToDevice, s), "copy x")) return BKE_ERR_CUDA;
        if (k0.P_out != k0.P && check_cuda(cudaMemcpyAsync(k0.P_out, k0.P, (size_t)N * n * n * es, cudaMemcpyDeviceToDevice, s), "copy P")) return BKE_ERR_CUDA;
    }
    return BKE_OK;
}

}  // namespace

int launch_kf_batch(const bke_kf_batch_args &a, cudaStream_t s)
{
    const bke_kf_args &k = a.step;
    const bool no_ctrl = !(k.B && k.u);
    const bool al = aligned16(k.x_out) && aligned16(k.P_out) && aligned16(a.means) && aligned16(a.covariances) &&
                    aligned16(a.means_p) && aligned16(a.covariances_p);
    if (no_ctrl && al && a.n_steps > 0) {
        if (k.dtype == BKE_F32 && k.dim_x == 4 && k.dim_z == 2) return launch_reg<float, 4, 2>(a, s);
        if (k.dtype == BKE_F32 && k.dim_x == 2 && k.dim_z == 1) return launch_reg<float, 2, 1>(a, s);
        if (k.dtype == BKE_F64 && k.dim_x == 2 && k.dim_z == 1) return launch_reg<double, 2, 1>(a, s);
        if (k.dtype == BKE_F64 && k.dim_x == 4 && k.dim_z == 2) return launch_reg<double, 4, 2>(a, s);
    }
    return launch_host_loop(a, s);
}

}  // namespace bke
