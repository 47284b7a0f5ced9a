// mix.cu — bank-level model mixing for multiple-model estimators: a bank of N tracks, each
// followed by the same M filters (one KalmanFilter bank per model).  The reference loops over a
// Python list of filter objects for ONE track (filterpy/kalman/IMM.py:160-249,
// filterpy/kalman/mmae.py:140-210); here every step is one launch over all tracks.
//
//   bke_mm_probabilities   IMM.py:178-184 + :239-247  (mu = cbar * L; normalise; cbar = mu M;
//                                                      omega[i,j] = M[i,j] mu[i] / cbar[j])
//                          mmae.py:180-184            (p *= L; p /= sum(p))
//                          with L = max(exp(log_likelihood), DBL_MIN)  (kalman_filter.py:1213-1223)
//   bke_mm_mix             IMM.py:201-213   mixed initial conditions x0_i, P0_i for every model i
//   bke_mm_estimate        IMM.py:228-237   x = sum mu_j x_j, P = sum mu_j ((x_j - x)(x_j - x)' + P_j)
//                          mmae.py:186-201  (with the reference's element-wise zip, see BKE_MM_MMAE)
//
// Work split: one thread per element of the x arrays, then of the P arrays, so that consecutive
// threads touch consecutive addresses of every model's bank arrays; the few per-track scalars (mu,
// omega) are re-read by the threads of a track from L1.  All HBM-bound: per track the mix reads and
// writes M (n + n^2) scalars.
#include <float.h>
#include "bke_internal.cuh"
#include "kf_rowio.cuh"

namespace bke {
namespace {

unsigned grid_for(int64_t work);

template <typename T>
struct MixP {
    int64_t N;
    int n, M;
    unsigned flags;
    const T *x[BKE_MM_MAX_MODELS], *P[BKE_MM_MAX_MODELS];
    T *xo[BKE_MM_MAX_MODELS], *Po[BKE_MM_MAX_MODELS];
    const T *ll[BKE_MM_MAX_MODELS];
    const double *w;             // omega[N,M,M] (mix) or mu[N,M] (estimate)
    int64_t sw;                  // per-track stride of w (0 = shared)
    double *mu, *cbar, *omega;   // probabilities kernel
    const double *trans;         // M[M,M]
};

// Element-parallel kernels: one thread per element of the concatenated x arrays (N*n) or of the
// concatenated P arrays (N*n*n), grid-stride; MM > 0 fixes the model count at compile time (loops
// unroll, per-model values stay in registers), MM == 0 is the run-time fallback (M <= 8).
// index / divisor with 32-bit arithmetic when the index fits (a 64-bit division costs ~80 instructions)
__device__ __forceinline__ int64_t div_idx(int64_t a, int b, bool small)
{
    return small ? (int64_t)((uint32_t)a / (uint32_t)b) : a / b;
}

template <int MM>
struct ModelCount {
    int m;
    __device__ __forceinline__ int get() const { return MM > 0 ? MM : m; }
};

// mixed initial conditions (IMM.py:201-213): for every target model i
//   x0_i = sum_j omega[j,i] x_j ;  P0_i = sum_j omega[j,i] ((x_j - x0_i)(x_j - x0_i)' + P_j)
template <typename T, int MM>
__global__ void __launch_bounds__(256) k_mm_mix(MixP<T> p)
{
    constexpr int MA = MM > 0 ? MM : BKE_MM_MAX_MODELS;
    const int n = p.n, nn = n * n;
    const int M = ModelCount<MM>{p.M}.get();
    const int64_t nx = p.N * n, total = nx + p.N * nn;
    const bool small = total <= 0xffffffffLL;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        if (g < nx) {
            const int64_t t = div_idx(g, n, small);
            const double *om = p.w + t * p.sw;
            T xj[MA];
#pragma unroll
            for (int j = 0; j < MA; j++) if (j < M) xj[j] = p.x[j][g];
#pragma unroll
            for (int i = 0; i < MA; i++) {
                if (i < M) {
                    T s = T(0);
#pragma unroll
                    for (int j = 0; j < MA; j++) if (j < M) s += xj[j] * (T)om[j * M + i];
                    p.xo[i][g] = s;
                }
            }
        } else {
            const int64_t q = g - nx;
            const int64_t t = div_idx(q, nn, small);
            const int rc = (int)(q - t * nn), r = rc / n, c = rc - r * n;
            const double *om = p.w + t * p.sw;
            T xr[MA], xc[MA], Pj[MA];
#pragma unroll
            for (int j = 0; j < MA; j++) {
                if (j < M) {
                    xr[j] = p.x[j][t * n + r];
                    xc[j] = p.x[j][t * n + c];
                    Pj[j] = p.P[j][q];
                }
            }
#pragma unroll
            for (int i = 0; i < MA; i++) {
                if (i < M) {
                    T w[MA];
                    T mr = T(0), mc = T(0);                 // the mixed mean, in the precision it is stored in
#pragma unroll
                    for (int j = 0; j < MA; j++) if (j < M) { w[j] = (T)om[j * M + i]; mr += xr[j] * w[j]; mc += xc[j] * w[j]; }
                    T s = T(0);
#pragma unroll
                    for (int j = 0; j < MA; j++) if (j < M) s += w[j] * ((xr[j] - mr) * (xc[j] - mc) + Pj[j]);
                    p.Po[i][q] = s;
                }
            }
        }
    }
}

// combined estimate (IMM.py:228-237; mmae.py:186-201 with BKE_MM_MMAE)
template <typename T, int MM>
__global__ void __launch_bounds__(256) k_mm_estimate(MixP<T> p)
{
    constexpr int MA = MM > 0 ? MM : BKE_MM_MAX_MODELS;
    const int n = p.n, nn = n * n;
    const int M = ModelCount<MM>{p.M}.get();
    const bool mmae = p.flags & BKE_MM_MMAE;
    const int64_t nx = p.N * n, total = nx + p.N * nn;
    const bool small = total <= 0xffffffffLL;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        if (g < nx) {
            const double *mu = p.w + div_idx(g, n, small) * p.sw;
            T s = T(0);
#pragma unroll
            for (int j = 0; j < MA; j++) if (j < M) s += p.x[j][g] * (T)mu[j];
            p.xo[0][g] = s;
        } else {
            const int64_t q = g - nx;
            const int64_t t = div_idx(q, nn, small);
            const int rc = (int)(q - t * nn), r = rc / n, c = rc - r * n;
            const double *mu = p.w + t * p.sw;
            T s = T(0);
            if (!mmae) {
                T xr[MA], xc[MA], w[MA], mr = T(0), mc = T(0);
#pragma unroll
                for (int j = 0; j < MA; j++) {
                    if (j < M) {
                        xr[j] = p.x[j][t * n + r]; xc[j] = p.x[j][t * n + c]; w[j] = (T)mu[j];
                        mr += xr[j] * w[j]; mc += xc[j] * w[j];
                    }
                }
#pragma unroll
                for (int j = 0; j < MA; j++) if (j < M) s += w[j] * ((xr[j] - mr) * (xc[j] - mc) + p.P[j][q]);
            } else {
                // mmae.py:197-199 zips the COMPONENTS of the mixed x with the filters: term j uses
                // y = f_j.x - x[j] (a scalar), and only min(dim_x, M) terms exist
                const int terms = M < n ? M : n;
                for (int j = 0; j < terms; j++) {
                    T mj = T(0);
                    for (int k = 0; k < M; k++) mj += p.x[k][t * n + j] * (T)mu[k];
                    s += (T)mu[j] * ((p.x[j][t * n + r] - mj) * (p.x[j][t * n + c] - mj) + p.P[j][q]);
                }
            }
            p.Po[0][q] = s;
        }
    }
}

// Row-parallel kernels for compile-time (dim_x, model count): one thread per (track, row r of P).  It
// loads each model's whole x and row r of its P with 16-byte loads, forms the mixed mean once and
// writes row r of every output covariance (plus element r of the mean): no redundant work across
// the threads of a row, a quarter of the threads of the element-parallel form.
// MIX = true: IMM.py:201-213 for every target model; MIX = false: IMM.py:228-237 (one output)
template <typename T, int NX, int MM, bool MIX>
__global__ void __launch_bounds__(256) k_mm_rows(MixP<T> p)
{
    const int64_t total = p.N * NX;
    for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t t = g / NX;
        const int r = (int)(g - t * NX);
        T xv[MM][NX], Pr[MM][NX];
#pragma unroll
        for (int j = 0; j < MM; j++) {
            ldv<T, NX>(xv[j], p.x[j] + t * NX);
            ldv<T, NX>(Pr[j], p.P[j] + g * NX);
        }
        const double *wd = p.w + t * p.sw;
        constexpr int OUTS = MIX ? MM : 1;
#pragma unroll
        for (int i = 0; i < OUTS; i++) {
            T w[MM], m[NX];
#pragma unroll
            for (int j = 0; j < MM; j++) w[j] = (T)(MIX ? wd[j * MM + i] : wd[j]);
#pragma unroll
            for (int c = 0; c < NX; c++) {
                T a = T(0);
#pragma unroll
                for (int j = 0; j < MM; j++) a += xv[j][c] * w[j];
                m[c] = a;
            }
            T mr = T(0), xr[MM];
#pragma unroll
            for (int c = 0; c < NX; c++) if (c == r) mr = m[c];
#pragma unroll
            for (int j = 0; j < MM; j++) {
                T v = T(0);
#pragma unroll
                for (int c = 0; c < NX; c++) if (c == r) v = xv[j][c];
                xr[j] = v - mr;
            }
            T out[NX];
#pragma unroll
            for (int c = 0; c < NX; c++) {
                T sacc = T(0);
#pragma unroll
                for (int j = 0; j < MM; j++) sacc += w[j] * (xr[j] * (xv[j][c] - m[c]) + Pr[j][c]);
                out[c] = sacc;
            }
            stv<T, NX>(p.Po[i] + g * NX, out);
            p.xo[i][g] = mr;
        }
    }
}

template <typename T, int NX, int MM>
bool launch_rows(const MixP<T> &p, int op, cudaStream_t s)
{
    const unsigned grid = grid_for(p.N * NX);
    if (op == 1) k_mm_rows<T, NX, MM, true><<<grid, 256, 0, s>>>(p);
    else k_mm_rows<T, NX, MM, false><<<grid, 256, 0, s>>>(p);
    return true;
}

template <typename T, int NX>
bool launch_rows_m(const MixP<T> &p, int op, cudaStream_t s)
{
    switch (p.M) {
    case 2: return launch_rows<T, NX, 2>(p, op, s);
    case 3: return launch_rows<T, NX, 3>(p, op, s);
    case 4: return launch_rows<T, NX, 4>(p, op, s);
    default: return false;
    }
}

// mode probabilities, one thread per track
template <typename T>
__global__ void __launch_bounds__(256) k_mm_probabilities(MixP<T> p)
{
    const int M = p.M;
    const bool mmae = p.flags & BKE_MM_MMAE, from_mu = p.flags & BKE_MM_FROM_MU;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < p.N; t += (int64_t)gridDim.x * blockDim.x) {
        double mu[BKE_MM_MAX_MODELS];
        if (from_mu) {
            for (int j = 0; j < M; j++) mu[j] = p.mu[t * M + j];
        } else {
            double sum = 0.0;
            for (int j = 0; j < M; j++) {
                double L = exp((double)p.ll[j][t]);
                if (L == 0.0) L = DBL_MIN;                       // kalman_filter.py:1221-1222
                const double prior = mmae ? p.mu[t * M + j] : p.cbar[t * M + j];
                mu[j] = prior * L;
                sum += mu[j];
            }
            const double rs = 1.0 / sum;                    // one division per track; the products differ from x / sum by <= 1 ulp
            for (int j = 0; j < M; j++) { mu[j] *= rs; p.mu[t * M + j] = mu[j]; }
        }
        if (mmae) continue;
        double cb[BKE_MM_MAX_MODELS];
        for (int j = 0; j < M; j++) {
            double s = 0.0;
            for (int i = 0; i < M; i++) s += mu[i] * p.trans[i * M + j];
            cb[j] = 1.0 / s;
            p.cbar[t * M + j] = s;
        }
        for (int i = 0; i < M; i++)
            for (int j = 0; j < M; j++) p.omega[(t * M + i) * M + j] = (p.trans[i * M + j] * mu[i]) * cb[j];
    }
}

unsigned grid_for(int64_t work)
{
    int64_t b = (work + 255) / 256;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (b > cap) b = cap;
    return (unsigned)(b < 1 ? 1 : b);
}

template <typename T>
int launch_t(const bke_mm_args &a, int op, cudaStream_t s)
{
    MixP<T> p;
    p.N = a.n_tracks; p.n = a.dim_x; p.M = a.n_models; p.flags = a.flags;
    for (int j = 0; j < BKE_MM_MAX_MODELS; j++) {
        p.x[j] = (const T *)a.x[j]; p.P[j] = (const T *)a.P[j];
        p.xo[j] = (T *)a.x_out[j]; p.Po[j] = (T *)a.P_out[j];
        p.ll[j] = (const T *)a.log_likelihood[j];
    }
    p.mu = a.mu; p.cbar = a.cbar; p.omega = a.omega; p.trans = a.trans;
    const int64_t E = a.dim_x + (int64_t)a.dim_x * a.dim_x;
    const unsigned ge = grid_for((p.N * E + 1) / 2);
    if (op != 0 && !(a.flags & BKE_MM_MMAE)) {
        // row-parallel form for the common shapes, when 16-byte accesses are possible
        bool aligned = true;
        for (int j = 0; j < p.M; j++)
            aligned = aligned && ((reinterpret_cast<uintptr_t>(p.x[j]) | reinterpret_cast<uintptr_t>(p.P[j])) & 15) == 0;
        const int outs = op == 1 ? p.M : 1;
        for (int j = 0; j < outs; j++) aligned = aligned && (reinterpret_cast<uintptr_t>(p.Po[j]) & 15) == 0;
        p.w = op == 1 ? a.omega : a.mu; p.sw = a.weights_stride;
        bool done = false;
        if (aligned && p.n == 4) done = launch_rows_m<T, 4>(p, op, s);
        else if (aligned && p.n == 6) done = launch_rows_m<T, 6>(p, op, s);
        else if (aligned && p.n == 2) done = launch_rows_m<T, 2>(p, op, s);
        if (done) return check_cuda(cudaGetLastError(), "mm launch");
    }
    if (op == 0) {
        k_mm_probabilities<T><<<grid_for(p.N), 256, 0, s>>>(p);
    } else if (op == 1) {
        p.w = a.omega; p.sw = a.weights_stride;
        switch (p.M) {
        case 2: k_mm_mix<T, 2><<<ge, 256, 0, s>>>(p); break;
        case 3: k_mm_mix<T, 3><<<ge, 256, 0, s>>>(p); break;
        case 4: k_mm_mix<T, 4><<<ge, 256, 0, s>>>(p); break;
        default: k_mm_mix<T, 0><<<ge, 256, 0, s>>>(p);
        }
    } else {
        p.w = a.mu; p.sw = a.weights_stride;
        switch (p.M) {
        case 2: k_mm_estimate<T, 2><<<ge, 256, 0, s>>>(p); break;
        case 3: k_mm_estimate<T, 3><<<ge, 256, 0, s>>>(p); break;
        case 4: k_mm_estimate<T, 4><<<ge, 256, 0, s>>>(p); break;
        default: k_mm_estimate<T, 0><<<ge, 256, 0, s>>>(p);
        }
    }
    return check_cuda(cudaGetLastError(), "mm launch");
}

int validate(const bke_mm_args *args, int op)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    const bke_mm_args &a = *args;
    if (a.n_tracks < 0) { set_error("n_tracks < 0"); return BKE_ERR_BAD_ARG; }
    if (a.n_models < 1 || a.n_models > BKE_MM_MAX_MODELS) { set_error("n_models must be in [1, %d]", BKE_MM_MAX_MODELS); return BKE_ERR_UNSUPPORTED; }
    if (int rc = check_dtype(a.dtype)) return rc;
    if (op != 0 && (a.dim_x < 1 || a.dim_x > 64)) { set_error("dim_x must be in [1, 64]"); return BKE_ERR_BAD_ARG; }
    if (a.n_tracks == 0) return BKE_OK;
    const int M = a.n_models;
    if (op == 0) {
        if (!(a.flags & BKE_MM_FROM_MU))
            for (int j = 0; j < M; j++) if (!a.log_likelihood[j]) { set_error("log_likelihood[%d] is NULL", j); return BKE_ERR_BAD_ARG; }
        if (!a.mu) { set_error("mu is NULL"); return BKE_ERR_BAD_ARG; }
        if (!(a.flags & BKE_MM_MMAE) && (!a.cbar || !a.omega || !a.trans)) { set_error("cbar, omega and trans are required"); return BKE_ERR_BAD_ARG; }
    } else {
        for (int j = 0; j < M; j++) if (!a.x[j] || !a.P[j]) { set_error("x[%d] / P[%d] is NULL", j, j); return BKE_ERR_BAD_ARG; }
        const int outs = op == 1 ? M : 1;
        for (int j = 0; j < outs; j++) {
            if (!a.x_out[j] || !a.P_out[j]) { set_error("x_out[%d] / P_out[%d] is NULL", j, j); return BKE_ERR_BAD_ARG; }
            for (int q = 0; q < M; q++)
                if (a.x_out[j] == a.x[q] || a.P_out[j] == a.P[q]) { set_error("outputs must not alias the inputs"); return BKE_ERR_BAD_ARG; }
        }
        if (op == 1 && !a.omega) { set_error("omega is NULL"); return BKE_ERR_BAD_ARG; }
        if (op == 2 && !a.mu) { set_error("mu is NULL"); return BKE_ERR_BAD_ARG; }
        if (a.weights_stride < 0) { set_error("negative stride"); return BKE_ERR_BAD_ARG; }
    }
    if (int rc = require_device()) return rc;
    return -1;      // go
}

int run(const bke_mm_args *args, int op, void *stream)
{
    const int v = validate(args, op);
    if (v >= 0) return v;
    return args->dtype == BKE_F32 ? launch_t<float>(*args, op, (cudaStream_t)stream)
                                  : launch_t<double>(*args, op, (cudaStream_t)stream);
}

}  // namespace
}  // namespace bke

extern "C" {
int bke_mm_probabilities(const bke_mm_args *args, void *stream) { return bke::run(args, 0, stream); }
int bke_mm_mix(const bke_mm_args *args, void *stream) { return bke::run(args, 1, stream); }
int bke_mm_estimate(const bke_mm_args *args, void *stream) { return bke::run(args, 2, stream); }
}
