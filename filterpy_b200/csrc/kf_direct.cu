// kf_direct.cu — thread-per-filter predict/update with the filter's arrays loaded straight from
// global memory into a register tile (csrc/kf_regtile.cuh), for the small shapes that have neither
// the TMA-staged kernel (4/2 fp32, csrc/kf_fast.cu) nor a good fit in the row-block kernel:
// 4/2 fp64 (the reference's default dtype), 1/1, 2/1, 2/2, 3/1, 4/1, 4/4, and 6/3, 6/2 in fp32.
//
// Same arithmetic as kf_fast.cu (filterpy/kalman/kalman_filter.py:471-478 predict, :533-556
// update); every thread reads its own rows of the AoS arrays with 16-byte loads — a row is 32-128
// contiguous bytes, so every fetched sector is used — and writes the posterior the same way.
// Shared (stride 0) models are read through the same pointers (all threads hit one line).
// Optional outputs, z_valid and the three predict/update modes are supported; a control input
// (B, u) and update-first go to the catch-all kernel.
#include "bke_internal.cuh"
#include "kf_regtile.cuh"
#include "kf_rowio.cuh"

namespace bke {
namespace {

template <typename T>
struct DirP {
    int64_t N;
    unsigned flags;
    T alpha_sq;
    const T *x, *P, *F, *Q, *H, *R, *z;
    int64_t sF, sQ, sH, sR;
    const uint8_t *valid;
    T *x_out, *P_out, *x_prior, *P_prior, *K, *y, *S, *SI, *ll;
    int32_t *status;
};

// EX: the optional outputs are compiled in (a separate instantiation keeps their tests and live
// ranges out of the plain kernel)
template <typename T, int N, int M, bool EX>
__global__ void __launch_bounds__(128) kf_direct_kernel(DirP<T> p)
{
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= p.N) return;
    const bool do_p = p.flags & BKE_DO_PREDICT, do_u = p.flags & BKE_DO_UPDATE;
    T x[N], P[N][N];
    ldv_rw<T, N>(x, p.x + f * N);
    ldv_rw<T, N * N>(&P[0][0], p.P + f * N * N);
    int st = BKE_STATUS_OK;
    if (do_p) {
        T F[N][N], Q[N][N];
        ldv<T, N * N>(&F[0][0], p.F + f * p.sF);
        ldv<T, N * N>(&Q[0][0], p.Q + f * p.sQ);
        reg_predict<T, N>(x, P, F, Q, p.alpha_sq);
        if (EX && p.x_prior) stv<T, N>(p.x_prior + f * N, x);
        if (EX && p.P_prior) stv<T, N * N>(p.P_prior + f * N * N, &P[0][0]);
    }
    if (do_u) {
        const bool has_z = p.valid == nullptr || p.valid[f] != 0;
        if (!has_z) {
            if (EX && p.y) { T zero[M]; for (int a = 0; a < M; a++) zero[a] = T(0); stv<T, M>(p.y + f * M, zero); }
        } else {
            T H[M][N], R[M][M], z[M];
            ldv<T, M * N>(&H[0][0], p.H + f * p.sH);
            ldv<T, M * M>(&R[0][0], p.R + f * p.sR);
            ldv<T, M>(z, p.z + f * M);
            KfUpdateOut<T, N, M> o;
            reg_update<T, N, M>(x, P, H, R, z, o);
            if (!o.ok) st = BKE_STATUS_SINGULAR_S;
            if (EX && p.S) stv<T, M * M>(p.S + f * M * M, &o.S[0][0]);
            if (EX && o.ok) {
                if (p.y) stv<T, M>(p.y + f * M, o.y);
                if (p.SI) stv<T, M * M>(p.SI + f * M * M, &o.SI[0][0]);
                if (p.K) stv<T, N * M>(p.K + f * N * M, &o.K[0][0]);
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
        }
    }
    stv<T, N>(p.x_out + f * N, x);
    stv<T, N * N>(p.P_out + f * N * N, &P[0][0]);
    if (p.status && (st != BKE_STATUS_OK || !(p.flags & BKE_STATUS_STICKY))) p.status[f] = st;
}

template <typename T, int N, int M>
int launch_inst(const bke_kf_args &a, cudaStream_t s)
{
    if (!(vec_ok<T, N>(a.x) && vec_ok<T, N * N>(a.P) && vec_ok<T, N * N>(a.F, a.F_stride) && vec_ok<T, N * N>(a.Q, a.Q_stride) &&
          vec_ok<T, M * N>(a.H, a.H_stride) && vec_ok<T, M * M>(a.R, a.R_stride) && vec_ok<T, M>(a.z) && vec_ok<T, N>(a.x_out) &&
          vec_ok<T, N * N>(a.P_out) && vec_ok<T, N>(a.x_prior) && vec_ok<T, N * N>(a.P_prior) && vec_ok<T, N * M>(a.K) &&
          vec_ok<T, M>(a.y) && vec_ok<T, M * M>(a.S) && vec_ok<T, M * M>(a.SI)))
        return BKE_ERR_UNSUPPORTED;
    DirP<T> p;
    p.N = a.n_filters; p.flags = a.flags; p.alpha_sq = (T)a.alpha_sq;
    p.x = (const T *)a.x; p.P = (const T *)a.P; p.F = (const T *)a.F; p.Q = (const T *)a.Q;
    p.H = (const T *)a.H; p.R = (const T *)a.R; p.z = (const T *)a.z;
    p.sF = a.F_stride; p.sQ = a.Q_stride; p.sH = a.H_stride; p.sR = a.R_stride;
    p.valid = a.z_valid;
    p.x_out = (T *)a.x_out; p.P_out = (T *)a.P_out; p.x_prior = (T *)a.x_prior; p.P_prior = (T *)a.P_prior;
    p.K = (T *)a.K; p.y = (T *)a.y; p.S = (T *)a.S; p.SI = (T *)a.SI; p.ll = (T *)a.log_likelihood;
    p.status = a.status;
    const bool ex = a.x_prior || a.P_prior || a.K || a.y || a.S || a.SI || a.log_likelihood;
    if (ex) kf_direct_kernel<T, N, M, true><<<(unsigned)((p.N + 127) / 128), 128, 0, s>>>(p);
    else kf_direct_kernel<T, N, M, false><<<(unsigned)((p.N + 127) / 128), 128, 0, s>>>(p);
    return check_cuda(cudaGetLastError(), "kf_direct_kernel launch");
}

template <typename T>
int dispatch(const bke_kf_args &a, cudaStream_t s)
{
    if (a.dim_x == 4 && a.dim_z == 2) return launch_inst<T, 4, 2>(a, s);
    if (a.dim_x == 2 && a.dim_z == 1) return launch_inst<T, 2, 1>(a, s);
    if (a.dim_x == 1 && a.dim_z == 1) return launch_inst<T, 1, 1>(a, s);
    if (a.dim_x == 2 && a.dim_z == 2) return launch_inst<T, 2, 2>(a, s);
    if (a.dim_x == 3 && a.dim_z == 1) return launch_inst<T, 3, 1>(a, s);
    if (a.dim_x == 4 && a.dim_z == 1) return launch_inst<T, 4, 1>(a, s);
    if (a.dim_x == 4 && a.dim_z == 4) return launch_inst<T, 4, 4>(a, s);
    if constexpr (sizeof(T) == 4) {      // a 6 x 6 fp64 tile does not fit the register file: row-block kernel
        if (a.dim_x == 6 && a.dim_z == 3) return launch_inst<T, 6, 3>(a, s);
        if (a.dim_x == 6 && a.dim_z == 2) return launch_inst<T, 6, 2>(a, s);
    }
    return BKE_ERR_UNSUPPORTED;
}

}  // namespace

int launch_kf_direct(const bke_kf_args &a, cudaStream_t s)
{
    static const int enabled = [] { const char *e = getenv("BKE_KF_DIRECT"); return e ? atoi(e) : 1; }();
    if (!enabled) return BKE_ERR_UNSUPPORTED;
    if (a.B != nullptr && a.u != nullptr) return BKE_ERR_UNSUPPORTED;
    if (a.flags & BKE_UPDATE_FIRST) return BKE_ERR_UNSUPPORTED;
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

}  // namespace bke
