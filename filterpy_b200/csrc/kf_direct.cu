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
//
// The same kernel, with the update form a template parameter, runs the two other measurement
// updates of the reference class (DESIGN.md §3.10): update_correlated (FORM_CORRELATED, :730-748)
// and the row block of update_sequential (FORM_ROWS, :778-824), where M is the block's row count L
// and the bank's dim_z enters only as the pitch of y, K and the z record.
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
    const T *Mc; int64_t sM;          // FORM_CORRELATED: the cross-correlation M [N,n,m]
    int m, start, rpitch;             // FORM_ROWS: the bank's dim_z, the block's first row, R's row pitch
    T *zrec;                          // FORM_ROWS: the z record [N,m] (H, R, z point at the block)
};

enum { FORM_PLAIN = 0, FORM_CORRELATED = 1, FORM_ROWS = 2 };

// EX: the optional outputs are compiled in (a separate instantiation keeps their tests and live
// ranges out of the plain kernel)
template <typename T, int N, int M, bool EX, int FORM = FORM_PLAIN>
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
    if constexpr (FORM == FORM_ROWS) {
      if (do_u && (p.valid == nullptr || p.valid[f] != 0)) {
        // the block's H_i [L,n] is contiguous; R_i is read with its row pitch (m in the bank's own R)
        T H[M][N], R[M][M], z[M];
#pragma unroll
        for (int e = 0; e < M * N; e++) (&H[0][0])[e] = __ldg(p.H + f * p.sH + e);
#pragma unroll
        for (int a = 0; a < M; a++)
#pragma unroll
            for (int b = 0; b < M; b++) R[a][b] = __ldg(p.R + f * p.sR + a * p.rpitch + b);
#pragma unroll
        for (int a = 0; a < M; a++) z[a] = __ldg(p.z + f * M + a);
        KfUpdateOut<T, N, M> o;
        reg_update<T, N, M, M == 1>(x, P, H, R, z, o);
        if (M > 1 && !o.ok) st = BKE_STATUS_SINGULAR_S;
        else {
            const int64_t row = f * p.m + p.start;
#pragma unroll
            for (int a = 0; a < M; a++) {
                if (p.y) p.y[row + a] = o.y[a];
                if (p.zrec) p.zrec[row + a] = z[a];
#pragma unroll
                for (int i = 0; i < N; i++)
                    if (p.K) p.K[(f * N + i) * p.m + p.start + a] = o.K[i][a];
            }
        }
      }
    } else if (do_u) {
        const bool has_z = p.valid == nullptr || p.valid[f] != 0;
        if (!has_z) {
            if (EX && p.y) { T zero[M]; for (int a = 0; a < M; a++) zero[a] = T(0); stv<T, M>(p.y + f * M, zero); }
        } else {
            T H[M][N], R[M][M], z[M];
            ldv<T, M * N>(&H[0][0], p.H + f * p.sH);
            ldv<T, M * M>(&R[0][0], p.R + f * p.sR);
            ldv<T, M>(z, p.z + f * M);
            KfUpdateOut<T, N, M> o;
            if constexpr (FORM == FORM_CORRELATED) {
                T Mc[N][M];
                ldv<T, N * M>(&Mc[0][0], p.Mc + f * p.sM);
                reg_update_correlated<T, N, M>(x, P, H, R, Mc, z, o);
            } else {
                reg_update<T, N, M>(x, P, H, R, z, o);
            }
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

template <typename T, int N, int M, int FORM = FORM_PLAIN>
int launch_inst(const bke_kf_args &a, cudaStream_t s, const DirP<T> *form = nullptr)
{
    if (!(vec_ok<T, N>(a.x) && vec_ok<T, N * N>(a.P) && vec_ok<T, N * N>(a.F, a.F_stride) && vec_ok<T, N * N>(a.Q, a.Q_stride) &&
          vec_ok<T, M * N>(a.H, a.H_stride) && vec_ok<T, M * M>(a.R, a.R_stride) && vec_ok<T, M>(a.z) && vec_ok<T, N>(a.x_out) &&
          vec_ok<T, N * N>(a.P_out) && vec_ok<T, N>(a.x_prior) && vec_ok<T, N * N>(a.P_prior) && vec_ok<T, N * M>(a.K) &&
          vec_ok<T, M>(a.y) && vec_ok<T, M * M>(a.S) && vec_ok<T, M * M>(a.SI)))
        return BKE_ERR_UNSUPPORTED;
    DirP<T> p = form ? *form : DirP<T>{};
    p.N = a.n_filters; p.flags = a.flags; p.alpha_sq = (T)a.alpha_sq;
    p.x = (const T *)a.x; p.P = (const T *)a.P; p.F = (const T *)a.F; p.Q = (const T *)a.Q;
    p.H = (const T *)a.H; p.R = (const T *)a.R; p.z = (const T *)a.z;
    p.sF = a.F_stride; p.sQ = a.Q_stride; p.sH = a.H_stride; p.sR = a.R_stride;
    p.valid = a.z_valid;
    p.x_out = (T *)a.x_out; p.P_out = (T *)a.P_out; p.x_prior = (T *)a.x_prior; p.P_prior = (T *)a.P_prior;
    p.K = (T *)a.K; p.y = (T *)a.y; p.S = (T *)a.S; p.SI = (T *)a.SI; p.ll = (T *)a.log_likelihood;
    p.status = a.status;
    if constexpr (FORM == FORM_ROWS) { p.H = form->H; p.R = form->R; p.z = form->z; p.K = form->K; p.y = form->y; }
    const bool ex = a.x_prior || a.P_prior || a.K || a.y || a.S || a.SI || a.log_likelihood;
    if (FORM == FORM_ROWS || ex) kf_direct_kernel<T, N, M, true, FORM><<<(unsigned)((p.N + 127) / 128), 128, 0, s>>>(p);
    else kf_direct_kernel<T, N, M, false, FORM><<<(unsigned)((p.N + 127) / 128), 128, 0, s>>>(p);
    return check_cuda(cudaGetLastError(), "kf_direct_kernel launch");
}

// update_correlated: the shapes of dispatch()
template <typename T>
int dispatch_correlated(const bke_kf_args &a, const void *M, int64_t M_stride, cudaStream_t s)
{
    DirP<T> p{};
    p.Mc = (const T *)M; p.sM = M_stride;
    const int n = a.dim_x, m = a.dim_z;
#define BKE_CORR(NN, MM) if (n == NN && m == MM) return vec_ok<T, NN * MM>(M, M_stride) ? \
        launch_inst<T, NN, MM, FORM_CORRELATED>(a, s, &p) : BKE_ERR_UNSUPPORTED;
    BKE_CORR(4, 2) BKE_CORR(2, 1) BKE_CORR(1, 1) BKE_CORR(2, 2) BKE_CORR(3, 1) BKE_CORR(4, 1) BKE_CORR(4, 4)
    if constexpr (sizeof(T) == 4) { BKE_CORR(6, 3) BKE_CORR(6, 2) }
#undef BKE_CORR
    return BKE_ERR_UNSUPPORTED;
}

// a row block of L rows: every (dim_x, L) that dispatch()'s shapes allow, for any dim_z.  `a` carries the
// block (dim_z = L, H and R at the block's first entry, z = z_i); the record's pitch is m.
template <typename T>
int dispatch_rows(const bke_kf_args &a, int m, int start, int rpitch, void *zrec, cudaStream_t s)
{
    DirP<T> p{};
    p.m = m; p.start = start; p.rpitch = rpitch; p.zrec = (T *)zrec;
    // the block's H, R, y, K are not at 16-byte boundaries in general: they are read and written per element
    bke_kf_args b = a;
    b.K = b.y = nullptr; b.H = b.R = nullptr; b.z = nullptr;
    p.H = (const T *)a.H; p.R = (const T *)a.R; p.z = (const T *)a.z; p.K = (T *)a.K; p.y = (T *)a.y;
    const int n = a.dim_x, L = a.dim_z;
#define BKE_ROWS(NN, LL) if (n == NN && L == LL) return launch_inst<T, NN, LL, FORM_ROWS>(b, s, &p);
    BKE_ROWS(1, 1) BKE_ROWS(2, 1) BKE_ROWS(2, 2) BKE_ROWS(3, 1)
    BKE_ROWS(4, 1) BKE_ROWS(4, 2) BKE_ROWS(4, 3) BKE_ROWS(4, 4)
    if constexpr (sizeof(T) == 4) { BKE_ROWS(6, 1) BKE_ROWS(6, 2) BKE_ROWS(6, 3) }
#undef BKE_ROWS
    return BKE_ERR_UNSUPPORTED;
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
    if (a.B != nullptr && a.u != nullptr) return BKE_ERR_UNSUPPORTED;
    if (a.flags & BKE_UPDATE_FIRST) return BKE_ERR_UNSUPPORTED;
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

int launch_kf_direct_correlated(const bke_kf_args &a, const void *M, int64_t M_stride, cudaStream_t s)
{
    if (a.B != nullptr && a.u != nullptr) return BKE_ERR_UNSUPPORTED;
    return a.dtype == BKE_F32 ? dispatch_correlated<float>(a, M, M_stride, s) : dispatch_correlated<double>(a, M, M_stride, s);
}

int launch_kf_direct_rows(const bke_kf_args &a, int m, int start, int rpitch, void *zrec, cudaStream_t s)
{
    if (a.B != nullptr && a.u != nullptr) return BKE_ERR_UNSUPPORTED;
    return a.dtype == BKE_F32 ? dispatch_rows<float>(a, m, start, rpitch, zrec, s)
                              : dispatch_rows<double>(a, m, start, rpitch, zrec, s);
}

}  // namespace bke
