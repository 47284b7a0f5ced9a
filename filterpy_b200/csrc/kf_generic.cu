// kf_generic.cu — linear Kalman filter bank, any (dim_x, dim_z, dim_u), fp32/fp64.
//
// One warp owns one filter at a time.  The filter's matrices live in the warp's private slice of
// shared memory; the 32 lanes split the output elements of every small dense product and
// synchronise with __syncwarp() only (no block barriers, warps are independent).
// This is the catch-all path behind bke_kf_step: the shapes the benchmark configurations use
// have register-tiled specialisations in kf_fast.cu.
//
// Arithmetic follows filterpy/kalman/kalman_filter.py (reference @ 3b51149):
//   predict  :471-478   x = Fx (+Bu);  P = alpha_sq * F P F' + Q
//   update   :515-561   y = z - Hx; S = H P H' + R; SI = inv(S); K = P H' SI; x += K y;
//                       P = (I-KH) P (I-KH)' + K R K'      (Joseph form)
//   z is None:515-520   posterior := prior
// and, with the update form a template parameter (DESIGN.md §3.10):
//   update_correlated  :730-748   S = H P H' + H M + M' H' + R; K = (P H' + M) SI; P = P - K (H P + M')
//   update_sequential  :778-824   the Joseph update of rows start .. start+L-1 (m = L here), K = P H' (1 / S)
//                                 for L = 1; y, K and the z record are written in the block's rows / columns
#include "bke_internal.cuh"
#include "kf_warp.cuh"

namespace bke {
namespace {

template <typename T>
struct KfP {
    int64_t N;
    int n, m, du;
    unsigned flags;
    T alpha_sq;
    const T *x, *P;
    T *x_out, *P_out;
    const T *F, *H, *Q, *R, *B, *u, *z;
    int64_t sF, sH, sQ, sR, sB, su;
    const uint8_t *valid;
    T *x_prior, *P_prior, *K, *y, *S, *SI, *ll;
    int32_t *status;
    int sticky;                       // BKE_STATUS_STICKY: write status only on failure
    const T *Mc; int64_t sM;          // FORM_CORRELATED: the cross-correlation M [N,n,m]
    int mfull, start, rpitch;         // FORM_ROWS: the bank's dim_z, the block's first row, R's row pitch
    T *zrec;                          // FORM_ROWS: the z record [N,mfull]
};

enum { FORM_PLAIN = 0, FORM_CORRELATED = 1, FORM_ROWS = 2 };

template <typename T, int FORM = FORM_PLAIN>
__global__ void __launch_bounds__(128) kf_generic_kernel(KfP<T> p, int per_warp_elems)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const int wpb = blockDim.x >> 5;
    T *w = reinterpret_cast<T *>(smem_raw) + (size_t)wib * per_warp_elems;
    const int n = p.n, m = p.m, nn = n * n, nm = n * m, mm = m * m;
    T *x = w;            T *xp = x + n;
    T *P = xp + n;       T *F = P + nn;
    T *T1 = F + nn;      T *T2 = T1 + nn;
    T *H = T2 + nn;      T *PHT = H + nm;
    T *K = PHT + nm;     T *R = K + nm;
    T *S = R + mm;       T *SI = S + mm;
    T *SA = SI + mm;     T *y = SA + mm;
    T *col = y + m;
    T *Mc = col + m;     // FORM_CORRELATED only: M [n,m] and G = H P + M' [m,n]
    T *G = Mc + nm;

    const bool do_predict = p.flags & BKE_DO_PREDICT;
    const bool do_update = p.flags & BKE_DO_UPDATE;
    const bool update_first = p.flags & BKE_UPDATE_FIRST;

    const int64_t warp_global = (int64_t)blockIdx.x * wpb + wib;
    const int64_t warp_stride = (int64_t)gridDim.x * wpb;

    for (int64_t f = warp_global; f < p.N; f += warp_stride) {
        warp_copy_in(x, p.x + f * n, n, lane);
        warp_copy_in(P, p.P + f * nn, nn, lane);
        int st = BKE_STATUS_OK;
        __syncwarp();

        auto predict = [&]() {
            warp_copy_in(F, p.F + f * p.sF, nn, lane);
            __syncwarp();
            // xp = F x (+ B u)
            for (int i = lane; i < n; i += 32) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += F[i * n + q] * x[q];
                if (p.B != nullptr && p.u != nullptr) {
                    const T *Bf = p.B + f * p.sB, *uf = p.u + f * p.su;
                    T b = T(0);
                    for (int q = 0; q < p.du; q++) b += Bf[i * p.du + q] * uf[q];
                    s += b;
                }
                xp[i] = s;
            }
            warp_mm<false>(F, P, n, n, n, lane, [&](int e, int, int, T s) { T1[e] = s; });
            __syncwarp();
            const T *Qf = p.Q + f * p.sQ;
            warp_mm<true>(T1, F, n, n, n, lane, [&](int e, int, int, T s) { P[e] = p.alpha_sq * s + Qf[e]; });
            for (int i = lane; i < n; i += 32) x[i] = xp[i];
            __syncwarp();
            if (p.x_prior) for (int i = lane; i < n; i += 32) p.x_prior[f * n + i] = x[i];
            if (p.P_prior) for (int e = lane; e < nn; e += 32) p.P_prior[f * nn + e] = P[e];
        };

        // kalman_filter.py:730-748
        auto update_correlated = [&]() {
            if (p.valid != nullptr && p.valid[f] == 0) {   // :705-710 — y = 0, posterior = prior
                if (p.y) for (int a = lane; a < m; a += 32) p.y[f * m + a] = T(0);
                return;
            }
            warp_copy_in(H, p.H + f * p.sH, nm, lane);
            warp_copy_in(R, p.R + f * p.sR, mm, lane);
            warp_copy_in(Mc, p.Mc + f * p.sM, nm, lane);
            __syncwarp();
            for (int a = lane; a < m; a += 32) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += H[a * n + q] * x[q];
                y[a] = p.z[f * m + a] - s;
            }
            warp_mm<true>(P, H, n, n, m, lane, [&](int e, int, int, T s) { PHT[e] = s; });
            __syncwarp();
            // S = H PHT + H M + M' H' + R, with (M' H')[a][b] = (H M)[b][a]
            for (int e = lane; e < mm; e += 32) {
                const int a = e / m, b = e - a * m;
                T s = T(0), hm = T(0), mh = T(0);
                for (int q = 0; q < n; q++) {
                    s += H[a * n + q] * PHT[q * m + b];
                    hm += H[a * n + q] * Mc[q * m + b];
                    mh += H[b * n + q] * Mc[q * m + a];
                }
                S[e] = s + hm + mh + R[e]; SA[e] = S[e];
            }
            __syncwarp();
            if (p.S) for (int e = lane; e < mm; e += 32) p.S[f * mm + e] = S[e];
            T logdet = T(0);
            bool ok = warp_inverse(SA, SI, col, m, lane, logdet);
            if (!ok) { st = BKE_STATUS_SINGULAR_S; return; }
            for (int e = lane; e < nm; e += 32) PHT[e] += Mc[e];
            __syncwarp();
            warp_mm<false>(PHT, SI, n, m, m, lane, [&](int e, int, int, T s) { K[e] = s; });
            __syncwarp();
            for (int i = lane; i < n; i += 32) {
                T s = T(0);
                for (int q = 0; q < m; q++) s += K[i * m + q] * y[q];
                xp[i] = x[i] + s;
            }
            warp_mm<false>(H, P, m, n, n, lane, [&](int e, int a, int j, T s) { G[e] = s + Mc[j * m + a]; });
            __syncwarp();
            for (int i = lane; i < n; i += 32) x[i] = xp[i];
            warp_mm<false>(K, G, n, m, n, lane, [&](int e, int, int, T s) { F[e] = P[e] - s; });
            __syncwarp();
            for (int e = lane; e < nn; e += 32) P[e] = F[e];
            if (p.K) for (int e = lane; e < nm; e += 32) p.K[f * nm + e] = K[e];
            if (p.y) for (int a = lane; a < m; a += 32) p.y[f * m + a] = y[a];
            if (p.SI) for (int e = lane; e < mm; e += 32) p.SI[f * mm + e] = SI[e];
            if (p.ll && lane == 0) {
                T q = T(0);
                for (int a = 0; a < m; a++) {
                    T s = T(0);
                    for (int b = 0; b < m; b++) s += SI[a * m + b] * y[b];
                    q += y[a] * s;
                }
                p.ll[f] = T(-0.5) * (q + logdet + T(m) * T(LOG_2PI));
            }
            __syncwarp();
        };

        auto update = [&]() {
            const bool has_z = (p.valid == nullptr) || (p.valid[f] != 0);
            if (!has_z) {   // kalman_filter.py:515-520 — y = 0, posterior = prior
                if (FORM != FORM_ROWS && p.y) for (int a = lane; a < m; a += 32) p.y[f * m + a] = T(0);
                return;
            }
            warp_copy_in(H, p.H + f * p.sH, nm, lane);
            if constexpr (FORM == FORM_ROWS) {
                for (int e = lane; e < mm; e += 32) R[e] = p.R[f * p.sR + (e / m) * p.rpitch + e % m];
            } else {
                warp_copy_in(R, p.R + f * p.sR, mm, lane);
            }
            __syncwarp();
            for (int a = lane; a < m; a += 32) {
                T s = T(0);
                for (int q = 0; q < n; q++) s += H[a * n + q] * x[q];
                y[a] = p.z[f * m + a] - s;
            }
            warp_mm<true>(P, H, n, n, m, lane, [&](int e, int, int, T s) { PHT[e] = s; });
            __syncwarp();
            warp_mm<false>(H, PHT, m, n, m, lane, [&](int e, int, int, T s) { S[e] = s + R[e]; SA[e] = s + R[e]; });
            __syncwarp();
            if (p.S) for (int e = lane; e < mm; e += 32) p.S[f * mm + e] = S[e];
            T logdet = T(0);
            if (FORM == FORM_ROWS && m == 1) {
                if (lane == 0) SI[0] = T(1) / SA[0];                 // PH' (1 / S): inf for S = 0, no LinAlgError
                __syncwarp();
            } else {
                bool ok = warp_inverse(SA, SI, col, m, lane, logdet);   // SA = scratch copy of S
                if (!ok) { st = BKE_STATUS_SINGULAR_S; return; }
            }
            warp_mm<false>(PHT, SI, n, m, m, lane, [&](int e, int, int, T s) { K[e] = s; });
            __syncwarp();
            for (int i = lane; i < n; i += 32) {
                T s = T(0);
                for (int q = 0; q < m; q++) s += K[i * m + q] * y[q];
                xp[i] = x[i] + s;
            }
            // T1 = I - K H
            warp_mm<false>(K, H, n, m, n, lane, [&](int e, int i, int j, T s) { T1[e] = (i == j ? T(1) : T(0)) - s; });
            __syncwarp();
            for (int i = lane; i < n; i += 32) x[i] = xp[i];
            // T2 = T1 P ;  PHT <- K R
            warp_mm<false>(T1, P, n, n, n, lane, [&](int e, int, int, T s) { T2[e] = s; });
            warp_mm<false>(K, R, n, m, m, lane, [&](int e, int, int, T s) { PHT[e] = s; });
            __syncwarp();
            // P = T2 T1' + (K R) K'
            for (int e = lane; e < nn; e += 32) {
                int i = e / n, j = e - i * n;
                T s1 = T(0), s2 = T(0);
                for (int q = 0; q < n; q++) s1 += T2[i * n + q] * T1[j * n + q];
                for (int q = 0; q < m; q++) s2 += PHT[i * m + q] * K[j * m + q];
                F[e] = s1 + s2;                 // F is free: use it as the staging buffer
            }
            __syncwarp();
            for (int e = lane; e < nn; e += 32) P[e] = F[e];
            if constexpr (FORM == FORM_ROWS) {
                const int M = p.mfull;
                if (p.K) for (int e = lane; e < nm; e += 32) p.K[(f * n + e / m) * M + p.start + e % m] = K[e];
                for (int a = lane; a < m; a += 32) {
                    if (p.y) p.y[f * M + p.start + a] = y[a];
                    if (p.zrec) p.zrec[f * M + p.start + a] = p.z[f * m + a];
                }
                __syncwarp();
                return;
            }
            if (p.K) for (int e = lane; e < nm; e += 32) p.K[f * nm + e] = K[e];
            if (p.y) for (int a = lane; a < m; a += 32) p.y[f * m + a] = y[a];
            if (p.SI) for (int e = lane; e < mm; e += 32) p.SI[f * mm + e] = SI[e];
            if (p.ll && lane == 0) {
                T q = T(0);
                for (int a = 0; a < m; a++) {
                    T s = T(0);
                    for (int b = 0; b < m; b++) s += SI[a * m + b] * y[b];
                    q += y[a] * s;
                }
                p.ll[f] = T(-0.5) * (q + logdet + T(m) * T(LOG_2PI));
            }
            __syncwarp();
        };

        auto run_update = [&]() {
            if constexpr (FORM == FORM_CORRELATED) update_correlated();
            else update();
        };
        if (update_first) {
            if (do_update) run_update();
            __syncwarp();
            if (do_predict) predict();
        } else {
            if (do_predict) predict();
            __syncwarp();
            if (do_update) run_update();
        }
        __syncwarp();
        for (int i = lane; i < n; i += 32) p.x_out[f * n + i] = x[i];
        for (int e = lane; e < nn; e += 32) p.P_out[f * nn + e] = P[e];
        if (p.status && lane == 0 && (st != BKE_STATUS_OK || !p.sticky)) p.status[f] = st;
        __syncwarp();
    }
}

template <typename T, int FORM = FORM_PLAIN>
int launch_t(const bke_kf_args &a, cudaStream_t s, const KfP<T> *form = nullptr)
{
    KfP<T> p = form ? *form : KfP<T>{};
    p.N = a.n_filters; p.n = a.dim_x; p.m = a.dim_z; p.du = a.dim_u; p.flags = a.flags;
    p.alpha_sq = (T)a.alpha_sq;
    p.x = (const T *)a.x; p.P = (const T *)a.P; p.x_out = (T *)a.x_out; p.P_out = (T *)a.P_out;
    p.F = (const T *)a.F; p.H = (const T *)a.H; p.Q = (const T *)a.Q; p.R = (const T *)a.R;
    p.B = (const T *)a.B; p.u = (const T *)a.u; p.z = (const T *)a.z;
    p.sF = a.F_stride; p.sH = a.H_stride; p.sQ = a.Q_stride; p.sR = a.R_stride; p.sB = a.B_stride; p.su = a.u_stride;
    p.valid = a.z_valid;
    p.x_prior = (T *)a.x_prior; p.P_prior = (T *)a.P_prior; p.K = (T *)a.K; p.y = (T *)a.y;
    p.S = (T *)a.S; p.SI = (T *)a.SI; p.ll = (T *)a.log_likelihood; p.status = a.status;
    p.sticky = (a.flags & BKE_STATUS_STICKY) ? 1 : 0;

    const int n = p.n, m = p.m;
    // layout must match the kernel: x, xp, P, F, T1, T2, H, PHT, K, R, S, SI, SA, y, col (, Mc, G)
    int per_warp = 2 * n + 4 * (n * n) + 3 * (n * m) + 4 * (m * m) + 2 * m + (FORM == FORM_CORRELATED ? 2 * n * m : 0);
    per_warp = (per_warp + 3) & ~3;
    const size_t bytes_per_warp = (size_t)per_warp * sizeof(T), budget = 200 * 1024;
    WarpShape w;
    if (int rc = warp_shape((const void *)kf_generic_kernel<T, FORM>, bytes_per_warp, budget, p.N, w)) {
        // named after the entry point that made the call (a row block's m is its row count)
        const char *entry = FORM == FORM_CORRELATED ? "bke_kf_step_correlated"
                          : FORM == FORM_ROWS       ? "bke_kf_update_rows" : "bke_kf_step";
        if (rc == BKE_ERR_UNSUPPORTED)
            set_error("%s: dim_x=%d %s=%d needs %zu B of shared memory per filter (> %zu)", entry, n,
                      FORM == FORM_ROWS ? "rows" : "dim_z", m, bytes_per_warp, budget);
        return rc;
    }
    kf_generic_kernel<T, FORM><<<w.grid, w.wpb * 32, w.smem, s>>>(p, per_warp);
    return check_cuda(cudaGetLastError(), "kf_generic_kernel launch");
}

}  // namespace

int launch_kf_generic(const bke_kf_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? launch_t<float>(a, s) : launch_t<double>(a, s);
}

template <typename T>
static int correlated_t(const bke_kf_args &a, const void *M, int64_t M_stride, cudaStream_t s)
{
    KfP<T> p{};
    p.Mc = (const T *)M; p.sM = M_stride;
    return launch_t<T, FORM_CORRELATED>(a, s, &p);
}

int launch_kf_generic_correlated(const bke_kf_args &a, const void *M, int64_t M_stride, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? correlated_t<float>(a, M, M_stride, s) : correlated_t<double>(a, M, M_stride, s);
}

template <typename T>
static int rows_t(const bke_kf_args &a, int m, int start, int rpitch, void *zrec, cudaStream_t s)
{
    KfP<T> p{};
    p.mfull = m; p.start = start; p.rpitch = rpitch; p.zrec = (T *)zrec;
    return launch_t<T, FORM_ROWS>(a, s, &p);
}

int launch_kf_generic_rows(const bke_kf_args &a, int m, int start, int rpitch, void *zrec, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? rows_t<float>(a, m, start, rpitch, zrec, s) : rows_t<double>(a, m, start, rpitch, zrec, s);
}

}  // namespace bke
