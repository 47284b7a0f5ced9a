// api.cu — the extern "C" boundary declared in include/bke.h: argument validation, error
// text, dispatch to the sm_90a kernels.  No torch types, no allocation, no host sync.
#include <stdarg.h>
#include <string.h>
#include "bke_internal.cuh"

namespace bke {

static thread_local char g_err[8192] = "";     // room for an NVRTC log (bke_ukf_model_compile)

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_cuda(cudaError_t e, const char *what)
{
    if (e == cudaSuccess) return BKE_OK;
    set_error("%s: %s", what, cudaGetErrorString(e));
    return BKE_ERR_CUDA;
}

int launch_kernel(const void *kern, unsigned grid, unsigned block, size_t smem, void *params, cudaStream_t s, const char *what)
{
    if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
    void *args[] = {params};
    return check_cuda(cudaLaunchKernel(kern, dim3(grid), dim3(block), args, smem, s), what);
}

int sm_count()
{
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (cached[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

int warp_shape(const void *kern, size_t bytes_per_warp, size_t budget, int64_t items, WarpShape &w)
{
    int wpb = 4;
    while (wpb > 1 && bytes_per_warp * wpb > budget) wpb >>= 1;
    if (bytes_per_warp * wpb > budget) return BKE_ERR_UNSUPPORTED;
    const size_t smem = bytes_per_warp * wpb;
    if (smem > 48 * 1024 &&
        check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute"))
        return BKE_ERR_CUDA;
    const int64_t want = (items + wpb - 1) / wpb, cap = (int64_t)sm_count() * 16;
    w = {wpb, smem, (int)(want < cap ? (want > 0 ? want : 1) : cap)};
    return BKE_OK;
}

int require_device()
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        set_error("no CUDA device available (%s); the engine has no CPU fallback",
                  e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
        return BKE_ERR_CUDA;
    }
    return BKE_OK;
}

int check_dtype(int32_t dtype)
{
    if (dtype != BKE_F32 && dtype != BKE_F64) { set_error("dtype must be BKE_F32 or BKE_F64"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int check_bank(int64_t n, int64_t dim_x, int64_t dim_z, int64_t dim_u)
{
    const char *why = n < 0 ? "n_filters < 0" : dim_x < 1 ? "dim_x must be 1 or greater" : dim_z < 1 ? "dim_z must be 1 or greater"
                    : dim_u < 0 ? "dim_u must be 0 or greater" : nullptr;
    if (!why) return BKE_OK;
    set_error("bad dimensions: %s", why);
    return BKE_ERR_BAD_ARG;
}

int check_predict_update(uint32_t flags)
{
    if (!(flags & (BKE_DO_PREDICT | BKE_DO_UPDATE))) { set_error("flags selects neither predict nor update"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int check_flag_bits(uint32_t flags, uint32_t allowed)
{
    if (!(flags & ~allowed)) return BKE_OK;
    set_error("flags may only hold the bits this call takes, here only%s%s%s%s", allowed & BKE_DO_PREDICT ? " BKE_DO_PREDICT" : "",
              allowed & BKE_DO_UPDATE ? " BKE_DO_UPDATE" : "", allowed & BKE_STATUS_STICKY ? " BKE_STATUS_STICKY" : "",
              allowed & BKE_REVERSE_TILES ? " BKE_REVERSE_TILES" : "");
    return BKE_ERR_BAD_ARG;
}

int check_strides(std::initializer_list<std::pair<int64_t, int64_t>> strides)
{
    for (const auto &s : strides)
        if (s.first != 0 && s.first != s.second) { set_error("model strides must be 0 (shared) or the dense per-filter size"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int check_control(const void *B, const void *u, int64_t dim_u)
{
    if ((B || u) && (!B || !u || dim_u < 1)) { set_error("a control input needs B, u and dim_u >= 1"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

static int validate_kf(const bke_kf_args &a, bool need_z)
{
    int rc;
    if ((rc = check_bank(a.n_filters, a.dim_x, a.dim_z, a.dim_u)) || (rc = check_dtype(a.dtype)) || (rc = check_predict_update(a.flags)))
        return rc;                                                       // kalman_filter.py:388-392
    if (!a.x || !a.P || !a.x_out || !a.P_out) { set_error("x, P, x_out, P_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_PREDICT) && (!a.F || !a.Q)) { set_error("predict needs F and Q"); return BKE_ERR_BAD_ARG; }
    if (a.flags & BKE_DO_UPDATE) {
        if (!a.H || !a.R) { set_error("update needs H and R"); return BKE_ERR_BAD_ARG; }
        if (need_z && !a.z) { set_error("update needs z"); return BKE_ERR_BAD_ARG; }
    }
    const int64_t n = a.dim_x, m = a.dim_z;
    return check_strides({{a.F_stride, n * n}, {a.Q_stride, n * n}, {a.H_stride, m * n}, {a.R_stride, m * m}});
}

static int validate_srkf(const bke_srkf_args &a)
{
    int rc;
    if ((rc = check_bank(a.n_filters, a.dim_x, a.dim_z, a.dim_u)) || (rc = check_dtype(a.dtype)) || (rc = check_predict_update(a.flags)) ||
        (rc = check_flag_bits(a.flags, BKE_DO_PREDICT | BKE_DO_UPDATE)))
        return rc;                                                       // square_root.py:128-133
    if (!a.x || !a.L || !a.x_out || !a.L_out) { set_error("x, L, x_out, L_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_PREDICT) && (!a.F || !a.Lq)) { set_error("predict needs F and Lq"); return BKE_ERR_BAD_ARG; }   // square_root.py:240-243
    if ((a.flags & BKE_DO_UPDATE) && (!a.H || !a.Lr || !a.z)) { set_error("update needs H, Lr and z"); return BKE_ERR_BAD_ARG; }   // :204-215
    if ((rc = check_control(a.B, a.u, a.dim_u))) return rc;                                           // :240
    const int64_t n = a.dim_x, m = a.dim_z, du = a.dim_u;
    return check_strides({{a.F_stride, n * n}, {a.Lq_stride, n * n}, {a.H_stride, m * n}, {a.Lr_stride, m * m}, {a.B_stride, n * du},
                          {a.u_stride, du}});
}

// the checks of bke_if_step
static int validate_if(const bke_if_args &a)
{
    int rc;
    if ((rc = check_bank(a.n_filters, a.dim_x, a.dim_z, a.dim_u)) || (rc = check_dtype(a.dtype)) || (rc = check_predict_update(a.flags)) ||
        (rc = check_flag_bits(a.flags, BKE_DO_PREDICT | BKE_DO_UPDATE | BKE_STATUS_STICKY)))
        return rc;                                                       // information_filter.py:132-137
    if (!a.x || !a.P_inv || !a.x_out || !a.P_inv_out) { set_error("x, P_inv, x_out, P_inv_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (!a.no_information) { set_error("no_information must be non-NULL (the per-filter flag is read and written)"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_PREDICT) && (!a.F || !a.F_inv || !a.Q)) { set_error("predict needs F, F_inv and Q"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_UPDATE) && (!a.H || !a.R_inv || !a.z)) { set_error("update needs H, R_inv and z"); return BKE_ERR_BAD_ARG; }
    if ((rc = check_control(a.B, a.u, a.dim_u))) return rc;                                           // information_filter.py:274
    const int64_t n = a.dim_x, m = a.dim_z, du = a.dim_u;
    if ((rc = check_strides({{a.F_stride, n * n}, {a.F_inv_stride, n * n}, {a.Q_stride, n * n}, {a.H_stride, m * n},
                             {a.R_inv_stride, m * m}, {a.B_stride, n * du}, {a.u_stride, du}})))
        return rc;
    if (a.ll_mode != BKE_IF_LL_NONE && a.ll_mode != BKE_IF_LL_FULL && a.ll_mode != BKE_IF_LL_BROADCAST) {
        set_error("ll_mode must be BKE_IF_LL_NONE, BKE_IF_LL_FULL or BKE_IF_LL_BROADCAST");
        return BKE_ERR_BAD_ARG;
    }
    if ((a.ll_mode == BKE_IF_LL_FULL && m != n) || (a.ll_mode == BKE_IF_LL_BROADCAST && m != 1)) {
        set_error("ll_mode %s needs %s", a.ll_mode == BKE_IF_LL_FULL ? "BKE_IF_LL_FULL" : "BKE_IF_LL_BROADCAST",
                  a.ll_mode == BKE_IF_LL_FULL ? "dim_z == dim_x" : "dim_z == 1");
        return BKE_ERR_BAD_ARG;
    }
    if (a.ll_mode != BKE_IF_LL_NONE && !a.log_likelihood) { set_error("ll_mode needs log_likelihood"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

// the checks of bke_poly_filter
static int validate_poly(const bke_poly_args &a)
{
    int rc;
    if ((rc = check_bank(a.n_filters))) return rc;
    if (a.n_steps < 1) { set_error("n_steps must be 1 or greater"); return BKE_ERR_BAD_ARG; }
    if ((rc = check_dtype(a.dtype))) return rc;
    const int fam = a.family;
    if (fam < BKE_POLY_GH || fam > BKE_POLY_FADING) { set_error("family must be one of BKE_POLY_*"); return BKE_ERR_BAD_ARG; }
    const bool gh = fam == BKE_POLY_GH || fam == BKE_POLY_GHK;
    if (!gh && (a.order < 0 || a.order > 2)) { set_error("order must be between 0 and 2"); return BKE_ERR_BAD_ARG; }
    if (a.mode != BKE_POLY_UPDATE && a.mode != BKE_POLY_BATCH) { set_error("mode must be BKE_POLY_UPDATE or BKE_POLY_BATCH"); return BKE_ERR_BAD_ARG; }
    const bool batch = a.mode == BKE_POLY_BATCH;
    const int ord = fam == BKE_POLY_GH ? 1 : fam == BKE_POLY_GHK ? 2 : a.order;
    if (a.n_filters == 0) return BKE_OK;
    // what the instance reads
    const bool need_dx = gh, need_ddx = fam == BKE_POLY_GHK && !batch;
    const bool need_g = fam != BKE_POLY_LSQ;
    const bool need_h = gh || (ord >= 1 && fam != BKE_POLY_LSQ);
    const bool need_k = (fam == BKE_POLY_GHK && !batch) || (ord == 2 && (fam == BKE_POLY_GH_ORDER || fam == BKE_POLY_FADING));
    const bool need_dt = ord >= 1;
    const bool need_dt2 = (fam == BKE_POLY_GHK && !batch) || (!gh && ord == 2);
    const bool need_hdt2 = fam == BKE_POLY_LSQ && ord == 2;
    if (!a.x || !a.z || (need_dx && !a.dx) || (need_ddx && !a.ddx)) { set_error("the state and z must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((need_g && !a.g) || (need_h && !a.h) || (need_k && !a.k) || (need_dt && !a.dt) || (need_dt2 && !a.dt2) ||
        (need_hdt2 && !a.hdt2)) {
        set_error("a parameter this family and order read is NULL");
        return BKE_ERR_BAD_ARG;
    }
    // a parameter per filter is one element; the stride of an absent one is not read
    if ((rc = check_strides({{a.g ? a.g_stride : 0, 1}, {a.h ? a.h_stride : 0, 1}, {a.k ? a.k_stride : 0, 1},
                             {a.dt ? a.dt_stride : 0, 1}, {a.dt2 ? a.dt2_stride : 0, 1}, {a.hdt2 ? a.hdt2_stride : 0, 1}})))
        return rc;
    // the outputs each family and mode have
    if (a.predictions && !(gh && batch)) { set_error("predictions is an output of the GH / GHK batch_filter only"); return BKE_ERR_BAD_ARG; }
    if (a.y && (batch || fam == BKE_POLY_LSQ || fam == BKE_POLY_FADING)) {
        set_error("y is an output of the GH, GHK and GH_ORDER update only");      // least_squares.py:128 never stores y
        return BKE_ERR_BAD_ARG;
    }
    if ((a.x_prediction || a.dx_prediction) && !(gh && !batch)) { set_error("x_prediction / dx_prediction are outputs of the GH / GHK update only"); return BKE_ERR_BAD_ARG; }
    if (a.ddx_prediction && !(fam == BKE_POLY_GHK && !batch)) { set_error("ddx_prediction is an output of the GHK update only"); return BKE_ERR_BAD_ARG; }
    if (a.K && !(fam == BKE_POLY_LSQ && !batch)) { set_error("K is an output of the LSQ update only"); return BKE_ERR_BAD_ARG; }
    if (fam == BKE_POLY_LSQ) {
        if (!a.n) { set_error("LSQ needs the counter n"); return BKE_ERR_BAD_ARG; }
        // the largest counter the call reaches, and the product of it the order's gains form (least_squares.py:131-145)
        int64_t top, p;
        if (a.n_max < 0 || __builtin_add_overflow(a.n_max, a.n_steps, &top) ||
            (ord >= 1 && __builtin_mul_overflow(top, top + 1, &p)) ||
            (ord == 2 && (__builtin_mul_overflow(p, top + 2, &p) || __builtin_mul_overflow(top, 3 * top, &p)))) {
            set_error("the LSQ counter n_max + n_steps overflows int64 in n(n+1)(n+2) (or the product its order forms)");
            return BKE_ERR_BAD_ARG;
        }
    }
    return BKE_OK;
}

// the checks of bke_imm_batch_filter; -1 = go
static int validate_imm(const bke_imm_batch_args *a)
{
    if (!a) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    int rc;
    if ((rc = check_bank(a->n_tracks, a->dim_x, a->dim_z))) return rc;
    if (a->n_steps < 0) { set_error("n_steps < 0"); return BKE_ERR_BAD_ARG; }
    if ((rc = check_dtype(a->dtype))) return rc;
    if (a->n_models < 2 || a->n_models > BKE_MM_MAX_MODELS) { set_error("n_models must be in [2, %d]", BKE_MM_MAX_MODELS); return BKE_ERR_BAD_ARG; }
    if ((rc = check_flag_bits(a->flags, BKE_STATUS_STICKY))) return rc;
    const int M = a->n_models;
    const int64_t N = a->n_tracks, T = a->n_steps, n = a->dim_x, m = a->dim_z;
    for (int j = 0; j < M; j++)
        if ((rc = check_strides({{a->F_stride[j], n * n}, {a->Q_stride[j], n * n}, {a->H_stride[j], m * n}, {a->R_stride[j], m * m}})))
            return rc;
    if (N == 0 || T == 0) return BKE_OK;
    for (int j = 0; j < M; j++) {
        if (!a->x[j] || !a->P[j] || !a->F[j] || !a->Q[j] || !a->H[j] || !a->R[j] || !a->S[j] || !a->log_likelihood[j] ||
            !a->K[j] || !a->y[j] || !a->SI[j] || !a->x_prior[j] || !a->P_prior[j] || !a->status[j]) {
            set_error("model %d: an array the call reads or writes is NULL", j);
            return BKE_ERR_BAD_ARG;
        }
    }
    if (!a->mu || !a->cbar || !a->omega || !a->trans || !a->zs || !a->means || !a->covariances || !a->means_p ||
        !a->covariances_p || !a->mus) {
        set_error("mu, cbar, omega, trans, zs and the five outputs must be non-NULL");
        return BKE_ERR_BAD_ARG;
    }
    // every array the call writes must be clear of every other array it touches
    struct Span { const void *p; int64_t bytes; bool written; };
    const int64_t es = a->dtype == BKE_F32 ? 4 : 8;
    Span sp[14 * BKE_MM_MAX_MODELS + 11];      // 14 arrays per model, 11 shared (zs_valid among them)
    int ns = 0;
    auto add = [&](const void *p, int64_t elems, bool written) { sp[ns++] = Span{p, elems, written}; };
    for (int j = 0; j < M; j++) {
        add(a->x[j], N * n * es, true); add(a->P[j], N * n * n * es, true);
        add(a->F[j], (a->F_stride[j] ? N : 1) * n * n * es, false); add(a->Q[j], (a->Q_stride[j] ? N : 1) * n * n * es, false);
        add(a->H[j], (a->H_stride[j] ? N : 1) * m * n * es, false); add(a->R[j], (a->R_stride[j] ? N : 1) * m * m * es, false);
        add(a->S[j], N * m * m * es, true); add(a->log_likelihood[j], N * es, true); add(a->K[j], N * n * m * es, true);
        add(a->y[j], N * m * es, true); add(a->SI[j], N * m * m * es, true); add(a->x_prior[j], N * n * es, true);
        add(a->P_prior[j], N * n * n * es, true); add(a->status[j], N * 4, true);
    }
    add(a->mu, N * M * 8, true); add(a->cbar, N * M * 8, true); add(a->omega, N * M * M * 8, true);
    add(a->trans, (int64_t)M * M * 8, false); add(a->zs, T * N * m * es, false);
    if (a->zs_valid) add(a->zs_valid, T * N, false);
    add(a->means, T * N * n * es, true); add(a->covariances, T * N * n * n * es, true);
    add(a->means_p, T * N * n * es, true); add(a->covariances_p, T * N * n * n * es, true);
    add(a->mus, T * N * M * 8, true);
    for (int i = 0; i < ns; i++) {
        for (int k = i + 1; k < ns; k++) {
            if (!sp[i].written && !sp[k].written) continue;
            const uintptr_t p0 = (uintptr_t)sp[i].p, p1 = (uintptr_t)sp[k].p;
            if (p0 < p1 + (uintptr_t)sp[k].bytes && p1 < p0 + (uintptr_t)sp[i].bytes) {
                set_error("an array bke_imm_batch_filter writes overlaps another of its arrays");
                return BKE_ERR_BAD_ARG;
            }
        }
    }
    if (!imm_batch_has_instance(a->dim_x, a->dim_z, a->dtype)) {
        set_error("bke_imm_batch_filter: no fused instance for dim_x=%d, dim_z=%d in this dtype", a->dim_x, a->dim_z);
        return BKE_ERR_UNSUPPORTED;
    }
    auto al16 = [](const void *p) { return ((uintptr_t)p & 15u) == 0; };
    bool al = al16(a->means) && al16(a->covariances) && al16(a->means_p) && al16(a->covariances_p);
    for (int j = 0; j < M; j++)
        al = al && al16(a->x[j]) && al16(a->P[j]) && al16(a->S[j]) && al16(a->log_likelihood[j]) && al16(a->K[j]) &&
             al16(a->y[j]) && al16(a->SI[j]) && al16(a->x_prior[j]) && al16(a->P_prior[j]);
    if (!al) { set_error("bke_imm_batch_filter: the state, diagnostic and output arrays must be 16-byte aligned"); return BKE_ERR_UNSUPPORTED; }
    return -1;
}

template <typename Args>
static int check_candidates(const Args &a, int64_t N, int64_t m);

// the checks of bke_score_measurements
static int validate_score(const bke_score_args &a)
{
    if (a.n_tracks < 0 || a.n_candidates < 0) { set_error("n_tracks and n_candidates must be 0 or greater"); return BKE_ERR_BAD_ARG; }
    if (int rc = check_dtype(a.dtype)) return rc;
    const bool uses_n = a.x || a.P;
    if (a.dim_z < 1 || a.dim_z > 1024 || (uses_n && (a.dim_x < 1 || a.dim_x > 1024))) {
        set_error("dim_z (and dim_x, when x or P is given) must be between 1 and 1024");
        return BKE_ERR_BAD_ARG;
    }
    const int64_t n = a.dim_x, m = a.dim_z;
    if (!a.x == !a.mean) { set_error("exactly one of x and mean must be given"); return BKE_ERR_BAD_ARG; }
    if (a.P && a.S) { set_error("at most one of P and S may be given"); return BKE_ERR_BAD_ARG; }
    if (a.H && !uses_n) { set_error("H maps x or P: it is read only with one of them"); return BKE_ERR_BAD_ARG; }
    if (uses_n && !a.H && n != m) { set_error("without H (the identity) dim_x must equal dim_z"); return BKE_ERR_BAD_ARG; }
    if (a.P && !a.R) { set_error("S = H P H' + R needs R"); return BKE_ERR_BAD_ARG; }
    if (a.R && !a.P) { set_error("R is read only with P"); return BKE_ERR_BAD_ARG; }
    if (int rc = check_strides({{a.H ? a.H_stride : 0, m * n}, {a.R ? a.R_stride : 0, m * m}, {a.S ? a.S_stride : 0, m * m}})) return rc;
    const bool scores = a.d2 || a.mahalanobis || a.log_likelihood || a.likelihood;
    if (!(a.zhat || a.y || scores || a.status)) { set_error("no output is requested"); return BKE_ERR_BAD_ARG; }
    if ((scores || a.status) && !a.P && !a.S) { set_error("the scores and status need a covariance: P or S"); return BKE_ERR_BAD_ARG; }
    return check_candidates(a, a.n_tracks, m);
}

// the candidates and outputs of the measurement scores (bke_score_args and bke_ukf_score_args alike)
template <typename Args>
static int check_candidates(const Args &a, int64_t N, int64_t m)
{
    const bool scores = a.d2 || a.mahalanobis || a.log_likelihood || a.likelihood;
    if ((a.y || scores) && !a.z) { set_error("y and the scores need z"); return BKE_ERR_BAD_ARG; }
    if (a.z_track_stride < 0 || a.z_cand_stride < 0) { set_error("z strides must be 0 or greater"); return BKE_ERR_BAD_ARG; }
    // every offset the kernel forms fits int64: pair * m, and z's last element
    int64_t pairs, t, u, last;
    if (__builtin_mul_overflow(N, a.n_candidates, &pairs) || __builtin_mul_overflow(pairs, m, &t) ||
        (N > 0 && __builtin_mul_overflow(N - 1, a.z_track_stride, &t)) ||
        (a.n_candidates > 0 && __builtin_mul_overflow(a.n_candidates - 1, a.z_cand_stride, &u)) ||
        (N > 0 && a.n_candidates > 0 && __builtin_add_overflow(t, u, &last)) ||
        (N > 0 && a.n_candidates > 0 && __builtin_add_overflow(last, m, &last))) {
        set_error("N * K * dim_z or the z offsets overflow int64");
        return BKE_ERR_BAD_ARG;
    }
    return BKE_OK;
}

// bke_ukf_score and bke_ukf_score_model: the bank as a UKF step reads it, then the candidates as the linear scores
int validate_ukf_score(const bke_ukf_score_args &a)
{
    int rc;
    if (a.n_candidates < 0) { set_error("n_candidates must be 0 or greater"); return BKE_ERR_BAD_ARG; }
    if ((rc = check_bank(a.n_filters, a.dim_x, a.dim_z)) || (rc = check_dtype(a.dtype))) return rc;
    if (a.flags & ~BKE_UKF_SIMPLEX) { set_error("flags must be 0 or BKE_UKF_SIMPLEX"); return BKE_ERR_BAD_ARG; }
    if (!a.x || !a.P || !a.R) { set_error("x, P and R must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model == BKE_HX_LINEAR && !a.H) { set_error("BKE_HX_LINEAR needs H"); return BKE_ERR_BAD_ARG; }
    const int64_t n = a.dim_x, m = a.dim_z;
    if ((rc = check_strides({{a.R_stride, m * m}, {a.hx_model == BKE_HX_LINEAR ? a.H_stride : 0, m * n}}))) return rc;
    const double lam_n = a.alpha * a.alpha * (a.dim_x + a.kappa);
    if (!(a.flags & BKE_UKF_SIMPLEX) && !(lam_n != 0.0)) { set_error("alpha^2 (n + kappa) must be non-zero"); return BKE_ERR_BAD_ARG; }
    if (!(a.zhat || a.y || a.d2 || a.mahalanobis || a.log_likelihood || a.likelihood || a.status)) {
        set_error("no output is requested");
        return BKE_ERR_BAD_ARG;
    }
    return check_candidates(a, a.n_filters, m);
}

// the checks every sigma-point step (UKF, CKF, EnKF; pre-built and run-time compiled) makes
template <typename Args>
static int validate_sigma(const Args &a)
{
    int rc;
    if ((rc = check_dtype(a.dtype)) || (rc = check_predict_update(a.flags))) return rc;
    if (!a.x || !a.P || !a.x_out || !a.P_out) { set_error("x, P, x_out, P_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_PREDICT) && !a.Q) { set_error("predict needs Q"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_UPDATE) && (!a.R || !a.z)) { set_error("update needs R and z"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model == BKE_FX_LINEAR && (a.flags & BKE_DO_PREDICT) && !a.F) { set_error("BKE_FX_LINEAR needs F"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model == BKE_HX_LINEAR && (a.flags & BKE_DO_UPDATE) && !a.H) { set_error("BKE_HX_LINEAR needs H"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model == BKE_FX_CONST_VEL && (a.dim_x & 1)) { set_error("BKE_FX_CONST_VEL needs an even dim_x"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

// bke_ukf_step and bke_ukf_step_model (where the dimension and dtype checks cannot fail: the args matched
// a compiled model)
int validate_ukf(const bke_ukf_args &a)
{
    int rc;
    if ((rc = check_bank(a.n_filters, a.dim_x, a.dim_z)) || (rc = validate_sigma(a))) return rc;
    const double lam_n = a.alpha * a.alpha * (a.dim_x + a.kappa);
    if (!(a.flags & BKE_UKF_SIMPLEX) && !(lam_n != 0.0)) { set_error("alpha^2 (n + kappa) must be non-zero"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int validate_ckf(const bke_ckf_args &a)
{
    int rc;
    if ((rc = check_bank(a.n_filters, a.dim_x, a.dim_z)) || (rc = validate_sigma(a))) return rc;
    if ((a.flags & BKE_DO_UPDATE) && !(a.flags & BKE_DO_PREDICT) && !a.sigmas_f) {
        set_error("an update without predict reads the propagated points of the last predict: sigmas_f must be non-NULL");
        return BKE_ERR_BAD_ARG;
    }
    return BKE_OK;
}

int validate_enkf(const bke_enkf_args &a)
{
    int rc;
    if ((rc = check_bank(a.n_filters, a.dim_x, a.dim_z))) return rc;
    if (a.dim_x > 16) { set_error("bad dimensions: dim_x must be 16 or less"); return BKE_ERR_BAD_ARG; }
    if (a.n_members < 2) { set_error("n_members must be 2 or greater (the covariances divide by n_members - 1)"); return BKE_ERR_BAD_ARG; }
    if ((rc = validate_sigma(a)) || (rc = check_flag_bits(a.flags, BKE_DO_PREDICT | BKE_DO_UPDATE))) return rc;
    if (!a.sigmas || !a.sigmas_out) { set_error("sigmas and sigmas_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (a.Q_stride < 0 || a.R_stride < 0 || a.F_stride < 0 || a.H_stride < 0) { set_error("negative model stride"); return BKE_ERR_BAD_ARG; }
    if (a.n_members > (1 << 24)) { set_error("n_members must be at most 2^24"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

// the pre-built steps: the family's checks, then a known model id, and a range model at the shape it is written for
template <typename Args, int (*validate)(const Args &)>
static int validate_prebuilt(const Args &a)
{
    if (int rc = validate(a)) return rc;
    if (a.hx_model == BKE_HX_RANGE_AZ_EL && !(a.dim_x == 6 && a.dim_z == 3)) { set_error("BKE_HX_RANGE_AZ_EL needs dim_x=6, dim_z=3"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model == BKE_HX_RANGE_BEARING && !(a.dim_x == 4 && a.dim_z == 2)) { set_error("BKE_HX_RANGE_BEARING needs dim_x=4, dim_z=2"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model < 0 || a.fx_model > BKE_FX_CONST_VEL || a.hx_model < 0 || a.hx_model > BKE_HX_RANGE_BEARING) {
        set_error("unknown fx/hx model id"); return BKE_ERR_BAD_ARG;
    }
    return BKE_OK;
}

template <typename Args> static bool empty_bank(const Args &a) { return a.n_filters == 0; }
static bool empty_bank(const bke_kf_rows_args &a) { return a.step.n_filters == 0; }
static bool empty_bank(const bke_kf_batch_args &a) { return a.step.n_filters == 0; }
static bool empty_bank(const bke_fls_args &a) { return a.step.n_filters == 0; }
static bool empty_bank(const bke_score_args &a) { return a.n_tracks == 0 || a.n_candidates == 0; }
static bool empty_bank(const bke_ukf_score_args &a) { return a.n_filters == 0 || a.n_candidates == 0; }

// the body of an entry point: its argument checks, then the device, then an empty bank returns at once, then the launch
template <typename Args, typename Validate, typename Launch>
static int checked_launch(const Args *args, Validate validate, Launch launch, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    int rc = validate(*args);
    if (rc || (rc = require_device())) return rc;
    if (empty_bank(*args)) return BKE_OK;
    return launch(*args, (cudaStream_t)stream);
}

}  // namespace bke

using namespace bke;

namespace bke {
int launch_kf_any(const bke_kf_args &a, cudaStream_t s)
{
    int rc = launch_kf_tc(a, s);
    if (rc == BKE_ERR_UNSUPPORTED) rc = launch_kf_fast(a, s);
    if (rc == BKE_ERR_UNSUPPORTED) rc = launch_kf_direct(a, s);
    if (rc == BKE_ERR_UNSUPPORTED) rc = launch_kf_rowblock(a, s);
    if (rc == BKE_ERR_UNSUPPORTED) rc = launch_kf_generic(a, s);
    return rc;
}
}  // namespace bke

extern "C" {

int bke_abi_version(void) { return BKE_ABI_VERSION; }

const char *bke_last_error(void) { return g_err; }

int bke_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int bke_kf_step(const bke_kf_args *args, void *stream)
{
    return checked_launch(args, [](const bke_kf_args &a) { return validate_kf(a, true); }, launch_kf_any, stream);
}

// the flags of the two other update forms: an update, optionally after a predict
static int validate_update_form(const bke_kf_args &a)
{
    if (int rc = check_flag_bits(a.flags, BKE_DO_PREDICT | BKE_DO_UPDATE | BKE_STATUS_STICKY | BKE_REVERSE_TILES)) return rc;
    if (!(a.flags & BKE_DO_UPDATE)) { set_error("flags must hold BKE_DO_UPDATE"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int bke_kf_step_correlated(const bke_kf_args *args, const void *M, int64_t M_stride, void *stream)
{
    auto validate = [&](const bke_kf_args &a) {
        int rc;
        if ((rc = validate_kf(a, true)) || (rc = validate_update_form(a))) return rc;
        if (!M) { set_error("M is NULL"); return BKE_ERR_BAD_ARG; }
        return check_strides({{M_stride, (int64_t)a.dim_x * a.dim_z}});
    };
    auto launch = [&](const bke_kf_args &a, cudaStream_t s) {
        int rc = launch_kf_direct_correlated(a, M, M_stride, s);
        return rc == BKE_ERR_UNSUPPORTED ? launch_kf_generic_correlated(a, M, M_stride, s) : rc;
    };
    return checked_launch(args, validate, launch, stream);
}

static int validate_rows(const bke_kf_rows_args &r)
{
    const bke_kf_args &a = r.step;
    const int64_t n = a.dim_x, m = a.dim_z, L = r.rows, start = r.start;
    if (L < 1 || start < 0 || start + L > m) {
        set_error("the block of rows %lld .. %lld is not within the %lld rows of z", (long long)start, (long long)(start + L - 1), (long long)m);
        return BKE_ERR_BAD_ARG;
    }
    int rc;
    if ((rc = check_strides({{r.H_i_stride, L * n}, {r.R_i_stride, L * L}}))) return rc;
    if (a.S || a.SI || a.log_likelihood) { set_error("update_rows does not write S, SI or log_likelihood: they must be NULL"); return BKE_ERR_BAD_ARG; }
    // the checks of bke_kf_step on the bank's arrays; a caller-supplied block stands in for H or R there
    bke_kf_args chk = a;
    if (r.H_i) { chk.H = r.H_i; chk.H_stride = 0; }
    if (r.R_i) { chk.R = r.R_i; chk.R_stride = 0; }
    if ((rc = validate_kf(chk, true))) return rc;
    return validate_update_form(a);
}

// the block as an update of L rows: H_i is contiguous in the bank's H, R_i has the row pitch m there
static int launch_rows(const bke_kf_rows_args &r, cudaStream_t s)
{
    const bke_kf_args &a = r.step;
    const int64_t n = a.dim_x, m = a.dim_z, L = r.rows, start = r.start;
    const size_t es = a.dtype == BKE_F32 ? 4 : 8;
    bke_kf_args b = a;
    b.dim_z = (int32_t)L;
    if (r.H_i) { b.H = r.H_i; b.H_stride = r.H_i_stride; }
    else b.H = (const char *)a.H + start * n * es;
    int rpitch = (int)L;
    if (r.R_i) { b.R = r.R_i; b.R_stride = r.R_i_stride; }
    else { b.R = (const char *)a.R + (start * m + start) * es; rpitch = (int)m; }
    int rc = launch_kf_direct_rows(b, (int)m, (int)start, rpitch, r.z_record, s);
    if (rc == BKE_ERR_UNSUPPORTED) rc = launch_kf_generic_rows(b, (int)m, (int)start, rpitch, r.z_record, s);
    return rc;
}

int bke_kf_update_rows(const bke_kf_rows_args *args, void *stream) { return checked_launch(args, validate_rows, launch_rows, stream); }

size_t bke_kf_sym_models_bytes(int64_t n_filters) { return kf_sym_models_bytes(n_filters); }

int bke_kf_pack_sym_models(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dtype, const void *Q,
                           const void *R, void *record, int32_t *asymmetric, void *stream)
{
    if (int rc = check_bank(n_filters)) return rc;
    if (n_filters > 0 && (!Q || !R || !record)) { set_error("Q, R and record must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (!asymmetric) { set_error("asymmetric must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (!(dim_x == 4 && dim_z == 2 && dtype == BKE_F32)) {
        set_error("packed symmetric models exist for dim_x = 4, dim_z = 2, BKE_F32 only");
        return BKE_ERR_UNSUPPORTED;
    }
    int rc = require_device();
    if (rc) return rc;
    return launch_kf_pack_sym(n_filters, Q, R, record, asymmetric, (cudaStream_t)stream);
}

int bke_kf_step_sym(const bke_kf_args *args, const void *record, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    int rc = validate_kf(*args, true);
    if (rc) return rc;
    if (!record) { set_error("record is NULL"); return BKE_ERR_BAD_ARG; }
    if ((rc = require_device())) return rc;
    if (args->n_filters == 0) return BKE_OK;
    g_err[0] = '\0';
    rc = launch_kf_fast(*args, (cudaStream_t)stream, record);
    if (rc == BKE_ERR_UNSUPPORTED && g_err[0] == '\0')      // (launch_kf_fast names some causes itself)
        set_error("the packed symmetric models cover per-filter models of dim_x = 4, dim_z = 2, BKE_F32 banks "
                  "without control input, on 16-byte aligned arrays");
    return rc;
}

static int validate_models(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dtype, const void *F, const void *Q,
                           const void *H, const void *R)
{
    if (int rc = check_bank(n_filters)) return rc;
    if (n_filters > 0 && (!F || !Q || !H || !R)) { set_error("F, Q, H and R must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (!(dim_x == 4 && dim_z == 2 && dtype == BKE_F32)) {
        set_error("packed models exist for dim_x = 4, dim_z = 2, BKE_F32 only");
        return BKE_ERR_UNSUPPORTED;
    }
    return BKE_OK;
}

static bool bad_mask(uint64_t varying) { return (varying >> BKE_KF42_MODEL_WORDS) != 0; }

int bke_kf_scan_models(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dtype, const void *F, const void *Q,
                       const void *H, const void *R, bke_kf_model_map *map, void *stream)
{
    int rc = validate_models(n_filters, dim_x, dim_z, dtype, F, Q, H, R);
    if (rc) return rc;
    if (!map) { set_error("map must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((rc = require_device())) return rc;
    return launch_kf_scan_models(n_filters, F, Q, H, R, map, (cudaStream_t)stream);
}

size_t bke_kf_packed_models_bytes(int64_t n_filters, uint64_t varying) { return kf_packed_models_bytes(n_filters, varying); }

int bke_kf_pack_models(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dtype, const void *F, const void *Q,
                       const void *H, const void *R, uint64_t varying, void *record, void *stream)
{
    int rc = validate_models(n_filters, dim_x, dim_z, dtype, F, Q, H, R);
    if (rc) return rc;
    if (bad_mask(varying)) { set_error("varying has bits above word %d", BKE_KF42_MODEL_WORDS - 1); return BKE_ERR_BAD_ARG; }
    if (n_filters > 0 && varying && !record) { set_error("record must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((rc = require_device())) return rc;
    return launch_kf_pack_models(n_filters, F, Q, H, R, varying, record, (cudaStream_t)stream);
}

static int validate_packed(const void *record, const bke_kf_model_map *host_map)
{
    if (!host_map) { set_error("host_map is NULL"); return BKE_ERR_BAD_ARG; }
    if (bad_mask(host_map->varying)) { set_error("varying has bits above word %d", BKE_KF42_MODEL_WORDS - 1); return BKE_ERR_BAD_ARG; }
    if (host_map->varying && !record) { set_error("record is NULL"); return BKE_ERR_BAD_ARG; }
    int plane[BKE_KF42_MODEL_WORDS];
    return kf_model_planes(*host_map, plane);
}

int bke_kf_step_packed(const bke_kf_args *args, const void *record, const bke_kf_model_map *host_map, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    int rc = validate_kf(*args, true);
    if (rc) return rc;
    if ((rc = validate_packed(record, host_map))) return rc;
    if ((rc = require_device())) return rc;
    if (args->n_filters == 0) return BKE_OK;
    g_err[0] = '\0';
    rc = launch_kf_fast(*args, (cudaStream_t)stream, record, host_map);
    if (rc == BKE_ERR_UNSUPPORTED && g_err[0] == '\0')      // (launch_kf_fast names some causes itself)
        set_error("the packed models cover per-filter models of dim_x = 4, dim_z = 2, BKE_F32 banks without "
                  "control input, on 16-byte aligned arrays");
    return rc;
}

int bke_kf_steps_packed(const bke_kf_args *args, const void *record, const bke_kf_model_map *host_map,
                        const void *const *zs, int32_t n_steps, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    int rc = validate_kf(*args, false);
    if (rc) return rc;
    if ((rc = validate_packed(record, host_map))) return rc;
    if (!zs) { set_error("zs is NULL"); return BKE_ERR_BAD_ARG; }
    if (reinterpret_cast<uintptr_t>(args->tile_order) & 3u) { set_error("tile_order must be 4-byte aligned"); return BKE_ERR_BAD_ARG; }
    // what only the fused ring refuses (launch_kf_fast refuses the rest), before anything is launched
    const bke_kf_args &a = *args;
    auto refuse = [](const char *why) { set_error("bke_kf_steps_packed: %s", why); return BKE_ERR_UNSUPPORTED; };
    if (n_steps < 1 || n_steps > BKE_KF42_MAX_RING) return refuse("n_steps must be 1 .. BKE_KF42_MAX_RING");
    if ((a.flags & ~BKE_REVERSE_TILES) != (BKE_DO_PREDICT | BKE_DO_UPDATE)) return refuse("flags must be BKE_DO_PREDICT | BKE_DO_UPDATE");
    if (a.z_valid) return refuse("z_valid is not taken");
    if (a.B || a.u) return refuse("a control input is not taken");
    if (a.x_prior || a.P_prior || a.K || a.y || a.S || a.SI || a.log_likelihood || a.status)
        return refuse("status and the optional outputs are not written");
    if (a.x_out != a.x || a.P_out != a.P) return refuse("the state is stepped in place (x_out = x, P_out = P)");
    const char *x0 = (const char *)a.x, *P0 = (const char *)a.P;
    for (int k = 0; k < n_steps; k++) {
        const char *z = (const char *)zs[k];
        if (!z) { set_error("zs[%d] is NULL", k); return BKE_ERR_BAD_ARG; }
        if (reinterpret_cast<uintptr_t>(z) & 15u) return refuse("every z must be 16-byte aligned");
        if ((z < x0 + a.n_filters * 16 && x0 < z + a.n_filters * 8) || (z < P0 + a.n_filters * 64 && P0 < z + a.n_filters * 8))
            return refuse("a z overlaps x or P");
    }
    if ((rc = require_device())) return rc;
    if (a.n_filters == 0) return BKE_OK;
    bke_kf_args st = a;
    st.z = zs[0];
    g_err[0] = '\0';
    rc = launch_kf_fast(st, (cudaStream_t)stream, record, host_map, zs, n_steps);
    if (rc == BKE_ERR_UNSUPPORTED && g_err[0] == '\0')     // (launch_kf_fast names some causes itself)
        set_error("the fused ring covers per-filter models of dim_x = 4, dim_z = 2, BKE_F32 banks on 16-byte aligned arrays");
    return rc;
}

int bke_capture_node_count(void *stream, int64_t *n_nodes)
{
    if (!n_nodes) { set_error("n_nodes is NULL"); return BKE_ERR_BAD_ARG; }
    int rc = require_device();
    if (rc) return rc;
    cudaStreamCaptureStatus status = cudaStreamCaptureStatusNone;
    cudaGraph_t graph = nullptr;
    if (check_cuda(cudaStreamGetCaptureInfo((cudaStream_t)stream, &status, nullptr, &graph, nullptr, nullptr),
                   "cudaStreamGetCaptureInfo")) return BKE_ERR_CUDA;
    if (status != cudaStreamCaptureStatusActive || !graph) { set_error("the stream is not capturing"); return BKE_ERR_BAD_ARG; }
    size_t n = 0;
    if (check_cuda(cudaGraphGetNodes(graph, nullptr, &n), "cudaGraphGetNodes")) return BKE_ERR_CUDA;
    *n_nodes = (int64_t)n;
    return BKE_OK;
}

static int validate_kf_batch(const bke_kf_batch_args &a)
{
    if (int rc = validate_kf(a.step, false)) return rc;
    if (a.n_steps < 0) { set_error("n_steps < 0"); return BKE_ERR_BAD_ARG; }
    if (a.n_steps > 0 && !a.zs) { set_error("zs is NULL"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int bke_kf_batch_filter(const bke_kf_batch_args *args, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    bke_kf_batch_args a = *args;
    a.step.flags |= BKE_DO_PREDICT | BKE_DO_UPDATE;
    return checked_launch(&a, validate_kf_batch, launch_kf_batch, stream);
}

size_t bke_fls_workspace_bytes(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dim_u, int32_t dtype, int64_t lag)
{
    return fls_workspace_bytes(n_filters, dim_x, dim_z, dim_u, dtype, lag);
}

static int validate_fls(const bke_fls_args &a)
{
    int rc;
    if ((rc = validate_kf(a.step, false))) return rc;
    if (a.n_steps < 1) { set_error("n_steps must be 1 or greater"); return BKE_ERR_BAD_ARG; }
    if (a.lag < 0) { set_error("lag < 0"); return BKE_ERR_BAD_ARG; }
    if (a.count < 0) { set_error("count < 0"); return BKE_ERR_BAD_ARG; }
    if (!a.zs) { set_error("zs is NULL"); return BKE_ERR_BAD_ARG; }
    if (!a.xs_smooth) { set_error("xs_smooth (the history) is NULL"); return BKE_ERR_BAD_ARG; }
    if (a.us && (rc = check_control(a.step.B, a.us, a.step.dim_u))) return rc;     // us stands in for u
    return BKE_OK;
}

int bke_fls_smooth(const bke_fls_args *args, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    bke_fls_args a = *args;
    a.step.flags = BKE_DO_PREDICT | BKE_DO_UPDATE;
    return checked_launch(&a, validate_fls, launch_fls, stream);
}

int bke_ukf_step(const bke_ukf_args *args, void *stream) { return checked_launch(args, validate_prebuilt<bke_ukf_args, validate_ukf>, launch_ukf, stream); }

int bke_ckf_step(const bke_ckf_args *args, void *stream) { return checked_launch(args, validate_prebuilt<bke_ckf_args, validate_ckf>, launch_ckf, stream); }

int bke_enkf_step(const bke_enkf_args *args, void *stream) { return checked_launch(args, validate_prebuilt<bke_enkf_args, validate_enkf>, launch_enkf, stream); }

int bke_enkf_initialize(int64_t n_filters, int32_t dim_x, int32_t n_members, int32_t dtype, uint32_t seed, uint32_t counter,
                        const void *x, const void *P, void *sigmas, int32_t *status, void *stream)
{
    int rc;
    if ((rc = check_bank(n_filters, dim_x))) return rc;
    if (dim_x > 16) { set_error("bke_enkf_initialize: 1 <= dim_x <= 16"); return BKE_ERR_BAD_ARG; }
    if (n_members < 2 || n_members > (1 << 24)) { set_error("bke_enkf_initialize: 2 <= n_members <= 2^24"); return BKE_ERR_BAD_ARG; }
    if ((rc = check_dtype(dtype))) return rc;
    if (!x || !P || !sigmas) { set_error("x, P and sigmas must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((rc = require_device())) return rc;
    if (n_filters == 0) return BKE_OK;
    return launch_enkf_init(n_filters, dim_x, n_members, dtype, seed, counter, x, P, sigmas, status, (cudaStream_t)stream);
}

int bke_srkf_step(const bke_srkf_args *args, void *stream) { return checked_launch(args, validate_srkf, launch_srkf, stream); }

int bke_cholesky_lower(int64_t n_filters, int32_t k, int32_t dtype, const void *A, int64_t stride, void *L,
                       int32_t *status, void *stream)
{
    int rc;
    if ((rc = check_bank(n_filters))) return rc;
    if (k < 1) { set_error("k must be 1 or greater"); return BKE_ERR_BAD_ARG; }
    if ((rc = check_dtype(dtype)) || (rc = check_strides({{stride, (int64_t)k * k}}))) return rc;
    if (n_filters > 0 && (!A || !L)) { set_error("A and L must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (k > BKE_CHOLESKY_MAX_DIM) {
        set_error("bke_cholesky_lower: k=%d is above BKE_CHOLESKY_MAX_DIM=%d", k, BKE_CHOLESKY_MAX_DIM);
        return BKE_ERR_UNSUPPORTED;
    }
    if ((rc = require_device())) return rc;
    if (n_filters == 0) return BKE_OK;
    return launch_cholesky_lower(n_filters, k, dtype, A, stride, L, status, (cudaStream_t)stream);
}

int bke_if_step(const bke_if_args *args, void *stream) { return checked_launch(args, validate_if, launch_if, stream); }

int bke_inverse(int64_t n_filters, int32_t k, int32_t dtype, const void *A, int64_t stride, void *Ai, int32_t *status,
                void *stream)
{
    int rc;
    if ((rc = check_bank(n_filters))) return rc;
    if (k < 1) { set_error("k must be 1 or greater"); return BKE_ERR_BAD_ARG; }
    if ((rc = check_dtype(dtype)) || (rc = check_strides({{stride, (int64_t)k * k}}))) return rc;
    if (n_filters > 0 && (!A || !Ai)) { set_error("A and Ai must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((rc = require_device())) return rc;
    if (n_filters == 0) return BKE_OK;
    return launch_inverse(n_filters, k, dtype, A, stride, Ai, status, (cudaStream_t)stream);
}

int bke_poly_filter(const bke_poly_args *args, void *stream) { return checked_launch(args, validate_poly, launch_poly, stream); }

int bke_imm_batch_filter(const bke_imm_batch_args *args, void *stream)
{
    const int v = validate_imm(args);
    if (v >= 0) return v;
    int rc = require_device();
    if (rc) return rc;
    return launch_imm_batch(*args, (cudaStream_t)stream);
}

int bke_score_measurements(const bke_score_args *args, void *stream) { return checked_launch(args, validate_score, launch_score, stream); }

// the pre-built hx models at the shapes they are written for
static int validate_ukf_score_prebuilt(const bke_ukf_score_args &a)
{
    if (int rc = validate_ukf_score(a)) return rc;
    if (a.hx_model == BKE_HX_RANGE_AZ_EL && !(a.dim_x == 6 && a.dim_z == 3)) { set_error("BKE_HX_RANGE_AZ_EL needs dim_x=6, dim_z=3"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model == BKE_HX_RANGE_BEARING && !(a.dim_x == 4 && a.dim_z == 2)) { set_error("BKE_HX_RANGE_BEARING needs dim_x=4, dim_z=2"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model < 0 || a.hx_model > BKE_HX_RANGE_BEARING) { set_error("unknown hx model id"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int bke_ukf_score(const bke_ukf_score_args *args, void *stream)
{
    return checked_launch(args, validate_ukf_score_prebuilt, launch_ukf_score, stream);
}

size_t bke_db_workspace_bytes(int64_t n_bins, int32_t dtype) { return check_dtype(dtype) ? 0 : db_workspace_bytes(n_bins, dtype); }

// the checks of bke_db_step; -1 = go
static int validate_db(const bke_db_args *a)
{
    if (!a) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    int rc;
    if (a->n_rows < 0 || a->n_bins < 1) { set_error("bad sizes: n_rows must be >= 0 and n_bins >= 1"); return BKE_ERR_BAD_ARG; }
    if (a->n_rows >= ((int64_t)1 << 31) || a->n_bins >= ((int64_t)1 << 31)) { set_error("n_rows and n_bins must be < 2^31"); return BKE_ERR_BAD_ARG; }
    if ((rc = check_dtype(a->dtype))) return rc;
    if (a->flags & ~(BKE_DB_NORMALIZE | BKE_DB_CONSTANT)) { set_error("flags may only hold BKE_DB_NORMALIZE and BKE_DB_CONSTANT"); return BKE_ERR_BAD_ARG; }
    if (a->kernel && a->kernel_len < 1) { set_error("kernel_len must be 1 or greater"); return BKE_ERR_BAD_ARG; }
    if (a->kernel && (rc = check_strides({{a->kernel_stride, a->kernel_len}}))) return rc;
    if (a->sums && !(a->flags & BKE_DB_NORMALIZE)) { set_error("sums is an output of BKE_DB_NORMALIZE only"); return BKE_ERR_BAD_ARG; }
    if (a->n_rows == 0) return BKE_OK;
    if (!a->pdf || !a->out) { set_error("pdf and out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    const int64_t B = a->n_rows, M = a->n_bins, es = a->dtype == BKE_F32 ? 4 : 8;
    const size_t need = db_workspace_bytes(M, a->dtype);
    if (need) {
        if (!a->workspace || ((uintptr_t)a->workspace & 255)) { set_error("workspace must be non-NULL and 256-byte aligned"); return BKE_ERR_BAD_ARG; }
        if (a->workspace_bytes < need) { set_error("workspace too small: %zu < %zu", a->workspace_bytes, need); return BKE_ERR_BAD_ARG; }
    }
    // out may be pdf itself; every array the call writes must otherwise be clear of every other array it touches
    struct Span { const void *p; int64_t bytes; bool written; };
    const Span sp[] = {{a->out, B * M * es, true}, {a->pdf, B * M * es, false}, {a->likelihood, B * M * es, false},
                       {a->kernel, (a->kernel_stride ? B : 1) * a->kernel_len * 8, false},
                       {a->offsets, B * 8, false}, {a->sums, B * 8, true},
                       {need ? a->workspace : nullptr, (int64_t)need, true}};
    const int ns = sizeof(sp) / sizeof(sp[0]);
    for (int i = 0; i < ns; i++) {
        for (int k = i + 1; k < ns; k++) {
            if (!sp[i].p || !sp[k].p || (!sp[i].written && !sp[k].written) || (i == 0 && k == 1 && sp[0].p == sp[1].p)) continue;
            if (!a->kernel && (i == 3 || k == 3)) continue;
            const uintptr_t p0 = (uintptr_t)sp[i].p, p1 = (uintptr_t)sp[k].p;
            if (p0 < p1 + (uintptr_t)sp[k].bytes && p1 < p0 + (uintptr_t)sp[i].bytes) {
                set_error("an array bke_db_step writes overlaps another of its arrays (only out == pdf may alias)");
                return BKE_ERR_BAD_ARG;
            }
        }
    }
    return -1;
}

int bke_db_step(const bke_db_args *args, void *stream)
{
    const int v = validate_db(args);
    if (v >= 0) return v;
    int rc = require_device();
    if (rc) return rc;
    return launch_db(*args, (cudaStream_t)stream);
}

}  // extern "C"
