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

static int require_device()
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

static int validate_kf(const bke_kf_args *a, bool need_z)
{
    if (!a) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    if (a->n_filters < 0) { set_error("n_filters < 0"); return BKE_ERR_BAD_ARG; }
    if (a->dim_x < 1) { set_error("dim_x must be 1 or greater"); return BKE_ERR_BAD_ARG; }   // kalman_filter.py:388
    if (a->dim_z < 1) { set_error("dim_z must be 1 or greater"); return BKE_ERR_BAD_ARG; }   // :390
    if (a->dim_u < 0) { set_error("dim_u must be 0 or greater"); return BKE_ERR_BAD_ARG; }   // :392
    if (a->dtype != BKE_F32 && a->dtype != BKE_F64) { set_error("dtype must be BKE_F32 or BKE_F64"); return BKE_ERR_BAD_ARG; }
    if (!(a->flags & (BKE_DO_PREDICT | BKE_DO_UPDATE))) { set_error("flags selects neither predict nor update"); return BKE_ERR_BAD_ARG; }
    if (!a->x || !a->P || !a->x_out || !a->P_out) { set_error("x, P, x_out, P_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (a->flags & BKE_DO_PREDICT) {
        if (!a->F || !a->Q) { set_error("predict needs F and Q"); return BKE_ERR_BAD_ARG; }
        if ((a->B == nullptr) != (a->u == nullptr) && a->dim_u > 0 && a->B && !a->u) { /* u=None: no control, kalman_filter.py:472 */ }
    }
    if (a->flags & BKE_DO_UPDATE) {
        if (!a->H || !a->R) { set_error("update needs H and R"); return BKE_ERR_BAD_ARG; }
        if (need_z && !a->z) { set_error("update needs z"); return BKE_ERR_BAD_ARG; }
    }
    const int64_t n = a->dim_x, m = a->dim_z;
    auto bad_stride = [](int64_t s, int64_t full) { return s != 0 && s != full; };
    if (bad_stride(a->F_stride, n * n) || bad_stride(a->Q_stride, n * n) || bad_stride(a->H_stride, m * n) ||
        bad_stride(a->R_stride, m * m)) {
        set_error("model strides must be 0 (shared) or the dense per-filter size");
        return BKE_ERR_BAD_ARG;
    }
    return BKE_OK;
}

static int validate_srkf(const bke_srkf_args *a)
{
    if (!a) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    if (a->n_filters < 0) { set_error("n_filters < 0"); return BKE_ERR_BAD_ARG; }
    if (a->dim_x < 1) { set_error("dim_x must be 1 or greater"); return BKE_ERR_BAD_ARG; }   // square_root.py:128-133
    if (a->dim_z < 1) { set_error("dim_z must be 1 or greater"); return BKE_ERR_BAD_ARG; }
    if (a->dim_u < 0) { set_error("dim_u must be 0 or greater"); return BKE_ERR_BAD_ARG; }
    if (a->dtype != BKE_F32 && a->dtype != BKE_F64) { set_error("dtype must be BKE_F32 or BKE_F64"); return BKE_ERR_BAD_ARG; }
    if (!(a->flags & (BKE_DO_PREDICT | BKE_DO_UPDATE))) { set_error("flags selects neither predict nor update"); return BKE_ERR_BAD_ARG; }
    if (a->flags & ~(BKE_DO_PREDICT | BKE_DO_UPDATE)) { set_error("flags may only hold BKE_DO_PREDICT and BKE_DO_UPDATE"); return BKE_ERR_BAD_ARG; }
    if (!a->x || !a->L || !a->x_out || !a->L_out) { set_error("x, L, x_out, L_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((a->flags & BKE_DO_PREDICT) && (!a->F || !a->Lq)) { set_error("predict needs F and Lq"); return BKE_ERR_BAD_ARG; }   // :240-243
    if ((a->flags & BKE_DO_UPDATE) && (!a->H || !a->Lr || !a->z)) { set_error("update needs H, Lr and z"); return BKE_ERR_BAD_ARG; }   // :204-215
    if ((a->B != nullptr || a->u != nullptr) && (!a->B || !a->u || a->dim_u < 1)) {
        set_error("a control input needs B, u and dim_u >= 1");                                       // :240
        return BKE_ERR_BAD_ARG;
    }
    const int64_t n = a->dim_x, m = a->dim_z, du = a->dim_u;
    auto bad_stride = [](int64_t s, int64_t full) { return s != 0 && s != full; };
    if (bad_stride(a->F_stride, n * n) || bad_stride(a->Lq_stride, n * n) || bad_stride(a->H_stride, m * n) ||
        bad_stride(a->Lr_stride, m * m) || bad_stride(a->B_stride, n * du) || bad_stride(a->u_stride, du)) {
        set_error("model strides must be 0 (shared) or the dense per-filter size");
        return BKE_ERR_BAD_ARG;
    }
    return BKE_OK;
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
    int rc = validate_kf(args, true);
    if (rc) return rc;
    if ((rc = require_device())) return rc;
    if (args->n_filters == 0) return BKE_OK;
    cudaStream_t s = (cudaStream_t)stream;
    return launch_kf_any(*args, s);
}

size_t bke_kf_sym_models_bytes(int64_t n_filters) { return kf_sym_models_bytes(n_filters); }

int bke_kf_pack_sym_models(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dtype, const void *Q,
                           const void *R, void *record, int32_t *asymmetric, void *stream)
{
    if (n_filters < 0) { set_error("n_filters < 0"); return BKE_ERR_BAD_ARG; }
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
    int rc = validate_kf(args, true);
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
    if (n_filters < 0) { set_error("n_filters < 0"); return BKE_ERR_BAD_ARG; }
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

int bke_kf_step_packed(const bke_kf_args *args, const void *record, const bke_kf_model_map *host_map, void *stream)
{
    int rc = validate_kf(args, true);
    if (rc) return rc;
    if (!host_map) { set_error("host_map is NULL"); return BKE_ERR_BAD_ARG; }
    if (bad_mask(host_map->varying)) { set_error("varying has bits above word %d", BKE_KF42_MODEL_WORDS - 1); return BKE_ERR_BAD_ARG; }
    if (host_map->varying && !record) { set_error("record is NULL"); return BKE_ERR_BAD_ARG; }
    if ((rc = require_device())) return rc;
    if (args->n_filters == 0) return BKE_OK;
    g_err[0] = '\0';
    rc = launch_kf_fast(*args, (cudaStream_t)stream, record, host_map);
    if (rc == BKE_ERR_UNSUPPORTED && g_err[0] == '\0')      // (launch_kf_fast names some causes itself)
        set_error("the packed models cover per-filter models of dim_x = 4, dim_z = 2, BKE_F32 banks without "
                  "control input, on 16-byte aligned arrays");
    return rc;
}

int bke_kf_batch_filter(const bke_kf_batch_args *args, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    bke_kf_args st = args->step;
    st.flags |= BKE_DO_PREDICT | BKE_DO_UPDATE;
    int rc = validate_kf(&st, false);
    if (rc) return rc;
    if (args->n_steps < 0) { set_error("n_steps < 0"); return BKE_ERR_BAD_ARG; }
    if (args->n_steps > 0 && !args->zs) { set_error("zs is NULL"); return BKE_ERR_BAD_ARG; }
    if ((rc = require_device())) return rc;
    if (st.n_filters == 0) return BKE_OK;
    bke_kf_batch_args a = *args;
    a.step = st;
    return launch_kf_batch(a, (cudaStream_t)stream);
}

int bke_ukf_step(const bke_ukf_args *args, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    const bke_ukf_args &a = *args;
    if (a.n_filters < 0 || a.dim_x < 1 || a.dim_z < 1) { set_error("bad dimensions"); return BKE_ERR_BAD_ARG; }
    if (a.dtype != BKE_F32 && a.dtype != BKE_F64) { set_error("dtype must be BKE_F32 or BKE_F64"); return BKE_ERR_BAD_ARG; }
    if (!(a.flags & (BKE_DO_PREDICT | BKE_DO_UPDATE))) { set_error("flags selects neither predict nor update"); return BKE_ERR_BAD_ARG; }
    if (!a.x || !a.P || !a.x_out || !a.P_out) { set_error("x, P, x_out, P_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_PREDICT) && !a.Q) { set_error("predict needs Q"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_UPDATE) && (!a.R || !a.z)) { set_error("update needs R and z"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model == BKE_FX_LINEAR && (a.flags & BKE_DO_PREDICT) && !a.F) { set_error("BKE_FX_LINEAR needs F"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model == BKE_HX_LINEAR && (a.flags & BKE_DO_UPDATE) && !a.H) { set_error("BKE_HX_LINEAR needs H"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model == BKE_FX_CONST_VEL && (a.dim_x & 1)) { set_error("BKE_FX_CONST_VEL needs an even dim_x"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model == BKE_HX_RANGE_AZ_EL && !(a.dim_x == 6 && a.dim_z == 3)) { set_error("BKE_HX_RANGE_AZ_EL needs dim_x=6, dim_z=3"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model == BKE_HX_RANGE_BEARING && !(a.dim_x == 4 && a.dim_z == 2)) { set_error("BKE_HX_RANGE_BEARING needs dim_x=4, dim_z=2"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model < 0 || a.fx_model > BKE_FX_CONST_VEL || a.hx_model < 0 || a.hx_model > BKE_HX_RANGE_BEARING) {
        set_error("unknown fx/hx model id"); return BKE_ERR_BAD_ARG;
    }
    double lam_n = a.alpha * a.alpha * (a.dim_x + a.kappa);
    if (!(lam_n != 0.0)) { set_error("alpha^2 (n + kappa) must be non-zero"); return BKE_ERR_BAD_ARG; }
    int rc = require_device();
    if (rc) return rc;
    if (a.n_filters == 0) return BKE_OK;
    return launch_ukf(a, (cudaStream_t)stream);
}

int bke_ckf_step(const bke_ckf_args *args, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    const bke_ckf_args &a = *args;
    int rc = validate_ckf(a);
    if (rc) return rc;
    if (a.hx_model == BKE_HX_RANGE_AZ_EL && !(a.dim_x == 6 && a.dim_z == 3)) { set_error("BKE_HX_RANGE_AZ_EL needs dim_x=6, dim_z=3"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model == BKE_HX_RANGE_BEARING && !(a.dim_x == 4 && a.dim_z == 2)) { set_error("BKE_HX_RANGE_BEARING needs dim_x=4, dim_z=2"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model < 0 || a.fx_model > BKE_FX_CONST_VEL || a.hx_model < 0 || a.hx_model > BKE_HX_RANGE_BEARING) {
        set_error("unknown fx/hx model id"); return BKE_ERR_BAD_ARG;
    }
    if ((rc = require_device())) return rc;
    if (a.n_filters == 0) return BKE_OK;
    return launch_ckf(a, (cudaStream_t)stream);
}

int bke_srkf_step(const bke_srkf_args *args, void *stream)
{
    int rc = validate_srkf(args);
    if (rc) return rc;
    if ((rc = require_device())) return rc;
    if (args->n_filters == 0) return BKE_OK;
    return launch_srkf(*args, (cudaStream_t)stream);
}

int bke_cholesky_lower(int64_t n_filters, int32_t k, int32_t dtype, const void *A, int64_t stride, void *L,
                       int32_t *status, void *stream)
{
    if (n_filters < 0) { set_error("n_filters < 0"); return BKE_ERR_BAD_ARG; }
    if (k < 1) { set_error("k must be 1 or greater"); return BKE_ERR_BAD_ARG; }
    if (dtype != BKE_F32 && dtype != BKE_F64) { set_error("dtype must be BKE_F32 or BKE_F64"); return BKE_ERR_BAD_ARG; }
    if (stride != 0 && stride != (int64_t)k * k) { set_error("stride must be 0 (shared) or k*k"); return BKE_ERR_BAD_ARG; }
    if (n_filters > 0 && (!A || !L)) { set_error("A and L must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (k > BKE_CHOLESKY_MAX_DIM) {
        set_error("bke_cholesky_lower: k=%d is above BKE_CHOLESKY_MAX_DIM=%d", k, BKE_CHOLESKY_MAX_DIM);
        return BKE_ERR_UNSUPPORTED;
    }
    int rc = require_device();
    if (rc) return rc;
    if (n_filters == 0) return BKE_OK;
    return launch_cholesky_lower(n_filters, k, dtype, A, stride, L, status, (cudaStream_t)stream);
}

}  // extern "C"
