// ukf_rts.cu — host side of UnscentedKalmanFilter.rts_smoother for a bank (kernel: ukf_rts_kernel.cuh).
#include "ukf_rts_kernel.cuh"
#include "ukf_rts_launch.cuh"

namespace bke {
namespace {

template <typename T>
int launch_t(const bke_ukf_rts_args &a, cudaStream_t s)
{
    UrP<T> p;
    ukf_rts_fill_params<T>(a, p);
    auto kern = (a.flags & BKE_UKF_SIMPLEX) ? ukf_rts_kernel<T, false, true> : ukf_rts_kernel<T, false>;
    kern<<<(unsigned)((p.N + 63) / 64), 64, 0, s>>>(p);
    return check_cuda(cudaGetLastError(), "ukf rts launch");
}

}  // namespace

int validate_ukf_rts(const bke_ukf_rts_args &a, bool user_fx)
{
    if (a.n_filters < 0 || a.n_steps < 0) { set_error("negative sizes"); return BKE_ERR_BAD_ARG; }
    if (a.dim_x < 1 || a.dim_x > UR_MAXN) { set_error("bke_ukf_rts_smoother: dim_x must be in [1, %d]", UR_MAXN); return BKE_ERR_UNSUPPORTED; }
    if (int rc = check_dtype(a.dtype)) return rc;
    const bool fx_ok = a.fx_model == BKE_FX_LINEAR || a.fx_model == BKE_FX_CONST_VEL || (user_fx && a.fx_model == BKE_FX_USER);
    if (!fx_ok) { set_error("unknown fx_model %d", a.fx_model); return BKE_ERR_UNSUPPORTED; }
    if (a.fx_model == BKE_FX_CONST_VEL && (a.dim_x & 1)) { set_error("BKE_FX_CONST_VEL needs an even dim_x"); return BKE_ERR_BAD_ARG; }
    if (a.n_filters == 0 || a.n_steps == 0) return BKE_OK;
    if (!a.Xs || !a.Ps || !a.Q || !a.x_out || !a.P_out) { set_error("NULL argument"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model == BKE_FX_LINEAR && !a.F) { set_error("BKE_FX_LINEAR needs F"); return BKE_ERR_BAD_ARG; }
    return -1;
}

}  // namespace bke

using namespace bke;

extern "C" int bke_ukf_rts_smoother(const bke_ukf_rts_args *args, void *stream)
{
    if (!args) { set_error("args is NULL"); return BKE_ERR_BAD_ARG; }
    const bke_ukf_rts_args &a = *args;
    const int v = validate_ukf_rts(a, false);
    if (v >= 0) return v;
    if (a.Q_stride < 0 || a.F_stride < 0) { set_error("negative stride"); return BKE_ERR_BAD_ARG; }
    if (int rc = require_device()) return rc;
    return a.dtype == BKE_F32 ? launch_t<float>(a, (cudaStream_t)stream) : launch_t<double>(a, (cudaStream_t)stream);
}
