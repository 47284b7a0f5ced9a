// ckf.cu — host side of the cubature Kalman filter bank: the closed set of pre-built (dim_x, dim_z, fx,
// hx) instances of the kernel in ckf_kernel.cuh, their launch and the argument checks shared by
// bke_ckf_step (api.cu) and bke_ckf_step_model (ukf_rtc.cu).
// (Instances around user-supplied fx / hx are compiled at run time: ukf_rtc.cu.)
#include "ckf_kernel.cuh"
#include "ckf_launch.cuh"

namespace bke {
namespace {
using namespace ckfk;

template <typename T, int N, int M, int FX, int HX>
int launch_inst(const bke_ckf_args &a, cudaStream_t s)
{
    CkfP<T> p;
    ckf_fill_params<T>(a, p);
    const size_t smem = ckf_smem_bytes<T>(N, M, FX == BKE_FX_LINEAR, a.F_stride == 0, HX == BKE_HX_LINEAR, a.H_stride == 0);
    constexpr int OCC = ckf_occupancy(N, sizeof(T) == 8);
    auto kern = ckf_has_extras(a) ? ckf_kernel<T, N, M, FX, HX, OCC, true> : ckf_kernel<T, N, M, FX, HX, OCC, false>;
    if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
    int64_t grid = (p.N + UB - 1) / UB;
    kern<<<(unsigned)grid, UB, smem, s>>>(p);
    return check_cuda(cudaGetLastError(), "ckf_kernel launch");
}

// the same (dim_x, dim_z, fx, hx) set as the UKF's (ukf.cu)
template <typename T>
int dispatch(const bke_ckf_args &a, cudaStream_t s)
{
    const int n = a.dim_x, m = a.dim_z, fx = a.fx_model, hx = a.hx_model;
#define BKE_CKF(NN, MM, FXX, HXX) \
    if (n == NN && m == MM && fx == FXX && hx == HXX) return launch_inst<T, NN, MM, FXX, HXX>(a, s);
    BKE_CKF(6, 3, BKE_FX_CONST_VEL, BKE_HX_RANGE_AZ_EL)
    BKE_CKF(6, 3, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
    BKE_CKF(6, 3, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_CKF(6, 3, BKE_FX_LINEAR, BKE_HX_RANGE_AZ_EL)
    BKE_CKF(4, 2, BKE_FX_CONST_VEL, BKE_HX_RANGE_BEARING)
    BKE_CKF(4, 2, BKE_FX_LINEAR, BKE_HX_RANGE_BEARING)
    BKE_CKF(4, 2, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
    BKE_CKF(4, 2, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_CKF(1, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_CKF(2, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_CKF(2, 1, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
    BKE_CKF(2, 2, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_CKF(3, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_CKF(3, 3, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_CKF(4, 4, BKE_FX_LINEAR, BKE_HX_LINEAR)
#undef BKE_CKF
    set_error("bke_ckf_step: no kernel instance for dim_x=%d dim_z=%d fx_model=%d hx_model=%d", n, m, fx, hx);
    return BKE_ERR_UNSUPPORTED;
}

}  // namespace

// checks common to bke_ckf_step and bke_ckf_step_model
int validate_ckf(const bke_ckf_args &a)
{
    if (a.n_filters < 0 || a.dim_x < 1 || a.dim_z < 1) { set_error("bad dimensions"); return BKE_ERR_BAD_ARG; }
    if (a.dtype != BKE_F32 && a.dtype != BKE_F64) { set_error("dtype must be BKE_F32 or BKE_F64"); return BKE_ERR_BAD_ARG; }
    if (!(a.flags & (BKE_DO_PREDICT | BKE_DO_UPDATE))) { set_error("flags selects neither predict nor update"); return BKE_ERR_BAD_ARG; }
    if (!a.x || !a.P || !a.x_out || !a.P_out) { set_error("x, P, x_out, P_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_PREDICT) && !a.Q) { set_error("predict needs Q"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_UPDATE) && (!a.R || !a.z)) { set_error("update needs R and z"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_UPDATE) && !(a.flags & BKE_DO_PREDICT) && !a.sigmas_f) {
        set_error("an update without predict reads the propagated points of the last predict: sigmas_f must be non-NULL");
        return BKE_ERR_BAD_ARG;
    }
    if (a.fx_model == BKE_FX_LINEAR && (a.flags & BKE_DO_PREDICT) && !a.F) { set_error("BKE_FX_LINEAR needs F"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model == BKE_HX_LINEAR && (a.flags & BKE_DO_UPDATE) && !a.H) { set_error("BKE_HX_LINEAR needs H"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model == BKE_FX_CONST_VEL && (a.dim_x & 1)) { set_error("BKE_FX_CONST_VEL needs an even dim_x"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int launch_ckf(const bke_ckf_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

}  // namespace bke
