// enkf.cu — host side of the ensemble Kalman filter bank: the closed set of pre-built (dim_x, dim_z, fx, hx)
// instances of the kernel in enkf_kernel.cuh, the initialize kernel for every dim_x <= 16, their launch and
// the argument checks shared by bke_enkf_step (api.cu) and bke_enkf_step_model (ukf_rtc.cu).
// (Instances around user-supplied fx / hx are compiled at run time: ukf_rtc.cu.)
#include "enkf_launch.cuh"

namespace bke {
namespace {
using namespace enkfk;

template <typename T, int N, int M, int FX, int HX>
int launch_inst(const bke_enkf_args &a, cudaStream_t s)
{
    EnkfP<T> p;
    enkf_fill_params<T>(a, p);
    const size_t smem = enkf_smem_bytes(N, a.n_members, sizeof(T));
    auto kern = enkf_has_extras(a) ? enkf_kernel<T, N, M, FX, HX, true> : enkf_kernel<T, N, M, FX, HX, false>;
    if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
    kern<<<enkf_grid(p.N), EB, smem, s>>>(p);
    return check_cuda(cudaGetLastError(), "enkf_kernel launch");
}

// the same (dim_x, dim_z, fx, hx) set as the UKF's and the CKF's
template <typename T>
int dispatch(const bke_enkf_args &a, cudaStream_t s)
{
    const int n = a.dim_x, m = a.dim_z, fx = a.fx_model, hx = a.hx_model;
#define BKE_ENKF(NN, MM, FXX, HXX) \
    if (n == NN && m == MM && fx == FXX && hx == HXX) return launch_inst<T, NN, MM, FXX, HXX>(a, s);
    BKE_ENKF(6, 3, BKE_FX_CONST_VEL, BKE_HX_RANGE_AZ_EL)
    BKE_ENKF(6, 3, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
    BKE_ENKF(6, 3, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_ENKF(6, 3, BKE_FX_LINEAR, BKE_HX_RANGE_AZ_EL)
    BKE_ENKF(4, 2, BKE_FX_CONST_VEL, BKE_HX_RANGE_BEARING)
    BKE_ENKF(4, 2, BKE_FX_LINEAR, BKE_HX_RANGE_BEARING)
    BKE_ENKF(4, 2, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
    BKE_ENKF(4, 2, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_ENKF(1, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_ENKF(2, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_ENKF(2, 1, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
    BKE_ENKF(2, 2, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_ENKF(3, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_ENKF(3, 3, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_ENKF(4, 4, BKE_FX_LINEAR, BKE_HX_LINEAR)
#undef BKE_ENKF
    set_error("bke_enkf_step: no kernel instance for dim_x=%d dim_z=%d fx_model=%d hx_model=%d", n, m, fx, hx);
    return BKE_ERR_UNSUPPORTED;
}

template <typename T, int N>
int launch_init_inst(const EnkfInitP<T> &p, cudaStream_t s)
{
    enkf_init_kernel<T, N><<<enkf_grid(p.N), EB, 0, s>>>(p);
    return check_cuda(cudaGetLastError(), "enkf_init_kernel launch");
}

template <typename T>
int init_dispatch(const EnkfInitP<T> &p, int n, cudaStream_t s)
{
    switch (n) {
#define BKE_ENKF_INIT(NN) case NN: return launch_init_inst<T, NN>(p, s);
    BKE_ENKF_INIT(1) BKE_ENKF_INIT(2) BKE_ENKF_INIT(3) BKE_ENKF_INIT(4) BKE_ENKF_INIT(5) BKE_ENKF_INIT(6) BKE_ENKF_INIT(7)
    BKE_ENKF_INIT(8) BKE_ENKF_INIT(9) BKE_ENKF_INIT(10) BKE_ENKF_INIT(11) BKE_ENKF_INIT(12) BKE_ENKF_INIT(13)
    BKE_ENKF_INIT(14) BKE_ENKF_INIT(15) BKE_ENKF_INIT(16)
#undef BKE_ENKF_INIT
    }
    set_error("bke_enkf_initialize: dim_x must be 1..16");
    return BKE_ERR_BAD_ARG;
}

}  // namespace

// checks common to bke_enkf_step and bke_enkf_step_model
int validate_enkf(const bke_enkf_args &a)
{
    if (a.n_filters < 0 || a.dim_x < 1 || a.dim_x > 16 || a.dim_z < 1) { set_error("bad dimensions (1 <= dim_x <= 16, 1 <= dim_z)"); return BKE_ERR_BAD_ARG; }
    if (a.n_members < 2) { set_error("n_members must be 2 or greater (the covariances divide by n_members - 1)"); return BKE_ERR_BAD_ARG; }
    if (a.dtype != BKE_F32 && a.dtype != BKE_F64) { set_error("dtype must be BKE_F32 or BKE_F64"); return BKE_ERR_BAD_ARG; }
    if (!(a.flags & (BKE_DO_PREDICT | BKE_DO_UPDATE))) { set_error("flags selects neither predict nor update"); return BKE_ERR_BAD_ARG; }
    if (a.flags & ~(BKE_DO_PREDICT | BKE_DO_UPDATE)) { set_error("flags: only BKE_DO_PREDICT and BKE_DO_UPDATE apply to the EnKF"); return BKE_ERR_BAD_ARG; }
    if (!a.x || !a.P || !a.x_out || !a.P_out) { set_error("x, P, x_out, P_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if (!a.sigmas || !a.sigmas_out) { set_error("sigmas and sigmas_out must be non-NULL"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_PREDICT) && !a.Q) { set_error("predict needs Q"); return BKE_ERR_BAD_ARG; }
    if ((a.flags & BKE_DO_UPDATE) && (!a.R || !a.z)) { set_error("update needs R and z"); return BKE_ERR_BAD_ARG; }
    if (a.Q_stride < 0 || a.R_stride < 0 || a.F_stride < 0 || a.H_stride < 0) { set_error("negative model stride"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model == BKE_FX_LINEAR && (a.flags & BKE_DO_PREDICT) && !a.F) { set_error("BKE_FX_LINEAR needs F"); return BKE_ERR_BAD_ARG; }
    if (a.hx_model == BKE_HX_LINEAR && (a.flags & BKE_DO_UPDATE) && !a.H) { set_error("BKE_HX_LINEAR needs H"); return BKE_ERR_BAD_ARG; }
    if (a.fx_model == BKE_FX_CONST_VEL && (a.dim_x & 1)) { set_error("BKE_FX_CONST_VEL needs an even dim_x"); return BKE_ERR_BAD_ARG; }
    if (a.n_members > (1 << 24)) { set_error("n_members must be at most 2^24"); return BKE_ERR_BAD_ARG; }
    return BKE_OK;
}

int launch_enkf(const bke_enkf_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

int launch_enkf_init(int64_t n_filters, int32_t dim_x, int32_t n_members, int32_t dtype, uint32_t seed, uint32_t counter,
                     const void *x, const void *P, void *sigmas, int32_t *status, cudaStream_t s)
{
    if (dtype == BKE_F32) {
        EnkfInitP<float> p{n_filters, n_members, seed, counter, (const float *)x, (const float *)P, (float *)sigmas, status};
        return init_dispatch<float>(p, dim_x, s);
    }
    EnkfInitP<double> p{n_filters, n_members, seed, counter, (const double *)x, (const double *)P, (double *)sigmas, status};
    return init_dispatch<double>(p, dim_x, s);
}

}  // namespace bke
