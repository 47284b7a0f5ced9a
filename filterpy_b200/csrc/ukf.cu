// ukf.cu — host side of the unscented Kalman filter bank: the closed set of pre-built (dim_x, dim_z,
// fx, hx) instances of the kernel in ukf_kernel.cuh and their launch (Merwe points here, the simplex set
// in ukf_simplex.cu).  (Instances around user-supplied fx / hx are compiled at run time: ukf_rtc.cu.)
#include "ukf_kernel.cuh"
#include "ukf_launch.cuh"

namespace bke {

// the simplex instances of the same (dim_x, dim_z, fx, hx) set (ukf_simplex.cu)
template <typename T, int N, int M, int FX, int HX>
int launch_ukf_simplex(const bke_ukf_args &a, cudaStream_t s);

namespace {
using namespace ukfk;

template <typename T, int N, int M, int FX, int HX>
int launch_inst(const bke_ukf_args &a, cudaStream_t s)
{
    if (a.flags & BKE_UKF_SIMPLEX) return launch_ukf_simplex<T, N, M, FX, HX>(a, s);      // ukf_simplex.cu
    UkfP<T> p;
    ukf_fill_params<T>(a, N, p);
    const size_t smem = ukf_smem_bytes<T>(N, M, 2 * N + 1, FX == BKE_FX_LINEAR, a.F_stride == 0, HX == BKE_HX_LINEAR, a.H_stride == 0);
    constexpr int OCC = ukf_occupancy(N, sizeof(T) == 8);
    const bool ex = a.x_prior || a.P_prior || a.K || a.y || a.S || a.SI || a.log_likelihood;
    auto kern = ex ? ukf_kernel<T, N, M, FX, HX, OCC, true> : ukf_kernel<T, N, M, FX, HX, OCC, false>;
    if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
    int64_t grid = (p.N + UB - 1) / UB;
    kern<<<(unsigned)grid, UB, smem, s>>>(p);
    return check_cuda(cudaGetLastError(), "ukf_kernel launch");
}

template <typename T>
int dispatch(const bke_ukf_args &a, cudaStream_t s)
{
    const int n = a.dim_x, m = a.dim_z, fx = a.fx_model, hx = a.hx_model;
#define BKE_UKF(NN, MM, FXX, HXX) \
    if (n == NN && m == MM && fx == FXX && hx == HXX) return launch_inst<T, NN, MM, FXX, HXX>(a, s);
    BKE_UKF(6, 3, BKE_FX_CONST_VEL, BKE_HX_RANGE_AZ_EL)
    BKE_UKF(6, 3, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
    BKE_UKF(6, 3, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_UKF(6, 3, BKE_FX_LINEAR, BKE_HX_RANGE_AZ_EL)
    BKE_UKF(4, 2, BKE_FX_CONST_VEL, BKE_HX_RANGE_BEARING)
    BKE_UKF(4, 2, BKE_FX_LINEAR, BKE_HX_RANGE_BEARING)
    BKE_UKF(4, 2, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
    BKE_UKF(4, 2, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_UKF(1, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_UKF(2, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_UKF(2, 1, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
    BKE_UKF(2, 2, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_UKF(3, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_UKF(3, 3, BKE_FX_LINEAR, BKE_HX_LINEAR)
    BKE_UKF(4, 4, BKE_FX_LINEAR, BKE_HX_LINEAR)
#undef BKE_UKF
    set_error("bke_ukf_step: no kernel instance for dim_x=%d dim_z=%d fx_model=%d hx_model=%d", n, m, fx, hx);
    return BKE_ERR_UNSUPPORTED;
}

}  // namespace

int launch_ukf(const bke_ukf_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

}  // namespace bke
