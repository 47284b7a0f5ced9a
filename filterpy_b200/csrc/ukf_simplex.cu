// ukf_simplex.cu — the SimplexSigmaPoints instances (BKE_UKF_SIMPLEX) of the pre-built UKF kernel: the same
// (dim_x, dim_z, fx, hx) set as ukf.cu's dispatch table, which calls launch_ukf_simplex from its launch_inst.
// A translation unit of their own leaves the code nvcc makes for the Merwe instances as it was.
#include "ukf_kernel.cuh"
#include "ukf_launch.cuh"

namespace bke {

template <typename T, int N, int M, int FX, int HX>
int launch_ukf_simplex(const bke_ukf_args &a, cudaStream_t s)
{
    using namespace ukfk;
    UkfP<T> p;
    ukf_fill_params<T>(a, N, p);
    const size_t smem = ukf_smem_bytes<T>(N, M, N + 1, FX == BKE_FX_LINEAR, a.F_stride == 0, HX == BKE_HX_LINEAR, a.H_stride == 0);
    constexpr int OCC = ukf_occupancy(N, sizeof(T) == 8, true, HX == BKE_HX_RANGE_AZ_EL || HX == BKE_HX_RANGE_BEARING);
    const bool ex = a.x_prior || a.P_prior || a.K || a.y || a.S || a.SI || a.log_likelihood;
    auto kern = ex ? ukf_kernel<T, N, M, FX, HX, OCC, true, true> : ukf_kernel<T, N, M, FX, HX, OCC, false, true>;
    if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "cudaFuncSetAttribute")) return BKE_ERR_CUDA;
    int64_t grid = (p.N + UB - 1) / UB;
    kern<<<(unsigned)grid, UB, smem, s>>>(p);
    return check_cuda(cudaGetLastError(), "ukf_kernel (simplex) launch");
}

// an instance missing here that ukf.cu dispatches is an undefined symbol at link time
#define BKE_UKF_SPX(NN, MM, FXX, HXX)                                                                  \
    template int launch_ukf_simplex<float, NN, MM, FXX, HXX>(const bke_ukf_args &, cudaStream_t);      \
    template int launch_ukf_simplex<double, NN, MM, FXX, HXX>(const bke_ukf_args &, cudaStream_t);
BKE_UKF_SPX(6, 3, BKE_FX_CONST_VEL, BKE_HX_RANGE_AZ_EL)
BKE_UKF_SPX(6, 3, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
BKE_UKF_SPX(6, 3, BKE_FX_LINEAR, BKE_HX_LINEAR)
BKE_UKF_SPX(6, 3, BKE_FX_LINEAR, BKE_HX_RANGE_AZ_EL)
BKE_UKF_SPX(4, 2, BKE_FX_CONST_VEL, BKE_HX_RANGE_BEARING)
BKE_UKF_SPX(4, 2, BKE_FX_LINEAR, BKE_HX_RANGE_BEARING)
BKE_UKF_SPX(4, 2, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
BKE_UKF_SPX(4, 2, BKE_FX_LINEAR, BKE_HX_LINEAR)
BKE_UKF_SPX(1, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
BKE_UKF_SPX(2, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
BKE_UKF_SPX(2, 1, BKE_FX_CONST_VEL, BKE_HX_LINEAR)
BKE_UKF_SPX(2, 2, BKE_FX_LINEAR, BKE_HX_LINEAR)
BKE_UKF_SPX(3, 1, BKE_FX_LINEAR, BKE_HX_LINEAR)
BKE_UKF_SPX(3, 3, BKE_FX_LINEAR, BKE_HX_LINEAR)
BKE_UKF_SPX(4, 4, BKE_FX_LINEAR, BKE_HX_LINEAR)
#undef BKE_UKF_SPX

}  // namespace bke
