// ukf_simplex.cu — the SimplexSigmaPoints instances (BKE_UKF_SIMPLEX) of the pre-built UKF kernel, one per
// row of BKE_SIGMA_INSTANCES; ukf.cu's launch_inst calls launch_ukf_simplex.
// A translation unit of their own leaves the code nvcc makes for the Merwe instances as it was.
#include "sigma_launch.cuh"

namespace bke {

template <typename T, int N, int M, int FX, int HX>
int launch_ukf_simplex(const bke_ukf_args &a, cudaStream_t s)
{
    using namespace ukfk;
    UkfP<T> p;
    ukf_fill_params<T>(a, N, p);
    const size_t smem = ukf_smem_bytes<T>(N, M, N + 1, FX == BKE_FX_LINEAR, a.F_stride == 0, HX == BKE_HX_LINEAR, a.H_stride == 0);
    constexpr int OCC = ukf_occupancy(N, sizeof(T) == 8, true, HX == BKE_HX_RANGE_AZ_EL || HX == BKE_HX_RANGE_BEARING);
    auto kern = has_extras(a) ? ukf_kernel<T, N, M, FX, HX, OCC, true, true> : ukf_kernel<T, N, M, FX, HX, OCC, false, true>;
    return launch_kernel((const void *)kern, ukf_grid(p.N), UB, smem, &p, s, "ukf_kernel (simplex) launch");
}

#define BKE_UKF_SPX(NN, MM, FXX, HXX)                                                                  \
    template int launch_ukf_simplex<float, NN, MM, FXX, HXX>(const bke_ukf_args &, cudaStream_t);      \
    template int launch_ukf_simplex<double, NN, MM, FXX, HXX>(const bke_ukf_args &, cudaStream_t);
BKE_SIGMA_INSTANCES(BKE_UKF_SPX)
#undef BKE_UKF_SPX

}  // namespace bke
