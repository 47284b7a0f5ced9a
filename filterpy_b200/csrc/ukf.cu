// ukf.cu — host side of the unscented Kalman filter bank: the pre-built instances (BKE_SIGMA_INSTANCES) of
// the kernel in ukf_kernel.cuh and their launch (Merwe points here, the simplex set in ukf_simplex.cu).
// (Instances around user-supplied fx / hx are compiled at run time: ukf_rtc.cu.)
#include "sigma_launch.cuh"

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
    auto kern = has_extras(a) ? ukf_kernel<T, N, M, FX, HX, OCC, true> : ukf_kernel<T, N, M, FX, HX, OCC, false>;
    return launch_kernel((const void *)kern, ukf_grid(p.N), UB, smem, &p, s, "ukf_kernel launch");
}

template <typename T>
int dispatch(const bke_ukf_args &a, cudaStream_t s)
{
    BKE_SIGMA_INSTANCES(BKE_SIGMA_DISPATCH_ROW)
    set_error("bke_ukf_step: no kernel instance for dim_x=%d dim_z=%d fx_model=%d hx_model=%d", a.dim_x, a.dim_z, a.fx_model, a.hx_model);
    return BKE_ERR_UNSUPPORTED;
}

}  // namespace

int launch_ukf(const bke_ukf_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

}  // namespace bke
