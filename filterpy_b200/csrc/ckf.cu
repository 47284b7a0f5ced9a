// ckf.cu — host side of the cubature Kalman filter bank: the pre-built instances (BKE_SIGMA_INSTANCES) of
// the kernel in ckf_kernel.cuh and their launch.
// (Instances around user-supplied fx / hx are compiled at run time: ukf_rtc.cu.)
#include "sigma_launch.cuh"

namespace bke {
namespace {
using namespace ckfk;

template <typename T, int N, int M, int FX, int HX>
int launch_inst(const bke_ckf_args &a, cudaStream_t s)
{
    CkfP<T> p;
    ckf_fill_params<T>(a, p);
    const size_t smem = ukf_smem_bytes<T>(N, M, 2 * N, FX == BKE_FX_LINEAR, a.F_stride == 0, HX == BKE_HX_LINEAR, a.H_stride == 0);
    constexpr int OCC = ckf_occupancy(N, sizeof(T) == 8);
    auto kern = has_extras(a) ? ckf_kernel<T, N, M, FX, HX, OCC, true> : ckf_kernel<T, N, M, FX, HX, OCC, false>;
    return launch_kernel((const void *)kern, ukf_grid(p.N), UB, smem, &p, s, "ckf_kernel launch");
}

template <typename T>
int dispatch(const bke_ckf_args &a, cudaStream_t s)
{
    BKE_SIGMA_INSTANCES(BKE_SIGMA_DISPATCH_ROW)
    set_error("bke_ckf_step: no kernel instance for dim_x=%d dim_z=%d fx_model=%d hx_model=%d", a.dim_x, a.dim_z, a.fx_model, a.hx_model);
    return BKE_ERR_UNSUPPORTED;
}

}  // namespace

int launch_ckf(const bke_ckf_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

}  // namespace bke
