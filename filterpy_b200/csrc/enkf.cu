// enkf.cu — host side of the ensemble Kalman filter bank: the pre-built instances (BKE_SIGMA_INSTANCES) of
// the kernel in enkf_kernel.cuh, the initialize kernel for every dim_x <= 16 and their launch.
// (Instances around user-supplied fx / hx are compiled at run time: ukf_rtc.cu.)
#include "sigma_launch.cuh"

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
    return launch_kernel((const void *)kern, enkf_grid(p.N), EB, smem, &p, s, "enkf_kernel launch");
}

template <typename T>
int dispatch(const bke_enkf_args &a, cudaStream_t s)
{
    BKE_SIGMA_INSTANCES(BKE_SIGMA_DISPATCH_ROW)
    set_error("bke_enkf_step: no kernel instance for dim_x=%d dim_z=%d fx_model=%d hx_model=%d", a.dim_x, a.dim_z, a.fx_model, a.hx_model);
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
