// ukf_score.cu — host side of bke_ukf_score: the pre-built instances of ukf_score_kernel.cuh, one per distinct
// (dim_x, dim_z, hx) of BKE_SIGMA_INSTANCES (the score does not run fx), for the Merwe and the simplex point set.
// A translation unit of its own leaves the code nvcc makes for the step instances (ukf.cu, ukf_simplex.cu) as it was.
// (The run-time compiled models carry their own instance: ukf_rtc.cu, bke_ukf_score_model.)
#include "sigma_launch.cuh"

namespace bke {
namespace {
using namespace ukfk;

template <typename T, int N, int M, int HX>
int launch_inst(const bke_ukf_score_args &a, cudaStream_t s)
{
    UkfScoreP<T> p;
    ukf_score_fill_params<T>(a, p);
    const bool spx = (a.flags & BKE_UKF_SIMPLEX) != 0, range = HX == BKE_HX_RANGE_AZ_EL || HX == BKE_HX_RANGE_BEARING;
    const size_t smem = ukf_score_smem_bytes<T>(N, M, spx, HX == BKE_HX_LINEAR, a.H_stride == 0);
    constexpr int OCC = ukf_occupancy(N, sizeof(T) == 8), OCC_SPX = ukf_occupancy(N, sizeof(T) == 8, true, range);
    const void *kern = spx ? (const void *)ukf_score_kernel<T, N, M, HX, OCC_SPX, true> : (const void *)ukf_score_kernel<T, N, M, HX, OCC, false>;
    return launch_kernel(kern, ukf_grid(p.N), UB, smem, &p, s, "ukf_score_kernel launch");
}

// a row of the instance table serves the score of its (dim_x, dim_z, hx); rows that differ in fx only repeat it
#define BKE_UKF_SCORE_ROW(NN, MM, FXX, HXX) \
    if (a.dim_x == NN && a.dim_z == MM && a.hx_model == HXX) return launch_inst<T, NN, MM, HXX>(a, s);

template <typename T>
int dispatch(const bke_ukf_score_args &a, cudaStream_t s)
{
    BKE_SIGMA_INSTANCES(BKE_UKF_SCORE_ROW)
    set_error("bke_ukf_score: no kernel instance for dim_x=%d dim_z=%d hx_model=%d", a.dim_x, a.dim_z, a.hx_model);
    return BKE_ERR_UNSUPPORTED;
}

#undef BKE_UKF_SCORE_ROW

}  // namespace

int launch_ukf_score(const bke_ukf_score_args &a, cudaStream_t s)
{
    return a.dtype == BKE_F32 ? dispatch<float>(a, s) : dispatch<double>(a, s);
}

}  // namespace bke
