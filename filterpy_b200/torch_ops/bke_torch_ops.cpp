// torch.ops.bke.* — the C-ABI of include/bke.h exposed as PyTorch operators on CUDA tensors (zero copy:
// the tensors' device pointers go straight into the bke_* calls on the current CUDA stream).
// asks for this twin of the ctypes binding: the same entry points, no arithmetic of its own.
//   bke::kf_step              bke_kf_step              KalmanFilter.predict + update, kalman_filter.py:437-561
//   bke::kf_predict           bke_kf_step (predict)    kalman_filter.py:437-482
//   bke::kf_step_correlated   bke_kf_step_correlated   predict + update_correlated, kalman_filter.py:437-482, 670-752
//   bke::kf_update_rows       bke_kf_update_rows       predict + update_sequential, kalman_filter.py:437-482, 754-824
//   bke::ukf_step             bke_ukf_step             UnscentedKalmanFilter.predict + update, UKF.py:364-491
//   bke::ckf_step             bke_ckf_step             CubatureKalmanFilter.predict + update, CubatureKalmanFilter.py:292-389
//   bke::enkf_step            bke_enkf_step            EnsembleKalmanFilter.predict + update, ensemble_kalman_filter.py:218-290
//   bke::srkf_step            bke_srkf_step            SquareRootKalmanFilter.predict + update, square_root.py:172-248
//   bke::if_step              bke_if_step              InformationFilter.predict + update, information_filter.py:178-289
//   bke::poly_filter          bke_poly_filter          GHFilter / GHKFilter / GHFilterOrder / LeastSquaresFilter / FadingMemoryFilter
//                                                      update (T epochs) and the g-h batch_filter, gh_filter.py, least_squares.py, fading_memory.py
//   bke::score_measurements   bke_score_measurements   stats.mahalanobis / log_likelihood / logpdf / NEES and
//                                                      KalmanFilter.log_likelihood_of, N tracks x K candidates
//   bke::ukf_score_measurements  bke_ukf_score        UnscentedKalmanFilter.score_measurements: the log_likelihood and
//                                                      mahalanobis of update(z_ik), N tracks x K candidates, UKF.py:459-477
//   bke::imm_batch_filter     bke_imm_batch_filter     IMMEstimator.batch_filter: T epochs of predict(); update(z), IMM.py:160-247
//   bke::fls_smooth_batch     bke_fls_smooth           FixedLagSmoother.smooth_batch, fixed_lag_smoother.py:217-311
//   bke::systematic_resample  bke_systematic_resample  monte_carlo/resampling.py:117-150
//   bke::stratified_resample  bke_stratified_resample  monte_carlo/resampling.py:80-114
//   bke::systematic_resample_bank  bke_resample_bank   resampling.py:117-150 on every row of weights[B, M]
//   bke::stratified_resample_bank  bke_resample_bank   resampling.py:80-114 on every row of weights[B, M]
//   bke::multinomial_resample_bank bke_multinomial_resample_bank       resampling.py:153-176 per row
//   bke::residual_resample_bank    bke_residual_resample_bank_prepare / _search   resampling.py:27-76 per row
//   bke::systematic_resample_bank_if_degenerate  bke_resample_bank_gated   normalise, neff, resample + gather where
//   bke::stratified_resample_bank_if_degenerate  bke_resample_bank_gated   neff < threshold, in place, per row
//   bke::discrete_bayes_step  bke_db_step              discrete_bayes.py predict / update / normalize of every row
//                                                      of pdf[B, M]
#include <limits>

#include <ATen/ATen.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>
#include <cstring>
#include <tuple>
#include <vector>
#include "../../include/bke.h"

namespace {

void check_rc(int rc, const char *what)
{
    TORCH_CHECK(rc == BKE_OK, what, ": ", bke_last_error());
}

int dtype_of(const at::Tensor &t)
{
    TORCH_CHECK(t.scalar_type() == at::kFloat || t.scalar_type() == at::kDouble, "bke: tensors must be float32 or float64");
    return t.scalar_type() == at::kFloat ? BKE_F32 : BKE_F64;
}

// a model is either shared by the bank ([r, c] -> stride 0) or dense per filter ([N, r, c])
const void *model(const at::Tensor &t, int64_t N, int64_t r, int64_t c, int64_t *stride, const at::Tensor &like, const char *name)
{
    TORCH_CHECK(t.is_cuda() && t.is_contiguous() && t.scalar_type() == like.scalar_type(), "bke: ", name, " must be a contiguous CUDA tensor of the state's dtype");
    if (t.dim() == 2) { TORCH_CHECK(t.size(0) == r && t.size(1) == c, "bke: bad shape for ", name); *stride = 0; }
    else { TORCH_CHECK(t.dim() == 3 && t.size(0) == N && t.size(1) == r && t.size(2) == c, "bke: bad shape for ", name); *stride = r * c; }
    return t.data_ptr();
}

// the form of update a kf_run call makes after its predict
struct KfForm {
    const at::Tensor *M = nullptr;          // update_correlated
    int64_t start = -1, rows = 0;           // update_sequential's block (z is then [N, rows])
};

std::tuple<at::Tensor, at::Tensor> kf_run(const at::Tensor &x, const at::Tensor &P, const at::Tensor &F, const at::Tensor &H,
                                          const at::Tensor &Q, const at::Tensor &R, const c10::optional<at::Tensor> &z,
                                          double alpha_sq, unsigned flags, const KfForm &form = KfForm())
{
    TORCH_CHECK(x.is_cuda() && P.is_cuda() && x.is_contiguous() && P.is_contiguous(), "bke: x and P must be contiguous CUDA tensors");
    TORCH_CHECK(x.dim() == 2 && P.dim() == 3 && P.size(0) == x.size(0) && P.size(1) == x.size(1) && P.size(2) == x.size(1), "bke: x is [N, n], P is [N, n, n]");
    TORCH_CHECK(P.scalar_type() == x.scalar_type(), "bke: x and P must share a dtype");
    c10::cuda::CUDAGuard guard(x.device());
    const int64_t N = x.size(0), n = x.size(1);
    bke_kf_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_filters = N; a.dim_x = (int32_t)n; a.dtype = dtype_of(x); a.flags = flags; a.alpha_sq = alpha_sq;
    at::Tensor x_out = at::empty_like(x), P_out = at::empty_like(P);
    a.x = x.data_ptr(); a.P = P.data_ptr(); a.x_out = x_out.data_ptr(); a.P_out = P_out.data_ptr();
    a.F = model(F, N, n, n, &a.F_stride, x, "F");
    a.Q = model(Q, N, n, n, &a.Q_stride, x, "Q");
    int64_t m = H.size(-2);
    a.dim_z = (int32_t)m;
    a.H = model(H, N, m, n, &a.H_stride, x, "H");
    a.R = model(R, N, m, m, &a.R_stride, x, "R");
    if (flags & BKE_DO_UPDATE) {
        TORCH_CHECK(z.has_value(), "bke: update needs z");
        const at::Tensor &zz = *z;
        const int64_t zm = form.start >= 0 ? form.rows : m;
        TORCH_CHECK(zz.is_cuda() && zz.is_contiguous() && zz.scalar_type() == x.scalar_type() && zz.dim() == 2 && zz.size(0) == N && zz.size(1) == zm, "bke: z is [N, m] (z_i [N, L] for a block)");
        a.z = zz.data_ptr();
    }
    void *stream = (void *)c10::cuda::getCurrentCUDAStream().stream();
    if (form.M) {
        int64_t sM = 0;
        const void *Mp = model(*form.M, N, n, m, &sM, x, "M");
        check_rc(bke_kf_step_correlated(&a, Mp, sM, stream), "bke_kf_step_correlated");
    } else if (form.start >= 0) {
        bke_kf_rows_args r;
        std::memset(&r, 0, sizeof(r));
        r.step = a; r.start = (int32_t)form.start; r.rows = (int32_t)form.rows;
        check_rc(bke_kf_update_rows(&r, stream), "bke_kf_update_rows");
    } else {
        check_rc(bke_kf_step(&a, stream), "bke_kf_step");
    }
    return std::make_tuple(x_out, P_out);
}

std::tuple<at::Tensor, at::Tensor> kf_step(const at::Tensor &x, const at::Tensor &P, const at::Tensor &F, const at::Tensor &H,
                                           const at::Tensor &Q, const at::Tensor &R, const at::Tensor &z, double alpha_sq)
{
    return kf_run(x, P, F, H, Q, R, z, alpha_sq, BKE_DO_PREDICT | BKE_DO_UPDATE);
}

std::tuple<at::Tensor, at::Tensor> kf_step_correlated(const at::Tensor &x, const at::Tensor &P, const at::Tensor &F, const at::Tensor &H,
                                                      const at::Tensor &Q, const at::Tensor &R, const at::Tensor &M, const at::Tensor &z,
                                                      double alpha_sq)
{
    KfForm form;
    form.M = &M;
    return kf_run(x, P, F, H, Q, R, z, alpha_sq, BKE_DO_PREDICT | BKE_DO_UPDATE, form);
}

// H and R are the bank's full [.,m,n] / [.,m,m]: the block's rows are read in place
std::tuple<at::Tensor, at::Tensor> kf_update_rows(const at::Tensor &x, const at::Tensor &P, const at::Tensor &F, const at::Tensor &H,
                                                  const at::Tensor &Q, const at::Tensor &R, const at::Tensor &z_i, int64_t start,
                                                  double alpha_sq)
{
    KfForm form;
    form.start = start;
    form.rows = z_i.dim() == 2 ? z_i.size(1) : 0;
    return kf_run(x, P, F, H, Q, R, z_i, alpha_sq, BKE_DO_PREDICT | BKE_DO_UPDATE, form);
}

std::tuple<at::Tensor, at::Tensor> kf_predict(const at::Tensor &x, const at::Tensor &P, const at::Tensor &F, const at::Tensor &Q, double alpha_sq)
{
    // H / R are not read by a predict-only call; hand the ABI placeholders of a legal shape
    at::Tensor H = at::zeros({1, x.size(1)}, x.options()), R = at::ones({1, 1}, x.options());
    return kf_run(x, P, F, H, Q, R, c10::nullopt, alpha_sq, BKE_DO_PREDICT);
}

std::tuple<at::Tensor, at::Tensor> ukf_step(const at::Tensor &x, const at::Tensor &P, const at::Tensor &Q, const at::Tensor &R,
                                            const at::Tensor &z, double dt, double alpha, double beta, double kappa,
                                            int64_t fx_model, int64_t hx_model, const c10::optional<at::Tensor> &F,
                                            const c10::optional<at::Tensor> &H, bool simplex)
{
    TORCH_CHECK(x.is_cuda() && P.is_cuda() && x.is_contiguous() && P.is_contiguous() && x.dim() == 2 && P.dim() == 3, "bke: x is [N, n], P is [N, n, n] on the GPU");
    c10::cuda::CUDAGuard guard(x.device());
    const int64_t N = x.size(0), n = x.size(1), m = z.size(1);
    bke_ukf_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_filters = N; a.dim_x = (int32_t)n; a.dim_z = (int32_t)m; a.dtype = dtype_of(x);
    a.flags = BKE_DO_PREDICT | BKE_DO_UPDATE; a.fx_model = (int32_t)fx_model; a.hx_model = (int32_t)hx_model;
    a.dt = dt; a.alpha = alpha; a.beta = beta; a.kappa = kappa;
    if (simplex) a.flags |= BKE_UKF_SIMPLEX;                   // SimplexSigmaPoints: alpha, beta, kappa ignored
    at::Tensor x_out = at::empty_like(x), P_out = at::empty_like(P);
    a.x = x.data_ptr(); a.P = P.data_ptr(); a.x_out = x_out.data_ptr(); a.P_out = P_out.data_ptr();
    a.Q = model(Q, N, n, n, &a.Q_stride, x, "Q");
    a.R = model(R, N, m, m, &a.R_stride, x, "R");
    if (F.has_value()) a.F = model(*F, N, n, n, &a.F_stride, x, "F");
    if (H.has_value()) a.H = model(*H, N, m, n, &a.H_stride, x, "H");
    TORCH_CHECK(z.is_cuda() && z.is_contiguous() && z.scalar_type() == x.scalar_type() && z.dim() == 2 && z.size(0) == N, "bke: z is [N, m]");
    a.z = z.data_ptr();
    check_rc(bke_ukf_step(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_ukf_step");
    return std::make_tuple(x_out, P_out);
}

std::tuple<at::Tensor, at::Tensor> ckf_step(const at::Tensor &x, const at::Tensor &P, const at::Tensor &Q, const at::Tensor &R,
                                            const at::Tensor &z, double dt, int64_t fx_model, int64_t hx_model,
                                            const c10::optional<at::Tensor> &F, const c10::optional<at::Tensor> &H)
{
    TORCH_CHECK(x.is_cuda() && P.is_cuda() && x.is_contiguous() && P.is_contiguous() && x.dim() == 2 && P.dim() == 3, "bke: x is [N, n], P is [N, n, n] on the GPU");
    c10::cuda::CUDAGuard guard(x.device());
    const int64_t N = x.size(0), n = x.size(1), m = z.size(1);
    bke_ckf_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_filters = N; a.dim_x = (int32_t)n; a.dim_z = (int32_t)m; a.dtype = dtype_of(x);
    a.flags = BKE_DO_PREDICT | BKE_DO_UPDATE; a.fx_model = (int32_t)fx_model; a.hx_model = (int32_t)hx_model;
    a.dt = dt;
    at::Tensor x_out = at::empty_like(x), P_out = at::empty_like(P);
    a.x = x.data_ptr(); a.P = P.data_ptr(); a.x_out = x_out.data_ptr(); a.P_out = P_out.data_ptr();
    a.Q = model(Q, N, n, n, &a.Q_stride, x, "Q");
    a.R = model(R, N, m, m, &a.R_stride, x, "R");
    if (F.has_value()) a.F = model(*F, N, n, n, &a.F_stride, x, "F");
    if (H.has_value()) a.H = model(*H, N, m, n, &a.H_stride, x, "H");
    TORCH_CHECK(z.is_cuda() && z.is_contiguous() && z.scalar_type() == x.scalar_type() && z.dim() == 2 && z.size(0) == N, "bke: z is [N, m]");
    a.z = z.data_ptr();
    check_rc(bke_ckf_step(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_ckf_step");
    return std::make_tuple(x_out, P_out);
}

// one fused EnKF epoch on sigmas[N, members, n]; the caller owns the noise stream's (seed, counter) and
// advances counter by 2 per call (a predict and an update draw)
std::tuple<at::Tensor, at::Tensor, at::Tensor> enkf_step(const at::Tensor &x, const at::Tensor &P, const at::Tensor &sigmas,
                                                         const at::Tensor &Q, const at::Tensor &R, const at::Tensor &z, double dt,
                                                         int64_t fx_model, int64_t hx_model, int64_t seed, int64_t counter,
                                                         const c10::optional<at::Tensor> &F, const c10::optional<at::Tensor> &H)
{
    TORCH_CHECK(x.is_cuda() && P.is_cuda() && x.is_contiguous() && P.is_contiguous() && x.dim() == 2 && P.dim() == 3, "bke: x is [N, n], P is [N, n, n] on the GPU");
    TORCH_CHECK(sigmas.is_cuda() && sigmas.is_contiguous() && sigmas.dim() == 3 && sigmas.size(0) == x.size(0) && sigmas.size(2) == x.size(1)
                && sigmas.scalar_type() == x.scalar_type(), "bke: sigmas is [N, members, n] of the state's dtype");
    TORCH_CHECK(seed >= 0 && seed <= 0xffffffffLL && counter >= 0 && counter <= 0xffffffffLL, "bke: seed and counter are uint32");
    c10::cuda::CUDAGuard guard(x.device());
    const int64_t N = x.size(0), n = x.size(1), m = z.size(1);
    bke_enkf_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_filters = N; a.dim_x = (int32_t)n; a.dim_z = (int32_t)m; a.n_members = (int32_t)sigmas.size(1); a.dtype = dtype_of(x);
    a.flags = BKE_DO_PREDICT | BKE_DO_UPDATE; a.fx_model = (int32_t)fx_model; a.hx_model = (int32_t)hx_model;
    a.seed = (uint32_t)seed; a.counter = (uint32_t)counter;
    a.dt = dt;
    at::Tensor x_out = at::empty_like(x), P_out = at::empty_like(P), s_out = at::empty_like(sigmas);
    a.x = x.data_ptr(); a.P = P.data_ptr(); a.x_out = x_out.data_ptr(); a.P_out = P_out.data_ptr();
    a.sigmas = sigmas.data_ptr(); a.sigmas_out = s_out.data_ptr();
    a.Q = model(Q, N, n, n, &a.Q_stride, x, "Q");
    a.R = model(R, N, m, m, &a.R_stride, x, "R");
    if (F.has_value()) a.F = model(*F, N, n, n, &a.F_stride, x, "F");
    if (H.has_value()) a.H = model(*H, N, m, n, &a.H_stride, x, "H");
    TORCH_CHECK(z.is_cuda() && z.is_contiguous() && z.scalar_type() == x.scalar_type() && z.dim() == 2 && z.size(0) == N, "bke: z is [N, m]");
    a.z = z.data_ptr();
    check_rc(bke_enkf_step(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_enkf_step");
    return std::make_tuple(x_out, P_out, s_out);
}

std::tuple<at::Tensor, at::Tensor> srkf_step(const at::Tensor &x, const at::Tensor &L, const at::Tensor &F, const at::Tensor &H,
                                             const at::Tensor &Lq, const at::Tensor &Lr, const at::Tensor &z)
{
    TORCH_CHECK(x.is_cuda() && L.is_cuda() && x.is_contiguous() && L.is_contiguous(), "bke: x and L must be contiguous CUDA tensors");
    TORCH_CHECK(x.dim() == 2 && L.dim() == 3 && L.size(0) == x.size(0) && L.size(1) == x.size(1) && L.size(2) == x.size(1), "bke: x is [N, n], L is [N, n, n]");
    TORCH_CHECK(L.scalar_type() == x.scalar_type(), "bke: x and L must share a dtype");
    c10::cuda::CUDAGuard guard(x.device());
    const int64_t N = x.size(0), n = x.size(1), m = H.size(-2);
    bke_srkf_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_filters = N; a.dim_x = (int32_t)n; a.dim_z = (int32_t)m; a.dtype = dtype_of(x);
    a.flags = BKE_DO_PREDICT | BKE_DO_UPDATE;
    at::Tensor x_out = at::empty_like(x), L_out = at::empty_like(L);
    a.x = x.data_ptr(); a.L = L.data_ptr(); a.x_out = x_out.data_ptr(); a.L_out = L_out.data_ptr();
    a.F = model(F, N, n, n, &a.F_stride, x, "F");
    a.H = model(H, N, m, n, &a.H_stride, x, "H");
    a.Lq = model(Lq, N, n, n, &a.Lq_stride, x, "Lq");
    a.Lr = model(Lr, N, m, m, &a.Lr_stride, x, "Lr");
    TORCH_CHECK(z.is_cuda() && z.is_contiguous() && z.scalar_type() == x.scalar_type() && z.dim() == 2 && z.size(0) == N && z.size(1) == m, "bke: z is [N, m]");
    a.z = z.data_ptr();
    check_rc(bke_srkf_step(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_srkf_step");
    return std::make_tuple(x_out, L_out);
}

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor> if_step(const at::Tensor &x, const at::Tensor &P_inv, const at::Tensor &no_information,
                                                       const at::Tensor &F, const at::Tensor &F_inv, const at::Tensor &Q,
                                                       const at::Tensor &H, const at::Tensor &R_inv, const at::Tensor &z)
{
    TORCH_CHECK(x.is_cuda() && P_inv.is_cuda() && x.is_contiguous() && P_inv.is_contiguous(), "bke: x and P_inv must be contiguous CUDA tensors");
    TORCH_CHECK(x.dim() == 2 && P_inv.dim() == 3 && P_inv.size(0) == x.size(0) && P_inv.size(1) == x.size(1) && P_inv.size(2) == x.size(1),
                "bke: x is [N, n], P_inv is [N, n, n]");
    TORCH_CHECK(P_inv.scalar_type() == x.scalar_type(), "bke: x and P_inv must share a dtype");
    TORCH_CHECK(no_information.is_cuda() && no_information.scalar_type() == at::kByte && no_information.dim() == 1 &&
                no_information.size(0) == x.size(0), "bke: no_information is a uint8 CUDA tensor [N]");
    c10::cuda::CUDAGuard guard(x.device());
    const int64_t N = x.size(0), n = x.size(1), m = H.size(-2);
    bke_if_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_filters = N; a.dim_x = (int32_t)n; a.dim_z = (int32_t)m; a.dtype = dtype_of(x);
    a.flags = BKE_DO_PREDICT | BKE_DO_UPDATE;
    a.ll_mode = BKE_IF_LL_NONE;
    at::Tensor x_out = at::empty_like(x), P_out = at::empty_like(P_inv), ni_out = no_information.contiguous().clone();
    at::Tensor status = at::empty({N}, x.options().dtype(at::kInt));   // BKE_STATUS_SINGULAR_S where an inv raises
    a.x = x.data_ptr(); a.P_inv = P_inv.data_ptr(); a.x_out = x_out.data_ptr(); a.P_inv_out = P_out.data_ptr();
    a.no_information = ni_out.data_ptr<uint8_t>();
    a.status = status.data_ptr<int32_t>();
    a.F = model(F, N, n, n, &a.F_stride, x, "F");
    a.F_inv = model(F_inv, N, n, n, &a.F_inv_stride, x, "F_inv");
    a.Q = model(Q, N, n, n, &a.Q_stride, x, "Q");
    a.H = model(H, N, m, n, &a.H_stride, x, "H");
    a.R_inv = model(R_inv, N, m, m, &a.R_inv_stride, x, "R_inv");
    TORCH_CHECK(z.is_cuda() && z.is_contiguous() && z.scalar_type() == x.scalar_type() && z.dim() == 2 && z.size(0) == N && z.size(1) == m, "bke: z is [N, m]");
    a.z = z.data_ptr();
    check_rc(bke_if_step(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_if_step");
    return std::make_tuple(x_out, P_out, ni_out, status);
}

// N tracks against K candidates (bke_score_measurements): z is [N, K, m] or [1, K, m] (one scan shared by every
// track); exactly one of x [N, n] and mean [N, m]; P (with R) or S; H, R, S shared [r, c] or per track [N, r, c];
// valid [N, K] uint8.  `outputs` names the outputs wanted, returned in that order: zhat, y, d2, mahalanobis,
// log_likelihood, likelihood, status.  Every tensor must be on z's device.
std::vector<at::Tensor> score_measurements(const at::Tensor &z, const c10::optional<at::Tensor> &x,
                                           const c10::optional<at::Tensor> &mean, const c10::optional<at::Tensor> &P,
                                           const c10::optional<at::Tensor> &S, const c10::optional<at::Tensor> &H,
                                           const c10::optional<at::Tensor> &R, const c10::optional<at::Tensor> &valid,
                                           c10::ArrayRef<c10::string_view> outputs)
{
    TORCH_CHECK(z.is_cuda() && z.is_contiguous() && z.dim() == 3, "bke: z is a contiguous CUDA tensor [N, K, m] or [1, K, m]");
    const int dt = dtype_of(z);
    auto given = [](const c10::optional<at::Tensor> &t) { return t.has_value() && t->defined(); };
    auto check = [&](const c10::optional<at::Tensor> &t, const char *name) {
        if (!given(t)) return (const void *)nullptr;
        TORCH_CHECK(t->is_cuda() && t->device() == z.device() && t->is_contiguous() && t->scalar_type() == z.scalar_type(),
                    "bke: ", name, " must be a contiguous CUDA tensor of z's dtype, on z's device");
        return (const void *)t->data_ptr();
    };
    TORCH_CHECK(given(x) != given(mean), "bke: exactly one of x and mean");
    const at::Tensor &src = given(x) ? *x : *mean;
    TORCH_CHECK(src.dim() == 2, "bke: x is [N, n], mean is [N, m]");
    const int64_t N = src.size(0), K = z.size(1), m = z.size(2);
    TORCH_CHECK(z.size(0) == N || z.size(0) == 1, "bke: z is [N, K, m] or [1, K, m]");
    const int64_t n = given(x) ? x->size(1) : (given(P) ? P->size(-1) : m);
    c10::cuda::CUDAGuard guard(z.device());
    bke_score_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_tracks = N; a.n_candidates = K; a.dim_x = (int32_t)n; a.dim_z = (int32_t)m; a.dtype = dt;
    a.x = check(x, "x"); a.mean = check(mean, "mean");
    if (given(mean)) TORCH_CHECK(mean->size(1) == m, "bke: mean is [N, m]");
    a.P = check(P, "P");
    if (given(P)) TORCH_CHECK(P->dim() == 3 && P->size(0) == N && P->size(1) == n && P->size(2) == n, "bke: P is [N, n, n]");
    if (given(S)) { check(S, "S"); a.S = model(*S, N, m, m, &a.S_stride, z, "S"); }
    if (given(H)) { check(H, "H"); a.H = model(*H, N, m, n, &a.H_stride, z, "H"); }
    if (given(R)) { check(R, "R"); a.R = model(*R, N, m, m, &a.R_stride, z, "R"); }
    a.z = z.data_ptr(); a.z_track_stride = z.size(0) == 1 ? 0 : K * m; a.z_cand_stride = m;
    if (given(valid)) {
        TORCH_CHECK(valid->is_cuda() && valid->device() == z.device() && valid->scalar_type() == at::kByte &&
                    valid->is_contiguous() && valid->numel() == N * K, "bke: valid is a contiguous uint8 CUDA tensor [N, K] on z's device");
        a.z_valid = valid->data_ptr<uint8_t>();
    }
    std::vector<at::Tensor> out;
    for (const auto &name : outputs) {
        at::Tensor t;
        if (name == "zhat") { t = at::empty({N, m}, z.options()); a.zhat = t.data_ptr(); }
        else if (name == "y") { t = at::empty({N, K, m}, z.options()); a.y = t.data_ptr(); }
        else if (name == "d2") { t = at::empty({N, K}, z.options()); a.d2 = t.data_ptr(); }
        else if (name == "mahalanobis") { t = at::empty({N, K}, z.options()); a.mahalanobis = t.data_ptr(); }
        else if (name == "log_likelihood") { t = at::empty({N, K}, z.options()); a.log_likelihood = t.data_ptr(); }
        else if (name == "likelihood") { t = at::empty({N, K}, z.options()); a.likelihood = t.data_ptr(); }
        else if (name == "status") { t = at::empty({N}, z.options().dtype(at::kInt)); a.status = t.data_ptr<int32_t>(); }
        else TORCH_CHECK(false, "bke: unknown output ", name);
        out.push_back(t);
    }
    if (N > 0 && K > 0)     // an empty tensor has no data pointer to pass
        check_rc(bke_score_measurements(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_score_measurements");
    return out;
}

// N UKF tracks against K candidates (bke_ukf_score, pre-built hx models): x [N, n], P [N, n, n], R and H shared
// [r, c] or per track [N, r, c], z [N, K, m] or [1, K, m], valid [N, K] uint8.  Returns (log_likelihood, mahalanobis,
// status), [N, K], [N, K] and [N].
std::tuple<at::Tensor, at::Tensor, at::Tensor> ukf_score_measurements(const at::Tensor &x, const at::Tensor &P, const at::Tensor &R,
                                                                      const at::Tensor &z, double alpha, double beta, double kappa,
                                                                      int64_t hx_model, const c10::optional<at::Tensor> &H,
                                                                      const c10::optional<at::Tensor> &valid, bool simplex)
{
    TORCH_CHECK(x.is_cuda() && P.is_cuda() && x.is_contiguous() && P.is_contiguous() && x.dim() == 2 && P.dim() == 3, "bke: x is [N, n], P is [N, n, n] on the GPU");
    TORCH_CHECK(z.is_cuda() && z.device() == x.device() && z.is_contiguous() && z.scalar_type() == x.scalar_type() && z.dim() == 3,
                "bke: z is a contiguous CUDA tensor [N, K, m] or [1, K, m] of x's dtype, on x's device");
    c10::cuda::CUDAGuard guard(x.device());
    const int64_t N = x.size(0), n = x.size(1), K = z.size(1), m = z.size(2);
    TORCH_CHECK(z.size(0) == N || z.size(0) == 1, "bke: z is [N, K, m] or [1, K, m]");
    bke_ukf_score_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_filters = N; a.n_candidates = K; a.dim_x = (int32_t)n; a.dim_z = (int32_t)m; a.dtype = dtype_of(x);
    a.flags = simplex ? BKE_UKF_SIMPLEX : 0u; a.hx_model = (int32_t)hx_model;
    a.alpha = alpha; a.beta = beta; a.kappa = kappa;
    a.x = x.data_ptr(); a.P = P.data_ptr();
    a.R = model(R, N, m, m, &a.R_stride, x, "R");
    if (H.has_value() && H->defined()) a.H = model(*H, N, m, n, &a.H_stride, x, "H");
    a.z = z.data_ptr(); a.z_track_stride = z.size(0) == 1 ? 0 : K * m; a.z_cand_stride = m;
    if (valid.has_value() && valid->defined()) {
        TORCH_CHECK(valid->is_cuda() && valid->device() == x.device() && valid->scalar_type() == at::kByte &&
                    valid->is_contiguous() && valid->numel() == N * K, "bke: valid is a contiguous uint8 CUDA tensor [N, K] on x's device");
        a.z_valid = valid->data_ptr<uint8_t>();
    }
    at::Tensor ll = at::empty({N, K}, x.options()), maha = at::empty({N, K}, x.options());
    at::Tensor status = at::empty({N}, x.options().dtype(at::kInt));
    a.log_likelihood = ll.data_ptr(); a.mahalanobis = maha.data_ptr(); a.status = status.data_ptr<int32_t>();
    if (N > 0 && K > 0)     // an empty tensor has no data pointer to pass
        check_rc(bke_ukf_score(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_ukf_score");
    return std::make_tuple(ll, maha, status);
}

// a polynomial tracker parameter: 0-d (shared, stride 0) or [N] (per filter, stride 1); undefined = not given
const void *poly_param(const c10::optional<at::Tensor> &t, int64_t N, int64_t *stride, const at::Tensor &like, const char *name)
{
    if (!t.has_value() || !t->defined()) return nullptr;
    TORCH_CHECK(t->is_cuda() && t->device() == like.device() && t->is_contiguous() && t->scalar_type() == like.scalar_type(),
                "bke: ", name, " must be a contiguous CUDA tensor of the state's dtype, on its device");
    TORCH_CHECK(t->dim() == 0 || (t->dim() == 1 && t->size(0) == N), "bke: ", name, " is 0-d (shared) or [N]");
    *stride = t->dim() == 0 ? 0 : 1;
    return t->data_ptr();
}

// T epochs of update() (batch = false) or batch_filter (batch = true) on z[T, N].  Returns (x, dx, ddx, n, results,
// predictions): the state after the call (the input state for batch), results[T+1, N, W] and, for the g-h batch,
// predictions[T, N]; what the family does not have is an empty tensor.  The inputs are not modified.
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> poly_filter(
    const at::Tensor &x, const c10::optional<at::Tensor> &dx, const c10::optional<at::Tensor> &ddx,
    const c10::optional<at::Tensor> &n, const at::Tensor &z, const c10::optional<at::Tensor> &g,
    const c10::optional<at::Tensor> &h, const c10::optional<at::Tensor> &k, const c10::optional<at::Tensor> &dt,
    const c10::optional<at::Tensor> &dt2, const c10::optional<at::Tensor> &hdt2, int64_t family, int64_t order, bool batch)
{
    TORCH_CHECK(family >= BKE_POLY_GH && family <= BKE_POLY_FADING, "bke: family must be one of BKE_POLY_*");
    const bool gh = family == BKE_POLY_GH || family == BKE_POLY_GHK;
    TORCH_CHECK(gh || (order >= 0 && order <= 2), "bke: order must be between 0 and 2");
    // the kernel indexes x as [N] (GH / GHK) or [N, order+1] and the call carries no size for it: check the shape here
    TORCH_CHECK(x.is_cuda(), "bke: x must be a CUDA tensor");
    if (gh) {
        TORCH_CHECK(x.dim() == 1, "bke: x of GH / GHK is [N] (dx and ddx are separate tensors)");
    } else {
        TORCH_CHECK(x.dim() == 2 && x.size(1) == order + 1, "bke: x is [N, order+1] = [N, ", order + 1, "], got ", x.sizes());
    }
    c10::cuda::CUDAGuard guard(x.device());
    const int64_t N = x.size(0);
    TORCH_CHECK(z.is_cuda() && z.device() == x.device() && z.is_contiguous() && z.scalar_type() == x.scalar_type() &&
                z.dim() == 2 && z.size(1) == N, "bke: z is [T, N] in the state's dtype, on x's device");
    bke_poly_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_filters = N; a.n_steps = z.size(0); a.family = (int32_t)family; a.order = (int32_t)order; a.dtype = dtype_of(x);
    a.mode = batch ? BKE_POLY_BATCH : BKE_POLY_UPDATE;
    auto state = [&](const c10::optional<at::Tensor> &t, const char *name) {
        if (!t.has_value() || !t->defined()) return at::Tensor();
        TORCH_CHECK(t->is_cuda() && t->device() == x.device() && t->scalar_type() == x.scalar_type() && t->dim() == 1 &&
                    t->size(0) == N, "bke: ", name, " is a CUDA tensor [N] of x's dtype, on x's device");
        return t->contiguous().clone();
    };
    at::Tensor x_out = x.contiguous().clone(), dx_out = state(dx, "dx"), ddx_out = state(ddx, "ddx"), n_out;
    a.x = x_out.data_ptr();
    a.dx = dx_out.defined() ? dx_out.data_ptr() : nullptr;
    a.ddx = ddx_out.defined() ? ddx_out.data_ptr() : nullptr;
    if (family == BKE_POLY_LSQ) {
        TORCH_CHECK(n.has_value() && n->is_cuda() && n->device() == x.device() && n->scalar_type() == at::kLong && n->dim() == 1 && n->size(0) == N,
                    "bke: LSQ needs the counter n, an int64 CUDA tensor [N]");
        n_out = n->contiguous().clone();
        a.n = n_out.data_ptr<int64_t>();
        a.n_max = N ? n_out.max().item<int64_t>() : 0;
    }
    a.g = poly_param(g, N, &a.g_stride, x, "g");
    a.h = poly_param(h, N, &a.h_stride, x, "h");
    a.k = poly_param(k, N, &a.k_stride, x, "k");
    a.dt = poly_param(dt, N, &a.dt_stride, x, "dt");
    a.dt2 = poly_param(dt2, N, &a.dt2_stride, x, "dt2");
    a.hdt2 = poly_param(hdt2, N, &a.hdt2_stride, x, "hdt2");
    a.z = z.data_ptr();
    const int64_t W = gh ? 2 : order + 1;
    at::Tensor results = at::empty({z.size(0) + 1, N, W}, x.options()), predictions;
    a.results = results.data_ptr();
    if (gh && batch) {
        predictions = at::empty({z.size(0), N}, x.options());
        a.predictions = predictions.data_ptr();
    }
    check_rc(bke_poly_filter(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_poly_filter");
    auto or_empty = [&](const at::Tensor &t) { return t.defined() ? t : at::empty({0}, x.options()); };
    return std::make_tuple(x_out, or_empty(dx_out), or_empty(ddx_out), or_empty(n_out), results, or_empty(predictions));
}

// T epochs of IMMEstimator predict(); update(z) for N tracks of M models (bke_imm_batch_filter).  x[j], P[j], S[j],
// log_likelihood[j] (model j's state, kept S and log-likelihood), mu and cbar are read and updated in place;
// the models' K, y, SI, x_prior, P_prior, status and omega are not returned.  Returns (means, covariances, means_p,
// covariances_p, mus).
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> imm_batch_filter(
    at::TensorList x, at::TensorList P, at::TensorList F, at::TensorList Q, at::TensorList H, at::TensorList R,
    at::ArrayRef<double> alpha_sq, at::TensorList S, at::TensorList log_likelihood, at::Tensor mu, at::Tensor cbar,
    const at::Tensor &trans, const at::Tensor &zs, const c10::optional<at::Tensor> &zs_valid)
{
    const int64_t M = (int64_t)x.size();
    TORCH_CHECK(M >= 2 && M <= BKE_MM_MAX_MODELS, "bke: 2 .. ", BKE_MM_MAX_MODELS, " models");
    TORCH_CHECK((int64_t)P.size() == M && (int64_t)F.size() == M && (int64_t)Q.size() == M && (int64_t)H.size() == M &&
                (int64_t)R.size() == M && (int64_t)alpha_sq.size() == M && (int64_t)S.size() == M &&
                (int64_t)log_likelihood.size() == M, "bke: one x, P, F, Q, H, R, alpha_sq, S and log_likelihood per model");
    const at::Tensor &x0 = x[0];
    TORCH_CHECK(x0.is_cuda() && x0.dim() == 2, "bke: x[j] is a CUDA tensor [N, n]");
    c10::cuda::CUDAGuard guard(x0.device());
    const int64_t N = x0.size(0), n = x0.size(1);
    TORCH_CHECK(zs.is_cuda() && zs.device() == x0.device() && zs.is_contiguous() && zs.scalar_type() == x0.scalar_type() &&
                zs.dim() == 3 && zs.size(1) == N, "bke: zs is [T, N, m] in the state's dtype, on x's device");
    const int64_t T = zs.size(0), m = zs.size(2);
    auto same = [&](const at::Tensor &t, std::vector<int64_t> shape, at::ScalarType st, const char *name) {
        TORCH_CHECK(t.is_cuda() && t.device() == x0.device() && t.is_contiguous() && t.scalar_type() == st &&
                    t.sizes().vec() == shape, "bke: ", name, " must be a contiguous CUDA tensor ", at::IntArrayRef(shape),
                    " of the right dtype, on x's device");
    };
    const auto dt = x0.scalar_type();
    bke_imm_batch_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_tracks = N; a.dim_x = (int32_t)n; a.dim_z = (int32_t)m; a.n_models = (int32_t)M; a.dtype = dtype_of(x0); a.n_steps = T;
    std::vector<at::Tensor> scratch;
    auto opts = x0.options();
    for (int64_t j = 0; j < M; j++) {
        same(x[j], {N, n}, dt, "x[j]"); same(P[j], {N, n, n}, dt, "P[j]");
        same(S[j], {N, m, m}, dt, "S[j]"); same(log_likelihood[j], {N}, dt, "log_likelihood[j]");
        a.x[j] = x[j].data_ptr(); a.P[j] = P[j].data_ptr(); a.S[j] = S[j].data_ptr(); a.log_likelihood[j] = log_likelihood[j].data_ptr();
        TORCH_CHECK(F[j].device() == x0.device() && Q[j].device() == x0.device() && H[j].device() == x0.device() &&
                    R[j].device() == x0.device(), "bke: the models must be on x's device");
        a.F[j] = model(F[j], N, n, n, &a.F_stride[j], x0, "F[j]");
        a.Q[j] = model(Q[j], N, n, n, &a.Q_stride[j], x0, "Q[j]");
        a.H[j] = model(H[j], N, m, n, &a.H_stride[j], x0, "H[j]");
        a.R[j] = model(R[j], N, m, m, &a.R_stride[j], x0, "R[j]");
        a.alpha_sq[j] = alpha_sq[j];
        scratch.push_back(at::zeros({N, n, m}, opts)); a.K[j] = scratch.back().data_ptr();
        scratch.push_back(at::zeros({N, m}, opts)); a.y[j] = scratch.back().data_ptr();
        scratch.push_back(at::zeros({N, m, m}, opts)); a.SI[j] = scratch.back().data_ptr();
        scratch.push_back(at::empty({N, n}, opts)); a.x_prior[j] = scratch.back().data_ptr();
        scratch.push_back(at::empty({N, n, n}, opts)); a.P_prior[j] = scratch.back().data_ptr();
        scratch.push_back(at::empty({N}, opts.dtype(at::kInt))); a.status[j] = scratch.back().data_ptr<int32_t>();
    }
    same(mu, {N, M}, at::kDouble, "mu"); same(cbar, {N, M}, at::kDouble, "cbar"); same(trans, {M, M}, at::kDouble, "trans");
    at::Tensor omega = at::empty({N, M, M}, opts.dtype(at::kDouble));
    a.mu = mu.data_ptr<double>(); a.cbar = cbar.data_ptr<double>(); a.omega = omega.data_ptr<double>(); a.trans = trans.data_ptr<double>();
    a.zs = zs.data_ptr();
    at::Tensor valid;
    if (zs_valid.has_value() && zs_valid->defined()) {
        TORCH_CHECK(zs_valid->device() == x0.device() && zs_valid->sizes() == at::IntArrayRef({T, N}), "bke: zs_valid is [T, N] on x's device");
        valid = zs_valid->to(at::kByte).contiguous();
        a.zs_valid = valid.data_ptr<uint8_t>();
    }
    at::Tensor means = at::empty({T, N, n}, opts), covs = at::empty({T, N, n, n}, opts);
    at::Tensor means_p = at::empty({T, N, n}, opts), covs_p = at::empty({T, N, n, n}, opts);
    at::Tensor mus = at::empty({T, N, M}, opts.dtype(at::kDouble));
    a.means = means.data_ptr(); a.covariances = covs.data_ptr(); a.means_p = means_p.data_ptr();
    a.covariances_p = covs_p.data_ptr(); a.mus = mus.data_ptr<double>();
    check_rc(bke_imm_batch_filter(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_imm_batch_filter");
    return std::make_tuple(means, covs, means_p, covs_p, mus);
}

// smooth_batch(zs, N) from (x, P): returns (xSmooth [T, N, n], xhat [T, N, n]); x and P are not changed
std::tuple<at::Tensor, at::Tensor> fls_smooth_batch(const at::Tensor &x, const at::Tensor &P, const at::Tensor &F, const at::Tensor &H,
                                                    const at::Tensor &Q, const at::Tensor &R, const at::Tensor &zs, int64_t lag)
{
    TORCH_CHECK(x.is_cuda() && P.is_cuda() && x.is_contiguous() && P.is_contiguous(), "bke: x and P must be contiguous CUDA tensors");
    TORCH_CHECK(x.dim() == 2 && P.dim() == 3 && P.size(0) == x.size(0) && P.size(1) == x.size(1) && P.size(2) == x.size(1), "bke: x is [N, n], P is [N, n, n]");
    TORCH_CHECK(P.scalar_type() == x.scalar_type(), "bke: x and P must share a dtype");
    c10::cuda::CUDAGuard guard(x.device());
    const int64_t N = x.size(0), n = x.size(1), m = H.size(-2);
    TORCH_CHECK(zs.is_cuda() && zs.is_contiguous() && zs.scalar_type() == x.scalar_type() && zs.dim() == 3 && zs.size(1) == N && zs.size(2) == m,
                "bke: zs is [T, N, m]");
    const int64_t T = zs.size(0);
    at::Tensor xs = at::empty({T, N, n}, x.options()), xhat = at::empty({T, N, n}, x.options());
    if (T == 0 || N == 0) return std::make_tuple(xs, xhat);
    bke_fls_args a;
    std::memset(&a, 0, sizeof(a));
    bke_kf_args &k = a.step;
    k.n_filters = N; k.dim_x = (int32_t)n; k.dim_z = (int32_t)m; k.dtype = dtype_of(x); k.alpha_sq = 1.0;
    at::Tensor x_out = at::empty_like(x), P_out = at::empty_like(P);
    k.x = x.data_ptr(); k.P = P.data_ptr(); k.x_out = x_out.data_ptr(); k.P_out = P_out.data_ptr();
    k.F = model(F, N, n, n, &k.F_stride, x, "F");
    k.H = model(H, N, m, n, &k.H_stride, x, "H");
    k.Q = model(Q, N, n, n, &k.Q_stride, x, "Q");
    k.R = model(R, N, m, m, &k.R_stride, x, "R");
    a.n_steps = T; a.lag = lag; a.count = 0;
    a.zs = zs.data_ptr(); a.xs_smooth = xs.data_ptr(); a.xhat = xhat.data_ptr();
    const size_t wsb = bke_fls_workspace_bytes(N, k.dim_x, k.dim_z, 0, k.dtype, lag);
    at::Tensor ws;
    if (wsb) {
        ws = at::empty({(int64_t)wsb}, x.options().dtype(at::kByte));      // the caching allocator aligns to 512 B
        a.workspace = ws.data_ptr(); a.workspace_bytes = wsb;
    }
    check_rc(bke_fls_smooth(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_fls_smooth");
    return std::make_tuple(xs, xhat);
}

at::Tensor resample(const at::Tensor &w, double u, const c10::optional<at::Tensor> &U)
{
    TORCH_CHECK(w.is_cuda() && w.is_contiguous() && w.scalar_type() == at::kDouble && w.dim() == 1, "bke: weights must be a contiguous 1-D float64 CUDA tensor");
    c10::cuda::CUDAGuard guard(w.device());
    const int64_t n = w.numel();
    at::Tensor idx = at::empty({n}, w.options().dtype(at::kInt));
    if (n == 0) return idx;
    const size_t wsb = bke_resample_workspace_bytes(n);
    at::Tensor ws = at::empty({(int64_t)wsb + 256}, w.options().dtype(at::kByte));
    char *wp = (char *)ws.data_ptr();
    wp += (256 - (reinterpret_cast<uintptr_t>(wp) & 255)) & 255;
    at::Tensor info = at::zeros({8}, w.options().dtype(at::kInt));
    void *st = (void *)c10::cuda::getCurrentCUDAStream().stream();
    if (U.has_value()) {
        const at::Tensor &uu = *U;
        TORCH_CHECK(uu.is_cuda() && uu.is_contiguous() && uu.scalar_type() == at::kDouble && uu.numel() == n, "bke: uniforms must match the weights");
        check_rc(bke_stratified_resample(n, (const double *)w.data_ptr(), (const double *)uu.data_ptr(), (int32_t *)idx.data_ptr(), wp, wsb,
                                         (int32_t *)info.data_ptr(), nullptr, st), "bke_stratified_resample");
    } else {
        check_rc(bke_systematic_resample(n, (const double *)w.data_ptr(), u, (int32_t *)idx.data_ptr(), wp, wsb, (int32_t *)info.data_ptr(),
                                         nullptr, st), "bke_systematic_resample");
    }
    // resampling.py:145: a position at or beyond cumsum[-1] is an IndexError in the reference
    TORCH_CHECK_INDEX(info[0].item<int>() == 0, "index ", n, " is out of bounds for axis 0 with size ", n);
    return idx;
}

at::Tensor systematic_resample(const at::Tensor &w, double u) { return resample(w, u, c10::nullopt); }
at::Tensor stratified_resample(const at::Tensor &w, const at::Tensor &U) { return resample(w, 0.0, U); }

at::Tensor resample_bank(const at::Tensor &w, const at::Tensor *u, const at::Tensor *U)
{
    TORCH_CHECK(w.is_cuda() && w.is_contiguous() && w.scalar_type() == at::kDouble && w.dim() == 2, "bke: weights must be a contiguous 2-D float64 CUDA tensor");
    c10::cuda::CUDAGuard guard(w.device());
    const int64_t B = w.size(0), M = w.size(1);
    const at::Tensor &r = u ? *u : *U;
    TORCH_CHECK(r.is_cuda() && r.is_contiguous() && r.scalar_type() == at::kDouble && r.device() == w.device(), "bke: uniforms must be a contiguous float64 CUDA tensor on the weights' device");
    if (u) {
        TORCH_CHECK(r.dim() == 1 && r.size(0) == B, "bke: u must be [n_sets]");
    } else {
        TORCH_CHECK(r.dim() == 2 && r.size(0) == B && r.size(1) == M, "bke: uniforms must be [n_sets, n_particles]");
    }
    at::Tensor idx = at::empty({B, M}, w.options().dtype(at::kInt));
    if (B == 0 || M == 0) return idx;
    at::Tensor status = at::empty({B}, w.options().dtype(at::kInt));
    bke_resample_bank_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_sets = B; a.n_particles = M; a.weights = (const double *)w.data_ptr();
    if (u) a.u = (const double *)r.data_ptr(); else a.uniforms = (const double *)r.data_ptr();
    a.indexes = (int32_t *)idx.data_ptr(); a.status = (int32_t *)status.data_ptr();
    check_rc(bke_resample_bank(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_resample_bank");
    // resampling.py:145: the first row whose positions run past its cumsum is where the reference loop raises
    const at::Tensor bad = status.nonzero();
    TORCH_CHECK_INDEX(bad.numel() == 0, "set ", bad.numel() ? bad[0][0].item<int64_t>() : 0, ": index ", M,
                      " is out of bounds for axis 0 with size ", M);
    return idx;
}

at::Tensor systematic_resample_bank(const at::Tensor &w, const at::Tensor &u) { return resample_bank(w, &u, nullptr); }
at::Tensor stratified_resample_bank(const at::Tensor &w, const at::Tensor &U) { return resample_bank(w, nullptr, &U); }

void check_bank_uniforms(const at::Tensor &w, const at::Tensor &U)
{
    TORCH_CHECK(w.is_cuda() && w.is_contiguous() && w.scalar_type() == at::kDouble && w.dim() == 2, "bke: weights must be a contiguous 2-D float64 CUDA tensor");
    TORCH_CHECK(U.is_cuda() && U.is_contiguous() && U.scalar_type() == at::kDouble && U.device() == w.device(), "bke: uniforms must be a contiguous float64 CUDA tensor on the weights' device");
    TORCH_CHECK(U.dim() == 2 && U.size(0) == w.size(0) && U.size(1) == w.size(1), "bke: uniforms must be [n_sets, n_particles]");
}

// resampling.py:173-176 on every row for the caller's uniforms[B, M]: int64 indexes
at::Tensor multinomial_resample_bank(const at::Tensor &w, const at::Tensor &U)
{
    check_bank_uniforms(w, U);
    c10::cuda::CUDAGuard guard(w.device());
    const int64_t B = w.size(0), M = w.size(1);
    TORCH_CHECK_INDEX(B == 0 || M > 0, "set 0: index -1 is out of bounds for axis 0 with size 0");
    at::Tensor idx = at::empty({B, M}, w.options().dtype(at::kLong));
    if (B == 0) return idx;
    at::Tensor status = at::empty({B}, w.options().dtype(at::kInt));
    const size_t wsb = bke_multinomial_resample_bank_workspace_bytes(B, M);
    at::Tensor ws = at::empty({(int64_t)(wsb / 8)}, w.options());
    bke_multinomial_resample_bank_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_sets = B; a.n_particles = M; a.weights = (const double *)w.data_ptr(); a.uniforms = (const double *)U.data_ptr();
    a.indexes = (int64_t *)idx.data_ptr(); a.status = (int32_t *)status.data_ptr();
    a.workspace = ws.data_ptr(); a.workspace_bytes = wsb;
    check_rc(bke_multinomial_resample_bank(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_multinomial_resample_bank");
    return idx;
}

// resampling.py:27-76 on every row; row b uses uniforms[b, :M - k_b]: int32 indexes
at::Tensor residual_resample_bank(const at::Tensor &w, const at::Tensor &U)
{
    check_bank_uniforms(w, U);
    c10::cuda::CUDAGuard guard(w.device());
    const int64_t B = w.size(0), M = w.size(1);
    TORCH_CHECK_INDEX(B == 0 || M > 0, "set 0: index -1 is out of bounds for axis 0 with size 0");
    at::Tensor idx = at::zeros({B, M}, w.options().dtype(at::kInt));
    if (B == 0) return idx;
    at::Tensor status = at::empty({B}, w.options().dtype(at::kInt));
    at::Tensor k = at::empty({B}, w.options().dtype(at::kLong));
    const size_t wsb = bke_residual_resample_bank_workspace_bytes(B, M);
    at::Tensor ws = at::empty({(int64_t)(wsb / 8)}, w.options());
    bke_residual_resample_bank_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_sets = B; a.n_particles = M; a.weights = (const double *)w.data_ptr(); a.uniforms = (const double *)U.data_ptr();
    a.indexes = (int32_t *)idx.data_ptr(); a.n_copies = (int64_t *)k.data_ptr(); a.status = (int32_t *)status.data_ptr();
    a.workspace = ws.data_ptr(); a.workspace_bytes = wsb;
    void *st = (void *)c10::cuda::getCurrentCUDAStream().stream();
    check_rc(bke_residual_resample_bank_prepare(&a, st), "bke_residual_resample_bank_prepare");
    check_rc(bke_residual_resample_bank_search(&a, st), "bke_residual_resample_bank_search");
    // resampling.py:61: the first row with k > M is where the reference loop raises
    const at::Tensor bad = status.bitwise_and(1).nonzero();
    TORCH_CHECK_INDEX(bad.numel() == 0, "set ", bad.numel() ? bad[0][0].item<int64_t>() : 0, ": index ", M,
                      " is out of bounds for axis 0 with size ", M);
    return idx;
}

// w <- w / np.sum(w), neff = 1 / np.sum(np.square(w)), and where neff < threshold: particles[b] <- particles[b][idx],
// w <- 1 / M (systematic for u[B], stratified for uniforms[B, M]); weights and particles in place
std::tuple<at::Tensor, at::Tensor> resample_bank_if_degenerate(const at::Tensor &w, const at::Tensor &parts,
                                                               const at::Tensor *u, const at::Tensor *U, double threshold)
{
    TORCH_CHECK(w.is_cuda() && w.is_contiguous() && w.scalar_type() == at::kDouble && w.dim() == 2, "bke: weights must be a contiguous 2-D float64 CUDA tensor");
    c10::cuda::CUDAGuard guard(w.device());
    const int64_t B = w.size(0), M = w.size(1);
    TORCH_CHECK(parts.is_cuda() && parts.is_contiguous() && parts.device() == w.device() && parts.dim() >= 2 &&
                parts.size(0) == B && parts.size(1) == M, "bke: particles must be a contiguous CUDA tensor [n_sets, n_particles, ...] on the weights' device");
    const at::Tensor &r = u ? *u : *U;
    TORCH_CHECK(r.is_cuda() && r.is_contiguous() && r.scalar_type() == at::kDouble && r.device() == w.device(), "bke: uniforms must be a contiguous float64 CUDA tensor on the weights' device");
    if (u) {
        TORCH_CHECK(r.dim() == 1 && r.size(0) == B, "bke: u must be [n_sets]");
    } else {
        TORCH_CHECK(r.dim() == 2 && r.size(0) == B && r.size(1) == M, "bke: uniforms must be [n_sets, n_particles]");
    }
    at::Tensor resampled = at::zeros({B}, w.options().dtype(at::kBool));
    at::Tensor neff = at::full({B}, std::numeric_limits<double>::infinity(), w.options());   // M = 0: 1 / sum([]) = inf
    if (B == 0 || M == 0) return {resampled, neff};
    at::Tensor idx = at::empty({B, M}, w.options().dtype(at::kInt));
    at::Tensor status = at::empty({B}, w.options().dtype(at::kInt));
    const size_t wsb = bke_resample_bank_gated_workspace_bytes(B);
    at::Tensor ws = at::empty({(int64_t)((wsb + 3) / 4)}, w.options().dtype(at::kInt));
    bke_resample_bank_gated_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_sets = B; a.n_particles = M; a.weights = (double *)w.data_ptr(); a.threshold = threshold;
    if (u) a.u = (const double *)r.data_ptr(); else a.uniforms = (const double *)r.data_ptr();
    a.particles = parts.data_ptr(); a.particle_bytes = parts.numel() / (B * M) * (int64_t)parts.element_size();
    a.indexes = (int32_t *)idx.data_ptr(); a.neff = (double *)neff.data_ptr();
    a.resampled = (uint8_t *)resampled.data_ptr(); a.status = (int32_t *)status.data_ptr();
    a.workspace = ws.data_ptr(); a.workspace_bytes = wsb;
    check_rc(bke_resample_bank_gated(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_resample_bank_gated");
    // resampling.py:145: the first resampled row whose positions run past its cumsum is where the loop raises
    const at::Tensor bad = status.nonzero();
    TORCH_CHECK_INDEX(bad.numel() == 0, "set ", bad.numel() ? bad[0][0].item<int64_t>() : 0, ": index ", M,
                      " is out of bounds for axis 0 with size ", M);
    return {resampled, neff};
}

std::tuple<at::Tensor, at::Tensor> systematic_resample_bank_if_degenerate(at::Tensor w, at::Tensor parts, const at::Tensor &u,
                                                                          double threshold)
{
    return resample_bank_if_degenerate(w, parts, &u, nullptr, threshold);
}

std::tuple<at::Tensor, at::Tensor> stratified_resample_bank_if_degenerate(at::Tensor w, at::Tensor parts, const at::Tensor &U,
                                                                          double threshold)
{
    return resample_bank_if_degenerate(w, parts, nullptr, &U, threshold);
}

}  // namespace

// discrete_bayes.py:26-128 on every row of pdf[B, M]: predict when kernel ([K] or [B, K], float64) is given (offsets
// [B] int64 per row, else `offset`), update when likelihood is given, then normalize when asked; a new tensor
at::Tensor discrete_bayes_step(const at::Tensor &pdf, const c10::optional<at::Tensor> &kernel,
                               const c10::optional<at::Tensor> &offsets, int64_t offset,
                               const c10::optional<at::Tensor> &likelihood, bool normalize, bool constant, double cval)
{
    TORCH_CHECK(pdf.is_cuda() && pdf.is_contiguous() && pdf.dim() == 2, "bke: pdf must be a contiguous 2-D CUDA tensor");
    const int dt = dtype_of(pdf);
    c10::cuda::CUDAGuard guard(pdf.device());
    const int64_t B = pdf.size(0), M = pdf.size(1);
    bke_db_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_rows = B; a.n_bins = M; a.dtype = dt;
    a.flags = (normalize ? BKE_DB_NORMALIZE : 0u) | (constant ? BKE_DB_CONSTANT : 0u);
    if (kernel) {
        const at::Tensor &k = *kernel;
        TORCH_CHECK(k.is_cuda() && k.is_contiguous() && k.scalar_type() == at::kDouble && k.device() == pdf.device() &&
                    (k.dim() == 1 || (k.dim() == 2 && k.size(0) == B)), "bke: kernel must be a contiguous float64 CUDA tensor [K] or [B, K]");
        a.kernel = (const double *)k.data_ptr(); a.kernel_len = k.size(-1); a.kernel_stride = k.dim() == 2 ? k.size(1) : 0;
        a.offset = offset; a.cval = cval;
        if (offsets) {
            TORCH_CHECK(offsets->is_cuda() && offsets->is_contiguous() && offsets->scalar_type() == at::kLong &&
                        offsets->dim() == 1 && offsets->size(0) == B && offsets->device() == pdf.device(),
                        "bke: offsets must be a contiguous int64 CUDA tensor [B]");
            a.offsets = (const int64_t *)offsets->data_ptr();
        }
    }
    if (likelihood) {
        TORCH_CHECK(likelihood->is_cuda() && likelihood->is_contiguous() && likelihood->scalar_type() == pdf.scalar_type() &&
                    likelihood->sizes() == pdf.sizes() && likelihood->device() == pdf.device(),
                    "bke: likelihood must be a contiguous CUDA tensor of the pdf's shape and dtype");
        a.likelihood = likelihood->data_ptr();
    }
    at::Tensor out = at::empty_like(pdf);
    a.pdf = pdf.data_ptr(); a.out = out.data_ptr();
    const size_t wsb = bke_db_workspace_bytes(M, dt);
    at::Tensor ws;
    if (wsb && B) {
        ws = at::empty({(int64_t)wsb + 256}, pdf.options().dtype(at::kByte));
        const uintptr_t p = (uintptr_t)ws.data_ptr();
        a.workspace = (void *)((p + 255) & ~(uintptr_t)255); a.workspace_bytes = wsb;
    }
    check_rc(bke_db_step(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_db_step");
    return out;
}

TORCH_LIBRARY(bke, m)
{
    m.def("kf_step(Tensor x, Tensor P, Tensor F, Tensor H, Tensor Q, Tensor R, Tensor z, float alpha_sq=1.0) -> (Tensor, Tensor)");
    m.def("kf_predict(Tensor x, Tensor P, Tensor F, Tensor Q, float alpha_sq=1.0) -> (Tensor, Tensor)");
    m.def("kf_step_correlated(Tensor x, Tensor P, Tensor F, Tensor H, Tensor Q, Tensor R, Tensor M, Tensor z, "
          "float alpha_sq=1.0) -> (Tensor, Tensor)");
    m.def("kf_update_rows(Tensor x, Tensor P, Tensor F, Tensor H, Tensor Q, Tensor R, Tensor z_i, int start, "
          "float alpha_sq=1.0) -> (Tensor, Tensor)");
    m.def("ukf_step(Tensor x, Tensor P, Tensor Q, Tensor R, Tensor z, float dt, float alpha, float beta, float kappa, "
          "int fx_model, int hx_model, Tensor? F=None, Tensor? H=None, bool simplex=False) -> (Tensor, Tensor)");
    m.def("ckf_step(Tensor x, Tensor P, Tensor Q, Tensor R, Tensor z, float dt, int fx_model, int hx_model, "
          "Tensor? F=None, Tensor? H=None) -> (Tensor, Tensor)");
    m.def("enkf_step(Tensor x, Tensor P, Tensor sigmas, Tensor Q, Tensor R, Tensor z, float dt, int fx_model, int hx_model, "
          "int seed, int counter, Tensor? F=None, Tensor? H=None) -> (Tensor, Tensor, Tensor)");
    m.def("srkf_step(Tensor x, Tensor L, Tensor F, Tensor H, Tensor Lq, Tensor Lr, Tensor z) -> (Tensor, Tensor)");
    m.def("if_step(Tensor x, Tensor P_inv, Tensor no_information, Tensor F, Tensor F_inv, Tensor Q, Tensor H, Tensor R_inv, "
          "Tensor z) -> (Tensor, Tensor, Tensor, Tensor)");
    m.def("poly_filter(Tensor x, Tensor? dx, Tensor? ddx, Tensor? n, Tensor z, Tensor? g, Tensor? h, Tensor? k, Tensor? dt, "
          "Tensor? dt2, Tensor? hdt2, int family, int order, bool batch=False) -> (Tensor, Tensor, Tensor, Tensor, Tensor, Tensor)");
    m.def("score_measurements(Tensor z, Tensor? x, Tensor? mean, Tensor? P, Tensor? S, Tensor? H, Tensor? R, Tensor? valid, "
          "str[] outputs) -> Tensor[]");
    m.def("ukf_score_measurements(Tensor x, Tensor P, Tensor R, Tensor z, float alpha, float beta, float kappa, int hx_model, "
          "Tensor? H=None, Tensor? valid=None, bool simplex=False) -> (Tensor, Tensor, Tensor)");
    m.def("imm_batch_filter(Tensor(a!)[] x, Tensor(b!)[] P, Tensor[] F, Tensor[] Q, Tensor[] H, Tensor[] R, float[] alpha_sq, "
          "Tensor(c!)[] S, Tensor(d!)[] log_likelihood, Tensor(e!) mu, Tensor(f!) cbar, Tensor trans, Tensor zs, "
          "Tensor? zs_valid=None) -> (Tensor, Tensor, Tensor, Tensor, Tensor)");
    m.def("fls_smooth_batch(Tensor x, Tensor P, Tensor F, Tensor H, Tensor Q, Tensor R, Tensor zs, int N) -> (Tensor, Tensor)");
    m.def("discrete_bayes_step(Tensor pdf, Tensor? kernel, Tensor? offsets, int offset, Tensor? likelihood, bool normalize, "
          "bool constant=False, float cval=0.0) -> Tensor");
    m.def("systematic_resample(Tensor weights, float u) -> Tensor");
    m.def("stratified_resample(Tensor weights, Tensor uniforms) -> Tensor");
    m.def("systematic_resample_bank(Tensor weights, Tensor u) -> Tensor");
    m.def("stratified_resample_bank(Tensor weights, Tensor uniforms) -> Tensor");
    m.def("multinomial_resample_bank(Tensor weights, Tensor uniforms) -> Tensor");
    m.def("residual_resample_bank(Tensor weights, Tensor uniforms) -> Tensor");
    m.def("systematic_resample_bank_if_degenerate(Tensor(a!) weights, Tensor(b!) particles, Tensor u, float threshold) "
          "-> (Tensor resampled, Tensor neff)");
    m.def("stratified_resample_bank_if_degenerate(Tensor(a!) weights, Tensor(b!) particles, Tensor uniforms, "
          "float threshold) -> (Tensor resampled, Tensor neff)");
}

TORCH_LIBRARY_IMPL(bke, CUDA, m)
{
    m.impl("discrete_bayes_step", &discrete_bayes_step);
    m.impl("kf_step", &kf_step);
    m.impl("kf_predict", &kf_predict);
    m.impl("kf_step_correlated", &kf_step_correlated);
    m.impl("kf_update_rows", &kf_update_rows);
    m.impl("ukf_step", &ukf_step);
    m.impl("ukf_score_measurements", &ukf_score_measurements);
    m.impl("ckf_step", &ckf_step);
    m.impl("enkf_step", &enkf_step);
    m.impl("srkf_step", &srkf_step);
    m.impl("if_step", &if_step);
    m.impl("poly_filter", &poly_filter);
    m.impl("score_measurements", &score_measurements);
    m.impl("imm_batch_filter", &imm_batch_filter);
    m.impl("fls_smooth_batch", &fls_smooth_batch);
    m.impl("systematic_resample", &systematic_resample);
    m.impl("stratified_resample", &stratified_resample);
    m.impl("systematic_resample_bank", &systematic_resample_bank);
    m.impl("stratified_resample_bank", &stratified_resample_bank);
    m.impl("multinomial_resample_bank", &multinomial_resample_bank);
    m.impl("residual_resample_bank", &residual_resample_bank);
    m.impl("systematic_resample_bank_if_degenerate", &systematic_resample_bank_if_degenerate);
    m.impl("stratified_resample_bank_if_degenerate", &stratified_resample_bank_if_degenerate);
}
