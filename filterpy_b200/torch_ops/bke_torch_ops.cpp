// torch.ops.bke.* — the C-ABI of include/bke.h exposed as PyTorch operators on CUDA tensors (zero copy:
// the tensors' device pointers go straight into the bke_* calls on the current CUDA stream).
// asks for this twin of the ctypes binding: the same entry points, no arithmetic of its own.
//   bke::kf_step              bke_kf_step              KalmanFilter.predict + update, kalman_filter.py:437-561
//   bke::kf_predict           bke_kf_step (predict)    kalman_filter.py:437-482
//   bke::ukf_step             bke_ukf_step             UnscentedKalmanFilter.predict + update, UKF.py:364-491
//   bke::ckf_step             bke_ckf_step             CubatureKalmanFilter.predict + update, CubatureKalmanFilter.py:292-389
//   bke::srkf_step            bke_srkf_step            SquareRootKalmanFilter.predict + update, square_root.py:172-248
//   bke::systematic_resample  bke_systematic_resample  monte_carlo/resampling.py:117-150
//   bke::stratified_resample  bke_stratified_resample  monte_carlo/resampling.py:80-114
#include <ATen/ATen.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>
#include <cstring>
#include <tuple>
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

std::tuple<at::Tensor, at::Tensor> kf_run(const at::Tensor &x, const at::Tensor &P, const at::Tensor &F, const at::Tensor &H,
                                          const at::Tensor &Q, const at::Tensor &R, const c10::optional<at::Tensor> &z,
                                          double alpha_sq, unsigned flags)
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
        TORCH_CHECK(zz.is_cuda() && zz.is_contiguous() && zz.scalar_type() == x.scalar_type() && zz.dim() == 2 && zz.size(0) == N && zz.size(1) == m, "bke: z is [N, m]");
        a.z = zz.data_ptr();
    }
    check_rc(bke_kf_step(&a, (void *)c10::cuda::getCurrentCUDAStream().stream()), "bke_kf_step");
    return std::make_tuple(x_out, P_out);
}

std::tuple<at::Tensor, at::Tensor> kf_step(const at::Tensor &x, const at::Tensor &P, const at::Tensor &F, const at::Tensor &H,
                                           const at::Tensor &Q, const at::Tensor &R, const at::Tensor &z, double alpha_sq)
{
    return kf_run(x, P, F, H, Q, R, z, alpha_sq, BKE_DO_PREDICT | BKE_DO_UPDATE);
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
                                            const c10::optional<at::Tensor> &H)
{
    TORCH_CHECK(x.is_cuda() && P.is_cuda() && x.is_contiguous() && P.is_contiguous() && x.dim() == 2 && P.dim() == 3, "bke: x is [N, n], P is [N, n, n] on the GPU");
    c10::cuda::CUDAGuard guard(x.device());
    const int64_t N = x.size(0), n = x.size(1), m = z.size(1);
    bke_ukf_args a;
    std::memset(&a, 0, sizeof(a));
    a.n_filters = N; a.dim_x = (int32_t)n; a.dim_z = (int32_t)m; a.dtype = dtype_of(x);
    a.flags = BKE_DO_PREDICT | BKE_DO_UPDATE; a.fx_model = (int32_t)fx_model; a.hx_model = (int32_t)hx_model;
    a.dt = dt; a.alpha = alpha; a.beta = beta; a.kappa = kappa;
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

}  // namespace

TORCH_LIBRARY(bke, m)
{
    m.def("kf_step(Tensor x, Tensor P, Tensor F, Tensor H, Tensor Q, Tensor R, Tensor z, float alpha_sq=1.0) -> (Tensor, Tensor)");
    m.def("kf_predict(Tensor x, Tensor P, Tensor F, Tensor Q, float alpha_sq=1.0) -> (Tensor, Tensor)");
    m.def("ukf_step(Tensor x, Tensor P, Tensor Q, Tensor R, Tensor z, float dt, float alpha, float beta, float kappa, "
          "int fx_model, int hx_model, Tensor? F=None, Tensor? H=None) -> (Tensor, Tensor)");
    m.def("ckf_step(Tensor x, Tensor P, Tensor Q, Tensor R, Tensor z, float dt, int fx_model, int hx_model, "
          "Tensor? F=None, Tensor? H=None) -> (Tensor, Tensor)");
    m.def("srkf_step(Tensor x, Tensor L, Tensor F, Tensor H, Tensor Lq, Tensor Lr, Tensor z) -> (Tensor, Tensor)");
    m.def("systematic_resample(Tensor weights, float u) -> Tensor");
    m.def("stratified_resample(Tensor weights, Tensor uniforms) -> Tensor");
}

TORCH_LIBRARY_IMPL(bke, CUDA, m)
{
    m.impl("kf_step", &kf_step);
    m.impl("kf_predict", &kf_predict);
    m.impl("ukf_step", &ukf_step);
    m.impl("ckf_step", &ckf_step);
    m.impl("srkf_step", &srkf_step);
    m.impl("systematic_resample", &systematic_resample);
    m.impl("stratified_resample", &stratified_resample);
}
