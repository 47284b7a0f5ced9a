// Internal helpers shared by the sm_90a kernels of the engine (not part of the C-ABI).
#pragma once
#ifndef __CUDACC_RTC__
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <initializer_list>
#include <utility>
#endif
#include "../../include/bke.h"

namespace bke {

#ifndef __CUDACC_RTC__
void set_error(const char *fmt, ...);
int check_cuda(cudaError_t e, const char *what);
// sets the kernel's dynamic shared-memory limit to smem bytes and launches it on grid x block threads with
// the one parameter block *params; `what` names the launch in the error
int launch_kernel(const void *kern, unsigned grid, unsigned block, size_t smem, void *params, cudaStream_t s, const char *what);

// the argument checks the filter-bank entry points share: each sets the error and returns BKE_ERR_BAD_ARG
// (require_device: BKE_ERR_CUDA), or BKE_OK
int require_device();                                    // the engine has no CPU fallback
int check_dtype(int32_t dtype);                          // BKE_F32 or BKE_F64
// n >= 0 filters, dim_x >= 1, dim_z >= 1, dim_u >= 0 (the defaults pass); upper bounds are the caller's
int check_bank(int64_t n, int64_t dim_x = 1, int64_t dim_z = 1, int64_t dim_u = 0);
int check_predict_update(uint32_t flags);                // flags select predict, update or both
int check_flag_bits(uint32_t flags, uint32_t allowed);   // no bit outside `allowed`
// each (stride, dense size): a model stride is 0 (one model shared by the bank) or the dense per-filter size
int check_strides(std::initializer_list<std::pair<int64_t, int64_t>> strides);
int check_control(const void *B, const void *u, int64_t dim_u);   // a control input needs B, u and dim_u >= 1

// Number of SMs of the current device (cached).
int sm_count();

// Launch shape of a kernel that gives each of `items` one warp and bytes_per_warp of dynamic shared memory:
// 4 warps per block, or 2 / 1 when their slices exceed `budget` bytes; grid = ceil(items / wpb) blocks, at
// least 1 and at most 16 per SM.  Raises the kernel's dynamic shared-memory limit when smem > 48 KB.
// Returns BKE_ERR_UNSUPPORTED, with no error text (the caller names what did not fit), when one warp's
// slice exceeds the budget.
struct WarpShape {
    int wpb;
    size_t smem;
    int grid;
};
int warp_shape(const void *kern, size_t bytes_per_warp, size_t budget, int64_t items, WarpShape &w);
#endif

constexpr unsigned FULL = 0xffffffffu;

template <typename T> struct DType;
template <> struct DType<float> { static constexpr int id = BKE_F32; };
template <> struct DType<double> { static constexpr int id = BKE_F64; };

// log(2*pi)
constexpr double LOG_2PI = 1.8378770664093454835606594728112;

#ifndef __CUDACC_RTC__
// ---- launchers implemented in the .cu files ---------------------------------------------
int launch_kf_generic(const bke_kf_args &a, cudaStream_t s);
// returns BKE_ERR_UNSUPPORTED when the specialised kernel does not cover the call.  Optional: `rec` alone is a
// record filled by launch_kf_pack_sym that replaces the per-filter Q and R; `rec` with the HOST copy of a map
// filled by launch_kf_scan_models is a record filled by launch_kf_pack_models that replaces F, Q, H and R;
// with `zs` on top, the launch runs n_steps (1 .. BKE_KF42_MAX_RING) predict+update pairs on the measurements
// zs[k] in turn (a.z is not read)
int launch_kf_fast(const bke_kf_args &a, cudaStream_t s, const void *rec = nullptr, const bke_kf_model_map *map = nullptr,
                   const void *const *zs = nullptr, int n_steps = 0);
size_t kf_sym_models_bytes(int64_t n_filters);
int launch_kf_pack_sym(int64_t n_filters, const void *Q, const void *R, void *record, int32_t *asym, cudaStream_t s);
size_t kf_packed_models_bytes(int64_t n_filters, uint64_t varying);
int launch_kf_scan_models(int64_t n_filters, const void *F, const void *Q, const void *H, const void *R,
                          bke_kf_model_map *map, cudaStream_t s);
int launch_kf_pack_models(int64_t n_filters, const void *F, const void *Q, const void *H, const void *R, uint64_t varying,
                          void *record, cudaStream_t s);
// the record plane each model word of a (host) map is read from: its own slot, or the representative slot of
// a copy flagged in map.duplicate (plane[e] = -1 for a shared word); BKE_ERR_BAD_ARG (with the error set) when
// a flagged bit has no representative or lies at or above popcount(varying)
int kf_model_planes(const bke_kf_model_map &map, int (&plane)[BKE_KF42_MODEL_WORDS]);
int launch_kf_rowblock(const bke_kf_args &a, cudaStream_t s);
int launch_kf_direct(const bke_kf_args &a, cudaStream_t s);
// update_correlated and update_sequential's row block (bke_kf_step_correlated, bke_kf_update_rows): register tiles
// for the shapes launch_kf_direct covers (BKE_ERR_UNSUPPORTED otherwise), the warp-per-filter kernel for any other.
// The rows calls take `a` with dim_z = L and H, R, z at the block; m is the bank's dim_z, the pitch of y, K and zrec.
int launch_kf_direct_correlated(const bke_kf_args &a, const void *M, int64_t M_stride, cudaStream_t s);
int launch_kf_generic_correlated(const bke_kf_args &a, const void *M, int64_t M_stride, cudaStream_t s);
int launch_kf_direct_rows(const bke_kf_args &a, int m, int start, int rpitch, void *zrec, cudaStream_t s);
int launch_kf_generic_rows(const bke_kf_args &a, int m, int start, int rpitch, void *zrec, cudaStream_t s);
// wgmma covariance propagation for shared-model fp32 banks with dim_x = 16 / 32 (kf_tc.cu); a fused step runs
// its update through launch_kf_any afterwards
int launch_kf_tc(const bke_kf_args &a, cudaStream_t s);
// the dispatch order of bke_kf_step: tensor-core predict (dim_x 16 / 32, shared models) -> TMA-staged 4/2 fp32 ->
// register tile with direct loads -> row-block -> catch-all
int launch_kf_any(const bke_kf_args &a, cudaStream_t s);
int launch_kf_batch(const bke_kf_batch_args &a, cudaStream_t s);
size_t fls_workspace_bytes(int64_t n_filters, int32_t dim_x, int32_t dim_z, int32_t dim_u, int32_t dtype, int64_t lag);
int launch_fls(const bke_fls_args &a, cudaStream_t s);
// the argument checks of each sigma-point family's step, pre-built and run-time compiled (api.cu)
int validate_ukf(const bke_ukf_args &a);
int validate_ckf(const bke_ckf_args &a);
int validate_enkf(const bke_enkf_args &a);
// bke_ukf_score and bke_ukf_score_model (api.cu)
int validate_ukf_score(const bke_ukf_score_args &a);
// the UKF smoother's, pre-built or compiled (user_fx: around a user fx, served besides the built-in ones); -1 = go
int validate_ukf_rts(const bke_ukf_rts_args &a, bool user_fx);
int launch_ukf(const bke_ukf_args &a, cudaStream_t s);
int launch_ckf(const bke_ckf_args &a, cudaStream_t s);
int launch_enkf(const bke_enkf_args &a, cudaStream_t s);
int launch_enkf_init(int64_t n_filters, int32_t dim_x, int32_t n_members, int32_t dtype, uint32_t seed, uint32_t counter,
                     const void *x, const void *P, void *sigmas, int32_t *status, cudaStream_t s);
int launch_srkf(const bke_srkf_args &a, cudaStream_t s);
int launch_cholesky_lower(int64_t n_filters, int32_t k, int32_t dtype, const void *A, int64_t stride, void *L,
                          int32_t *status, cudaStream_t s);
int launch_if(const bke_if_args &a, cudaStream_t s);
int launch_inverse(int64_t n_filters, int32_t k, int32_t dtype, const void *A, int64_t stride, void *Ai, int32_t *status,
                   cudaStream_t s);
int launch_poly(const bke_poly_args &a, cudaStream_t s);
int launch_score(const bke_score_args &a, cudaStream_t s);
int launch_ukf_score(const bke_ukf_score_args &a, cudaStream_t s);
// the (dim_x, dim_z, dtype) combinations bke_imm_batch_filter has a fused kernel for
bool imm_batch_has_instance(int dim_x, int dim_z, int dtype);
int launch_imm_batch(const bke_imm_batch_args &a, cudaStream_t s);
// np.cumsum(weights) bit for bit into cumsum_out (resample.cu's parity-map scan), its last element also to the
// device double *total_out when that is non-NULL (bke_cumsum_exact and the discrete Bayes rows too long to stage)
size_t cumsum_workspace_bytes(int64_t n);
int cumsum_exact(int64_t n, const double *weights, double *cumsum_out, int last_one, double *total_out, void *workspace,
                 size_t workspace_bytes, int32_t *info, cudaStream_t stream);
// bke_db_step after its argument checks (discrete_bayes.cu)
size_t db_workspace_bytes(int64_t n_bins, int32_t dtype);
int launch_db(const bke_db_args &a, cudaStream_t s);
#endif

}  // namespace bke
