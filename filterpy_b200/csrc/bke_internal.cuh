// Internal helpers shared by the sm_90a kernels of the engine (not part of the C-ABI).
#pragma once
#ifndef __CUDACC_RTC__
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#endif
#include "../../include/bke.h"

namespace bke {

#ifndef __CUDACC_RTC__
void set_error(const char *fmt, ...);
int check_cuda(cudaError_t e, const char *what);

// Number of SMs of the current device (cached).
int sm_count();
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
// filled by launch_kf_scan_models is a record filled by launch_kf_pack_models that replaces F, Q, H and R
int launch_kf_fast(const bke_kf_args &a, cudaStream_t s, const void *rec = nullptr, const bke_kf_model_map *map = nullptr);
size_t kf_sym_models_bytes(int64_t n_filters);
int launch_kf_pack_sym(int64_t n_filters, const void *Q, const void *R, void *record, int32_t *asym, cudaStream_t s);
size_t kf_packed_models_bytes(int64_t n_filters, uint64_t varying);
int launch_kf_scan_models(int64_t n_filters, const void *F, const void *Q, const void *H, const void *R,
                          bke_kf_model_map *map, cudaStream_t s);
int launch_kf_pack_models(int64_t n_filters, const void *F, const void *Q, const void *H, const void *R, uint64_t varying,
                          void *record, cudaStream_t s);
int launch_kf_rowblock(const bke_kf_args &a, cudaStream_t s);
int launch_kf_direct(const bke_kf_args &a, cudaStream_t s);
// wgmma covariance propagation for shared-model fp32 banks with dim_x = 16 / 32 (kf_tc.cu); a fused step runs
// its update through launch_kf_any afterwards
int launch_kf_tc(const bke_kf_args &a, cudaStream_t s);
// the dispatch order of bke_kf_step: tensor-core predict (dim_x 16 / 32, shared models) -> TMA-staged 4/2 fp32 ->
// register tile with direct loads -> row-block -> catch-all
int launch_kf_any(const bke_kf_args &a, cudaStream_t s);
int launch_kf_batch(const bke_kf_batch_args &a, cudaStream_t s);
int launch_ukf(const bke_ukf_args &a, cudaStream_t s);
int validate_ckf(const bke_ckf_args &a);
int launch_ckf(const bke_ckf_args &a, cudaStream_t s);
int launch_srkf(const bke_srkf_args &a, cudaStream_t s);
int launch_cholesky_lower(int64_t n_filters, int32_t k, int32_t dtype, const void *A, int64_t stride, void *L,
                          int32_t *status, cudaStream_t s);
#endif

}  // namespace bke
