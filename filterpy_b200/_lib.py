"""ctypes binding of the C-ABI in ``include/bke.h`` (the drop-in boundary).

The library is loaded from ``filterpy_b200/_C/libbke.so`` (built in-tree by ``_build.py``).
There is no CPU fallback: if the library is missing and cannot be built, or a compute entry
point reports no CUDA device, an exception is raised.
"""
import ctypes
import os
from ctypes import (POINTER, c_char_p, c_double, c_int, c_int32, c_int64, c_size_t, c_uint32, c_uint64,
                    c_void_p)

from . import _build

BKE_ABI_VERSION = 1
BKE_F32, BKE_F64 = 0, 1
BKE_OK, BKE_ERR_BAD_ARG, BKE_ERR_UNSUPPORTED, BKE_ERR_CUDA = 0, 1, 2, 3
BKE_STATUS_OK, BKE_STATUS_SINGULAR_S, BKE_STATUS_NOT_PD = 0, 1, 2
BKE_DO_PREDICT, BKE_DO_UPDATE, BKE_UPDATE_FIRST = 1, 2, 4
BKE_REVERSE_TILES = 16
BKE_UKF_SIMPLEX = 32             # bke_ukf_args.flags / bke_ukf_rts_args.flags: SimplexSigmaPoints
BKE_FX_LINEAR, BKE_FX_CONST_VEL = 0, 1
BKE_HX_LINEAR, BKE_HX_RANGE_AZ_EL, BKE_HX_RANGE_BEARING = 0, 1, 2
BKE_FX_USER = BKE_HX_USER = 100
# the UKF / CKF hooks compiled from source text (bke_ukf_model_compile_hooks)
BKE_HOOK_X_MEAN, BKE_HOOK_Z_MEAN, BKE_HOOK_RESIDUAL_X, BKE_HOOK_RESIDUAL_Z, BKE_HOOK_STATE_ADD = 1, 2, 4, 8, 16

class KfArgs(ctypes.Structure):
    _fields_ = [
        ("n_filters", c_int64),
        ("dim_x", c_int32), ("dim_z", c_int32), ("dim_u", c_int32),
        ("dtype", c_int32),
        ("flags", c_uint32), ("reserved", c_uint32),
        ("alpha_sq", c_double),
        ("x", c_void_p), ("P", c_void_p),
        ("x_out", c_void_p), ("P_out", c_void_p),
        ("F", c_void_p), ("F_stride", c_int64),
        ("H", c_void_p), ("H_stride", c_int64),
        ("Q", c_void_p), ("Q_stride", c_int64),
        ("R", c_void_p), ("R_stride", c_int64),
        ("B", c_void_p), ("B_stride", c_int64),
        ("u", c_void_p), ("u_stride", c_int64),
        ("z", c_void_p), ("z_valid", c_void_p),
        ("x_prior", c_void_p), ("P_prior", c_void_p),
        ("K", c_void_p), ("y", c_void_p), ("S", c_void_p), ("SI", c_void_p),
        ("log_likelihood", c_void_p),
        ("status", c_void_p),
        ("F_host", c_void_p), ("Q_host", c_void_p), ("H_host", c_void_p), ("R_host", c_void_p),
        ("tile_order", c_void_p),
    ]


class KfRowsArgs(ctypes.Structure):
    _fields_ = [
        ("step", KfArgs),
        ("start", c_int32), ("rows", c_int32),
        ("H_i", c_void_p), ("H_i_stride", c_int64),
        ("R_i", c_void_p), ("R_i_stride", c_int64),
        ("z_record", c_void_p),
    ]


BKE_KF42_MODEL_WORDS = 37
BKE_KF42_MAX_RING = 8


class KfModelMap(ctypes.Structure):
    _fields_ = [
        ("varying", c_uint64),
        ("asymmetric", c_int32), ("duplicate", c_uint32),
        ("words", ctypes.c_float * BKE_KF42_MODEL_WORDS),
    ]


class KfBatchArgs(ctypes.Structure):
    _fields_ = [
        ("step", KfArgs),
        ("n_steps", c_int64),
        ("zs", c_void_p), ("zs_valid", c_void_p),
        ("means", c_void_p), ("covariances", c_void_p),
        ("means_p", c_void_p), ("covariances_p", c_void_p),
    ]


BKE_FLS_FUSED_MAX_LAG = 16


class FlsArgs(ctypes.Structure):
    _fields_ = [
        ("step", KfArgs),
        ("n_steps", c_int64), ("lag", c_int64), ("count", c_int64),
        ("zs", c_void_p), ("us", c_void_p),
        ("xs_smooth", c_void_p), ("xhat", c_void_p),
        ("workspace", c_void_p), ("workspace_bytes", c_size_t),
    ]


class UkfArgs(ctypes.Structure):
    _fields_ = [
        ("n_filters", c_int64),
        ("dim_x", c_int32), ("dim_z", c_int32),
        ("dtype", c_int32), ("flags", c_uint32),
        ("fx_model", c_int32), ("hx_model", c_int32),
        ("dt", c_double),
        ("alpha", c_double), ("beta", c_double), ("kappa", c_double),
        ("x", c_void_p), ("P", c_void_p),
        ("x_out", c_void_p), ("P_out", c_void_p),
        ("Q", c_void_p), ("Q_stride", c_int64),
        ("R", c_void_p), ("R_stride", c_int64),
        ("F", c_void_p), ("F_stride", c_int64),
        ("H", c_void_p), ("H_stride", c_int64),
        ("z", c_void_p), ("z_valid", c_void_p),
        ("x_prior", c_void_p), ("P_prior", c_void_p),
        ("K", c_void_p), ("y", c_void_p), ("S", c_void_p), ("SI", c_void_p),
        ("log_likelihood", c_void_p),
        ("status", c_void_p),
    ]


class CkfArgs(ctypes.Structure):
    _fields_ = [
        ("n_filters", c_int64),
        ("dim_x", c_int32), ("dim_z", c_int32),
        ("dtype", c_int32), ("flags", c_uint32),
        ("fx_model", c_int32), ("hx_model", c_int32),
        ("dt", c_double),
        ("x", c_void_p), ("P", c_void_p),
        ("x_out", c_void_p), ("P_out", c_void_p),
        ("Q", c_void_p), ("Q_stride", c_int64),
        ("R", c_void_p), ("R_stride", c_int64),
        ("F", c_void_p), ("F_stride", c_int64),
        ("H", c_void_p), ("H_stride", c_int64),
        ("z", c_void_p), ("z_valid", c_void_p),
        ("x_prior", c_void_p), ("P_prior", c_void_p),
        ("K", c_void_p), ("y", c_void_p), ("S", c_void_p), ("SI", c_void_p),
        ("log_likelihood", c_void_p),
        ("status", c_void_p),
        ("sigmas_f", c_void_p),
    ]


class EnkfArgs(ctypes.Structure):
    _fields_ = [
        ("n_filters", c_int64),
        ("dim_x", c_int32), ("dim_z", c_int32),
        ("n_members", c_int32),
        ("dtype", c_int32), ("flags", c_uint32),
        ("fx_model", c_int32), ("hx_model", c_int32),
        ("seed", c_uint32), ("counter", c_uint32), ("reserved", c_uint32),
        ("dt", c_double),
        ("x", c_void_p), ("P", c_void_p),
        ("x_out", c_void_p), ("P_out", c_void_p),
        ("sigmas", c_void_p), ("sigmas_out", c_void_p),
        ("Q", c_void_p), ("Q_stride", c_int64),
        ("R", c_void_p), ("R_stride", c_int64),
        ("F", c_void_p), ("F_stride", c_int64),
        ("H", c_void_p), ("H_stride", c_int64),
        ("z", c_void_p), ("z_valid", c_void_p),
        ("x_prior", c_void_p), ("P_prior", c_void_p),
        ("K", c_void_p), ("S", c_void_p), ("SI", c_void_p),
        ("status", c_void_p),
    ]


class SrkfArgs(ctypes.Structure):
    _fields_ = [
        ("n_filters", c_int64),
        ("dim_x", c_int32), ("dim_z", c_int32), ("dim_u", c_int32),
        ("dtype", c_int32),
        ("flags", c_uint32), ("reserved", c_uint32),
        ("x", c_void_p), ("L", c_void_p),
        ("x_out", c_void_p), ("L_out", c_void_p),
        ("F", c_void_p), ("F_stride", c_int64),
        ("H", c_void_p), ("H_stride", c_int64),
        ("Lq", c_void_p), ("Lq_stride", c_int64),
        ("Lr", c_void_p), ("Lr_stride", c_int64),
        ("B", c_void_p), ("B_stride", c_int64),
        ("u", c_void_p), ("u_stride", c_int64),
        ("z", c_void_p), ("z_valid", c_void_p),
        ("x_prior", c_void_p), ("L_prior", c_void_p),
        ("K", c_void_p), ("y", c_void_p), ("S1_2", c_void_p), ("SI1_2", c_void_p),
        ("status", c_void_p),
    ]


BKE_CHOLESKY_MAX_DIM = 16

BKE_STATUS_STICKY = 8
BKE_IF_LL_NONE, BKE_IF_LL_FULL, BKE_IF_LL_BROADCAST = 0, 1, 2


class IfArgs(ctypes.Structure):
    _fields_ = [
        ("n_filters", c_int64),
        ("dim_x", c_int32), ("dim_z", c_int32), ("dim_u", c_int32),
        ("dtype", c_int32),
        ("flags", c_uint32), ("ll_mode", c_int32),
        ("x", c_void_p), ("P_inv", c_void_p),
        ("x_out", c_void_p), ("P_inv_out", c_void_p),
        ("no_information", c_void_p),
        ("F", c_void_p), ("F_stride", c_int64),
        ("F_inv", c_void_p), ("F_inv_stride", c_int64),
        ("Q", c_void_p), ("Q_stride", c_int64),
        ("H", c_void_p), ("H_stride", c_int64),
        ("R_inv", c_void_p), ("R_inv_stride", c_int64),
        ("B", c_void_p), ("B_stride", c_int64),
        ("u", c_void_p), ("u_stride", c_int64),
        ("z", c_void_p), ("z_valid", c_void_p),
        ("x_prior", c_void_p), ("P_inv_prior", c_void_p),
        ("K", c_void_p), ("y", c_void_p), ("S", c_void_p), ("log_likelihood", c_void_p),
        ("status", c_void_p),
    ]

BKE_POLY_GH, BKE_POLY_GHK, BKE_POLY_GH_ORDER, BKE_POLY_LSQ, BKE_POLY_FADING = 0, 1, 2, 3, 4
BKE_POLY_UPDATE, BKE_POLY_BATCH = 0, 1


class PolyArgs(ctypes.Structure):
    _fields_ = [
        ("n_filters", c_int64), ("n_steps", c_int64),
        ("family", c_int32), ("order", c_int32), ("dtype", c_int32), ("mode", c_int32),
        ("x", c_void_p), ("dx", c_void_p), ("ddx", c_void_p),
        ("g", c_void_p), ("g_stride", c_int64),
        ("h", c_void_p), ("h_stride", c_int64),
        ("k", c_void_p), ("k_stride", c_int64),
        ("dt", c_void_p), ("dt_stride", c_int64),
        ("dt2", c_void_p), ("dt2_stride", c_int64),
        ("hdt2", c_void_p), ("hdt2_stride", c_int64),
        ("n", c_void_p), ("n_max", c_int64),
        ("z", c_void_p),
        ("results", c_void_p), ("predictions", c_void_p), ("y", c_void_p),
        ("x_prediction", c_void_p), ("dx_prediction", c_void_p), ("ddx_prediction", c_void_p),
        ("K", c_void_p),
    ]


class ScoreArgs(ctypes.Structure):
    _fields_ = [
        ("n_tracks", c_int64), ("n_candidates", c_int64),
        ("dim_x", c_int32), ("dim_z", c_int32), ("dtype", c_int32), ("reserved", c_int32),
        ("x", c_void_p), ("mean", c_void_p), ("P", c_void_p),
        ("S", c_void_p), ("S_stride", c_int64),
        ("H", c_void_p), ("H_stride", c_int64),
        ("R", c_void_p), ("R_stride", c_int64),
        ("z", c_void_p), ("z_track_stride", c_int64), ("z_cand_stride", c_int64),
        ("z_valid", c_void_p),
        ("zhat", c_void_p), ("y", c_void_p), ("d2", c_void_p), ("mahalanobis", c_void_p),
        ("log_likelihood", c_void_p), ("likelihood", c_void_p),
        ("status", c_void_p),
    ]


class UkfScoreArgs(ctypes.Structure):
    _fields_ = [
        ("n_filters", c_int64), ("n_candidates", c_int64),
        ("dim_x", c_int32), ("dim_z", c_int32), ("dtype", c_int32), ("flags", c_uint32),
        ("hx_model", c_int32), ("reserved", c_int32),
        ("alpha", c_double), ("beta", c_double), ("kappa", c_double),
        ("x", c_void_p), ("P", c_void_p),
        ("R", c_void_p), ("R_stride", c_int64),
        ("H", c_void_p), ("H_stride", c_int64),
        ("z", c_void_p), ("z_track_stride", c_int64), ("z_cand_stride", c_int64),
        ("z_valid", c_void_p),
        ("zhat", c_void_p), ("y", c_void_p), ("d2", c_void_p), ("mahalanobis", c_void_p),
        ("log_likelihood", c_void_p), ("likelihood", c_void_p),
        ("status", c_void_p),
    ]


class ResampleShardArgs(ctypes.Structure):
    _fields_ = [
        ("n_local", c_int64), ("n_global", c_int64), ("j_offset", c_int64), ("capacity", c_int64),
        ("weights", c_void_p), ("uniforms", c_void_p),
        ("u", c_double),
        ("carry_approx", c_void_p), ("carry_exact", c_void_p),
        ("indexes", c_void_p), ("out_range", c_void_p), ("carry_out", c_void_p),
        ("workspace", c_void_p), ("workspace_bytes", c_size_t),
        ("info", c_void_p),
        ("is_last", c_int32), ("phase", c_int32),
    ]


class ResampleShardExt(ctypes.Structure):
    _fields_ = [
        ("shard_sum_out", c_void_p), ("shard_sums_all", c_void_p),
        ("composite_out", c_void_p), ("composites_all", c_void_p),
        ("carry_approx_buf", c_void_p), ("carry_exact_buf", c_void_p),
        ("compose_status", c_void_p),
        ("shard_rank", c_int32), ("n_shards", c_int32),
    ]


class ResampleBankArgs(ctypes.Structure):
    _fields_ = [
        ("n_sets", c_int64), ("n_particles", c_int64),
        ("weights", c_void_p), ("u", c_void_p), ("uniforms", c_void_p),
        ("indexes", c_void_p), ("status", c_void_p),
    ]


class ResampleBankGatedArgs(ctypes.Structure):
    _fields_ = [
        ("n_sets", c_int64), ("n_particles", c_int64),
        ("weights", c_void_p), ("u", c_void_p), ("uniforms", c_void_p),
        ("threshold", ctypes.c_double),
        ("particles", c_void_p), ("particle_bytes", c_int64),
        ("indexes", c_void_p), ("neff", c_void_p), ("resampled", c_void_p), ("status", c_void_p),
        ("workspace", c_void_p), ("workspace_bytes", c_size_t),
    ]


class MultinomialResampleBankArgs(ctypes.Structure):
    _fields_ = [
        ("n_sets", c_int64), ("n_particles", c_int64),
        ("weights", c_void_p), ("uniforms", c_void_p),
        ("indexes", c_void_p), ("status", c_void_p),
        ("workspace", c_void_p), ("workspace_bytes", c_size_t),
    ]


class ResidualResampleBankArgs(ctypes.Structure):
    _fields_ = [
        ("n_sets", c_int64), ("n_particles", c_int64),
        ("weights", c_void_p), ("uniforms", c_void_p),
        ("indexes", c_void_p), ("n_copies", c_void_p), ("status", c_void_p),
        ("workspace", c_void_p), ("workspace_bytes", c_size_t),
    ]


class RtsArgs(ctypes.Structure):
    _fields_ = [
        ("n_filters", c_int64), ("n_steps", c_int64),
        ("dim_x", c_int32), ("dtype", c_int32), ("model_shift", c_int32), ("reserved", c_int32),
        ("Xs", c_void_p), ("Ps", c_void_p),
        ("F", c_void_p), ("F_stride", c_int64), ("F_step_stride", c_int64),
        ("Q", c_void_p), ("Q_stride", c_int64), ("Q_step_stride", c_int64),
        ("x_out", c_void_p), ("P_out", c_void_p), ("K", c_void_p), ("Pp", c_void_p),
        ("status", c_void_p),
    ]


class UkfRtsArgs(ctypes.Structure):
    _fields_ = [
        ("n_filters", c_int64), ("n_steps", c_int64),
        ("dim_x", c_int32), ("dtype", c_int32), ("fx_model", c_int32), ("flags", c_uint32),
        ("alpha", c_double), ("beta", c_double), ("kappa", c_double), ("dt", c_double),
        ("dts", c_void_p),
        ("Xs", c_void_p), ("Ps", c_void_p),
        ("Q", c_void_p), ("Q_stride", c_int64),
        ("F", c_void_p), ("F_stride", c_int64),
        ("x_out", c_void_p), ("P_out", c_void_p), ("K", c_void_p),
        ("status", c_void_p),
    ]


BKE_MM_MAX_MODELS = 8
BKE_MM_MMAE = 1
BKE_MM_FROM_MU = 2


class MmArgs(ctypes.Structure):
    _fields_ = [
        ("n_tracks", c_int64),
        ("dim_x", c_int32), ("n_models", c_int32), ("dtype", c_int32), ("flags", c_uint32),
        ("x", c_void_p * BKE_MM_MAX_MODELS), ("P", c_void_p * BKE_MM_MAX_MODELS),
        ("log_likelihood", c_void_p * BKE_MM_MAX_MODELS),
        ("x_out", c_void_p * BKE_MM_MAX_MODELS), ("P_out", c_void_p * BKE_MM_MAX_MODELS),
        ("mu", c_void_p), ("cbar", c_void_p), ("omega", c_void_p), ("trans", c_void_p),
        ("weights_stride", c_int64),
    ]


_MM = BKE_MM_MAX_MODELS


class ImmBatchArgs(ctypes.Structure):
    _fields_ = [
        ("n_tracks", c_int64),
        ("dim_x", c_int32), ("dim_z", c_int32), ("n_models", c_int32), ("dtype", c_int32),
        ("n_steps", c_int64),
        ("flags", c_uint32), ("reserved", c_uint32),
        ("x", c_void_p * _MM), ("P", c_void_p * _MM),
        ("F", c_void_p * _MM), ("F_stride", c_int64 * _MM),
        ("Q", c_void_p * _MM), ("Q_stride", c_int64 * _MM),
        ("H", c_void_p * _MM), ("H_stride", c_int64 * _MM),
        ("R", c_void_p * _MM), ("R_stride", c_int64 * _MM),
        ("alpha_sq", ctypes.c_double * _MM),
        ("S", c_void_p * _MM), ("log_likelihood", c_void_p * _MM),
        ("K", c_void_p * _MM), ("y", c_void_p * _MM), ("SI", c_void_p * _MM),
        ("x_prior", c_void_p * _MM), ("P_prior", c_void_p * _MM),
        ("status", c_void_p * _MM),
        ("mu", c_void_p), ("cbar", c_void_p), ("omega", c_void_p), ("trans", c_void_p),
        ("zs", c_void_p), ("zs_valid", c_void_p),
        ("means", c_void_p), ("covariances", c_void_p), ("means_p", c_void_p), ("covariances_p", c_void_p),
        ("mus", c_void_p),
    ]


_MODEL = [c_int32] * 5        # dim_x, dim_z, dtype, fx_model, hx_model of the run-time compiled models

# Every prototype of include/bke.h, in header order: symbol -> (restype, argtypes).  A struct pointer is typed
# POINTER(its Structure) except where the caller passes device memory (bke_kf_scan_models' map).
_SIGNATURES = {
    "bke_abi_version": (c_int, []),
    "bke_last_error": (c_char_p, []),
    "bke_device_count": (c_int, []),
    "bke_kf_step": (c_int, [POINTER(KfArgs), c_void_p]),
    "bke_kf_step_correlated": (c_int, [POINTER(KfArgs), c_void_p, c_int64, c_void_p]),
    "bke_kf_update_rows": (c_int, [POINTER(KfRowsArgs), c_void_p]),
    "bke_kf_sym_models_bytes": (c_size_t, [c_int64]),
    "bke_kf_pack_sym_models": (c_int, [c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_void_p]),
    "bke_kf_step_sym": (c_int, [POINTER(KfArgs), c_void_p, c_void_p]),
    "bke_kf_scan_models": (c_int, [c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p]),
    "bke_kf_packed_models_bytes": (c_size_t, [c_int64, c_uint64]),
    "bke_kf_pack_models": (c_int, [c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_uint64, c_void_p, c_void_p]),
    "bke_kf_step_packed": (c_int, [POINTER(KfArgs), c_void_p, POINTER(KfModelMap), c_void_p]),
    "bke_kf_steps_packed": (c_int, [POINTER(KfArgs), c_void_p, POINTER(KfModelMap), POINTER(c_void_p), c_int32,
                                    c_void_p]),
    "bke_capture_node_count": (c_int, [c_void_p, POINTER(c_int64)]),
    "bke_kf_batch_filter": (c_int, [POINTER(KfBatchArgs), c_void_p]),
    "bke_fls_workspace_bytes": (c_size_t, [c_int64, c_int32, c_int32, c_int32, c_int32, c_int64]),
    "bke_fls_smooth": (c_int, [POINTER(FlsArgs), c_void_p]),
    "bke_ukf_step": (c_int, [POINTER(UkfArgs), c_void_p]),
    "bke_ukf_model_compile": (c_int, _MODEL + [c_char_p, c_char_p, POINTER(c_void_p)]),
    "bke_ukf_model_log": (c_char_p, [c_void_p]),
    "bke_ukf_model_registers": (c_int, [c_void_p, c_int32]),
    "bke_ukf_model_free": (None, [c_void_p]),
    "bke_ukf_step_model": (c_int, [POINTER(UkfArgs), c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p]),
    "bke_debug_ukf_model_cubin_bytes": (c_size_t, _MODEL + [c_char_p, c_char_p]),
    "bke_ukf_model_compile_hooks": (c_int, _MODEL + [c_uint32, c_char_p, c_char_p, POINTER(c_void_p)]),
    "bke_debug_ukf_model_hooks_cubin_bytes": (c_size_t, _MODEL + [c_uint32, c_char_p, c_char_p]),
    "bke_ukf_model_compile_points": (c_int, _MODEL + [c_uint32, c_uint32, c_char_p, c_char_p, POINTER(c_void_p)]),
    "bke_debug_ukf_model_points_cubin_bytes": (c_size_t, _MODEL + [c_uint32, c_uint32, c_char_p, c_char_p]),
    "bke_ckf_step": (c_int, [POINTER(CkfArgs), c_void_p]),
    "bke_ckf_model_compile": (c_int, _MODEL + [c_char_p, c_char_p, POINTER(c_void_p)]),
    "bke_ckf_step_model": (c_int, [POINTER(CkfArgs), c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p]),
    "bke_debug_ckf_model_cubin_bytes": (c_size_t, _MODEL + [c_char_p, c_char_p]),
    "bke_ckf_model_compile_hooks": (c_int, _MODEL + [c_uint32, c_char_p, c_char_p, POINTER(c_void_p)]),
    "bke_debug_ckf_model_hooks_cubin_bytes": (c_size_t, _MODEL + [c_uint32, c_char_p, c_char_p]),
    "bke_enkf_initialize": (c_int, [c_int64, c_int32, c_int32, c_int32, c_uint32, c_uint32, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p]),
    "bke_enkf_step": (c_int, [POINTER(EnkfArgs), c_void_p]),
    "bke_enkf_model_compile": (c_int, _MODEL + [c_char_p, c_char_p, POINTER(c_void_p)]),
    "bke_enkf_step_model": (c_int, [POINTER(EnkfArgs), c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p]),
    "bke_debug_enkf_model_cubin_bytes": (c_size_t, _MODEL + [c_char_p, c_char_p]),
    "bke_srkf_step": (c_int, [POINTER(SrkfArgs), c_void_p]),
    "bke_cholesky_lower": (c_int, [c_int64, c_int32, c_int32, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "bke_if_step": (c_int, [POINTER(IfArgs), c_void_p]),
    "bke_inverse": (c_int, [c_int64, c_int32, c_int32, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "bke_poly_filter": (c_int, [POINTER(PolyArgs), c_void_p]),
    "bke_score_measurements": (c_int, [POINTER(ScoreArgs), c_void_p]),
    "bke_ukf_score": (c_int, [POINTER(UkfScoreArgs), c_void_p]),
    "bke_ukf_score_model": (c_int, [POINTER(UkfScoreArgs), c_void_p, c_void_p, c_int64, c_void_p]),
    "bke_debug_ukf_score_model_cubin_bytes": (c_size_t, _MODEL + [c_uint32, c_uint32, c_char_p, c_char_p]),
    "bke_merwe_sigma_points": (c_int, [c_int64, c_int32, c_int32, c_double, c_double, c_double, c_void_p, c_void_p,
                                       c_void_p, c_void_p, c_void_p]),
    "bke_simplex_sigma_points": (c_int, [c_int64, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_void_p]),
    "bke_unscented_transform": (c_int, [c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_int64, c_void_p, c_void_p, c_void_p]),
    "bke_resample_workspace_bytes": (c_size_t, [c_int64]),
    "bke_systematic_resample": (c_int, [c_int64, c_void_p, c_double, c_void_p, c_void_p, c_size_t, c_void_p,
                                        c_void_p, c_void_p]),
    "bke_stratified_resample": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p,
                                        c_void_p, c_void_p]),
    "bke_resample_normalized": (c_int, [c_int64, c_void_p, c_double, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]),
    "bke_resample_shard": (c_int, [POINTER(ResampleShardArgs), c_void_p]),
    "bke_resample_composite_bytes": (c_size_t, []),
    "bke_resample_shard_stage": (c_int, [POINTER(ResampleShardArgs), POINTER(ResampleShardExt), c_int32,
                                         c_void_p]),
    "bke_resample_shard_compose": (c_int, [POINTER(ResampleShardArgs), c_void_p, c_void_p]),
    "bke_resample_compose_carry": (c_int, [c_int32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "bke_resample_bank": (c_int, [POINTER(ResampleBankArgs), c_void_p]),
    "bke_resample_bank_gated_workspace_bytes": (c_size_t, [c_int64]),
    "bke_resample_bank_gated": (c_int, [POINTER(ResampleBankGatedArgs), c_void_p]),
    "bke_resample_bank_gated_stats": (c_int, [POINTER(ResampleBankGatedArgs), c_void_p]),
    "bke_resample_bank_gated_apply": (c_int, [POINTER(ResampleBankGatedArgs), c_void_p]),
    "bke_multinomial_resample_bank_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "bke_multinomial_resample_bank": (c_int, [POINTER(MultinomialResampleBankArgs), c_void_p]),
    "bke_residual_resample_bank_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "bke_residual_resample_bank_prepare": (c_int, [POINTER(ResidualResampleBankArgs), c_void_p]),
    "bke_residual_resample_bank_search": (c_int, [POINTER(ResidualResampleBankArgs), c_void_p]),
    "bke_weights_sum": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "bke_weights_scale": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "bke_kf_rts_smoother": (c_int, [POINTER(RtsArgs), c_void_p]),
    "bke_ukf_rts_smoother": (c_int, [POINTER(UkfRtsArgs), c_void_p]),
    "bke_ukf_rts_smoother_model": (c_int, [POINTER(UkfRtsArgs), c_void_p, c_void_p, c_int64, c_void_p]),
    "bke_mm_probabilities": (c_int, [POINTER(MmArgs), c_void_p]),
    "bke_mm_mix": (c_int, [POINTER(MmArgs), c_void_p]),
    "bke_mm_estimate": (c_int, [POINTER(MmArgs), c_void_p]),
    "bke_imm_batch_filter": (c_int, [POINTER(ImmBatchArgs), c_void_p]),
    "bke_cumsum_exact": (c_int, [c_int64, c_void_p, c_void_p, c_int32, c_void_p, c_size_t, c_void_p, c_void_p]),
    "bke_searchsorted": (c_int, [c_int64, c_void_p, c_int64, c_void_p, c_int32, c_void_p, c_void_p]),
    "bke_multinomial_resample": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_size_t, c_void_p, c_void_p]),
    "bke_gather_rows": (c_int, [c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int32, c_void_p, c_void_p,
                                c_void_p]),
    "bke_gather_rows_bank": (c_int, [c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int32, c_void_p, c_void_p,
                                     c_void_p]),
    "bke_residual_workspace_bytes": (c_size_t, [c_int64]),
    "bke_residual_prepare": (c_int, [c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                     c_void_p]),
    "bke_searchsorted_bracket_sweep": (c_int, [c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                               c_void_p, c_void_p]),
}

# every symbol include/bke.h declares (build() and the tests check that the library exports all of them)
EXPORTED_SYMBOLS = list(_SIGNATURES)


class BkeError(RuntimeError):
    pass


_lib = None


def lib_path():
    return _build.LIB


def _point_at_nvrtc():
    """User-supplied UKF models are compiled by NVRTC, which libbke.so dlopens on first use: prefer the toolkit's
    copy, else the one pip installed next to torch's CUDA libraries (BKE_NVRTC_LIB overrides both)."""
    if os.environ.get("BKE_NVRTC_LIB"):
        return
    import glob
    import sys
    cands = sorted(glob.glob("/usr/local/cuda/lib64/libnvrtc.so.1*"))
    for sp in sys.path:
        cands += sorted(glob.glob(os.path.join(sp, "nvidia", "cuda_nvrtc", "lib", "libnvrtc.so.1*")))
    if cands:
        os.environ["BKE_NVRTC_LIB"] = cands[0]


def kernel_include_dirs():
    """Directories NVRTC reads the engine's kernel headers from (bke_ukf_model_compile)."""
    here = os.path.dirname(os.path.abspath(__file__))
    return os.path.join(here, "csrc") + ":" + os.path.join(os.path.dirname(here), "include")


def load():
    """Load (building first if the sources are newer) and type the library."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("BKE_LIB_PATH") or _build.LIB      # BKE_LIB_PATH: an explicitly chosen build (A/B measurements)
    if os.environ.get("BKE_LIB_PATH"):
        if not os.path.exists(path):
            raise BkeError("BKE_LIB_PATH=%s does not exist" % path)
    else:
        try:
            if _build.needs_build():
                _build.build()
        except Exception as e:  # stale or missing and not buildable
            if not os.path.exists(path):
                raise BkeError("libbke.so is missing and could not be built (%s); the engine has no "
                               "CPU fallback" % e)
    _point_at_nvrtc()
    lib = ctypes.CDLL(path)
    for name, (restype, argtypes) in _SIGNATURES.items():
        f = getattr(lib, name)
        f.restype, f.argtypes = restype, argtypes
    if lib.bke_abi_version() != BKE_ABI_VERSION:
        raise BkeError("libbke.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc):
    if rc != BKE_OK:
        msg = load().bke_last_error().decode("utf-8", "replace")
        if rc == BKE_ERR_BAD_ARG:
            raise ValueError(msg)
        if rc == BKE_ERR_UNSUPPORTED:
            raise NotImplementedError(msg)
        raise BkeError(msg)
