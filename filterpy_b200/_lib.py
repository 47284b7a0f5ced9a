"""ctypes binding of the C-ABI in ``include/bke.h`` (the drop-in boundary).

The library is loaded from ``filterpy_b200/_C/libbke.so`` (built in-tree by ``_build.py``).
There is no CPU fallback: if the library is missing and cannot be built, or a compute entry
point reports no CUDA device, an exception is raised.
"""
import ctypes
import os
from ctypes import c_double, c_int32, c_int64, c_size_t, c_uint32, c_uint64, c_void_p

from . import _build

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

# every symbol include/bke.h declares (tests check that the library exports all of them)
EXPORTED_SYMBOLS = [
    "bke_abi_version", "bke_last_error", "bke_device_count",
    "bke_kf_step", "bke_kf_step_correlated", "bke_kf_update_rows", "bke_kf_batch_filter", "bke_ukf_step",
    "bke_fls_workspace_bytes", "bke_fls_smooth",
    "bke_kf_sym_models_bytes", "bke_kf_pack_sym_models", "bke_kf_step_sym",
    "bke_kf_scan_models", "bke_kf_packed_models_bytes", "bke_kf_pack_models", "bke_kf_step_packed",
    "bke_kf_steps_packed", "bke_capture_node_count",
    "bke_resample_workspace_bytes", "bke_systematic_resample", "bke_stratified_resample",
    "bke_weights_sum", "bke_weights_scale", "bke_resample_shard", "bke_resample_normalized",
    "bke_resample_composite_bytes", "bke_resample_shard_compose", "bke_resample_compose_carry", "bke_resample_shard_stage",
    "bke_merwe_sigma_points", "bke_simplex_sigma_points", "bke_unscented_transform",
    "bke_ukf_model_compile_points", "bke_debug_ukf_model_points_cubin_bytes",
    "bke_ukf_model_compile", "bke_ukf_model_log", "bke_ukf_model_registers", "bke_ukf_model_free", "bke_ukf_step_model",
    "bke_debug_ukf_model_cubin_bytes", "bke_ukf_rts_smoother_model",
    "bke_ckf_step", "bke_ckf_model_compile", "bke_ckf_step_model", "bke_debug_ckf_model_cubin_bytes",
    "bke_ukf_model_compile_hooks", "bke_debug_ukf_model_hooks_cubin_bytes",
    "bke_ckf_model_compile_hooks", "bke_debug_ckf_model_hooks_cubin_bytes",
    "bke_enkf_initialize", "bke_enkf_step", "bke_enkf_model_compile", "bke_enkf_step_model", "bke_debug_enkf_model_cubin_bytes",
    "bke_srkf_step", "bke_cholesky_lower",
    "bke_if_step", "bke_inverse",
    "bke_poly_filter",
    "bke_imm_batch_filter",
    "bke_score_measurements",
    "bke_kf_rts_smoother", "bke_ukf_rts_smoother", "bke_mm_probabilities", "bke_mm_mix", "bke_mm_estimate", "bke_cumsum_exact", "bke_searchsorted", "bke_multinomial_resample", "bke_gather_rows",
    "bke_resample_bank", "bke_gather_rows_bank",
    "bke_multinomial_resample_bank_workspace_bytes", "bke_multinomial_resample_bank",
    "bke_residual_resample_bank_workspace_bytes", "bke_residual_resample_bank_prepare",
    "bke_residual_resample_bank_search",
    "bke_resample_bank_gated_workspace_bytes", "bke_resample_bank_gated", "bke_resample_bank_gated_stats",
    "bke_resample_bank_gated_apply",
    "bke_residual_workspace_bytes", "bke_residual_prepare", "bke_searchsorted_bracket_sweep",
]


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
    lib.bke_abi_version.restype = ctypes.c_int
    lib.bke_last_error.restype = ctypes.c_char_p
    lib.bke_device_count.restype = ctypes.c_int
    lib.bke_kf_step.argtypes = [ctypes.POINTER(KfArgs), c_void_p]
    lib.bke_kf_step.restype = ctypes.c_int
    lib.bke_kf_step_correlated.argtypes = [ctypes.POINTER(KfArgs), c_void_p, c_int64, c_void_p]
    lib.bke_kf_step_correlated.restype = ctypes.c_int
    lib.bke_kf_update_rows.argtypes = [ctypes.POINTER(KfRowsArgs), c_void_p]
    lib.bke_kf_update_rows.restype = ctypes.c_int
    lib.bke_kf_sym_models_bytes.argtypes = [c_int64]
    lib.bke_kf_sym_models_bytes.restype = c_size_t
    lib.bke_kf_pack_sym_models.argtypes = [c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p]
    lib.bke_kf_pack_sym_models.restype = ctypes.c_int
    lib.bke_kf_step_sym.argtypes = [ctypes.POINTER(KfArgs), c_void_p, c_void_p]
    lib.bke_kf_step_sym.restype = ctypes.c_int
    lib.bke_kf_scan_models.argtypes = [c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_void_p, c_void_p]
    lib.bke_kf_scan_models.restype = ctypes.c_int
    lib.bke_kf_packed_models_bytes.argtypes = [c_int64, c_uint64]
    lib.bke_kf_packed_models_bytes.restype = c_size_t
    lib.bke_kf_pack_models.argtypes = [c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_uint64, c_void_p, c_void_p]
    lib.bke_kf_pack_models.restype = ctypes.c_int
    lib.bke_kf_step_packed.argtypes = [ctypes.POINTER(KfArgs), c_void_p, ctypes.POINTER(KfModelMap), c_void_p]
    lib.bke_kf_step_packed.restype = ctypes.c_int
    lib.bke_kf_steps_packed.argtypes = [ctypes.POINTER(KfArgs), c_void_p, ctypes.POINTER(KfModelMap),
                                        ctypes.POINTER(c_void_p), c_int32, c_void_p]
    lib.bke_kf_steps_packed.restype = ctypes.c_int
    lib.bke_capture_node_count.argtypes = [c_void_p, ctypes.POINTER(c_int64)]
    lib.bke_capture_node_count.restype = ctypes.c_int
    lib.bke_kf_batch_filter.argtypes = [ctypes.POINTER(KfBatchArgs), c_void_p]
    lib.bke_kf_batch_filter.restype = ctypes.c_int
    lib.bke_fls_workspace_bytes.argtypes = [c_int64, c_int32, c_int32, c_int32, c_int32, c_int64]
    lib.bke_fls_workspace_bytes.restype = c_size_t
    lib.bke_fls_smooth.argtypes = [ctypes.POINTER(FlsArgs), c_void_p]
    lib.bke_fls_smooth.restype = ctypes.c_int
    lib.bke_ukf_step.argtypes = [ctypes.POINTER(UkfArgs), c_void_p]
    lib.bke_ukf_step.restype = ctypes.c_int
    lib.bke_ukf_model_compile.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, ctypes.c_char_p, ctypes.c_char_p,
                                          ctypes.POINTER(c_void_p)]
    lib.bke_ukf_model_compile.restype = ctypes.c_int
    lib.bke_ukf_model_log.argtypes = [c_void_p]
    lib.bke_ukf_model_log.restype = ctypes.c_char_p
    lib.bke_ukf_model_registers.argtypes = [c_void_p, c_int32]
    lib.bke_ukf_model_registers.restype = ctypes.c_int
    lib.bke_ukf_model_free.argtypes = [c_void_p]
    lib.bke_ukf_model_free.restype = None
    lib.bke_ukf_step_model.argtypes = [ctypes.POINTER(UkfArgs), c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p]
    lib.bke_ukf_step_model.restype = ctypes.c_int
    lib.bke_ukf_rts_smoother_model.argtypes = [ctypes.POINTER(UkfRtsArgs), c_void_p, c_void_p, c_int64, c_void_p]
    lib.bke_ukf_rts_smoother_model.restype = ctypes.c_int
    lib.bke_debug_ukf_model_cubin_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, ctypes.c_char_p, ctypes.c_char_p]
    lib.bke_debug_ukf_model_cubin_bytes.restype = c_size_t
    lib.bke_ukf_model_compile_points.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, c_uint32, c_uint32,
                                                 ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(c_void_p)]
    lib.bke_ukf_model_compile_points.restype = ctypes.c_int
    lib.bke_debug_ukf_model_points_cubin_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, c_uint32, c_uint32,
                                                           ctypes.c_char_p, ctypes.c_char_p]
    lib.bke_debug_ukf_model_points_cubin_bytes.restype = c_size_t
    for fam in ("ukf", "ckf"):
        f = getattr(lib, "bke_%s_model_compile_hooks" % fam)
        f.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, c_uint32, ctypes.c_char_p, ctypes.c_char_p,
                      ctypes.POINTER(c_void_p)]
        f.restype = ctypes.c_int
        f = getattr(lib, "bke_debug_%s_model_hooks_cubin_bytes" % fam)
        f.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, c_uint32, ctypes.c_char_p, ctypes.c_char_p]
        f.restype = c_size_t
    lib.bke_ckf_step.argtypes = [ctypes.POINTER(CkfArgs), c_void_p]
    lib.bke_ckf_step.restype = ctypes.c_int
    lib.bke_ckf_model_compile.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, ctypes.c_char_p, ctypes.c_char_p,
                                          ctypes.POINTER(c_void_p)]
    lib.bke_ckf_model_compile.restype = ctypes.c_int
    lib.bke_ckf_step_model.argtypes = [ctypes.POINTER(CkfArgs), c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p]
    lib.bke_ckf_step_model.restype = ctypes.c_int
    lib.bke_debug_ckf_model_cubin_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, ctypes.c_char_p, ctypes.c_char_p]
    lib.bke_debug_ckf_model_cubin_bytes.restype = c_size_t
    lib.bke_enkf_initialize.argtypes = [c_int64, c_int32, c_int32, c_int32, c_uint32, c_uint32, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p]
    lib.bke_enkf_initialize.restype = ctypes.c_int
    lib.bke_enkf_step.argtypes = [ctypes.POINTER(EnkfArgs), c_void_p]
    lib.bke_enkf_step.restype = ctypes.c_int
    lib.bke_enkf_model_compile.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, ctypes.c_char_p, ctypes.c_char_p,
                                           ctypes.POINTER(c_void_p)]
    lib.bke_enkf_model_compile.restype = ctypes.c_int
    lib.bke_enkf_step_model.argtypes = [ctypes.POINTER(EnkfArgs), c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p]
    lib.bke_enkf_step_model.restype = ctypes.c_int
    lib.bke_debug_enkf_model_cubin_bytes.argtypes = [c_int32, c_int32, c_int32, c_int32, c_int32, ctypes.c_char_p, ctypes.c_char_p]
    lib.bke_debug_enkf_model_cubin_bytes.restype = c_size_t
    lib.bke_srkf_step.argtypes = [ctypes.POINTER(SrkfArgs), c_void_p]
    lib.bke_srkf_step.restype = ctypes.c_int
    lib.bke_cholesky_lower.argtypes = [c_int64, c_int32, c_int32, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]
    lib.bke_cholesky_lower.restype = ctypes.c_int
    lib.bke_if_step.argtypes = [ctypes.POINTER(IfArgs), c_void_p]
    lib.bke_if_step.restype = ctypes.c_int
    lib.bke_inverse.argtypes = [c_int64, c_int32, c_int32, c_void_p, c_int64, c_void_p, c_void_p, c_void_p]
    lib.bke_inverse.restype = ctypes.c_int
    lib.bke_poly_filter.argtypes = [ctypes.POINTER(PolyArgs), c_void_p]
    lib.bke_poly_filter.restype = ctypes.c_int
    lib.bke_score_measurements.argtypes = [ctypes.POINTER(ScoreArgs), c_void_p]
    lib.bke_score_measurements.restype = ctypes.c_int
    lib.bke_resample_workspace_bytes.argtypes = [c_int64]
    lib.bke_resample_workspace_bytes.restype = c_size_t
    lib.bke_systematic_resample.argtypes = [c_int64, c_void_p, c_double, c_void_p, c_void_p, c_size_t,
                                            c_void_p, c_void_p, c_void_p]
    lib.bke_systematic_resample.restype = ctypes.c_int
    lib.bke_stratified_resample.argtypes = [c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                            c_void_p, c_void_p, c_void_p]
    lib.bke_stratified_resample.restype = ctypes.c_int
    lib.bke_resample_normalized.argtypes = [c_int64, c_void_p, c_double, c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_size_t, c_void_p, c_void_p, c_void_p]
    lib.bke_resample_normalized.restype = ctypes.c_int
    lib.bke_weights_sum.argtypes = [c_int64, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]
    lib.bke_weights_sum.restype = ctypes.c_int
    lib.bke_weights_scale.argtypes = [c_int64, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.bke_weights_scale.restype = ctypes.c_int
    lib.bke_resample_composite_bytes.argtypes = []
    lib.bke_resample_composite_bytes.restype = c_size_t
    lib.bke_resample_shard_compose.argtypes = [ctypes.POINTER(ResampleShardArgs), c_void_p, c_void_p]
    lib.bke_resample_shard_compose.restype = ctypes.c_int
    lib.bke_resample_compose_carry.argtypes = [c_int32, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.bke_resample_compose_carry.restype = ctypes.c_int
    lib.bke_resample_shard_stage.argtypes = [ctypes.POINTER(ResampleShardArgs), ctypes.POINTER(ResampleShardExt), c_int32, c_void_p]
    lib.bke_resample_shard_stage.restype = ctypes.c_int
    lib.bke_resample_shard.argtypes = [ctypes.POINTER(ResampleShardArgs), c_void_p]
    lib.bke_resample_shard.restype = ctypes.c_int
    lib.bke_merwe_sigma_points.argtypes = [c_int64, c_int32, c_int32, c_double, c_double, c_double,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.bke_merwe_sigma_points.restype = ctypes.c_int
    lib.bke_simplex_sigma_points.argtypes = [c_int64, c_int32, c_int32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.bke_simplex_sigma_points.restype = ctypes.c_int
    lib.bke_unscented_transform.argtypes = [c_int64, c_int32, c_int32, c_int32, c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_int64, c_void_p, c_void_p, c_void_p]
    lib.bke_unscented_transform.restype = ctypes.c_int
    lib.bke_kf_rts_smoother.argtypes = [ctypes.POINTER(RtsArgs), c_void_p]
    lib.bke_kf_rts_smoother.restype = ctypes.c_int
    lib.bke_ukf_rts_smoother.argtypes = [ctypes.POINTER(UkfRtsArgs), c_void_p]
    lib.bke_ukf_rts_smoother.restype = ctypes.c_int
    lib.bke_imm_batch_filter.argtypes = [ctypes.POINTER(ImmBatchArgs), c_void_p]
    lib.bke_imm_batch_filter.restype = ctypes.c_int
    for name in ("bke_mm_probabilities", "bke_mm_mix", "bke_mm_estimate"):
        getattr(lib, name).argtypes = [ctypes.POINTER(MmArgs), c_void_p]
        getattr(lib, name).restype = ctypes.c_int
    lib.bke_cumsum_exact.argtypes = [c_int64, c_void_p, c_void_p, c_int32, c_void_p, c_size_t, c_void_p, c_void_p]
    lib.bke_cumsum_exact.restype = ctypes.c_int
    lib.bke_searchsorted.argtypes = [c_int64, c_void_p, c_int64, c_void_p, c_int32, c_void_p, c_void_p]
    lib.bke_searchsorted.restype = ctypes.c_int
    lib.bke_multinomial_resample.argtypes = [c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                             c_size_t, c_void_p, c_void_p]
    lib.bke_multinomial_resample.restype = ctypes.c_int
    lib.bke_gather_rows.argtypes = [c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int32, c_void_p, c_void_p,
                                    c_void_p]
    lib.bke_gather_rows.restype = ctypes.c_int
    lib.bke_gather_rows_bank.argtypes = [c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int32, c_void_p, c_void_p,
                                         c_void_p]
    lib.bke_gather_rows_bank.restype = ctypes.c_int
    lib.bke_resample_bank.argtypes = [ctypes.POINTER(ResampleBankArgs), c_void_p]
    lib.bke_resample_bank.restype = ctypes.c_int
    for name in ("bke_multinomial_resample_bank_workspace_bytes", "bke_residual_resample_bank_workspace_bytes"):
        getattr(lib, name).argtypes = [c_int64, c_int64]
        getattr(lib, name).restype = c_size_t
    lib.bke_multinomial_resample_bank.argtypes = [ctypes.POINTER(MultinomialResampleBankArgs), c_void_p]
    lib.bke_multinomial_resample_bank.restype = ctypes.c_int
    lib.bke_resample_bank_gated_workspace_bytes.argtypes = [c_int64]
    lib.bke_resample_bank_gated_workspace_bytes.restype = c_size_t
    for name in ("bke_resample_bank_gated", "bke_resample_bank_gated_stats", "bke_resample_bank_gated_apply"):
        getattr(lib, name).argtypes = [ctypes.POINTER(ResampleBankGatedArgs), c_void_p]
        getattr(lib, name).restype = ctypes.c_int
    for name in ("bke_residual_resample_bank_prepare", "bke_residual_resample_bank_search"):
        getattr(lib, name).argtypes = [ctypes.POINTER(ResidualResampleBankArgs), c_void_p]
        getattr(lib, name).restype = ctypes.c_int
    lib.bke_residual_workspace_bytes.argtypes = [c_int64]
    lib.bke_residual_workspace_bytes.restype = c_size_t
    lib.bke_residual_prepare.argtypes = [c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                         c_void_p]
    lib.bke_residual_prepare.restype = ctypes.c_int
    lib.bke_searchsorted_bracket_sweep.argtypes = [c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                                   c_void_p, c_void_p]
    lib.bke_searchsorted_bracket_sweep.restype = ctypes.c_int
    if lib.bke_abi_version() != 1:
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
