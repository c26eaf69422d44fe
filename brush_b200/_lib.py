"""ctypes binding of libbrush_b200.so -- the C ABI declared in include/brush_b200.h.

There is no CPU fallback: if the CUDA library is missing or a symbol cannot be resolved the
import of any op fails loudly.  PyTorch is used by the callers only for device memory and
streams; no torch type crosses this boundary.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbrush_b200.so")

BG_OK, BG_ERR_NULL, BG_ERR_INVALID, BG_ERR_CUDA, BG_ERR_CAPACITY, BG_ERR_UNSUPPORTED = range(6)
PASS_FORWARD, PASS_BACKWARD, PASS_BACKWARD_SMOOTH = 0, 1, 2
PROJECTED_STRIDE = 16
VCOMBINED_STRIDE = 10
ABI_VERSION = 13
BILAGRID_L, BILAGRID_H, BILAGRID_W = 8, 16, 16
BILAGRID_FLOATS = BILAGRID_L * BILAGRID_H * BILAGRID_W * 12

_STATUS_NAMES = {1: "BG_ERR_NULL", 2: "BG_ERR_INVALID", 3: "BG_ERR_CUDA", 4: "BG_ERR_CAPACITY", 5: "BG_ERR_UNSUPPORTED"}


class BgError(RuntimeError):
    def __init__(self, status: int, where: str, detail: str):
        self.status = status
        super().__init__(f"{where}: {_STATUS_NAMES.get(status, status)} {detail}".strip())


class BgCamera(C.Structure):
    _fields_ = [
        ("viewmat", C.c_float * 12),
        ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
        ("cam_pos", C.c_float * 3),
        ("lim_pos_x", C.c_float), ("lim_pos_y", C.c_float), ("lim_neg_x", C.c_float), ("lim_neg_y", C.c_float),
        ("half_max_render_fov", C.c_float),
        ("camera_model", C.c_uint32),
        ("model_params", C.c_float * 8),
    ]


class BgRenderState(C.Structure):
    _fields_ = [
        ("projected", C.c_void_p),
        ("compact_gid_from_isect", C.c_void_p),
        ("global_from_compact_gid", C.c_void_p),
        ("compact_from_global_gid", C.c_void_p),
        ("tile_offsets", C.c_void_p),
        ("depths", C.c_void_p),
        ("tile_id_from_isect", C.c_void_p),
        ("counters_dev", C.c_void_p),
        ("counters_host", C.POINTER(C.c_uint32)),
        ("n", C.c_uint32), ("k", C.c_uint32), ("w", C.c_uint32), ("h", C.c_uint32),
        ("tiles_x", C.c_uint32), ("tiles_y", C.c_uint32),
        ("mip", C.c_int32), ("pass_", C.c_int32),
    ]


class BgTrainStepArgs(C.Structure):
    _fields_ = [
        ("cam", BgCamera),
        ("w", C.c_uint32), ("h", C.c_uint32), ("n", C.c_uint32), ("k", C.c_uint32),
        ("mip", C.c_int32),
        ("background", C.c_float * 3),
        ("transforms", C.c_void_p), ("sh", C.c_void_p), ("raw_opac", C.c_void_p),
        ("m_t", C.c_void_p), ("v_t", C.c_void_p), ("m_sh", C.c_void_p), ("v_sh", C.c_void_p), ("m_o", C.c_void_p), ("v_o", C.c_void_p),
        ("refine_norm", C.c_void_p), ("vis_weight", C.c_void_p), ("max_screen", C.c_void_p),
        ("gt_packed", C.c_void_p),
        ("l1_weight", C.c_float), ("ssim_weight", C.c_float),
        ("has_composite_bg", C.c_int32),
        ("composite_bg", C.c_float * 3),
        ("mask", C.c_int32), ("channels", C.c_int32),
        ("alpha_weight", C.c_float),
        ("lr_mean", C.c_float), ("lr_rotation", C.c_float), ("lr_scale", C.c_float), ("lr_coeffs_dc", C.c_float),
        ("lr_coeffs_sh_scale", C.c_float), ("lr_opac", C.c_float),
        ("noise_scale", C.c_float), ("median_scale", C.c_float),
        ("seed", C.c_uint64),
        ("step", C.c_int32),
        ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_uint64),
        ("loss_out", C.c_void_p),
        ("state_out", BgRenderState),
    ]


class BgDepthSupervision(C.Structure):
    _fields_ = [
        ("target", C.c_void_p),
        ("weight", C.c_float),
        ("valid_count", C.c_uint32),
        ("depth_loss_out", C.c_void_p),
    ]


class BgTrainUpdateArgs(C.Structure):
    _fields_ = [
        ("n", C.c_uint32), ("k", C.c_uint32),
        ("transforms", C.c_void_p), ("sh", C.c_void_p), ("raw_opac", C.c_void_p),
        ("m_t", C.c_void_p), ("v_t", C.c_void_p), ("m_sh", C.c_void_p), ("v_sh", C.c_void_p), ("m_o", C.c_void_p), ("v_o", C.c_void_p),
        ("refine_norm", C.c_void_p), ("vis_weight", C.c_void_p), ("max_screen", C.c_void_p),
        ("v_transforms", C.c_void_p), ("v_sh_grad", C.c_void_p), ("v_raw_opac", C.c_void_p),
        ("v_refine", C.c_void_p), ("visible", C.c_void_p), ("max_radius", C.c_void_p),
        ("lr_mean", C.c_float), ("lr_rotation", C.c_float), ("lr_scale", C.c_float), ("lr_coeffs_dc", C.c_float),
        ("lr_coeffs_sh_scale", C.c_float), ("lr_opac", C.c_float),
        ("noise_scale", C.c_float), ("median_scale", C.c_float),
        ("seed", C.c_uint64),
        ("step", C.c_int32),
        ("min_scale", C.c_void_p),
    ]


class BgRefineStats(C.Structure):
    _fields_ = [("num_added", C.c_uint32), ("num_split_oversized", C.c_uint32), ("num_split_high_grad", C.c_uint32),
                ("num_pruned", C.c_uint32), ("num_pruned_non_finite", C.c_uint32), ("total_splats", C.c_uint32)]


class BgRefineArgs(C.Structure):
    _fields_ = [
        ("n", C.c_uint32), ("k", C.c_uint32), ("capacity", C.c_uint32),
        ("transforms", C.c_void_p), ("sh", C.c_void_p), ("raw_opac", C.c_void_p),
        ("m_t", C.c_void_p), ("v_t", C.c_void_p), ("m_sh", C.c_void_p), ("v_sh", C.c_void_p), ("m_o", C.c_void_p), ("v_o", C.c_void_p),
        ("refine_norm", C.c_void_p), ("vis_weight", C.c_void_p), ("max_screen", C.c_void_p),
        ("transforms_out", C.c_void_p), ("sh_out", C.c_void_p), ("raw_opac_out", C.c_void_p),
        ("m_t_out", C.c_void_p), ("v_t_out", C.c_void_p), ("m_sh_out", C.c_void_p), ("v_sh_out", C.c_void_p), ("m_o_out", C.c_void_p),
        ("v_o_out", C.c_void_p),
        ("bounds_center", C.c_float * 3),
        ("max_allowed", C.c_float),
        ("split_at_screen_size", C.c_float), ("growth_grad_threshold", C.c_float), ("growth_select_fraction", C.c_float),
        ("max_splats", C.c_uint32),
        ("growth_enabled", C.c_int32),
        ("opac_decay_minus", C.c_float),
        ("seed", C.c_uint64),
        ("refine_index", C.c_uint32),
        ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_uint64),
    ]


class BgDecimateArgs(C.Structure):
    _fields_ = [
        ("n", C.c_uint32), ("k", C.c_uint32), ("target", C.c_uint32),
        ("scores", C.c_void_p),
        ("transforms", C.c_void_p), ("sh", C.c_void_p), ("raw_opac", C.c_void_p),
        ("min_scale", C.c_void_p),
        ("transforms_out", C.c_void_p), ("sh_out", C.c_void_p), ("raw_opac_out", C.c_void_p),
        ("min_scale_out", C.c_void_p),
        ("kept_ids_out", C.c_void_p),
        ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_uint64),
    ]


class BgCompressArgs(C.Structure):
    _fields_ = [
        ("n", C.c_uint32), ("k", C.c_uint32),
        ("transforms", C.c_void_p), ("sh", C.c_void_p), ("raw_opac", C.c_void_p),
        ("chunks_out", C.c_void_p),
        ("packed_out", C.c_void_p),
        ("sh_out", C.c_void_p),
        ("order_out", C.c_void_p),
        ("count_out", C.c_void_p),
        ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_uint64),
    ]


class BgTsdfGrid(C.Structure):
    _fields_ = [
        ("origin", C.c_float * 3), ("h", C.c_float),
        ("dims", C.c_uint32 * 3), ("trunc", C.c_float),
        ("tsdf", C.c_void_p), ("weight", C.c_void_p), ("rgb", C.c_void_p),
    ]


class BgSparseTsdfGrid(C.Structure):
    _fields_ = [
        ("origin", C.c_float * 3), ("h", C.c_float),
        ("dims", C.c_uint32 * 3), ("trunc", C.c_float),
        ("brick_slot", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_uint64),
        ("num_bricks", C.c_uint32),
        ("tsdf", C.c_void_p), ("weight", C.c_void_p), ("rgb", C.c_void_p),
    ]


class BgTrainViewsArgs(C.Structure):
    _fields_ = [
        ("w", C.c_uint32), ("h", C.c_uint32), ("n", C.c_uint32), ("k", C.c_uint32),
        ("mip", C.c_int32),
        ("background", C.c_float * 3),
        ("local_views", C.c_uint32),
        ("cams", C.POINTER(BgCamera)),
        ("gt_packed", C.POINTER(C.c_void_p)),
        ("transforms", C.c_void_p), ("sh", C.c_void_p), ("raw_opac", C.c_void_p),
        ("m_t", C.c_void_p), ("v_t", C.c_void_p), ("m_sh", C.c_void_p), ("v_sh", C.c_void_p), ("m_o", C.c_void_p), ("v_o", C.c_void_p),
        ("refine_norm", C.c_void_p), ("vis_weight", C.c_void_p), ("max_screen", C.c_void_p),
        ("min_scale", C.c_void_p),
        ("l1_weight", C.c_float), ("ssim_weight", C.c_float),
        ("has_composite_bg", C.c_int32),
        ("composite_bg", C.c_float * 3),
        ("mask", C.c_int32), ("channels", C.c_int32),
        ("alpha_weight", C.c_float),
        ("lr_mean", C.c_float), ("lr_rotation", C.c_float), ("lr_scale", C.c_float), ("lr_coeffs_dc", C.c_float),
        ("lr_coeffs_sh_scale", C.c_float), ("lr_opac", C.c_float),
        ("noise_scale", C.c_float), ("median_scale", C.c_float),
        ("seed", C.c_uint64),
        ("step", C.c_int32),
        ("chunks", C.c_uint32),
        ("workspace", C.c_void_p),
        ("workspace_bytes", C.c_uint64),
        ("loss_out", C.c_void_p),
        ("state_out", BgRenderState),
    ]


class BgBilagridStep(C.Structure):
    _fields_ = [
        ("grid", C.c_void_p), ("m", C.c_void_p), ("v", C.c_void_p),
        ("step", C.c_int32),
        ("lr", C.c_float), ("tv_weight", C.c_float),
        ("tv_loss_out", C.c_void_p),
    ]


class BgBilagridViews(C.Structure):
    _fields_ = [
        ("grids", C.c_void_p), ("m", C.c_void_p), ("v", C.c_void_p),
        ("steps", C.c_void_p),
        ("num_views", C.c_uint32),
        ("view_index", C.POINTER(C.c_uint32)),
        ("lr", C.c_float), ("tv_weight", C.c_float),
        ("tv_loss_out", C.c_void_p),
    ]


# name -> (restype, argtypes); one entry per function declared in include/brush_b200.h
_P, _U32, _U64, _I32, _I64, _F = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int32, C.c_int64, C.c_float
SIGNATURES = {
    "bg_abi_version": (_U32, []),
    "bg_last_error_string": (C.c_char_p, []),
    "bg_ctx_create": (_I32, [_I32, _U32, _U32, _U32, _U64, C.POINTER(_P)]),
    "bg_ctx_destroy": (_I32, [_P]),
    "bg_ctx_arena_bytes": (_U64, [_P]),
    "bg_render_forward": (_I32, [_P, _P, C.POINTER(BgCamera), _U32, _U32, _U32, _U32, _P, _P, _P, _I32,
                                 C.POINTER(_F), _I32, _P, _P, _P, C.POINTER(BgRenderState)]),
    "bg_rasterize_backward": (_I32, [_P, _P, C.POINTER(BgRenderState), _P, _P, C.POINTER(_F), _I32, _P, _U32]),
    "bg_render_forward_depth": (_I32, [_P, _P, C.POINTER(BgCamera), _U32, _U32, _U32, _U32, _P, _P, _P, _I32,
                                       C.POINTER(_F), _I32, _P, _P, _P, _P, C.POINTER(BgRenderState)]),
    "bg_rasterize_backward_depth": (_I32, [_P, _P, C.POINTER(BgRenderState), _P, _P, _P, _P, C.POINTER(_F), _I32, _P, _U32, _P]),
    "bg_project_backward_depth": (_I32, [_P, _P, C.POINTER(BgCamera), C.POINTER(BgRenderState), _P, _P, _P, _P, _P, _P, _P, _P,
                                         _P]),
    "bg_debug_blend_stats": (_I32, [_P, _P, C.POINTER(BgRenderState), _P, _P, C.POINTER(_F), _P, _P]),
    "bg_project_backward": (_I32, [_P, _P, C.POINTER(BgCamera), C.POINTER(BgRenderState), _P, _P, _P, _P, _P, _P, _P, _P]),
    "bg_normal_noise": (_I32, [_P, _P, C.c_uint64, C.c_uint64, C.c_uint64, _P]),
    "bg_train_step_workspace_bytes": (C.c_uint64, [_U32, _U32, _U32, _U32]),
    "bg_train_step": (_I32, [_P, _P, C.POINTER(BgTrainStepArgs)]),
    "bg_depth_loss_num_partials": (_U32, [_U32, _U32]),
    "bg_depth_loss_fused": (_I32, [_P, _P, _P, _P, _P, _U32, _U32, _F, _P, _P, _P]),
    "bg_train_step_depth_workspace_bytes": (_U64, [_U32, _U32, _U32, _U32]),
    "bg_train_step_depth": (_I32, [_P, _P, C.POINTER(BgTrainStepArgs), C.POINTER(BgDepthSupervision)]),
    "bg_train_update": (_I32, [_P, _P, C.POINTER(BgTrainUpdateArgs)]),
    "bg_dp_unique_id": (_I32, [_P]),
    "bg_dp_comm_create": (_I32, [_P, _P, _I32, _I32, C.POINTER(_P)]),
    "bg_dp_comm_destroy": (_I32, [_P]),
    "bg_dp_small_floats": (_U64, [_U32]),
    "bg_dp_stat_floats": (_U64, [_U32]),
    "bg_dp_record_floats": (_U64, [_U32, _U32]),
    "bg_dp_pack_view": (_I32, [_P, _P, _U32, _U32, _U32, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "bg_dp_exchange": (_I32, [_P, _P, _P, _U32, _U32, _P, _P, _P, _P, _U32]),
    "bg_train_step_views_workspace_bytes": (_U64, [_U32, _U32, _U32, _U32, _U32, _U32]),
    "bg_train_step_views": (_I32, [_P, _P, _P, C.POINTER(BgTrainViewsArgs)]),
    "bg_train_step_views_depth_workspace_bytes": (_U64, [_U32, _U32, _U32, _U32, _U32, _U32]),
    "bg_train_step_views_depth": (_I32, [_P, _P, _P, C.POINTER(BgTrainViewsArgs), C.POINTER(BgDepthSupervision)]),
    "bg_refine_workspace_bytes": (_U64, [_U32]),
    "bg_refine": (_I32, [_P, _P, C.POINTER(BgRefineArgs), C.POINTER(BgRefineStats)]),
    "bg_bounds_percentile": (_I32, [_P, _P, _U32, _P, _F, _P, _U64, C.POINTER(_F)]),
    "bg_compute_min_scale": (_I32, [_P, _P, _U32, _P, _P, _U32, _F, _P]),
    "bg_fold_min_scale_forward": (_I32, [_P, _P, _U32, _P, _P, _P, _P, _P]),
    "bg_fold_min_scale_backward": (_I32, [_P, _P, _U32, _P, _P, _P, _P, _P]),
    "bg_project_backward_factored": (_I32, [_P, _P, C.POINTER(BgCamera), C.POINTER(BgRenderState), _P, _P, _P, _P, _P, _P, _P, _P]),
    "bg_sh_grad_from_views": (_I32, [_P, _P, _U32, _U32, _P, C.POINTER(_F), _U32, _P, C.c_uint64, _F, _P]),
    "bg_radix_argsort_u32": (_I32, [_P, _P, _P, _P, _U32, _P, _U32, _P, _P]),
    "bg_inclusive_scan_u32": (_I32, [_P, _P, _P, _U32, _P]),
    "bg_image_loss_forward": (_I32, [_P, _P, _P, _P, _U32, _U32, _U32, _I64, _I64, _I64, _F, _F, C.POINTER(_F), _I32, _P]),
    "bg_image_loss_backward": (_I32, [_P, _P, _P, _P, _P, _U32, _U32, _U32, _I64, _I64, _I64, _F, _F, C.POINTER(_F), _I32, _P]),
    "bg_image_loss_num_partials": (_U32, [_U32, _U32, _U32]),
    "bg_image_loss_fused": (_I32, [_P, _P, _P, _P, _U32, _U32, _U32, _I64, _I64, _I64, _F, _F, C.POINTER(_F), _I32,
                                   C.POINTER(_F), _P, _P]),
    "bg_adam_step": (_I32, [_P, _P, _P, _P, _P, _P, _U64, _U32, _P, _F, _F, _F, _F, _I32, _I32]),
    "bg_refine_stats_noise": (_I32, [_P, _P, _U32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _F, _F]),
    "bg_pup_accumulate": (_I32, [_P, _P, _U32, _P, _I32, _P]),
    "bg_pup_log_det": (_I32, [_P, _P, _U32, _P, _P]),
    "bg_decimate_workspace_bytes": (_U64, [_U32]),
    "bg_decimate_to_count": (_I32, [_P, _P, C.POINTER(BgDecimateArgs)]),
    "bg_compress_workspace_bytes": (_U64, [_U32]),
    "bg_compress_splats": (_I32, [_P, _P, C.POINTER(BgCompressArgs)]),
    "bg_tsdf_integrate": (_I32, [_P, _P, C.POINTER(BgTsdfGrid), C.POINTER(BgCamera), _U32, _U32, _P, _P, C.c_float]),
    "bg_mesh_workspace_bytes": (_U64, [_U32, _U32, _U32]),
    "bg_mesh_count": (_I32, [_P, _P, C.POINTER(BgTsdfGrid), _P, _U64, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "bg_mesh_emit": (_I32, [_P, _P, C.POINTER(BgTsdfGrid), _P, _U64, _U32, _U32, _P, _P, _P]),
    "bg_sparse_tsdf_workspace_bytes": (_U64, [_U32, _U32, _U32, _U32, _U32]),
    "bg_sparse_tsdf_mark": (_I32, [_P, _P, C.POINTER(BgSparseTsdfGrid), C.POINTER(BgCamera), _U32, _U32, _P, _P, C.c_float]),
    "bg_sparse_tsdf_allocate": (_I32, [_P, _P, C.POINTER(BgSparseTsdfGrid), C.POINTER(C.c_uint32)]),
    "bg_sparse_tsdf_integrate": (_I32, [_P, _P, C.POINTER(BgSparseTsdfGrid), C.POINTER(BgCamera), _U32, _U32, _P, _P, C.c_float]),
    "bg_sparse_mesh_workspace_bytes": (_U64, [_U32]),
    "bg_sparse_mesh_count": (_I32, [_P, _P, C.POINTER(BgSparseTsdfGrid), _P, _U64, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "bg_sparse_mesh_emit": (_I32, [_P, _P, C.POINTER(BgSparseTsdfGrid), _P, _U64, _U32, _U32, _P, _P, _P]),
    "bg_bilagrid_slice": (_I32, [_P, _P, _P, _P, _U32, _U32, _P]),
    "bg_bilagrid_slice_backward": (_I32, [_P, _P, _P, _P, _P, _U32, _U32, _P, _P]),
    "bg_bilagrid_update": (_I32, [_P, _P, C.POINTER(BgBilagridStep), _P]),
    "bg_train_step_bilagrid_workspace_bytes": (_U64, [_U32, _U32, _U32, _U32]),
    "bg_train_step_bilagrid": (_I32, [_P, _P, C.POINTER(BgTrainStepArgs), C.POINTER(BgDepthSupervision), C.POINTER(BgBilagridStep)]),
    "bg_train_step_views_bilagrid_workspace_bytes": (_U64, [_U32, _U32, _U32, _U32, _U32, _U32]),
    "bg_train_step_views_bilagrid": (_I32, [_P, _P, _P, C.POINTER(BgTrainViewsArgs), C.POINTER(BgDepthSupervision),
                                            C.POINTER(BgBilagridViews)]),
    "bg_bilagrid_update_views": (_I32, [_P, _P, C.POINTER(BgBilagridViews), _U32, _P, _P]),
}

_lib = None


def load() -> C.CDLL:
    """Loads the library and binds every declared symbol; raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m brush_b200.build` (nvcc, sm_90a). "
            "brush_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.bg_abi_version() != ABI_VERSION:
        raise ImportError(f"ABI mismatch: library {lib.bg_abi_version()} != binding {ABI_VERSION}")
    _lib = lib
    return lib


def check(status: int, where: str):
    if status != BG_OK:
        detail = load().bg_last_error_string()
        raise BgError(status, where, detail.decode() if detail else "")


def camera_struct(u) -> BgCamera:
    """u: brush_b200.camera.ProjectUniforms."""
    c = BgCamera()
    for i in range(12):
        c.viewmat[i] = float(u.viewmat[i])
    c.fx, c.fy, c.cx, c.cy = u.fx, u.fy, u.cx, u.cy
    for i in range(3):
        c.cam_pos[i] = float(u.cam_pos[i])
    c.lim_pos_x, c.lim_pos_y, c.lim_neg_x, c.lim_neg_y = u.lim_pos_x, u.lim_pos_y, u.lim_neg_x, u.lim_neg_y
    c.half_max_render_fov = u.half_max_render_fov
    c.camera_model = u.camera_model
    for i, v in enumerate(getattr(u, "model_params", ())):
        c.model_params[i] = float(v)
    return c
