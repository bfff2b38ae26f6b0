"""ctypes binding of libsgn_raster.so (include/sgn_raster.h).

The product path has NO CPU fallback: if the shared library is missing or a call fails this module
raises.  The library is built in-tree by build.py (nvcc, sm_90a).
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsgn_raster.so")
MAX_FOURIER = 8
RECORD_FLOATS = 12


class SgnError(RuntimeError):
    pass


class Segment(C.Structure):
    _fields_ = [
        ("row0", C.c_int32), ("count", C.c_int32), ("F", C.c_int32), ("cls", C.c_int32),
        ("has_pose", C.c_int32), ("chunk0", C.c_int32),
        ("R", C.c_float * 9), ("t", C.c_float * 3), ("q", C.c_float * 4), ("idft", C.c_float * MAX_FOURIER),
        ("means", C.c_void_p), ("scales", C.c_void_p), ("quats", C.c_void_p),
        ("features_dc", C.c_void_p), ("features_rest", C.c_void_p), ("opacities", C.c_void_p),
    ]


class SegmentGrads(C.Structure):
    _fields_ = [
        ("means", C.c_void_p), ("scales", C.c_void_p), ("quats", C.c_void_p),
        ("features_dc", C.c_void_p), ("features_rest", C.c_void_p), ("opacities", C.c_void_p),
    ]


class CameraStruct(C.Structure):
    _fields_ = [
        ("viewmat", C.c_float * 12),
        ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
        ("width", C.c_int32), ("height", C.c_int32),
        ("cam_pos", C.c_float * 3),
        ("limx", C.c_float), ("limy", C.c_float),
        ("clip_thresh", C.c_float),
        ("block_width", C.c_int32),
        ("sh_degree", C.c_int32), ("sh_degree_to_use", C.c_int32),
        ("antialiased", C.c_int32),  # rasterize_mode: 0 classic (zero-initialised), 1 antialiased
        ("filter_3d", C.c_void_p),   # device array of per-segment 3D filter pointers; NULL (zero-initialised) = off
    ]


class FilterView(C.Structure):
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
                ("width", C.c_int32), ("height", C.c_int32)]


class FilterXform(C.Structure):
    _fields_ = [("M", C.c_double * 12), ("present", C.c_int32), ("pad", C.c_int32)]


class FilterSub(C.Structure):
    _fields_ = [("means", C.c_void_p), ("out", C.c_void_p), ("count", C.c_int32), ("chunk0", C.c_int32)]


class BlendOpts(C.Structure):
    _fields_ = [
        ("alpha_clamp_fwd", C.c_float), ("alpha_clamp_bwd", C.c_float),
        ("class_streams", C.c_int32), ("has_sky", C.c_int32), ("eval_clamp", C.c_int32),
        ("split_fwd_main", C.c_int32), ("split_fwd_acc", C.c_int32), ("split_bwd_main", C.c_int32),
        ("split_bwd_acc", C.c_int32),
        ("raw_mode", C.c_int32), ("background", C.c_float * 4), ("tuning", C.c_int32),
    ]


class AdamTensor(C.Structure):
    _fields_ = [
        ("param", C.c_void_p), ("arena_offset", C.c_int64), ("grad_offset", C.c_int64), ("numel", C.c_int64), ("chunk0", C.c_int32),
        ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("step_size", C.c_float),
        ("sqrt_bc2", C.c_float), ("one_minus_beta1", C.c_float), ("one_minus_beta2", C.c_float),
    ]


class DensifySegment(C.Structure):
    _fields_ = [
        ("row0", C.c_int32), ("count", C.c_int32), ("first", C.c_int32), ("pad", C.c_int32),
        ("xys_grad_norm", C.c_void_p), ("vis_counts", C.c_void_p), ("max_2Dsize", C.c_void_p),
    ]


class RefineConfig(C.Structure):
    _fields_ = [
        ("densify", C.c_int32), ("n_split_samples", C.c_int32), ("use_screen_size", C.c_int32), ("cull_big", C.c_int32),
        ("max_size", C.c_float), ("densify_grad_thresh", C.c_float), ("densify_size_thresh", C.c_float),
        ("split_screen_size", C.c_float), ("cull_alpha_thresh", C.c_float), ("cull_scale_thresh", C.c_float),
        ("cull_screen_size", C.c_float), ("inv_size_fac", C.c_float),
    ]


class RefineTensors(C.Structure):
    _fields_ = [
        ("src", C.c_void_p * 6), ("dst", C.c_void_p * 6), ("src_m", C.c_void_p * 6), ("dst_m", C.c_void_p * 6),
        ("src_v", C.c_void_p * 6), ("dst_v", C.c_void_p * 6), ("width", C.c_int32 * 6),
    ]


class MCMCSub(C.Structure):
    _fields_ = [
        ("means", C.c_void_p), ("scales", C.c_void_p), ("quats", C.c_void_p), ("opacities", C.c_void_p),
        ("count", C.c_int32), ("chunk0", C.c_int32), ("row0", C.c_int32), ("index", C.c_int32), ("noise_lr", C.c_float), ("pad", C.c_int32),
    ]


MCMC_MAX_TENSORS = 16  # SGN_MCMC_MAX_TENSORS
MCMC_NOISE, MCMC_RELOCATE, MCMC_ADD = 0, 1, 2  # SGN_MCMC_*: the purpose word of the Philox counter


class MCMCTensors(C.Structure):
    _fields_ = [("data", C.c_void_p * MCMC_MAX_TENSORS), ("width", C.c_int32 * MCMC_MAX_TENSORS), ("count", C.c_int32), ("pad", C.c_int32)]


# flag bits of sgn_refine_decide (csrc/sgn_refine_rules.cuh)
RF_SPLIT, RF_DUP, RF_KEEP_ORIG, RF_KEEP_SPLIT, RF_KEEP_DUP, RF_HIGH_GRAD, RF_ALPHA, RF_TOOBIG = (1 << i for i in range(8))


class LossIn(C.Structure):
    _fields_ = [
        ("rgb", C.c_void_p), ("gt_u8", C.c_void_p), ("gt_f32", C.c_void_p), ("mask", C.c_void_p),
        ("accumulation", C.c_void_p), ("sky_mask", C.c_void_p), ("object_acc", C.c_void_p),
        ("w_l1", C.c_float), ("w_sky", C.c_float), ("w_entropy", C.c_float),
    ]


class BlendFwdOut(C.Structure):
    _fields_ = [
        ("rgb", C.c_void_p), ("accumulation", C.c_void_p), ("depth", C.c_void_p),
        ("object_acc", C.c_void_p), ("background_acc", C.c_void_p),
        ("raw", C.c_void_p), ("final_T", C.c_void_p), ("final_idx", C.c_void_p), ("tile_depth", C.c_void_p),
        ("sched", C.c_void_p), ("staged", C.c_void_p),
    ]


class BlendBwdIn(C.Structure):
    _fields_ = [
        ("v_rgb", C.c_void_p), ("v_accumulation", C.c_void_p), ("v_depth", C.c_void_p),
        ("v_object_acc", C.c_void_p), ("v_background_acc", C.c_void_p),
        ("raw", C.c_void_p), ("final_T", C.c_void_p), ("final_idx", C.c_void_p), ("tile_depth", C.c_void_p),
        ("sched", C.c_void_p), ("sky", C.c_void_p), ("v_sky", C.c_void_p),
        ("v_fixed", C.c_void_p), ("fixed_scale", C.c_void_p), ("num_gaussians", C.c_int64),
    ]


_lib = None

EXPORTS = [
    "sgn_last_error", "sgn_abi_version", "sgn_launch_count", "sgn_sizeof_segment", "sgn_sizeof_segment_grads", "sgn_sizeof_camera",
    "sgn_upload", "sgn_bin_count", "sgn_project_fwd", "sgn_project_bwd", "sgn_l1_project_fwd", "sgn_l1_project_bwd", "sgn_l1_project_bwd_comp", "sgn_l1_sh", "sgn_bin_scan_scratch_bytes", "sgn_bin_scan",
    "sgn_bin_sort_scratch_bytes", "sgn_bin_sort", "sgn_bin_class_scratch_bytes", "sgn_bin_class_lists", "sgn_blend_sched_ints",
    "sgn_blend_fwd", "sgn_blend_bwd", "sgn_sizeof_adam_tensor", "sgn_adam_chunk_elems", "sgn_adam_step",
    "sgn_loss_scratch_bytes", "sgn_loss_fwd", "sgn_loss_bwd", "sgn_ssim_workspace_bytes", "sgn_ssim_fwd", "sgn_ssim_bwd",
    "sgn_metrics_scratch_bytes", "sgn_metrics", "sgn_sky_fwd", "sgn_sky_bwd", "sgn_cube_texture_fwd", "sgn_cube_texture_bwd",
    "sgn_sky_det_scratch_bytes", "sgn_sky_bwd_det", "sgn_cube_texture_bwd_det",
    "sgn_sizeof_densify_segment", "sgn_densify_stats",
    "sgn_sizeof_refine_config", "sgn_sizeof_refine_tensors", "sgn_refine_decide", "sgn_refine_apply",
    "sgn_bin_local_cap", "sgn_bin_local_scratch_bytes", "sgn_bin_local_count", "sgn_bin_local_sort",
    "sgn_project_bwd_range", "sgn_allreduce_sym", "sgn_blend_extra_fwd", "sgn_blend_extra_bwd", "sgn_blend_extra_bwd_det",
    "sgn_bin_sort_capped", "sgn_visible_flags", "sgn_visible_union", "sgn_project_bwd_pose", "sgn_pose_grad_reduce",
    "sgn_project_fwd_view", "sgn_project_bwd_view", "sgn_view_grad_reduce", "sgn_sky_fwd_view", "sgn_sky_bwd_view",
    "sgn_sky_bwd_det_view", "sgn_camera_adjust_fwd", "sgn_camera_adjust_bwd", "sgn_cube_texture_bwd_uv", "sgn_cube_texture_bwd_uv_det",
    "sgn_sky_rot_scratch_bytes", "sgn_sky_bwd_view_rot", "sgn_sky_bwd_det_view_rot", "sgn_knn_scratch_bytes", "sgn_knn",
    "sgn_lidar_depth_map", "sgn_depth_scratch_bytes", "sgn_depth_loss_fwd", "sgn_depth_loss_bwd", "sgn_depth_metrics",
    "sgn_semantic_scratch_bytes", "sgn_semantic_loss_fwd", "sgn_semantic_loss_bwd", "sgn_semantic_metrics", "sgn_refine_carry",
    "sgn_scale_reg_scratch_bytes", "sgn_scale_reg_fwd", "sgn_scale_reg_bwd", "sgn_sizeof_filter_xform", "sgn_filter3d",
    "sgn_bilagrid_slice_fwd", "sgn_bilagrid_slice_bwd_scratch_bytes", "sgn_bilagrid_slice_bwd", "sgn_bilagrid_tv_scratch_bytes",
    "sgn_bilagrid_tv_fwd", "sgn_bilagrid_tv_bwd", "sgn_sizeof_mcmc_sub", "sgn_sizeof_mcmc_tensors", "sgn_mcmc_noise",
    "sgn_mcmc_sample_scratch_bytes", "sgn_mcmc_sample", "sgn_mcmc_relocate", "sgn_mcmc_copy_rows", "sgn_mcmc_reg_scratch_bytes",
    "sgn_mcmc_reg_fwd", "sgn_mcmc_reg_bwd",
]
VIEW_FLOATS = 12  # SGN_VIEW_FLOATS: the view's cotangent, viewmat[12] row-major; the device view itself is 12 + 3 (cam_pos) floats
POSE_FLOATS = 16  # SGN_POSE_FLOATS: a segment's pose (and its cotangent) as R[9] row-major, t[3], q[4]
AR_MAX_SLICES = 48  # SGN_AR_MAX_SLICES


def load():
    """Load libsgn_raster.so; raise loudly if it is not there (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("SGN_RASTER_LIB", LIB_PATH)  # developer A/B of two builds of the same ABI (tools/)
    if not os.path.exists(path):
        raise SgnError(
            f"{path} is missing. Build it with `python street-gaussians-ns_b200/build.py` "
            "(or __graft_entry__.build()). There is no CPU fallback for the rasterizer.")
    L = C.CDLL(path)
    vp, i32, i64, sz = C.c_void_p, C.c_int, C.c_int64, C.c_size_t
    L.sgn_last_error.restype = C.c_char_p
    L.sgn_abi_version.restype = C.c_int
    L.sgn_launch_count.restype = C.c_longlong
    for f in ("sgn_sizeof_segment", "sgn_sizeof_segment_grads", "sgn_sizeof_camera", "sgn_sizeof_filter_xform"):
        getattr(L, f).restype = sz
    L.sgn_filter3d.argtypes = [vp, i32, i32, vp, i32, vp, C.c_double, C.c_double, vp, vp]
    L.sgn_filter3d.restype = C.c_int
    L.sgn_upload.argtypes = [vp, sz, vp, vp]
    L.sgn_project_fwd.argtypes = [vp, i32, i32, i32, C.POINTER(CameraStruct), vp, vp, vp, vp, vp, vp, vp]
    L.sgn_project_bwd.argtypes = [vp, vp, i32, i32, i32, C.POINTER(CameraStruct), vp, vp, vp, vp]
    L.sgn_project_bwd_range.argtypes = [vp, vp, i32, i32, i32, C.POINTER(CameraStruct), vp, vp, vp, i32, i32, vp]
    L.sgn_project_bwd_range.restype = C.c_int
    L.sgn_project_bwd_pose.argtypes = [vp, vp, i32, i32, i32, C.POINTER(CameraStruct), vp, vp, vp, i32, i32, vp, vp]
    L.sgn_pose_grad_reduce.argtypes = [vp, i32, i32, vp, vp, vp]
    L.sgn_project_bwd_pose.restype = L.sgn_pose_grad_reduce.restype = C.c_int
    L.sgn_project_fwd_view.argtypes = [vp, i32, i32, i32, C.POINTER(CameraStruct), vp, vp, vp, vp, vp, vp, vp, vp]
    L.sgn_project_bwd_view.argtypes = [vp, vp, i32, i32, i32, C.POINTER(CameraStruct), vp, vp, vp, vp, i32, i32, vp, vp, vp]
    L.sgn_view_grad_reduce.argtypes = [i32, vp, vp, vp]
    L.sgn_camera_adjust_fwd.argtypes = [vp, i32, i32, C.POINTER(C.c_float), C.c_float, C.c_float, vp, vp, vp, vp]
    L.sgn_camera_adjust_bwd.argtypes = [vp, i32, i32, C.POINTER(C.c_float), C.c_float, C.c_float, vp, vp, vp, vp]
    for f in ("sgn_project_fwd_view", "sgn_project_bwd_view", "sgn_view_grad_reduce", "sgn_camera_adjust_fwd", "sgn_camera_adjust_bwd"):
        getattr(L, f).restype = C.c_int
    L.sgn_allreduce_sym.argtypes = [vp, vp, vp, i32, i32, i32, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                    C.POINTER(C.c_int64), C.POINTER(C.c_int64), vp, C.c_float, i32, vp]
    L.sgn_visible_flags.argtypes = [vp, i64, vp, vp]
    L.sgn_visible_union.argtypes = [vp, i64, i32, i64, vp, vp]
    L.sgn_allreduce_sym.restype = L.sgn_visible_flags.restype = L.sgn_visible_union.restype = C.c_int
    L.sgn_blend_extra_fwd.argtypes = [C.POINTER(CameraStruct), C.POINTER(BlendOpts), vp, vp, vp, vp, vp, vp, i32, vp, vp]
    L.sgn_blend_extra_bwd.argtypes = [C.POINTER(CameraStruct), C.POINTER(BlendOpts), vp, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp]
    L.sgn_blend_extra_bwd_det.argtypes = [C.POINTER(CameraStruct), C.POINTER(BlendOpts), vp, vp, vp, vp, vp, vp, i32, i64, vp, vp, vp,
                                          vp, vp, vp, vp]
    L.sgn_blend_extra_fwd.restype = L.sgn_blend_extra_bwd.restype = L.sgn_blend_extra_bwd_det.restype = C.c_int
    fl = C.c_float
    L.sgn_l1_project_fwd.argtypes = [i32, vp, vp, fl, vp, C.POINTER(CameraStruct), vp, vp, vp, vp, vp, vp, vp, vp]
    L.sgn_l1_project_bwd.argtypes = [i32, vp, vp, fl, vp, C.POINTER(CameraStruct), vp, vp, vp, vp, vp, vp, vp, vp]
    L.sgn_l1_project_bwd_comp.argtypes = [i32, vp, vp, fl, vp, C.POINTER(CameraStruct), vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.sgn_l1_sh.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp, vp]
    for f in ("sgn_l1_project_fwd", "sgn_l1_project_bwd", "sgn_l1_project_bwd_comp", "sgn_l1_sh"):
        getattr(L, f).restype = C.c_int
    L.sgn_bin_scan_scratch_bytes.argtypes = [i32]
    L.sgn_bin_scan_scratch_bytes.restype = sz
    L.sgn_bin_scan.argtypes = [i32, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.sgn_bin_count.argtypes = [i32, C.POINTER(CameraStruct), vp, vp, vp, vp, vp, vp]
    L.sgn_bin_count.restype = C.c_int
    L.sgn_bin_sort_scratch_bytes.argtypes = [i64]
    L.sgn_bin_sort_scratch_bytes.restype = sz
    L.sgn_bin_sort.argtypes = [i32, i64, C.POINTER(CameraStruct), vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.sgn_bin_sort_capped.argtypes = [i32, i64, vp, vp, C.POINTER(CameraStruct), vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.sgn_bin_sort_capped.restype = C.c_int
    L.sgn_bin_local_cap.restype = C.c_int
    L.sgn_bin_local_scratch_bytes.argtypes = [i64, i32]
    L.sgn_bin_local_scratch_bytes.restype = sz
    L.sgn_bin_local_count.argtypes = [i32, C.POINTER(CameraStruct), vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.sgn_bin_local_count.restype = C.c_int
    L.sgn_bin_local_sort.argtypes = [i32, i64, i32, C.POINTER(CameraStruct), vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.sgn_bin_local_sort.restype = C.c_int
    L.sgn_bin_class_scratch_bytes.argtypes = [i32]
    L.sgn_bin_class_scratch_bytes.restype = sz
    L.sgn_bin_class_lists.argtypes = [C.POINTER(CameraStruct), i64, vp, vp, vp, vp, vp, sz, vp]
    L.sgn_blend_sched_ints.argtypes = [i32]
    L.sgn_blend_sched_ints.restype = sz
    L.sgn_blend_fwd.argtypes = [C.POINTER(CameraStruct), C.POINTER(BlendOpts), vp, vp, vp, i64, vp, vp, vp,
                                C.POINTER(BlendFwdOut), vp]
    L.sgn_blend_bwd.argtypes = [C.POINTER(CameraStruct), C.POINTER(BlendOpts), vp, vp, vp, i64, vp, vp,
                                C.POINTER(BlendBwdIn), vp, vp]
    for f in ("sgn_upload", "sgn_project_fwd", "sgn_project_bwd", "sgn_bin_scan", "sgn_bin_sort", "sgn_bin_class_lists",
              "sgn_blend_fwd", "sgn_blend_bwd"):
        getattr(L, f).restype = C.c_int
    L.sgn_sizeof_densify_segment.restype = sz
    L.sgn_densify_stats.argtypes = [vp, i32, i32, vp, vp, i32, i32, vp]
    L.sgn_densify_stats.restype = C.c_int
    L.sgn_loss_scratch_bytes.restype = sz
    L.sgn_loss_fwd.argtypes = [i32, i32, C.POINTER(LossIn), vp, vp, sz, vp]
    L.sgn_loss_fwd.restype = C.c_int
    L.sgn_loss_bwd.argtypes = [i32, i32, C.POINTER(LossIn), vp, vp, vp, vp, vp]
    L.sgn_loss_bwd.restype = C.c_int
    L.sgn_ssim_workspace_bytes.argtypes = [i32, i32]
    L.sgn_ssim_workspace_bytes.restype = sz
    L.sgn_ssim_fwd.argtypes = [i32, i32, C.POINTER(LossIn), fl, vp, vp, sz, vp]
    L.sgn_ssim_bwd.argtypes = [i32, i32, C.POINTER(LossIn), fl, vp, vp, vp, vp]
    L.sgn_ssim_fwd.restype = L.sgn_ssim_bwd.restype = C.c_int
    L.sgn_metrics_scratch_bytes.restype = sz
    L.sgn_metrics.argtypes = [i32, i32, C.POINTER(LossIn), vp, i32, i32, i32, vp, vp, vp, sz, vp]
    L.sgn_metrics.restype = C.c_int
    L.sgn_sky_fwd.argtypes = [C.POINTER(CameraStruct), vp, vp, vp, i32, vp, vp, vp]
    L.sgn_sky_bwd.argtypes = [C.POINTER(CameraStruct), vp, vp, i32, vp, vp, vp]
    L.sgn_cube_texture_fwd.argtypes = [i32, vp, vp, i32, vp, vp]
    L.sgn_cube_texture_bwd.argtypes = [i32, vp, i32, vp, vp, vp]
    L.sgn_sky_det_scratch_bytes.argtypes = [i32]
    L.sgn_sky_det_scratch_bytes.restype = sz
    L.sgn_sky_bwd_det.argtypes = [C.POINTER(CameraStruct), vp, vp, i32, vp, vp, vp, sz, vp]
    L.sgn_cube_texture_bwd_det.argtypes = [i32, vp, i32, vp, vp, vp, sz, vp]
    L.sgn_sky_fwd_view.argtypes = [C.POINTER(CameraStruct), vp, vp, vp, vp, i32, vp, vp, vp]
    L.sgn_sky_bwd_view.argtypes = [C.POINTER(CameraStruct), vp, vp, vp, i32, vp, vp, vp]
    L.sgn_sky_bwd_det_view.argtypes = [C.POINTER(CameraStruct), vp, vp, vp, i32, vp, vp, vp, sz, vp]
    L.sgn_cube_texture_bwd_uv.argtypes = [i32, vp, vp, i32, vp, vp, vp, vp]
    L.sgn_cube_texture_bwd_uv_det.argtypes = [i32, vp, vp, i32, vp, vp, vp, vp, sz, vp]
    L.sgn_sky_rot_scratch_bytes.argtypes = [i32, i32]
    L.sgn_sky_rot_scratch_bytes.restype = sz
    L.sgn_sky_bwd_view_rot.argtypes = [C.POINTER(CameraStruct), vp, vp, vp, vp, i32, vp, vp, vp, sz, vp, vp]
    L.sgn_sky_bwd_det_view_rot.argtypes = [C.POINTER(CameraStruct), vp, vp, vp, vp, i32, vp, vp, vp, sz, vp, sz, vp, vp]
    for f in ("sgn_sky_fwd", "sgn_sky_bwd", "sgn_cube_texture_fwd", "sgn_cube_texture_bwd", "sgn_sky_bwd_det", "sgn_cube_texture_bwd_det",
              "sgn_sky_fwd_view", "sgn_sky_bwd_view", "sgn_sky_bwd_det_view", "sgn_cube_texture_bwd_uv", "sgn_cube_texture_bwd_uv_det",
              "sgn_sky_bwd_view_rot", "sgn_sky_bwd_det_view_rot"):
        getattr(L, f).restype = C.c_int
    L.sgn_knn_scratch_bytes.argtypes = [i64, i64]
    L.sgn_knn_scratch_bytes.restype = sz
    L.sgn_knn.argtypes = [vp, i64, vp, i64, i32, vp, vp, vp, vp, sz, vp]
    L.sgn_knn.restype = C.c_int
    L.sgn_lidar_depth_map.argtypes = [vp, i64, C.POINTER(CameraStruct), vp, vp, vp]
    L.sgn_depth_scratch_bytes.restype = sz
    L.sgn_depth_loss_fwd.argtypes = [i32, i32, vp, vp, vp, fl, vp, vp, vp, sz, vp]
    L.sgn_depth_loss_bwd.argtypes = [i32, i32, vp, vp, vp, fl, vp, vp, vp, vp]
    L.sgn_depth_metrics.argtypes = [i32, i32, vp, vp, vp, vp, vp, sz, vp]
    for f in ("sgn_lidar_depth_map", "sgn_depth_loss_fwd", "sgn_depth_loss_bwd", "sgn_depth_metrics"):
        getattr(L, f).restype = C.c_int
    L.sgn_semantic_scratch_bytes.restype = sz
    L.sgn_semantic_loss_fwd.argtypes = [i32, i32, i32, vp, vp, vp, fl, vp, vp, vp, sz, vp]
    L.sgn_semantic_loss_bwd.argtypes = [i32, i32, i32, vp, vp, vp, fl, vp, vp, vp, vp]
    L.sgn_semantic_metrics.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp]
    L.sgn_refine_carry.argtypes = [i32, C.POINTER(RefineConfig), vp, vp, C.POINTER(C.c_int32), vp, vp, i32, vp, vp, vp, vp, vp]
    for f in ("sgn_semantic_loss_fwd", "sgn_semantic_loss_bwd", "sgn_semantic_metrics", "sgn_refine_carry"):
        getattr(L, f).restype = C.c_int
    L.sgn_scale_reg_scratch_bytes.restype = sz
    L.sgn_scale_reg_fwd.argtypes = [vp, i32, i32, i32, fl, vp, vp, sz, vp]
    L.sgn_scale_reg_bwd.argtypes = [vp, vp, i32, i32, i32, fl, vp, vp]
    L.sgn_scale_reg_fwd.restype = L.sgn_scale_reg_bwd.restype = C.c_int
    L.sgn_bilagrid_slice_fwd.argtypes = [vp, i32, i32, i32, vp, i32, i32, vp, vp]
    L.sgn_bilagrid_slice_bwd_scratch_bytes.argtypes = [i32, i32, i32, i32, i32]
    L.sgn_bilagrid_slice_bwd_scratch_bytes.restype = sz
    L.sgn_bilagrid_slice_bwd.argtypes = [vp, i32, i32, i32, vp, vp, i32, i32, vp, vp, vp, sz, vp]
    L.sgn_bilagrid_tv_scratch_bytes.restype = sz
    L.sgn_bilagrid_tv_fwd.argtypes = [vp, i32, i32, i32, i32, vp, vp, sz, vp]
    L.sgn_bilagrid_tv_bwd.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp]
    for f in ("sgn_bilagrid_slice_fwd", "sgn_bilagrid_slice_bwd", "sgn_bilagrid_tv_fwd", "sgn_bilagrid_tv_bwd"):
        getattr(L, f).restype = C.c_int
    u64 = C.c_uint64
    L.sgn_sizeof_mcmc_sub.restype = L.sgn_sizeof_mcmc_tensors.restype = sz
    L.sgn_mcmc_noise.argtypes = [vp, i32, i32, fl, u64, i32, vp, vp]
    L.sgn_mcmc_sample_scratch_bytes.argtypes = [i32]
    L.sgn_mcmc_sample_scratch_bytes.restype = sz
    L.sgn_mcmc_sample.argtypes = [vp, i32, fl, i32, i32, vp, u64, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    L.sgn_mcmc_relocate.argtypes = [vp, vp, i32, vp, fl, C.POINTER(MCMCTensors), vp]
    L.sgn_mcmc_copy_rows.argtypes = [C.POINTER(MCMCTensors), vp, i32, vp, i32, vp, vp]
    L.sgn_mcmc_reg_scratch_bytes.restype = sz
    L.sgn_mcmc_reg_fwd.argtypes = [vp, i32, i32, i32, fl, fl, vp, vp, sz, vp]
    L.sgn_mcmc_reg_bwd.argtypes = [vp, vp, i32, i32, i32, fl, fl, vp, vp, vp]
    for f in ("sgn_mcmc_noise", "sgn_mcmc_sample", "sgn_mcmc_relocate", "sgn_mcmc_copy_rows", "sgn_mcmc_reg_fwd", "sgn_mcmc_reg_bwd"):
        getattr(L, f).restype = C.c_int
    L.sgn_sizeof_adam_tensor.restype = sz
    L.sgn_adam_chunk_elems.restype = C.c_int
    L.sgn_adam_step.argtypes = [vp, i32, i32, vp, vp, vp, vp]
    L.sgn_adam_step.restype = C.c_int
    L.sgn_sizeof_refine_config.restype = sz
    L.sgn_sizeof_refine_tensors.restype = sz
    L.sgn_refine_decide.argtypes = [i32, C.POINTER(RefineConfig), vp, vp, vp, vp, vp, vp, vp, vp]
    L.sgn_refine_decide.restype = C.c_int
    L.sgn_refine_apply.argtypes = [i32, C.POINTER(RefineConfig), C.POINTER(RefineTensors), vp, vp, C.POINTER(C.c_int32), vp, vp]
    L.sgn_refine_apply.restype = C.c_int
    assert L.sgn_sizeof_refine_config() == C.sizeof(RefineConfig), "sgn_refine_config layout mismatch"
    assert L.sgn_sizeof_refine_tensors() == C.sizeof(RefineTensors), "sgn_refine_tensors layout mismatch"
    assert L.sgn_sizeof_adam_tensor() == C.sizeof(AdamTensor), "sgn_adam_tensor layout mismatch"
    assert L.sgn_sizeof_segment() == C.sizeof(Segment), "sgn_segment layout mismatch between header and ctypes"
    assert L.sgn_sizeof_segment_grads() == C.sizeof(SegmentGrads)
    assert L.sgn_sizeof_camera() == C.sizeof(CameraStruct), "sgn_camera layout mismatch"
    assert L.sgn_sizeof_mcmc_sub() == C.sizeof(MCMCSub), "sgn_mcmc_sub layout mismatch"
    assert L.sgn_sizeof_mcmc_tensors() == C.sizeof(MCMCTensors), "sgn_mcmc_tensors layout mismatch"
    _lib = L
    return L


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().sgn_last_error().decode("utf-8", "replace")
        raise SgnError(f"{what} failed (status {rc}): {msg}")
