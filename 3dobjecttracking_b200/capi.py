"""ctypes binding of libm3t_b200.so (include/m3t_b200.h) + a Workload -> context helper.

This is the CUDA path and the only compute path of the package: loading fails loudly when the
library is missing and every call raises M3TBError on a non-zero status (no CPU fallback).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _build
from .synth import Intrinsics, Workload

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libm3t_b200.so")
MAX_SCHEDULE = 8

fp = C.POINTER(C.c_float)


class M3TBError(RuntimeError):
    pass


class RegionParams(C.Structure):
    _fields_ = [("n_lines_max", C.c_int32), ("use_adaptive_coverage", C.c_int32),
                ("reference_contour_length", C.c_float), ("min_continuous_distance", C.c_float),
                ("function_length", C.c_int32), ("distribution_length", C.c_int32),
                ("function_amplitude", C.c_float), ("function_slope", C.c_float), ("learning_rate", C.c_float),
                ("n_global_iterations", C.c_int32), ("n_scales", C.c_int32), ("scales", C.c_int32 * MAX_SCHEDULE),
                ("n_standard_deviations", C.c_int32), ("standard_deviations", C.c_float * MAX_SCHEDULE),
                ("n_histogram_bins", C.c_int32), ("learning_rate_f", C.c_float), ("learning_rate_b", C.c_float),
                ("unconsidered_line_length", C.c_float), ("max_considered_line_length", C.c_float),
                ("measure_occlusions", C.c_int32), ("measured_depth_offset_radius", C.c_float),
                ("measured_occlusion_radius", C.c_float), ("measured_occlusion_threshold", C.c_float),
                ("n_unoccluded_iterations", C.c_int32), ("min_n_unoccluded_lines", C.c_int32),
                ("model_occlusions", C.c_int32), ("modeled_depth_offset_radius", C.c_float),
                ("modeled_occlusion_radius", C.c_float), ("modeled_occlusion_threshold", C.c_float),
                ("use_region_checking", C.c_int32)]


class DepthParams(C.Structure):
    _fields_ = [("n_points_max", C.c_int32), ("use_adaptive_coverage", C.c_int32), ("use_depth_scaling", C.c_int32),
                ("reference_surface_area", C.c_float), ("stride_length", C.c_float),
                ("n_considered_distances", C.c_int32), ("considered_distances", C.c_float * MAX_SCHEDULE),
                ("n_standard_deviations", C.c_int32), ("standard_deviations", C.c_float * MAX_SCHEDULE),
                ("measure_occlusions", C.c_int32), ("measured_depth_offset_radius", C.c_float),
                ("measured_occlusion_radius", C.c_float), ("measured_occlusion_threshold", C.c_float),
                ("n_unoccluded_iterations", C.c_int32), ("min_n_unoccluded_points", C.c_int32),
                ("model_occlusions", C.c_int32), ("modeled_depth_offset_radius", C.c_float),
                ("modeled_occlusion_radius", C.c_float), ("modeled_occlusion_threshold", C.c_float),
                ("use_silhouette_checking", C.c_int32)]


class RenderingArg(C.Structure):
    """m3tb_rendering"""
    _fields_ = [("image", C.c_void_p), ("image_size", C.c_int32), ("pitch", C.c_size_t), ("corner_u", C.c_float),
                ("corner_v", C.c_float), ("scale", C.c_float), ("projection_term_a", C.c_float),
                ("projection_term_b", C.c_float), ("id", C.c_int32), ("visible", C.c_int32)]


class OptimizerParams(C.Structure):
    _fields_ = [("tikhonov_parameter_rotation", C.c_float), ("tikhonov_parameter_translation", C.c_float)]


class Link(C.Structure):
    """m3tb_link (m3t::Link, link.h:150-156)."""
    _fields_ = [("body", C.c_int32), ("parent", C.c_int32), ("body2joint", C.c_float * 12),
                ("joint2parent", C.c_float * 12), ("link2world", C.c_float * 12), ("free_directions", C.c_int32 * 6),
                ("fixed_body2joint_pose", C.c_int32), ("n_extra_bodies", C.c_int32), ("extra_bodies", C.c_int32 * 3)]


class Constraint(C.Structure):
    """m3tb_constraint (m3t::Constraint / m3t::SoftConstraint)."""
    _fields_ = [("link1", C.c_int32), ("link2", C.c_int32), ("body12joint1", C.c_float * 12),
                ("body22joint2", C.c_float * 12), ("directions", C.c_int32 * 6), ("soft", C.c_int32),
                ("max_distance_rotation", C.c_float), ("max_distance_translation", C.c_float),
                ("standard_deviation_rotation", C.c_float), ("standard_deviation_translation", C.c_float)]


DESCRIPTOR_DAISY, DESCRIPTOR_SIFT, DESCRIPTOR_ORB = 1, 3, 4  # M3TB_DESCRIPTOR_*


def texture_params_default():
    p = TextureParams()
    lib().m3tb_texture_params_default(C.byref(p))
    return p


class TextureParams(C.Structure):
    """m3tb_texture_params (m3t::TextureModality, texture_modality.h:400-436)."""
    _fields_ = [("descriptor_type", C.c_int32), ("focused_image_size", C.c_int32),
                ("descriptor_distance_threshold", C.c_float), ("tukey_norm_constant", C.c_float),
                ("n_standard_deviations", C.c_int32), ("standard_deviations", C.c_float * 8),
                ("max_keyframe_rotation_difference", C.c_float), ("max_keyframe_age", C.c_int32),
                ("n_keyframes", C.c_int32), ("measure_occlusions", C.c_int32), ("measured_occlusion_radius", C.c_float),
                ("measured_occlusion_threshold", C.c_float), ("model_occlusions", C.c_int32),
                ("modeled_occlusion_radius", C.c_float), ("modeled_occlusion_threshold", C.c_float),
                ("n_features_max", C.c_int32)]  # device capacity: 512 .. 4096 features per upload


DESCRIPTOR_ORB = 4
TEXTURE_POINT_LIMIT = 8 * 4096  # a full deque of 8 keyframes at n_features_max 4096


class DeviceFeatures(C.Structure):
    """m3tb_device_features: one body's keypoints (x[i * xy_stride], y[i * xy_stride], crop coordinates) and descriptor
    rows (descriptor_pitch bytes apart; 32-byte ORB rows with length 0, `length` floats for SIFT / DAISY) in device
    memory."""
    _fields_ = [("n", C.c_int), ("length", C.c_int), ("x", C.c_void_p), ("y", C.c_void_p), ("xy_stride", C.c_int),
                ("descriptors", C.c_void_p), ("descriptor_pitch", C.c_size_t)]


class OrbParams(C.Structure):
    """m3tb_orb_params: cv::ORB's n_features, scale_factor and n_levels (300, 1.2, 3 by default)."""
    _fields_ = [("n_features", C.c_int32), ("scale_factor", C.c_float), ("n_levels", C.c_int32)]


TEXTURE_POINT_DTYPE = np.dtype([("center_f_body", "<f4", 3), ("correspondence_center", "<f4", 2), ("center", "<f4", 2)])

REGION_LINE_DTYPE = np.dtype([("model_index", "<i4"), ("valid", "<i4"), ("center_f_body", "<f4", 3),
                              ("center_u", "<f4"), ("center_v", "<f4"), ("normal_u", "<f4"), ("normal_v", "<f4"),
                              ("delta_r", "<f4"), ("normal_component_to_scale", "<f4"), ("distribution", "<f4", 12),
                              ("mean", "<f4"), ("measured_variance", "<f4")])
DEPTH_POINT_DTYPE = np.dtype([("model_index", "<i4"), ("valid", "<i4"), ("center_f_body", "<f4", 3),
                              ("normal_f_body", "<f4", 3), ("correspondence_center_f_camera", "<f4", 3)])

# every symbol include/m3t_b200.h declares (tests check the library exports all of them)
SYMBOLS = [
    "m3tb_region_params_default", "m3tb_depth_params_default", "m3tb_optimizer_params_default", "m3tb_create",
    "m3tb_destroy", "m3tb_set_stream", "m3tb_synchronize", "m3tb_last_error", "m3tb_launch_count",
    "m3tb_set_region_model", "m3tb_set_depth_model", "m3tb_set_color_camera", "m3tb_set_depth_camera",
    "m3tb_upload_color", "m3tb_upload_depth", "m3tb_upload_color_device", "m3tb_upload_depth_device",
    "m3tb_upload_color_batch", "m3tb_upload_depth_batch", "m3tb_set_body", "m3tb_n_bodies", "m3tb_set_poses",
    "m3tb_get_poses", "m3tb_set_histograms", "m3tb_get_histograms", "m3tb_tracking_step", "m3tb_corr_iteration",
    "m3tb_start_modalities", "m3tb_calculate_results", "m3tb_region_correspondences",
    "m3tb_region_gradient_hessian", "m3tb_depth_correspondences", "m3tb_depth_gradient_hessian",
    "m3tb_calculate_optimization", "m3tb_get_region_lines", "m3tb_get_depth_points", "m3tb_get_closest_views",
    "m3tb_debug_phase_clocks", "m3tb_last_ingest_bytes", "m3tb_set_structure", "m3tb_clear_structures",
    "m3tb_n_structures", "m3tb_calculate_consistent_poses", "m3tb_refine_poses", "m3tb_get_link_poses", "m3tb_get_structure_theta",
    "m3tb_set_gradient_hessian", "m3tb_debug_rigid_solve", "m3tb_reset_joint_poses", "m3tb_prefetch_frames", "m3tb_detach_frames",
    "m3tb_debug_closest_view", "m3tb_upload_depth_rendering", "m3tb_upload_silhouette_rendering",
    "m3tb_share_color_histograms", "m3tb_debug_last_launch", "m3tb_set_body_geometry", "m3tb_set_focused_renderer",
    "m3tb_attach_renderer", "m3tb_render", "m3tb_get_rendering", "m3tb_model_params_default", "m3tb_model_views",
    "m3tb_generate_depth_model", "m3tb_get_depth_model", "m3tb_debug_render_model_view", "m3tb_debug_resources",
    "m3tb_generate_region_model", "m3tb_get_region_model", "m3tb_debug_region_model_view", "m3tb_set_viewer",
    "m3tb_update_viewers", "m3tb_get_viewer_image", "m3tb_set_full_renderer", "m3tb_render_full",
    "m3tb_get_full_rendering", "m3tb_undistortion_map", "m3tb_set_camera_undistortion", "m3tb_get_camera_image",
    "m3tb_texture_params_default", "m3tb_set_texture_modality", "m3tb_get_texture_focus", "m3tb_upload_texture_features",
    "m3tb_upload_texture_float_features",
    "m3tb_texture_correspondences", "m3tb_texture_gradient_hessian", "m3tb_get_texture_points",
    "m3tb_get_texture_keyframes", "m3tb_texture_crop", "m3tb_upload_texture_features_device",
    "m3tb_get_texture_feature_flags", "m3tb_orb_params_default", "m3tb_texture_detect_orb",
    "m3tb_get_texture_detections", "m3tb_get_texture_orb_keypoints",
]

KERNEL_NAMES = {0: None, 1: "k_track", 2: "k_track2", 3: "k_track_cluster"}


class LaunchInfo(C.Structure):
    """m3tb_launch_info: the tracking-kernel variant of the last tracking launch."""
    _fields_ = [("kernel", C.c_int32), ("threads", C.c_int32), ("items_per_thread", C.c_int32), ("lut_smem", C.c_int32),
                ("occ", C.c_int32), ("tiles", C.c_int32), ("tma_mode", C.c_int32)]


class ModelParams(C.Structure):
    """m3tb_model_params (model.h:161-167)."""
    _fields_ = [("sphere_radius", C.c_float), ("n_divides", C.c_int32), ("n_points", C.c_int32),
                ("max_radius_depth_offset", C.c_float), ("stride_depth_offset", C.c_float),
                ("use_random_seed", C.c_int32), ("image_size", C.c_int32)]


_lib = None


def lib():
    """Loads libm3t_b200.so; builds it in-tree with nvcc when it is missing. When the sources are newer than the
    library it is rebuilt only with M3TB_AUTO_REBUILD=1 (never under torchrun: ranks would race) - otherwise a
    warning is printed, because a stale binary silently running is worse than a loud one. Raises if loading fails."""
    global _lib, LIB_PATH
    if _lib is not None:
        return _lib
    if os.environ.get("M3TB_LIB"):  # A/B experiments: another build of the same library
        LIB_PATH = os.environ["M3TB_LIB"]
        if not os.path.exists(LIB_PATH):
            raise M3TBError(f"M3TB_LIB names a library that does not exist: {LIB_PATH}")
    if not os.path.exists(LIB_PATH):
        _build.build_cuda()
    elif _build._stale(LIB_PATH, _build.cuda_sources()):
        if os.environ.get("M3TB_AUTO_REBUILD") == "1" and int(os.environ.get("WORLD_SIZE", "1")) == 1:
            _build.build_cuda()
        else:
            import sys
            print("3dobjecttracking_b200.capi: WARNING libm3t_b200.so is older than its sources "
                  "(python __graft_entry__.py rebuilds it)", file=sys.stderr)
    L = C.CDLL(LIB_PATH)
    vp, ci = C.c_void_p, C.c_int
    L.m3tb_region_params_default.argtypes = [C.POINTER(RegionParams)]
    L.m3tb_depth_params_default.argtypes = [C.POINTER(DepthParams)]
    L.m3tb_optimizer_params_default.argtypes = [C.POINTER(OptimizerParams)]
    L.m3tb_create.argtypes = [ci, ci, ci, ci, C.POINTER(vp)]
    L.m3tb_destroy.argtypes = [vp]
    L.m3tb_set_stream.argtypes = [vp, vp]
    L.m3tb_synchronize.argtypes = [vp]
    L.m3tb_last_error.argtypes = [vp]
    L.m3tb_last_error.restype = C.c_char_p
    L.m3tb_launch_count.argtypes = [vp]
    L.m3tb_launch_count.restype = C.c_int64
    for n in ("m3tb_set_region_model", "m3tb_set_depth_model"):
        getattr(L, n).argtypes = [vp, ci, ci, ci, fp, fp, vp, C.c_float, C.c_float]
    L.m3tb_set_color_camera.argtypes = [vp, ci, C.POINTER(Intrinsics), fp]
    L.m3tb_set_depth_camera.argtypes = [vp, ci, C.POINTER(Intrinsics), fp, C.c_float]
    for n in ("m3tb_upload_color", "m3tb_upload_depth", "m3tb_upload_color_device", "m3tb_upload_depth_device"):
        getattr(L, n).argtypes = [vp, ci, vp, C.c_size_t]
    for n in ("m3tb_upload_color_batch", "m3tb_upload_depth_batch"):
        getattr(L, n).argtypes = [vp, ci, ci, vp, C.c_size_t, C.c_size_t]
    L.m3tb_set_body.argtypes = [vp, ci, C.POINTER(RegionParams), C.POINTER(DepthParams), C.POINTER(OptimizerParams),
                                ci, ci, ci, ci]
    L.m3tb_n_bodies.argtypes = [vp]
    L.m3tb_set_poses.argtypes = [vp, ci, ci, fp]
    L.m3tb_get_poses.argtypes = [vp, ci, ci, fp]
    L.m3tb_set_histograms.argtypes = [vp, ci, fp, fp]
    L.m3tb_get_histograms.argtypes = [vp, ci, fp, fp]
    L.m3tb_share_color_histograms.argtypes = [vp, ci, ci]
    L.m3tb_tracking_step.argtypes = [vp, ci, ci, ci]
    L.m3tb_corr_iteration.argtypes = [vp, ci, ci, ci]
    L.m3tb_start_modalities.argtypes = [vp, ci]
    L.m3tb_calculate_results.argtypes = [vp, ci]
    L.m3tb_region_correspondences.argtypes = [vp, ci, ci]
    L.m3tb_depth_correspondences.argtypes = [vp, ci, ci]
    L.m3tb_region_gradient_hessian.argtypes = [vp, ci, ci, ci, fp, fp]
    L.m3tb_depth_gradient_hessian.argtypes = [vp, ci, ci, ci, fp, fp]
    L.m3tb_calculate_optimization.argtypes = [vp, ci, ci, ci]
    L.m3tb_get_region_lines.argtypes = [vp, ci, vp, ci, C.POINTER(ci)]
    L.m3tb_get_depth_points.argtypes = [vp, ci, vp, ci, C.POINTER(ci)]
    L.m3tb_get_closest_views.argtypes = [vp, ci, C.POINTER(ci), C.POINTER(ci)]
    L.m3tb_set_structure.argtypes = [vp, ci, C.POINTER(Link), ci, C.POINTER(Constraint), ci, C.POINTER(OptimizerParams)]
    L.m3tb_clear_structures.argtypes = [vp]
    L.m3tb_n_structures.argtypes = [vp]
    L.m3tb_calculate_consistent_poses.argtypes = [vp]
    L.m3tb_refine_poses.argtypes = [vp, C.POINTER(ci), ci, C.POINTER(ci), ci, ci, ci]
    L.m3tb_reset_joint_poses.argtypes = [vp]
    L.m3tb_prefetch_frames.argtypes = [vp]
    L.m3tb_detach_frames.argtypes = [vp]
    L.m3tb_upload_depth_rendering.argtypes = [vp, ci, ci, C.POINTER(RenderingArg)]
    L.m3tb_upload_silhouette_rendering.argtypes = [vp, ci, ci, C.POINTER(RenderingArg)]
    ip = C.POINTER(C.c_int)
    L.m3tb_debug_closest_view.argtypes = [fp, ci, fp, ci, ip, ip, ip, ip]
    L.m3tb_get_link_poses.argtypes = [vp, ci, fp, fp, fp]
    L.m3tb_get_structure_theta.argtypes = [vp, ci, fp, ci, C.POINTER(ci), C.POINTER(ci)]
    L.m3tb_set_gradient_hessian.argtypes = [vp, ci, fp, fp]
    L.m3tb_debug_rigid_solve.argtypes = [vp, ci, ci, fp, fp, fp, fp, C.POINTER(ci)]
    L.m3tb_debug_last_launch.argtypes = [vp, C.POINTER(LaunchInfo)]
    L.m3tb_set_body_geometry.argtypes = [vp, ci, fp, ci, fp, C.c_float, ci, ci, ci]
    L.m3tb_set_focused_renderer.argtypes = [vp, ci, ci, ci, ci, C.c_float, C.c_float, ci, ip, ci, ip, ci]
    L.m3tb_attach_renderer.argtypes = [vp, ci, ci, ci, ci]
    L.m3tb_render.argtypes = [vp]
    L.m3tb_get_rendering.argtypes = [vp, ci, vp, vp, fp, fp, fp, fp, fp, ip]
    L.m3tb_model_params_default.argtypes = [C.POINTER(ModelParams)]
    L.m3tb_model_views.argtypes = [C.POINTER(ModelParams), fp, ci, ip]
    L.m3tb_generate_depth_model.argtypes = [vp, ci, ci, ip, ci, C.POINTER(ModelParams)]
    L.m3tb_get_depth_model.argtypes = [vp, ci, ip, ip, fp, fp, vp, fp, fp]
    L.m3tb_debug_render_model_view.argtypes = [vp, ci, ip, ci, C.POINTER(ModelParams), ci, vp, vp, vp]
    L.m3tb_generate_region_model.argtypes = [vp, ci, ci, vp, ci, C.POINTER(ModelParams)]
    L.m3tb_get_region_model.argtypes = [vp, ci, ip, ip, fp, fp, vp, fp, fp]
    L.m3tb_debug_region_model_view.argtypes = [vp, ci, vp, ci, C.POINTER(ModelParams), ci, vp, ip, vp, vp, vp, ci, ip,
                                               ip]
    L.m3tb_debug_resources.argtypes = [ci, C.POINTER(C.c_longlong)]
    L.m3tb_set_viewer.argtypes = [vp, ci, ci, ci, ip, ci, C.c_float, C.c_float, C.c_float]
    L.m3tb_update_viewers.argtypes = [vp]
    L.m3tb_get_viewer_image.argtypes = [vp, ci, vp, C.c_size_t, vp, C.c_size_t]
    L.m3tb_set_full_renderer.argtypes = [vp, ci, ci, ci, C.c_float, C.c_float, ci, ip, ci]
    L.m3tb_render_full.argtypes = [vp]
    L.m3tb_texture_params_default.argtypes = [C.POINTER(TextureParams)]
    L.m3tb_set_texture_modality.argtypes = [vp, ci, C.POINTER(TextureParams), ci]
    L.m3tb_get_texture_focus.argtypes = [vp, ci, ci, ip, fp, ip]
    L.m3tb_upload_texture_features.argtypes = [vp, ci, fp, vp, ci, ci, ci, C.c_float]
    L.m3tb_upload_texture_float_features.argtypes = [vp, ci, fp, fp, ci, ci, ci, ci, C.c_float]
    L.m3tb_texture_correspondences.argtypes = [vp, ci, ci]
    L.m3tb_texture_gradient_hessian.argtypes = [vp, ci, ci, ci, fp, fp]
    L.m3tb_get_texture_points.argtypes = [vp, ci, vp, ci, C.POINTER(ci)]
    L.m3tb_get_texture_keyframes.argtypes = [vp, ci, C.POINTER(ci), ip, fp, vp, ci, C.POINTER(ci), fp]
    L.m3tb_texture_crop.argtypes = [vp, ip, ci, vp, C.c_size_t, C.c_size_t, ci, ci, ip, fp, ip, ip]
    L.m3tb_upload_texture_features_device.argtypes = [vp, ip, C.POINTER(DeviceFeatures), ci]
    L.m3tb_get_texture_feature_flags.argtypes = [vp, ci, ci, ip]
    L.m3tb_orb_params_default.argtypes = [C.POINTER(OrbParams)]
    L.m3tb_orb_params_default.restype = None
    L.m3tb_texture_detect_orb.argtypes = [vp, ip, ci, C.POINTER(OrbParams)]
    L.m3tb_get_texture_detections.argtypes = [vp, ci, ci, ip]
    L.m3tb_get_texture_orb_keypoints.argtypes = [vp, ci, fp, fp, fp, ip, vp, ci, C.POINTER(ci)]
    L.m3tb_get_full_rendering.argtypes = [vp, ci, vp, C.c_size_t, vp, C.c_size_t, vp, C.c_size_t, fp, fp]
    L.m3tb_undistortion_map.argtypes = [C.POINTER(Intrinsics), fp, C.POINTER(Intrinsics), vp, C.c_size_t]
    L.m3tb_set_camera_undistortion.argtypes = [vp, ci, ci, vp, C.c_size_t, ci, C.c_int32]
    L.m3tb_get_camera_image.argtypes = [vp, ci, ci, vp, C.c_size_t]
    _lib = L
    return L


def debug_resources(fail_after=-1):
    """m3tb_debug_resources: the number of CUDA resources the library holds across all contexts (device and pinned
    allocations, streams, events). fail_after > 0 arms the n-th resource creation from now on to fail as an allocation
    failure, 0 disarms, negative only queries."""
    live = C.c_longlong(0)
    lib().m3tb_debug_resources(int(fail_after), C.byref(live))
    return int(live.value)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return a.ctypes.data_as(fp)


def model_params(**kw) -> ModelParams:
    """m3tb_model_params_default with the given fields replaced (sphere_radius, n_divides, n_points,
    max_radius_depth_offset, stride_depth_offset, use_random_seed, image_size)."""
    p = ModelParams()
    lib().m3tb_model_params_default(C.byref(p))
    for k, v in kw.items():
        if k not in dict(ModelParams._fields_):
            raise TypeError(f"unknown model parameter {k}")
        setattr(p, k, v)
    return p


def associated_bodies(associated):
    """m3tb_associated_body records [n, 3] int32 (body, movable, same_region) of a list of triples."""
    a = np.ascontiguousarray(np.asarray(associated, np.int32).reshape(-1, 3))
    return a


def model_views(params=None):
    """Geodesic camera2body poses [n,3,4] float32 of a model (m3tb_model_views, host only); the view orientation is
    column 2."""
    p = params if params is not None else model_params()
    n = C.c_int(0)
    ip = C.POINTER(C.c_int)
    if lib().m3tb_model_views(C.byref(p), None, 0, C.cast(C.byref(n), ip)) != 0:
        raise M3TBError("m3tb_model_views: bad parameters")
    out = np.zeros((n.value, 3, 4), np.float32)
    lib().m3tb_model_views(C.byref(p), _p(out), n.value, C.cast(C.byref(n), ip))
    return out


def undistortion_map(raw, coefficients, rectified):
    """m3tb_undistortion_map (host only): the (H, W, 2) int16 map of cv::initUndistortRectifyMap(CV_32FC1) +
    cv::convertMaps(CV_16SC2, nninterpolation=True) for camera matrix `raw`, coefficients k1, k2, p1, p2, k3, k4, k5, k6
    and new camera matrix `rectified` (both Intrinsics of the same size)."""
    k = _f32(coefficients).reshape(8)
    out = np.zeros((rectified.height, rectified.width, 2), np.int16)
    if lib().m3tb_undistortion_map(C.byref(raw), _p(k), C.byref(rectified), out.ctypes.data, out.strides[0]) != 0:
        raise M3TBError("m3tb_undistortion_map: bad arguments")
    return out


_KINDS = {"color": 0, "depth": 1}


def region_params(settings=None) -> RegionParams:
    p = RegionParams()
    lib().m3tb_region_params_default(C.byref(p))
    if settings is None:
        return p
    for k in ("n_lines_max", "min_continuous_distance", "function_amplitude", "function_slope", "learning_rate",
              "n_global_iterations", "n_histogram_bins", "learning_rate_f", "learning_rate_b",
              "unconsidered_line_length", "max_considered_line_length", "reference_contour_length",
              "measured_depth_offset_radius", "measured_occlusion_radius", "measured_occlusion_threshold",
              "n_unoccluded_iterations", "min_n_unoccluded_lines", "modeled_depth_offset_radius",
              "modeled_occlusion_radius", "modeled_occlusion_threshold"):
        setattr(p, k, getattr(settings, k))
    p.model_occlusions = int(settings.model_occlusions)
    p.use_region_checking = int(settings.use_region_checking)
    p.use_adaptive_coverage = int(settings.use_adaptive_coverage)
    p.measure_occlusions = int(settings.measure_occlusions)
    p.n_scales = len(settings.scales)
    p.n_standard_deviations = len(settings.standard_deviations)
    for i, s in enumerate(settings.scales):
        p.scales[i] = int(s)
    for i, s in enumerate(settings.standard_deviations):
        p.standard_deviations[i] = float(s)
    return p


def depth_params(settings=None) -> DepthParams:
    p = DepthParams()
    lib().m3tb_depth_params_default(C.byref(p))
    if settings is None:
        return p
    p.n_points_max = settings.n_points_max
    p.stride_length = settings.stride_length
    p.use_adaptive_coverage = int(settings.use_adaptive_coverage)
    p.reference_surface_area = settings.reference_surface_area
    p.use_depth_scaling = int(settings.use_depth_scaling)
    p.measure_occlusions = int(settings.measure_occlusions)
    for k in ("measured_depth_offset_radius", "measured_occlusion_radius", "measured_occlusion_threshold",
              "n_unoccluded_iterations", "min_n_unoccluded_points", "modeled_depth_offset_radius",
              "modeled_occlusion_radius", "modeled_occlusion_threshold"):
        setattr(p, k, getattr(settings, k))
    p.model_occlusions = int(settings.model_occlusions)
    p.use_silhouette_checking = int(settings.use_silhouette_checking)
    p.n_considered_distances = len(settings.considered_distances)
    p.n_standard_deviations = len(settings.standard_deviations)
    for i, s in enumerate(settings.considered_distances):
        p.considered_distances[i] = float(s)
    for i, s in enumerate(settings.standard_deviations):
        p.standard_deviations[i] = float(s)
    return p


class Context:
    """Thin object wrapper over an m3tb_ctx."""

    def __init__(self, device=0, max_bodies=1, max_cameras=1, max_models=1, stream=None):
        self.L = lib()
        h = C.c_void_p()
        rc = self.L.m3tb_create(device, max_bodies, max_cameras, max_models, C.byref(h))
        if rc != 0:
            raise M3TBError(f"m3tb_create failed with status {rc} (no usable sm_90 CUDA device?)")
        self.h = h
        self.n_bodies = 0
        self._texture_length = {}  # SIFT / DAISY bodies: descriptor length of their uploads (0 before the first)
        if stream is not None:
            self.set_stream(stream)

    def _ck(self, rc):
        if rc != 0:
            raise M3TBError(f"status {rc}: {self.L.m3tb_last_error(self.h).decode()}")

    def close(self):
        if self.h:
            self.L.m3tb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream_handle):
        self._ck(self.L.m3tb_set_stream(self.h, C.c_void_p(cuda_stream_handle)))

    def synchronize(self):
        self._ck(self.L.m3tb_synchronize(self.h))

    @property
    def launch_count(self):
        return int(self.L.m3tb_launch_count(self.h))

    def set_region_model(self, model_id, m):
        self._ck(self.L.m3tb_set_region_model(self.h, model_id, m.n_views, m.n_points, _p(m.orientations),
                                              _p(m.view_scalars), m.points.ctypes.data_as(C.c_void_p),
                                              m.stride_depth_offset, m.max_radius_depth_offset))

    def set_depth_model(self, model_id, m):
        self._ck(self.L.m3tb_set_depth_model(self.h, model_id, m.n_views, m.n_points, _p(m.orientations),
                                             _p(m.view_scalars), m.points.ctypes.data_as(C.c_void_p),
                                             m.stride_depth_offset, m.max_radius_depth_offset))

    def set_color_camera(self, cam, intr, w2c):
        w = _f32(w2c).reshape(12)
        self._ck(self.L.m3tb_set_color_camera(self.h, cam, C.byref(intr), _p(w)))

    def set_depth_camera(self, cam, intr, w2c, depth_scale):
        w = _f32(w2c).reshape(12)
        self._ck(self.L.m3tb_set_depth_camera(self.h, cam, C.byref(intr), _p(w), depth_scale))

    def upload_color(self, cam, frame):
        self._ck(self.L.m3tb_upload_color(self.h, cam, frame.ctypes.data_as(C.c_void_p), frame.strides[0]))

    def upload_depth(self, cam, frame):
        self._ck(self.L.m3tb_upload_depth(self.h, cam, frame.ctypes.data_as(C.c_void_p), frame.strides[0]))

    def upload_color_batch(self, first, frames):
        """frames: [n,H,pitch] u8 (numpy or a pinned torch tensor's numpy view)."""
        self._ck(self.L.m3tb_upload_color_batch(self.h, first, frames.shape[0], C.c_void_p(frames.ctypes.data),
                                                frames.strides[0], frames.strides[1]))

    def upload_depth_batch(self, first, frames):
        self._ck(self.L.m3tb_upload_depth_batch(self.h, first, frames.shape[0], C.c_void_p(frames.ctypes.data),
                                                frames.strides[0], frames.strides[1]))

    def upload_batch_ptr(self, color, first, count, ptr, frame_stride, pitch):
        f = self.L.m3tb_upload_color_batch if color else self.L.m3tb_upload_depth_batch
        self._ck(f(self.h, first, count, C.c_void_p(ptr), frame_stride, pitch))

    def set_camera_undistortion(self, camera_kind, cam, map_xy, channels, depth_value_offset=0):
        """Every later upload to camera `cam` (camera_kind "color" | "depth", or 0 | 1) takes the raw frame (`channels`
        bytes per colour pixel: 4 BGRA or 3 BGR; 1 for depth) and rectifies it through map_xy ([H, W, 2] int16, e.g.
        undistortion_map()); depth_value_offset is added to every depth pixel with saturation. map_xy None removes it."""
        kind = _KINDS.get(camera_kind, camera_kind)
        if map_xy is None:
            self._ck(self.L.m3tb_set_camera_undistortion(self.h, int(kind), cam, None, 0, int(channels), 0))
            return
        m = np.ascontiguousarray(map_xy, np.int16)
        self._ck(self.L.m3tb_set_camera_undistortion(self.h, int(kind), cam, m.ctypes.data, m.strides[0], int(channels),
                                                     int(depth_value_offset)))

    def get_camera_image(self, camera_kind, cam, width, height):
        """Camera::image(): the frame camera `cam` holds, [H, W, 3] u8 BGR (colour) or [H, W] u16 (depth)."""
        kind = _KINDS.get(camera_kind, camera_kind)
        out = np.zeros((height, width, 3), np.uint8) if kind == 0 else np.zeros((height, width), np.uint16)
        self.get_camera_image_to(kind, cam, out.ctypes.data, out.strides[0])
        return out

    def get_camera_image_to(self, camera_kind, cam, ptr, pitch):
        """The frame camera `cam` holds into caller memory, host or device (e.g. a torch tensor's data_ptr()), rows
        `pitch` bytes apart."""
        kind = _KINDS.get(camera_kind, camera_kind)
        self._ck(self.L.m3tb_get_camera_image(self.h, int(kind), cam, C.c_void_p(ptr), pitch))

    def prefetch_frames(self):
        self._ck(self.L.m3tb_prefetch_frames(self.h))

    def detach_frames(self):
        self._ck(self.L.m3tb_detach_frames(self.h))

    def upload_rendering(self, body, key, r):
        """key: "region_depth" | "region_silhouette" | "depth_depth" | "depth_silhouette"; r: synth.Rendering."""
        a = RenderingArg()
        a.image = r.image.ctypes.data
        a.image_size = r.image.shape[0]
        a.pitch = r.image.strides[0]
        a.corner_u, a.corner_v, a.scale = r.corner_u, r.corner_v, r.scale
        a.projection_term_a, a.projection_term_b = r.projection_term_a, r.projection_term_b
        a.id, a.visible = int(r.id), int(r.visible)
        modality = 0 if key.startswith("region") else 1
        f = self.L.m3tb_upload_depth_rendering if key.endswith("depth") else self.L.m3tb_upload_silhouette_rendering
        self._ck(f(self.h, body, modality, C.byref(a)))

    def set_body_geometry(self, body, triangles, geometry2body=None, maximum_body_diameter=None, enable_culling=True,
                          body_id=0, region_id=0):
        """Body + RendererGeometry::AddBody: triangles [n,3,3] (metres, geometry frame, counter-clockwise seen from
        outside). The diameter defaults to twice the largest vertex distance from the body origin."""
        t = _f32(triangles).reshape(-1, 9)
        g2b = _f32(np.eye(4)[:3] if geometry2body is None else geometry2body).reshape(12)
        if maximum_body_diameter is None:
            v = t.reshape(-1, 3).astype(np.float64) @ g2b.reshape(3, 4)[:, :3].T.astype(np.float64) + g2b.reshape(3, 4)[:, 3]
            maximum_body_diameter = 2.0 * float(np.linalg.norm(v, axis=1).max())
        self._ck(self.L.m3tb_set_body_geometry(self.h, body, _p(t), t.shape[0], _p(g2b), maximum_body_diameter,
                                               int(enable_culling), int(body_id), int(region_id)))

    def set_focused_renderer(self, renderer, camera_kind, camera, geometry_bodies, referenced_bodies, image_size=200,
                             z_min=0.02, z_max=10.0, id_type="body"):
        """camera_kind: "color" | "depth" (or 0 | 1); id_type: "body" | "region" (or 0 | 1)."""
        kind = {"color": 0, "depth": 1}.get(camera_kind, camera_kind)
        idt = {"body": 0, "region": 1}.get(id_type, id_type)
        g = np.ascontiguousarray(geometry_bodies, np.int32)
        r = np.ascontiguousarray(referenced_bodies, np.int32)
        ip = C.POINTER(C.c_int)
        self._ck(self.L.m3tb_set_focused_renderer(self.h, renderer, int(kind), camera, image_size, z_min, z_max, int(idt),
                                                  g.ctypes.data_as(ip), g.size, r.ctypes.data_as(ip), r.size))
        self._renderer_refs = getattr(self, "_renderer_refs", {})
        self._renderer_refs[renderer] = (image_size, r.size)

    def attach_renderer(self, body, key, renderer):
        """key: "region_depth" | "region_silhouette" | "depth_depth" | "depth_silhouette" | "texture_depth" |
        "texture_silhouette"; renderer -1 detaches."""
        modality = 0 if key.startswith("region") else 2 if key.startswith("texture") else 1
        kind = 0 if key.endswith("depth") else 1
        self._ck(self.L.m3tb_attach_renderer(self.h, body, modality, kind, renderer))

    def render(self):
        self._ck(self.L.m3tb_render(self.h))

    def get_rendering(self, renderer):
        """dict(depth [S,S] u16, silhouette [S,S] u8, corner_u, corner_v, scale, projection_term_a / b (float32),
        visible [n_referenced] int32)."""
        S, n_ref = self._renderer_refs[renderer]
        depth = np.zeros((S, S), np.uint16)
        sil = np.zeros((S, S), np.uint8)
        f = [C.c_float(0.0) for _ in range(5)]
        vis = np.zeros(n_ref, np.int32)
        self._ck(self.L.m3tb_get_rendering(self.h, renderer, depth.ctypes.data, sil.ctypes.data, *[C.byref(x) for x in f],
                                           vis.ctypes.data_as(C.POINTER(C.c_int))))
        out = dict(zip(("corner_u", "corner_v", "scale", "projection_term_a", "projection_term_b"),
                       (np.float32(x.value) for x in f)))
        out.update(depth=depth, silhouette=sil, visible=vis)
        return out

    def set_viewer(self, viewer, kind, camera, geometry_bodies, opacity=0.5, min_depth=0.0, max_depth=1.0):
        """NormalColorViewer (kind "color" / 0) or NormalDepthViewer ("depth" / 1) of camera `camera` drawing
        `geometry_bodies` in that order. The image size is the camera's at the next update."""
        k = {"color": 0, "depth": 1}.get(kind, kind)
        g = np.ascontiguousarray(geometry_bodies, np.int32)
        self._ck(self.L.m3tb_set_viewer(self.h, viewer, int(k), camera, g.ctypes.data_as(C.POINTER(C.c_int)), g.size,
                                        opacity, min_depth, max_depth))

    def update_viewers(self):
        """Tracker::UpdateViewers: every viewer from the current poses and camera frames."""
        self._ck(self.L.m3tb_update_viewers(self.h))

    def get_viewer_image(self, viewer, width, height):
        """(blended BGR8 image [H,W,3], normal image [H,W,4] in GL_BGRA order) of the viewer's last update."""
        bgr = np.zeros((height, width, 3), np.uint8)
        normal = np.zeros((height, width, 4), np.uint8)
        self._ck(self.L.m3tb_get_viewer_image(self.h, viewer, bgr.ctypes.data, bgr.strides[0], normal.ctypes.data,
                                              normal.strides[0]))
        return bgr, normal

    def set_full_renderer(self, renderer, camera_kind, camera, geometry_bodies, z_min=0.02, z_max=10.0,
                          id_type="body"):
        """FullBasicDepthRenderer / FullSilhouetteRenderer / FullNormalRenderer of camera `camera` (camera_kind
        "color" | "depth", or 0 | 1) drawing `geometry_bodies` in that order; id_type "body" | "region" (or 0 | 1). The
        image size is the camera's at the next render_full."""
        kind = {"color": 0, "depth": 1}.get(camera_kind, camera_kind)
        idt = {"body": 0, "region": 1}.get(id_type, id_type)
        g = np.ascontiguousarray(geometry_bodies, np.int32)
        self._ck(self.L.m3tb_set_full_renderer(self.h, renderer, int(kind), camera, z_min, z_max, int(idt),
                                               g.ctypes.data_as(C.POINTER(C.c_int)), g.size))

    def render_full(self):
        """FullRenderer::StartRendering of every full renderer from the current poses."""
        self._ck(self.L.m3tb_render_full(self.h))

    def get_full_rendering(self, renderer, width, height):
        """dict(depth [H,W] u16, silhouette [H,W] u8, normal [H,W,4] u8 in GL_BGRA order, projection_term_a / b
        (float32)) of the renderer's last render."""
        depth = np.zeros((height, width), np.uint16)
        sil = np.zeros((height, width), np.uint8)
        normal = np.zeros((height, width, 4), np.uint8)
        out = self.get_full_rendering_to(renderer, depth.ctypes.data, depth.strides[0], sil.ctypes.data,
                                          sil.strides[0], normal.ctypes.data, normal.strides[0])
        out.update(depth=depth, silhouette=sil, normal=normal)
        return out

    def get_full_rendering_to(self, renderer, depth_ptr=None, depth_pitch=0, silhouette_ptr=None,
                              silhouette_pitch=0, normal_ptr=None, normal_pitch=0):
        """The images into caller memory, host or device (e.g. torch tensors' data_ptr(), pitch in bytes); a None
        pointer skips that image. Returns dict(projection_term_a, projection_term_b)."""
        a, b = C.c_float(0.0), C.c_float(0.0)
        self._ck(self.L.m3tb_get_full_rendering(self.h, renderer, depth_ptr, depth_pitch, silhouette_ptr,
                                                silhouette_pitch, normal_ptr, normal_pitch, C.byref(a), C.byref(b)))
        return dict(projection_term_a=np.float32(a.value), projection_term_b=np.float32(b.value))

    def generate_depth_model(self, model_id, body, occlusion_bodies=(), params=None):
        """DepthModel::GenerateModel on the device from the geometry of m3tb_set_body_geometry (params: ModelParams,
        default model_params())."""
        p = params if params is not None else model_params()
        occ = np.ascontiguousarray(occlusion_bodies, np.int32)
        self._ck(self.L.m3tb_generate_depth_model(self.h, model_id, body, occ.ctypes.data_as(C.POINTER(C.c_int)),
                                                  occ.size, C.byref(p)))

    def get_depth_model(self, model_id):
        """A generated depth model as synth.Model (orientations, surface areas, [nv, np, 36] DataPoints, and the
        stride_depth_offset / max_radius_depth_offset it was generated with)."""
        from .synth import Model
        nv, npt = C.c_int(0), C.c_int(0)
        stride, radius = C.c_float(0.0), C.c_float(0.0)
        ip = C.POINTER(C.c_int)
        self._ck(self.L.m3tb_get_depth_model(self.h, model_id, C.cast(C.byref(nv), ip), C.cast(C.byref(npt), ip),
                                             None, None, None, C.byref(stride), C.byref(radius)))
        ori = np.zeros((nv.value, 3), np.float32)
        area = np.zeros(nv.value, np.float32)
        pts = np.zeros((nv.value, npt.value, 36), np.float32)
        self._ck(self.L.m3tb_get_depth_model(self.h, model_id, None, None, _p(ori), _p(area), pts.ctypes.data, None,
                                             None))
        return Model("depth", ori, area, pts, stride_depth_offset=float(np.float32(stride.value)),
                     max_radius_depth_offset=float(np.float32(radius.value)))

    def debug_render_model_view(self, body, view, occlusion_bodies=(), params=None):
        """dict(normal [S,S,4] u8 BGRA, depth [S,S] u16, silhouette [S,S] u8) of one generation view."""
        p = params if params is not None else model_params()
        S = p.image_size
        occ = np.ascontiguousarray(occlusion_bodies, np.int32)
        normal = np.zeros((S, S, 4), np.uint8)
        depth = np.zeros((S, S), np.uint16)
        sil = np.zeros((S, S), np.uint8)
        self._ck(self.L.m3tb_debug_render_model_view(self.h, body, occ.ctypes.data_as(C.POINTER(C.c_int)), occ.size,
                                                     C.byref(p), view, normal.ctypes.data, depth.ctypes.data,
                                                     sil.ctypes.data))
        return dict(normal=normal, depth=depth, silhouette=sil)

    def generate_region_model(self, model_id, body, associated=(), params=None):
        """RegionModel::GenerateModel on the device. associated: (body, movable, same_region) triples in
        RegionModel::AddAssociatedBody order (params: ModelParams, default model_params())."""
        p = params if params is not None else model_params()
        a = associated_bodies(associated)
        self._ck(self.L.m3tb_generate_region_model(self.h, model_id, body, a.ctypes.data, len(a), C.byref(p)))

    def get_region_model(self, model_id):
        """A generated region model as synth.Model (orientations, contour lengths, [nv, np, 38] DataPoints, and the
        stride_depth_offset / max_radius_depth_offset it was generated with)."""
        from .synth import Model
        nv, npt = C.c_int(0), C.c_int(0)
        stride, radius = C.c_float(0.0), C.c_float(0.0)
        ip = C.POINTER(C.c_int)
        self._ck(self.L.m3tb_get_region_model(self.h, model_id, C.cast(C.byref(nv), ip), C.cast(C.byref(npt), ip),
                                              None, None, None, C.byref(stride), C.byref(radius)))
        ori = np.zeros((nv.value, 3), np.float32)
        length = np.zeros(nv.value, np.float32)
        pts = np.zeros((nv.value, npt.value, 38), np.float32)
        self._ck(self.L.m3tb_get_region_model(self.h, model_id, None, None, _p(ori), _p(length), pts.ctypes.data, None,
                                              None))
        return Model("region", ori, length, pts, stride_depth_offset=float(np.float32(stride.value)),
                     max_radius_depth_offset=float(np.float32(radius.value)))

    def debug_region_model_view(self, body, view, associated=(), params=None):
        """dict(silhouettes [n_renderers,S,S] u8 (main, same-region, occlusion, foreground, background, as used),
        depth [S,S] u16, contours: list of [n,2] int32 (x, y)) of one region-generation view."""
        p = params if params is not None else model_params()
        S = p.image_size
        a = associated_bodies(associated)
        ip = C.POINTER(C.c_int)
        n_sil, n_pts, n_c = C.c_int(0), C.c_int(0), C.c_int(0)
        args = (self.h, body, a.ctypes.data, len(a), C.byref(p), view)
        self._ck(self.L.m3tb_debug_region_model_view(*args, None, C.cast(C.byref(n_sil), ip), None, None, None, 0,
                                                     C.cast(C.byref(n_pts), ip), C.cast(C.byref(n_c), ip)))
        sil = np.zeros((n_sil.value, S, S), np.uint8)
        depth = np.zeros((S, S), np.uint16)
        pts = np.zeros((max(n_pts.value, 1), 2), np.int32)
        offs = np.zeros(max(n_pts.value, 1) + 1, np.int32)
        self._ck(self.L.m3tb_debug_region_model_view(*args, sil.ctypes.data, None, depth.ctypes.data, pts.ctypes.data,
                                                     offs.ctypes.data, max(n_pts.value, 1), None, None))
        contours = [pts[offs[k]:offs[k + 1]].copy() for k in range(n_c.value)]
        return dict(silhouettes=sil, depth=depth, contours=contours)

    def set_body(self, body, region, depth, optimizer, region_model=0, depth_model=0, color_camera=0, depth_camera=0):
        self._ck(self.L.m3tb_set_body(self.h, body, C.byref(region) if region is not None else None,
                                      C.byref(depth) if depth is not None else None,
                                      C.byref(optimizer) if optimizer is not None else None, region_model,
                                      depth_model, color_camera, depth_camera))
        self.n_bodies = max(self.n_bodies, body + 1)

    def set_poses(self, poses, first=0):
        p = _f32(poses).reshape(-1, 12)
        self._ck(self.L.m3tb_set_poses(self.h, first, p.shape[0], _p(p)))

    def get_poses(self, first=0, count=None):
        count = self.n_bodies - first if count is None else count
        out = np.zeros((count, 12), np.float32)
        self._ck(self.L.m3tb_get_poses(self.h, first, count, _p(out)))
        return out.reshape(count, 3, 4)

    def share_color_histograms(self, body, owner_body):
        """RegionModality::UseSharedColorHistograms: `body` uses the ColorHistograms object of `owner_body` (-1: its own again)."""
        self._ck(self.L.m3tb_share_color_histograms(self.h, body, owner_body))

    def set_histograms(self, body, hf, hb):
        hf, hb = _f32(hf), _f32(hb)
        self._ck(self.L.m3tb_set_histograms(self.h, body, _p(hf), _p(hb)))
        self.synchronize()  # hf / hb are temporaries

    def get_histograms(self, body, n_bins):
        hf = np.zeros(n_bins ** 3, np.float32)
        hb = np.zeros(n_bins ** 3, np.float32)
        self._ck(self.L.m3tb_get_histograms(self.h, body, _p(hf), _p(hb)))
        return hf, hb

    def tracking_step(self, iteration, n_corr, n_update):
        self._ck(self.L.m3tb_tracking_step(self.h, iteration, n_corr, n_update))

    def corr_iteration(self, iteration, corr, n_update):
        self._ck(self.L.m3tb_corr_iteration(self.h, iteration, corr, n_update))

    def start_modalities(self, iteration):
        self._ck(self.L.m3tb_start_modalities(self.h, iteration))

    def calculate_results(self, iteration):
        self._ck(self.L.m3tb_calculate_results(self.h, iteration))

    def region_correspondences(self, iteration, corr):
        self._ck(self.L.m3tb_region_correspondences(self.h, iteration, corr))

    def depth_correspondences(self, iteration, corr):
        self._ck(self.L.m3tb_depth_correspondences(self.h, iteration, corr))

    def region_gradient_hessian(self, iteration, corr, opt):
        g = np.zeros((self.n_bodies, 6), np.float32)
        H = np.zeros((self.n_bodies, 6, 6), np.float32)
        self._ck(self.L.m3tb_region_gradient_hessian(self.h, iteration, corr, opt, _p(g), _p(H)))
        return g, H

    def depth_gradient_hessian(self, iteration, corr, opt):
        g = np.zeros((self.n_bodies, 6), np.float32)
        H = np.zeros((self.n_bodies, 6, 6), np.float32)
        self._ck(self.L.m3tb_depth_gradient_hessian(self.h, iteration, corr, opt, _p(g), _p(H)))
        return g, H

    def calculate_optimization(self, iteration, corr, opt):
        self._ck(self.L.m3tb_calculate_optimization(self.h, iteration, corr, opt))

    # -- kinematic structures (Optimizer with Link tree / Constraints / SoftConstraints) --
    def set_structure(self, index, spec, body_offset=0):
        """spec: synth.StructureSpec (links in pre-order). body_offset is subtracted from the link body indices
        (a context that holds bodies [first, first+count) of a workload)."""
        nl = len(spec.links)
        links = (Link * nl)()
        for i, l in enumerate(spec.links):
            K = links[i]
            K.body = l.body - body_offset if l.body >= 0 else -1
            K.parent = l.parent
            K.body2joint[:] = np.asarray(l.body2joint, np.float32).reshape(12).tolist()
            K.joint2parent[:] = np.asarray(l.joint2parent, np.float32).reshape(12).tolist()
            l2w = l.link2world if l.link2world is not None else np.eye(4, dtype=np.float32)[:3]
            K.link2world[:] = np.asarray(l2w, np.float32).reshape(12).tolist()
            K.free_directions[:] = [int(bool(d)) for d in l.free_directions]
            K.fixed_body2joint_pose = int(l.fixed_body2joint_pose)
            extra = tuple(getattr(l, "extra_bodies", ()) or ())
            K.n_extra_bodies = len(extra)
            for k, e in enumerate(extra):
                K.extra_bodies[k] = int(e) - body_offset
        nc = len(spec.constraints)
        cons = (Constraint * max(nc, 1))()
        for i, c in enumerate(spec.constraints):
            K = cons[i]
            K.link1, K.link2 = c.link1, c.link2
            K.body12joint1[:] = np.asarray(c.body12joint1, np.float32).reshape(12).tolist()
            K.body22joint2[:] = np.asarray(c.body22joint2, np.float32).reshape(12).tolist()
            K.directions[:] = [int(bool(d)) for d in c.directions]
            K.soft = int(c.soft)
            K.max_distance_rotation, K.max_distance_translation = c.max_distance_rotation, c.max_distance_translation
            K.standard_deviation_rotation = c.standard_deviation_rotation
            K.standard_deviation_translation = c.standard_deviation_translation
        op = OptimizerParams(spec.tikhonov_rotation, spec.tikhonov_translation)
        self._ck(self.L.m3tb_set_structure(self.h, index, links, nl, cons, nc, C.byref(op)))

    def set_gradient_hessian(self, modality, g, H):
        """modality: 0 region, 1 depth, 2 texture."""
        g = np.ascontiguousarray(g, np.float32)
        H = np.ascontiguousarray(H, np.float32)
        self._ck(self.L.m3tb_set_gradient_hessian(self.h, modality, _p(g), _p(H)))

    def debug_rigid_solve(self, solve, a, b, poses):
        """Test aid: the device rigid-body solve, on the shared-memory layout of k_track (solve 0) or k_track2 (solve 1),
        on systems a [n, 6, 6] (lower triangle read), b [n, 6] from start poses [n, 3, 4]: (theta [n, 6], updated [n]
        bool, poses [n, 3, 4])."""
        a = np.ascontiguousarray(a, np.float32).reshape(-1, 36)
        n = a.shape[0]
        b = np.ascontiguousarray(b, np.float32).reshape(n, 6)
        p = np.array(poses, np.float32).reshape(n, 12)
        theta = np.zeros((n, 6), np.float32)
        upd = np.zeros(n, np.int32)
        self._ck(self.L.m3tb_debug_rigid_solve(self.h, solve, n, _p(a), _p(b), _p(p), _p(theta),
                                               upd.ctypes.data_as(C.POINTER(C.c_int))))
        return theta, upd.astype(bool), p.reshape(n, 3, 4)

    def clear_structures(self):
        self._ck(self.L.m3tb_clear_structures(self.h))

    def n_structures(self):
        return self.L.m3tb_n_structures(self.h)

    def reset_joint_poses(self):
        self._ck(self.L.m3tb_reset_joint_poses(self.h))

    def calculate_consistent_poses(self):
        self._ck(self.L.m3tb_calculate_consistent_poses(self.h))

    def refine_poses(self, bodies=(), structures=(), n_corr_iterations=7, n_update_iterations=2):
        """Refiner::RefinePoses for the rigid bodies `bodies` and the kinematic structures `structures`; every other
        body and structure keeps its state. Nothing is launched when both are empty."""
        b = np.ascontiguousarray(list(bodies), dtype=np.int32)
        s = np.ascontiguousarray(list(structures), dtype=np.int32)
        ip = C.POINTER(C.c_int)
        self._ck(self.L.m3tb_refine_poses(self.h, b.ctypes.data_as(ip), len(b), s.ctypes.data_as(ip), len(s),
                                          n_corr_iterations, n_update_iterations))

    def get_link_poses(self, structure, n_links):
        """(body2joint, joint2parent, link2world), each [n_links, 3, 4]."""
        out = [np.zeros((n_links, 3, 4), np.float32) for _ in range(3)]
        self._ck(self.L.m3tb_get_link_poses(self.h, structure, _p(out[0]), _p(out[1]), _p(out[2])))
        return tuple(out)

    def get_structure_theta(self, structure, capacity=128):
        th = np.zeros(capacity, np.float32)
        n, upd = C.c_int(0), C.c_int(0)
        self._ck(self.L.m3tb_get_structure_theta(self.h, structure, _p(th), capacity, C.byref(n), C.byref(upd)))
        return th[:n.value], bool(upd.value)

    def get_region_lines(self, body, capacity):
        out = np.zeros(capacity, REGION_LINE_DTYPE)
        n = C.c_int(0)
        self._ck(self.L.m3tb_get_region_lines(self.h, body, out.ctypes.data_as(C.c_void_p), capacity, C.byref(n)))
        return out[:min(n.value, capacity)]

    # ---- texture modality (TextureModality) --------------------------------------------------------------------------
    def set_texture_modality(self, body, params, color_camera=0):
        """params: TextureParams (None removes the modality)."""
        self._ck(self.L.m3tb_set_texture_modality(self.h, body, C.byref(params) if params is not None else None,
                                                  color_camera))
        self._texture_length.pop(body, None)
        if params is not None and params.descriptor_type in (DESCRIPTOR_DAISY, DESCRIPTOR_SIFT):
            self._texture_length[body] = 0

    def get_texture_focus(self, first=0, count=None):
        """(roi [count, 4] int32 x, y, width, height; scale [count] float32; valid [count] bool)."""
        count = self.n_bodies - first if count is None else count
        roi = np.zeros((max(count, 1), 4), np.int32)
        scale = np.zeros(max(count, 1), np.float32)
        valid = np.zeros(max(count, 1), np.int32)
        ip = C.POINTER(C.c_int)
        self._ck(self.L.m3tb_get_texture_focus(self.h, first, count, roi.ctypes.data_as(ip), _p(scale),
                                               valid.ctypes.data_as(ip)))
        return roi[:count], scale[:count], valid[:count].astype(bool)

    def upload_texture_features(self, body, keypoints_xy, descriptors, roi_x, roi_y, scale):
        """keypoints_xy [n, 2] float32 in crop coordinates; descriptors [n, 32] uint8 (ORB) or [n, length] float32
        (SIFT / DAISY, m3tb_upload_texture_float_features)."""
        xy = np.ascontiguousarray(np.asarray(keypoints_xy, np.float32).reshape(-1, 2))
        if isinstance(descriptors, np.ndarray) and descriptors.dtype == np.float32:
            d = np.ascontiguousarray(descriptors)
            assert d.ndim == 2, "float descriptors are [n, length]"
            self._ck(self.L.m3tb_upload_texture_float_features(self.h, body, _p(xy), _p(d), xy.shape[0], d.shape[1],
                                                               int(roi_x), int(roi_y), float(scale)))
            if self._texture_length.get(body) == 0:
                self._texture_length[body] = d.shape[1]
            return
        d = np.ascontiguousarray(np.asarray(descriptors, np.uint8).reshape(-1, 32))
        self._ck(self.L.m3tb_upload_texture_features(self.h, body, _p(xy), d.ctypes.data_as(C.c_void_p), xy.shape[0],
                                                     int(roi_x), int(roi_y), float(scale)))

    def texture_crop(self, bodies, ptr, pitch, body_stride, capacity_width, capacity_height):
        """The focused grey images of `bodies` into device memory at ptr (e.g. a torch uint8 tensor's data_ptr()):
        body k's crop at ptr + k * body_stride, rows `pitch` bytes apart, at most capacity_width x capacity_height.
        Returns (roi [n, 4] int32, scale [n] float32, size [n, 2] int32 width, height, valid [n] bool)."""
        ids = np.ascontiguousarray(bodies, np.int32).reshape(-1)
        n = len(ids)
        roi = np.zeros((max(n, 1), 4), np.int32)
        scale = np.zeros(max(n, 1), np.float32)
        size = np.zeros((max(n, 1), 2), np.int32)
        valid = np.zeros(max(n, 1), np.int32)
        ip = C.POINTER(C.c_int)
        self._ck(self.L.m3tb_texture_crop(self.h, ids.ctypes.data_as(ip), n, C.c_void_p(ptr), pitch, body_stride,
                                          capacity_width, capacity_height, roi.ctypes.data_as(ip), _p(scale),
                                          size.ctypes.data_as(ip), valid.ctypes.data_as(ip)))
        return roi[:n], scale[:n], size[:n], valid[:n].astype(bool)

    def upload_texture_features_device(self, bodies, features):
        """features: one DeviceFeatures per body (m3tb_upload_texture_features_device); does not synchronise."""
        ids = np.ascontiguousarray(bodies, np.int32).reshape(-1)
        arr = (DeviceFeatures * max(len(ids), 1))(*features)
        self._ck(self.L.m3tb_upload_texture_features_device(self.h, ids.ctypes.data_as(C.POINTER(C.c_int)), arr,
                                                            len(ids)))
        for b, f in zip(ids, features):
            if f.length and self._texture_length.get(int(b)) == 0:
                self._texture_length[int(b)] = f.length

    def get_texture_feature_flags(self, first=0, count=None):
        """[count] bool: the body's last device upload held a non-finite descriptor value and was dropped."""
        count = self.n_bodies - first if count is None else count
        out = np.zeros(max(count, 1), np.int32)
        self._ck(self.L.m3tb_get_texture_feature_flags(self.h, first, count, out.ctypes.data_as(C.POINTER(C.c_int))))
        return out[:count].astype(bool)

    def texture_detect_orb(self, bodies, params=None):
        """cv::ORB detect + compute on the device for the ORB bodies `bodies` (m3tb_texture_detect_orb): the focused
        crop of each body's current frame, its keypoints and descriptors stored in the body's feature slot. params:
        None (defaults), one (n_features, scale_factor, n_levels) tuple / OrbParams for all, or one per body."""
        ids = np.ascontiguousarray(bodies, np.int32).reshape(-1)
        arr = None
        if params is not None:
            if isinstance(params, (OrbParams, tuple)):
                params = [params] * len(ids)
            arr = (OrbParams * max(len(ids), 1))(*[p if isinstance(p, OrbParams) else OrbParams(int(p[0]), float(p[1]), int(p[2]))
                                                   for p in params])
        self._ck(self.L.m3tb_texture_detect_orb(self.h, ids.ctypes.data_as(C.POINTER(C.c_int)), len(ids), arr))

    def get_texture_detections(self, first=0, count=None):
        """[count] int32: the keypoints cv::ORB kept at each body's last device detection (m3tb_get_texture_detections)."""
        count = self.n_bodies - first if count is None else count
        out = np.zeros(max(count, 1), np.int32)
        self._ck(self.L.m3tb_get_texture_detections(self.h, first, count, out.ctypes.data_as(C.POINTER(C.c_int))))
        return out[:count]

    def get_texture_orb_keypoints(self, body, capacity=4096):
        """The body's last device detection in canonical order (m3tb_get_texture_orb_keypoints): a dict of xy [n, 2]
        (crop coordinates), angle, response (float32), octave (int32) and descriptors [n, 32] (uint8)."""
        xy = np.zeros((capacity, 2), np.float32)
        angle = np.zeros(capacity, np.float32)
        response = np.zeros(capacity, np.float32)
        octave = np.zeros(capacity, np.int32)
        desc = np.zeros((capacity, 32), np.uint8)
        n = C.c_int(0)
        self._ck(self.L.m3tb_get_texture_orb_keypoints(self.h, body, _p(xy), _p(angle), _p(response),
                                                        octave.ctypes.data_as(C.POINTER(C.c_int)),
                                                        desc.ctypes.data_as(C.c_void_p), capacity, C.byref(n)))
        k = n.value
        return {"xy": xy[:k], "angle": angle[:k], "response": response[:k], "octave": octave[:k],
                "descriptors": desc[:k]}

    def texture_correspondences(self, iteration, corr_iteration):
        self._ck(self.L.m3tb_texture_correspondences(self.h, iteration, corr_iteration))

    def texture_gradient_hessian(self, iteration, corr_iteration, opt_iteration):
        g = np.zeros((self.n_bodies, 6), np.float32)
        H = np.zeros((self.n_bodies, 6, 6), np.float32)
        self._ck(self.L.m3tb_texture_gradient_hessian(self.h, iteration, corr_iteration, opt_iteration, _p(g), _p(H)))
        return g, H

    def get_texture_points(self, body, capacity=TEXTURE_POINT_LIMIT):
        out = np.zeros(capacity, TEXTURE_POINT_DTYPE)
        n = C.c_int(0)
        self._ck(self.L.m3tb_get_texture_points(self.h, body, out.ctypes.data_as(C.c_void_p), capacity, C.byref(n)))
        return out[:min(n.value, capacity)]

    def get_texture_keyframes(self, body, capacity=TEXTURE_POINT_LIMIT):
        """dict(sizes [n_keyframes], points [total, 3] float32, descriptors, age, orientation [3]). descriptors:
        [total, 32] uint8 for ORB; [total, length] float32 for a SIFT / DAISY body, length that of its uploads."""
        length = self._texture_length.get(body)
        nk, age = C.c_int(0), C.c_int(0)
        sizes = np.zeros(8, np.int32)
        pts = np.zeros((capacity, 3), np.float32)
        desc = np.zeros((capacity, 32), np.uint8) if length is None else np.zeros((capacity, length), np.float32)
        o = np.zeros(3, np.float32)
        self._ck(self.L.m3tb_get_texture_keyframes(self.h, body, C.byref(nk), sizes.ctypes.data_as(C.POINTER(C.c_int)),
                                                   _p(pts), desc.ctypes.data_as(C.c_void_p), capacity, C.byref(age),
                                                   _p(o)))
        sizes = sizes[:nk.value]
        total = min(int(sizes.sum()), capacity)
        return dict(sizes=sizes, points=pts[:total], descriptors=desc[:total], age=age.value, orientation=o)

    def get_depth_points(self, body, capacity):
        out = np.zeros(capacity, DEPTH_POINT_DTYPE)
        n = C.c_int(0)
        self._ck(self.L.m3tb_get_depth_points(self.h, body, out.ctypes.data_as(C.c_void_p), capacity, C.byref(n)))
        return out[:min(n.value, capacity)]

    def last_ingest_bytes(self):
        v = C.c_ulonglong(0)
        self.L.m3tb_last_ingest_bytes.argtypes = [C.c_void_p, C.POINTER(C.c_ulonglong)]
        self._ck(self.L.m3tb_last_ingest_bytes(self.h, C.byref(v)))
        return int(v.value)

    def phase_clocks(self, body, n=128):
        out = np.zeros(n, np.int64)
        self.L.m3tb_debug_phase_clocks.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
        self._ck(self.L.m3tb_debug_phase_clocks(self.h, body, out.ctypes.data_as(C.c_void_p), n))
        return out

    def last_launch(self):
        """The tracking-kernel variant of the last tracking launch as a dict (kernel: "k_track2" | "k_track" |
        "k_track_cluster" | None before the first launch)."""
        info = LaunchInfo()
        self._ck(self.L.m3tb_debug_last_launch(self.h, C.byref(info)))
        d = {k: int(getattr(info, k)) for k, _ in LaunchInfo._fields_}
        d["kernel"] = KERNEL_NAMES.get(d["kernel"], d["kernel"])
        return d

    def get_closest_views(self, body):
        a, b = C.c_int(0), C.c_int(0)
        self._ck(self.L.m3tb_get_closest_views(self.h, body, C.byref(a), C.byref(b)))
        return a.value, b.value


def debug_closest_view(orientations, queries, prev=None):
    """(scan, pruned, n_evaluated) of m3tb_debug_closest_view: host-only check of the pruned GetClosestView."""
    ori = _f32(orientations).reshape(-1, 3)
    q = _f32(queries).reshape(-1, 3)
    n = q.shape[0]
    pv = np.ascontiguousarray(prev if prev is not None else np.zeros(n), np.int32)
    out = [np.zeros(n, np.int32) for _ in range(3)]
    ip = C.POINTER(C.c_int)
    rc = lib().m3tb_debug_closest_view(_p(ori), ori.shape[0], _p(q), n, pv.ctypes.data_as(ip),
                                       *[o.ctypes.data_as(ip) for o in out])
    if rc != 0:
        raise M3TBError(f"m3tb_debug_closest_view: status {rc}")
    return tuple(out)


def context_from_workload(wl: Workload, device=0, stream=None, upload_frames=True, first=0, count=None) -> Context:
    """One context holding bodies [first, first+count) of a workload: one colour + one depth camera per
    body (one RGB-D pair per body, SURVEY §8d), models shared."""
    count = wl.n_bodies - first if count is None else count
    ctx = Context(device, max_bodies=count, max_cameras=count, max_models=1, stream=stream)
    if wl.region:
        ctx.set_region_model(0, wl.region_model)
    if wl.depth:
        ctx.set_depth_model(0, wl.depth_model)
    rp = region_params(wl.region) if wl.region else None
    dp = depth_params(wl.depth) if wl.depth else None
    op = OptimizerParams(wl.tikhonov_rotation, wl.tikhonov_translation)
    # the depth camera serves the depth modality and RegionModality::MeasureOcclusions
    need_depth_camera = bool(wl.depth) or bool(wl.region and wl.region.measure_occlusions and wl.depth_frames is not None)
    cw = getattr(wl, "color_world2camera_per_body", None)
    dw = getattr(wl, "depth_world2camera_per_body", None)
    for b in range(count):
        if wl.region:
            ctx.set_color_camera(b, wl.color_intrinsics, wl.color_world2camera if cw is None else cw[first + b])
        if need_depth_camera:
            ctx.set_depth_camera(b, wl.depth_intrinsics, wl.depth_world2camera if dw is None else dw[first + b], wl.depth_scale)
    if upload_frames:
        if wl.region:
            ctx.upload_color_batch(0, wl.color_frames[first:first + count])
        if need_depth_camera:
            ctx.upload_depth_batch(0, wl.depth_frames[first:first + count])
    for b in range(count):
        ctx.set_body(b, rp, dp, op, 0, 0, b, b)
    if getattr(wl, "histogram_owner", None) is not None:
        for b in range(count):
            o = int(wl.histogram_owner[first + b])
            if o >= 0:
                ctx.share_color_histograms(b, o - first)
    for b, per in (getattr(wl, "renderings", None) or {}).items():  # FocusedRenderer outputs, where the workload has them
        if first <= b < first + count:
            for key, r in per.items():
                ctx.upload_rendering(b - first, key, r)
    ctx.set_poses(wl.start_body2world[first:first + count])
    if getattr(wl, "structures", None):  # structures whose bodies all lie inside [first, first+count)
        k = 0
        for sp in wl.structures:
            ids = [l.body for l in sp.links if l.body >= 0] + [e for l in sp.links for e in (getattr(l, "extra_bodies", ()) or ())]
            if ids and (min(ids) < first or max(ids) >= first + count):
                continue
            ctx.set_structure(k, sp, body_offset=first)
            k += 1
    ctx.synchronize()
    return ctx
