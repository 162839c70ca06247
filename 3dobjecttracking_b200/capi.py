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
    "m3tb_n_structures", "m3tb_calculate_consistent_poses", "m3tb_get_link_poses", "m3tb_get_structure_theta",
    "m3tb_set_gradient_hessian", "m3tb_reset_joint_poses", "m3tb_prefetch_frames", "m3tb_detach_frames",
    "m3tb_debug_closest_view", "m3tb_upload_depth_rendering", "m3tb_upload_silhouette_rendering",
    "m3tb_share_color_histograms",
]

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
    _lib = L
    return L


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return a.ctypes.data_as(fp)


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
        g = np.ascontiguousarray(g, np.float32)
        H = np.ascontiguousarray(H, np.float32)
        self._ck(self.L.m3tb_set_gradient_hessian(self.h, modality, _p(g), _p(H)))

    def clear_structures(self):
        self._ck(self.L.m3tb_clear_structures(self.h))

    def n_structures(self):
        return self.L.m3tb_n_structures(self.h)

    def reset_joint_poses(self):
        self._ck(self.L.m3tb_reset_joint_poses(self.h))

    def calculate_consistent_poses(self):
        self._ck(self.L.m3tb_calculate_consistent_poses(self.h))

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
