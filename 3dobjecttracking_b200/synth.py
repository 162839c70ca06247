"""Seeded synthetic workloads for the M3T pose-optimisation hot path (SURVEY.md §8d).

ctypes wrapper around synth/libm3t_synth.so (analytic sparse-viewpoint models of the reference's
triangle prism, synthetic 640x480 BGR8 / U16 frames, ground-truth + perturbed start poses) plus the
BASELINE.json workload presets C1..C4. Pure data tooling: no CUDA, no oracle.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "synth", "libm3t_synth.so")
_lib = None

REGION_POINT_FLOATS = 38  # 152 B, RegionModel::DataPoint (region_model.h:89-95)
DEPTH_POINT_FLOATS = 36   # 144 B, DepthModel::DataPoint (depth_model.h:67-71)


class Intrinsics(C.Structure):
    """m3t::Intrinsics (common.h:25-29); layout shared by m3tb_intrinsics / orc_intrinsics."""
    _fields_ = [("fu", C.c_float), ("fv", C.c_float), ("ppu", C.c_float), ("ppv", C.c_float),
                ("width", C.c_int32), ("height", C.c_int32)]

    def copy(self):
        return Intrinsics(self.fu, self.fv, self.ppu, self.ppv, self.width, self.height)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            from . import _build
            _build.build_synth()
        L = C.CDLL(_LIB_PATH)
        fp = C.POINTER(C.c_float)
        L.m3ts_n_views.restype = C.c_int
        L.m3ts_n_views.argtypes = [C.c_int]
        for name in ("m3ts_generate_region_model", "m3ts_generate_depth_model"):
            f = getattr(L, name)
            f.restype = C.c_int
            f.argtypes = [C.c_int, C.c_int, C.c_float, C.c_uint64, fp, fp, C.c_void_p]
        L.m3ts_ground_truth_pose.restype = None
        L.m3ts_ground_truth_pose.argtypes = [C.c_uint64, C.c_int, C.POINTER(Intrinsics), C.c_float, C.c_float,
                                             C.c_float, fp]
        L.m3ts_perturb_pose.restype = None
        L.m3ts_perturb_pose.argtypes = [C.c_uint64, C.c_int, C.c_float, C.c_float, fp, fp]
        L.m3ts_render_color.restype = None
        L.m3ts_render_color.argtypes = [C.POINTER(Intrinsics), fp, C.c_uint64, C.POINTER(C.c_uint8),
                                        C.POINTER(C.c_uint8), C.c_float, C.c_void_p, C.c_size_t]
        L.m3ts_render_depth.restype = None
        L.m3ts_render_depth.argtypes = [C.POINTER(Intrinsics), fp, C.c_uint64, C.c_float, C.c_float, C.c_float,
                                        C.c_float, C.c_void_p, C.c_size_t]
        _lib = L
    return _lib


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


@dataclass
class Model:
    """Sparse viewpoint model in the reference's layout (views x points x DataPoint)."""
    kind: str                    # "region" | "depth"
    orientations: np.ndarray     # [nv,3] f32
    view_scalars: np.ndarray     # [nv] f32: contour_length / surface_area
    points: np.ndarray           # [nv,np,38|36] f32
    stride_depth_offset: float = 0.002   # model.h:161-167
    max_radius_depth_offset: float = 0.05

    @property
    def n_views(self):
        return self.points.shape[0]

    @property
    def n_points(self):
        return self.points.shape[1]


def generate_region_model(n_divides=4, n_points=200, sphere_radius=0.8, seed=0) -> Model:
    nv = lib().m3ts_n_views(n_divides)
    ori = np.zeros((nv, 3), np.float32)
    cl = np.zeros(nv, np.float32)
    pts = np.zeros((nv, n_points, REGION_POINT_FLOATS), np.float32)
    r = lib().m3ts_generate_region_model(n_divides, n_points, sphere_radius, seed, _fp(ori), _fp(cl),
                                         pts.ctypes.data_as(C.c_void_p))
    assert r == nv, r
    return Model("region", ori, cl, pts)


def generate_depth_model(n_divides=4, n_points=200, sphere_radius=0.8, seed=0) -> Model:
    nv = lib().m3ts_n_views(n_divides)
    ori = np.zeros((nv, 3), np.float32)
    sa = np.zeros(nv, np.float32)
    pts = np.zeros((nv, n_points, DEPTH_POINT_FLOATS), np.float32)
    r = lib().m3ts_generate_depth_model(n_divides, n_points, sphere_radius, seed, _fp(ori), _fp(sa),
                                        pts.ctypes.data_as(C.c_void_p))
    assert r == nv, r
    return Model("depth", ori, sa, pts)


def pose_mul(a, b):
    """[R|t] x [R|t] for float32 [3,4] arrays (float64 internally; data prep only)."""
    A = np.eye(4); A[:3] = a
    B = np.eye(4); B[:3] = b
    return (A @ B)[:3].astype(np.float32)


def pose_inv(a):
    A = np.eye(4); A[:3] = a
    return np.linalg.inv(A)[:3].astype(np.float32)


def ground_truth_pose(seed, index, intr, margin_px, z_min, z_max):
    out = np.zeros(12, np.float32)
    lib().m3ts_ground_truth_pose(seed, index, C.byref(intr), margin_px, z_min, z_max, _fp(out))
    return out.reshape(3, 4)


def perturb_pose(seed, index, rot_deg, trans_m, pose):
    src = np.ascontiguousarray(pose, np.float32).reshape(12)
    out = np.zeros(12, np.float32)
    lib().m3ts_perturb_pose(seed, index, rot_deg, trans_m, _fp(src), _fp(out))
    return out.reshape(3, 4)


def render_color(intr, body2camera, seed, fg_mean=(40, 80, 200), bg_mean=(120, 120, 120), sigma=10.0, out=None):
    """BGR8 frame [H, pitch] with pitch = 3*W rounded up to 16 B (cv::Mat-style row pitch)."""
    pitch = (3 * intr.width + 15) // 16 * 16
    if out is None:
        out = np.zeros((intr.height, pitch), np.uint8)
    fg = (C.c_uint8 * 3)(*fg_mean)
    bg = (C.c_uint8 * 3)(*bg_mean)
    b2c = np.ascontiguousarray(body2camera, np.float32).reshape(12)
    lib().m3ts_render_color(C.byref(intr), _fp(b2c), seed, fg, bg, sigma, out.ctypes.data_as(C.c_void_p), out.strides[0])
    return out


def render_depth(intr, body2camera, seed, background_z=1.0, noise_sigma=0.001, invalid_fraction=0.01,
                 depth_scale=0.001, out=None):
    if out is None:
        out = np.zeros((intr.height, intr.width), np.uint16)
    b2c = np.ascontiguousarray(body2camera, np.float32).reshape(12)
    lib().m3ts_render_depth(C.byref(intr), _fp(b2c), seed, background_z, noise_sigma, invalid_fraction, depth_scale,
                            out.ctypes.data_as(C.c_void_p), out.strides[0])
    return out


# --------------------------------------------------------------------------------------------------
# Workload presets (BASELINE.json configs; parameters from SURVEY.md §8d)
# --------------------------------------------------------------------------------------------------
@dataclass
class RegionSettings:
    n_lines_max: int = 200
    min_continuous_distance: float = 3.0
    function_amplitude: float = 0.43
    function_slope: float = 0.5
    learning_rate: float = 1.3
    n_global_iterations: int = 1
    scales: tuple = (6, 4, 2, 1)
    standard_deviations: tuple = (15.0, 5.0, 3.5, 1.5)
    n_histogram_bins: int = 16
    learning_rate_f: float = 0.2
    learning_rate_b: float = 0.2
    unconsidered_line_length: float = 0.5
    max_considered_line_length: float = 20.0
    use_adaptive_coverage: bool = False
    reference_contour_length: float = 0.0
    # measured occlusion handling (region_modality.h:432-443)
    measure_occlusions: bool = False
    measured_depth_offset_radius: float = 0.01
    measured_occlusion_radius: float = 0.01
    measured_occlusion_threshold: float = 0.03
    n_unoccluded_iterations: int = 10
    min_n_unoccluded_lines: int = 0
    # checks on renderer images (region_modality.h:424-431)
    model_occlusions: bool = False
    modeled_depth_offset_radius: float = 0.01
    modeled_occlusion_radius: float = 0.01
    modeled_occlusion_threshold: float = 0.03
    use_region_checking: bool = False


@dataclass
class DepthSettings:
    n_points_max: int = 200
    stride_length: float = 0.005
    considered_distances: tuple = (0.05, 0.02, 0.01)
    standard_deviations: tuple = (0.05, 0.03, 0.02)
    use_adaptive_coverage: bool = False
    reference_surface_area: float = 0.0
    use_depth_scaling: bool = False
    # measured occlusion handling (depth_modality.h:313-321)
    measure_occlusions: bool = False
    measured_depth_offset_radius: float = 0.01
    measured_occlusion_radius: float = 0.01
    measured_occlusion_threshold: float = 0.03
    n_unoccluded_iterations: int = 10
    min_n_unoccluded_points: int = 0
    # checks on renderer images (depth_modality.h:305-312)
    model_occlusions: bool = False
    modeled_depth_offset_radius: float = 0.01
    modeled_occlusion_radius: float = 0.01
    modeled_occlusion_threshold: float = 0.03
    use_silhouette_checking: bool = False


@dataclass
class Rendering:
    """One FocusedRenderer output for one body in one camera (renderer.h:156-230): `image` is the focused depth image
    (u16, depth = a / (b - value), renderer.cpp:511-513) or the focused silhouette image (u8 ids); the focused image
    shows the square [corner, corner + image_size / scale) of the camera image."""
    image: np.ndarray
    corner_u: float
    corner_v: float
    scale: float
    projection_term_a: float = 0.0
    projection_term_b: float = 0.0
    id: int = 0
    visible: bool = True


@dataclass
class Workload:
    name: str
    n_bodies: int
    region: RegionSettings | None
    depth: DepthSettings | None
    tikhonov_rotation: float
    tikhonov_translation: float
    n_corr_iterations: int
    n_update_iterations: int
    color_intrinsics: Intrinsics
    depth_intrinsics: Intrinsics
    color_world2camera: np.ndarray          # [3,4]
    depth_world2camera: np.ndarray          # [3,4]
    depth_scale: float
    region_model: Model | None
    depth_model: Model | None
    color_frames: np.ndarray | None         # [nb,H,pitch] u8 (one frame per body)
    depth_frames: np.ndarray | None         # [nb,H,W] u16
    gt_body2world: np.ndarray               # [nb,3,4]
    start_body2world: np.ndarray            # [nb,3,4]
    seed: int = 0
    notes: dict = field(default_factory=dict)
    structures: list | None = None          # [StructureSpec] (kinematic structures, config 5); None = rigid bodies
    color_world2camera_per_body: np.ndarray | None = None   # [nb,3,4]: multi-camera rigs (default: one pose for all)
    depth_world2camera_per_body: np.ndarray | None = None
    histogram_owner: np.ndarray | None = None   # [nb] int: body whose ColorHistograms object this body uses (-1: its own)
    renderings: dict | None = None          # {body: {"region_depth" | "region_silhouette" | "depth_depth" | "depth_silhouette": Rendering}}

    @property
    def lines_per_body(self):
        return self.region.n_lines_max if self.region else 0

    @property
    def points_per_body(self):
        return self.depth.n_points_max if self.depth else 0


@dataclass
class LinkSpec:
    """One m3t::Link (link.h:150-156). body: index into the workload's bodies or -1; parent: index into the
    structure's link list (links are listed in Optimizer::ReferencedLinks() order, parent < own index) or -1."""
    body: int
    parent: int
    body2joint: np.ndarray = None           # [3,4]
    joint2parent: np.ndarray = None         # [3,4]
    free_directions: tuple = (1, 1, 1, 1, 1, 1)
    fixed_body2joint_pose: bool = True
    link2world: np.ndarray = None           # [3,4], links without a body only
    extra_bodies: tuple = ()                # further modality sets (bodies) of the same physical body (link.h:151)


@dataclass
class ConstraintSpec:
    """m3t::Constraint (constraint.h:109-112), or m3t::SoftConstraint when `soft` (soft_constraint.h:128-136)."""
    link1: int
    link2: int
    body12joint1: np.ndarray = None
    body22joint2: np.ndarray = None
    directions: tuple = (0, 0, 0, 0, 0, 0)
    soft: bool = False
    max_distance_rotation: float = 0.0
    max_distance_translation: float = 0.0
    standard_deviation_rotation: float = 0.01
    standard_deviation_translation: float = 0.001


@dataclass
class StructureSpec:
    """One m3t::Optimizer with its link tree and constraints."""
    links: list
    constraints: list = field(default_factory=list)
    tikhonov_rotation: float = 1000.0
    tikhonov_translation: float = 30000.0

    @property
    def dof(self):
        return sum(int(sum(1 for d in l.free_directions if d)) for l in self.links)

    @property
    def n_constraint_rows(self):
        return sum(int(sum(1 for d in c.directions if d)) for c in self.constraints if not c.soft)


def identity_pose():
    p = np.zeros((3, 4), np.float32)
    p[:, :3] = np.eye(3, dtype=np.float32)
    return p


def translation_pose(x=0.0, y=0.0, z=0.0):
    p = identity_pose()
    p[:, 3] = (x, y, z)
    return p


def rotation_pose(axis, deg):
    p = identity_pose()
    p[:, :3] = _rot(axis, deg)
    return p


def fill_depth_offsets(model: Model, seed=0):
    """Synthetic DataPoint::depth_offsets (the analytic generator leaves them at 0): non-negative and non-decreasing
    with the radius index, like Model::CalculateDepthOffsets (model.cpp:338-384) produces them. In place."""
    first = 8 if model.kind == "region" else 6
    rng = np.random.default_rng([seed, 0x4F46, model.n_views, model.n_points])
    slope = rng.uniform(0.0, 0.6, size=model.points.shape[:2]).astype(np.float32)
    k = np.arange(30, dtype=np.float32)
    model.points[:, :, first:first + 30] = slope[:, :, None] * (k * np.float32(model.stride_depth_offset))[None, None, :]


def add_occluder(wl: Workload, body: int, side="left", cover=0.45, gap_m=0.12, color_mean=(60, 170, 70), sigma=8.0, seed=0):
    """Paints a fronto-parallel occluder (a plane patch in the colour camera's frame, gap_m in front of the body) over
    `cover` of the body's image extent into the body's colour and depth frames, consistently in both cameras."""
    b2w = wl.gt_body2world[body]
    T = lambda p: np.vstack([np.asarray(p, np.float64), [0, 0, 0, 1]])
    b2c = (T(wl.color_world2camera) @ T(b2w))[:3]
    zc = b2c[2, 3]
    z_occ = zc - gap_m
    r = 0.045  # prism circumradius
    cx, cy = b2c[0, 3], b2c[1, 3]
    if side == "left":
        x0, x1, y0, y1 = cx - 3 * r, cx - r + 2 * r * cover, cy - 3 * r, cy + 3 * r
    else:
        x0, x1, y0, y1 = cx - 3 * r, cx + 3 * r, cy - 3 * r, cy - r + 2 * r * cover
    # the patch is given at the body's depth; seen from the camera it is the cone through it cut at z_occ
    x0, x1, y0, y1 = (v * z_occ / zc for v in (x0, x1, y0, y1))
    rng = np.random.default_rng([seed, 0x4F43, body])
    ci, di = wl.color_intrinsics, wl.depth_intrinsics
    if wl.color_frames is not None:
        v, u = np.mgrid[0:ci.height, 0:ci.width]
        X = (u - ci.ppu) / ci.fu * z_occ
        Y = (v - ci.ppv) / ci.fv * z_occ
        m = (X >= x0) & (X <= x1) & (Y >= y0) & (Y <= y1)
        img = wl.color_frames[body][:, :3 * ci.width].reshape(ci.height, ci.width, 3)
        noise = rng.normal(0.0, sigma, size=(int(m.sum()), 3))
        img[m] = np.clip(np.rint(np.asarray(color_mean, np.float64)[None, :] + noise), 0, 255).astype(np.uint8)
    if wl.depth_frames is not None:
        # plane z = z_occ of the colour camera expressed in the depth camera: n . X = d
        c2d = T(wl.depth_world2camera) @ np.linalg.inv(T(wl.color_world2camera))
        n = c2d[:3, :3] @ np.array([0.0, 0.0, 1.0])
        p0 = c2d[:3, :3] @ np.array([0.0, 0.0, z_occ]) + c2d[:3, 3]
        d = float(n @ p0)
        v, u = np.mgrid[0:di.height, 0:di.width]
        ray = np.stack([(u - di.ppu) / di.fu, (v - di.ppv) / di.fv, np.ones_like(u, np.float64)], -1)
        t = d / (ray @ n)
        P = ray * t[..., None]
        Pc = (P - c2d[:3, 3]) @ c2d[:3, :3]      # back into the colour camera frame (R^T (P - t))
        m = (t > 0) & (Pc[..., 0] >= x0) & (Pc[..., 0] <= x1) & (Pc[..., 1] >= y0) & (Pc[..., 1] <= y1)
        z = P[..., 2] + rng.normal(0.0, 0.001, size=P.shape[:2])
        wl.depth_frames[body][m] = np.clip(np.rint(z[m] / wl.depth_scale), 1, 65535).astype(np.uint16)
    wl.notes.setdefault("occluders", []).append(dict(body=body, side=side, cover=cover, z=z_occ))


def add_renderings(wl: Workload, image_size=200, z_min=0.02, z_max=5.0, occluder_bodies=(), region_id=7, seed=0):
    """Synthetic stand-ins for what FocusedDepthRenderer / FocusedSilhouetteRenderer hand to the modalities (the
    OpenGL renderers stay with the caller): for every body and both cameras a focused depth image and a focused
    silhouette image of the body AT ITS START POSE, computed by the same ray caster that makes the frames, with
    FocusedRenderer's geometry (corner, scale: renderer.cpp:385-395; projection terms: :568-569). For bodies listed
    in occluder_bodies a nearer fronto-parallel plane covers the left part of the focused images (another body's id in
    the silhouette, its depth in the depth rendering), so that the checks reject some lines / points."""
    wl.renderings = {}
    a = z_max * z_min * 65535.0 / (z_max - z_min)
    b = z_max * 65535.0 / (z_max - z_min)
    for body in range(wl.n_bodies):
        per = {}
        for kind, intr, w2c in (("region", wl.color_intrinsics, wl.color_world2camera),
                                ("depth", wl.depth_intrinsics, wl.depth_world2camera)):
            if (kind == "region" and not wl.region) or (kind == "depth" and not wl.depth):
                continue
            b2c = pose_mul(w2c, wl.start_body2world[body])
            z = float(b2c[2, 3])
            cu, cv = b2c[0, 3] * intr.fu / z + intr.ppu, b2c[1, 3] * intr.fv / z + intr.ppv
            r = 0.05  # a little more than the prism's circumradius (renderer.cpp: 2 r fu / z = the focused square)
            d = 2.0 * r * intr.fu / z
            corner_u, corner_v, scale = float(cu - 0.5 * d), float(cv - 0.5 * d), float(image_size / d)
            # the focused image is a pinhole image with intrinsics (f * scale, (pp - corner) * scale)
            fi = Intrinsics(intr.fu * scale, intr.fv * scale, (intr.ppu - corner_u) * scale, (intr.ppv - corner_v) * scale,
                            image_size, image_size)
            depth_mm = render_depth(fi, b2c, seed * 7919 + body, background_z=0.0, noise_sigma=0.0, invalid_fraction=0.0,
                                    depth_scale=0.0001)  # 0.1 mm units, 0 = background
            zmap = depth_mm.astype(np.float64) * 0.0001
            on_body = depth_mm > 0
            zmap[~on_body] = z_max
            sil = np.where(on_body, region_id, 0).astype(np.uint8)
            if body in occluder_bodies:
                cols = slice(0, int(image_size * 0.45))
                zmap[:, cols] = np.minimum(zmap[:, cols], z - 0.15)
                sil[:, cols] = region_id + 1
            value = np.clip(np.rint(b - a / zmap), 0, 65535).astype(np.uint16)
            per[f"{kind}_depth"] = Rendering(np.ascontiguousarray(value), corner_u, corner_v, scale, float(np.float32(a)),
                                             float(np.float32(b)), 0, True)
            per[f"{kind}_silhouette"] = Rendering(np.ascontiguousarray(sil), corner_u, corner_v, scale, 0.0, 0.0, region_id, True)
        wl.renderings[body] = per
    return wl


# ---- triangle soups for the device renderers (m3tb_set_body_geometry) -------------------------------------------------
# the reference's triangle prism in the body frame (synth/m3t_synth.cpp kVerts / kFaces: data/_body/triangle.obj with
# geometry2body's z offset applied)
PRISM_VERTICES = np.array([[-0.038305, 0.0, -0.006], [-0.038305, 0.0, 0.006], [0.019152, -0.033231, -0.006],
                           [0.019152, -0.033231, 0.006], [0.019152, 0.033231, -0.006], [0.019152, 0.033231, 0.006]])
PRISM_FACES = np.array([[0, 2, 3], [2, 4, 3], [3, 5, 1], [4, 0, 1], [0, 4, 2], [1, 0, 3], [4, 5, 3], [5, 4, 1]])


def _outward(vertices, faces):
    """[n,3,3] float32 soup of a convex body around the origin, every triangle counter-clockwise seen from outside."""
    tri = np.asarray(vertices, np.float64)[np.asarray(faces)]
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    flip = np.einsum("ij,ij->i", n, tri.mean(axis=1)) < 0
    tri[flip] = tri[flip][:, [0, 2, 1]]
    return tri.astype(np.float32)


def prism_triangles():
    """The prism (8 triangles) and its maximum body diameter (twice the largest vertex distance, as float32)."""
    return _outward(PRISM_VERTICES, PRISM_FACES), float(np.float32(2.0 * np.linalg.norm(PRISM_VERTICES, axis=1).max()))


def icosphere_triangles(radius=0.04, n_divides=4):
    """A closed subdivided icosahedron (20 * 4^n_divides triangles; 5120 at the default) and its diameter."""
    t = (1.0 + 5.0 ** 0.5) / 2.0
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1),
         (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
         (9, 8, 1)]
    tri = np.array([[v[i] for i in face] for face in f], np.float64)
    tri /= np.linalg.norm(tri, axis=2, keepdims=True)
    for _ in range(n_divides):
        a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
        ab, bc, ca = [m / np.linalg.norm(m, axis=1, keepdims=True) for m in (a + b, b + c, c + a)]
        tri = np.concatenate([np.stack(x, 1) for x in ((a, ab, ca), (ab, b, bc), (ca, bc, c), (ab, bc, ca))])
    tri *= radius
    return _outward(tri.reshape(-1, 3), np.arange(tri.shape[0] * 3).reshape(-1, 3)), float(np.float32(2.0 * radius))


PRESETS = {
    # name: (n_bodies, n_lines, n_points, rbot_shape)
    "c1": dict(n_bodies=1, n_lines=200, n_points=0, rbot=False),
    "c2": dict(n_bodies=1, n_lines=200, n_points=200, rbot=False),
    "c3": dict(n_bodies=64, n_lines=300, n_points=0, rbot=True),
    "c4": dict(n_bodies=128, n_lines=512, n_points=512, rbot=False),  # per-GPU shard of 1024 bodies / 8 GPUs
}


def default_color_intrinsics(rbot=False):
    if rbot:  # rbot_evaluator.h:40-41 re-centred to a 640x480 frame
        return Intrinsics(650.048, 647.183, 319.5, 239.5, 640, 480)
    return Intrinsics(614.0, 614.5, 321.3, 238.9, 640, 480)


def default_depth_intrinsics():
    return Intrinsics(385.7, 385.9, 322.1, 241.6, 640, 480)


def _rot(axis, deg):
    a = np.deg2rad(deg)
    x, y, z = np.asarray(axis, float) / np.linalg.norm(axis)
    c, s, Cc = np.cos(a), np.sin(a), 1 - np.cos(a)
    return np.array([[c + x * x * Cc, x * y * Cc - z * s, x * z * Cc + y * s],
                     [y * x * Cc + z * s, c + y * y * Cc, y * z * Cc - x * s],
                     [z * x * Cc - y * s, z * y * Cc + x * s, c + z * z * Cc]])


def make_chain_workload(n_chains=2, n_links=8, n_lines=300, n_points=300, variant="projected", n_divides=4, seed=0,
                        rot_deg=3.0, trans_m=0.005, joint_deg=3.0, color_sigma=10.0, first_chain=0, frames=True,
                        models=None, soft=False) -> Workload:
    """BASELINE.json configs[4] shape (SURVEY §8d C5): n_chains instances of an n_links serial chain, RTB-shape
    parameters (examples/evaluate_rtb_dataset.cpp:27-66), chain geometry of examples/optimization_time.cpp.

    variant "projected" (optimization_time.cpp:48-56): root link with 6 DoF, every further link is the child of the
    previous one with joint2parent = Tx(0.01) and one revolute DoF about x -> 6 + (n_links-1) unknowns.
    variant "constrained" (optimization_time.cpp:32-46): every link is a 6-DoF child of the root and consecutive
    links are tied by a Constraint with body12joint1 = Tx(-0.01), directions (0,1,1,1,1,1) -> 6 n_links unknowns + 5
    (n_links-1) constraint rows. soft=True uses SoftConstraints instead of Constraints in the constrained variant.
    Bodies are numbered chain * n_links + link. Every link is observed in its own RGB-D pair by the same camera pair
    (deviation from "one pair per instance": the links of this chain geometry overlap in space, rendering them into
    one frame would make the silhouettes meaningless; the arithmetic of the path is unaffected)."""
    nb = n_chains * n_links
    region = RegionSettings(n_lines_max=n_lines, scales=(9, 7, 5, 2), standard_deviations=(25.0, 15.0, 10.0)) if n_lines else None
    depth = DepthSettings(n_points_max=n_points, stride_length=0.008, considered_distances=(0.1, 0.08, 0.05),
                          standard_deviations=(0.05, 0.03, 0.02)) if n_points else None
    ci, di = default_color_intrinsics(False), default_depth_intrinsics()
    c_w2c = np.zeros((3, 4), np.float32)
    c_w2c[:, :3] = _rot((0.2, 1.0, 0.1), 4.0)
    c_w2c[:, 3] = (0.01, -0.02, 0.03)
    d_rel = np.zeros((3, 4), np.float32)
    d_rel[:, :3] = _rot((1.0, 0.3, -0.2), 0.6)
    d_rel[:, 3] = (-0.015, 0.001, 0.002)
    d_w2c = pose_mul(d_rel, c_w2c)
    c_c2w = pose_inv(c_w2c)
    if models is not None:
        region_model, depth_model = models
    else:
        region_model = generate_region_model(n_divides, max(n_lines, 1), 0.8, seed) if region else None
        depth_model = generate_depth_model(n_divides, max(n_points, 1), 0.8, seed) if depth else None
    gt = np.zeros((nb, 3, 4), np.float32)
    start = np.zeros((nb, 3, 4), np.float32)
    pitch = (3 * ci.width + 15) // 16 * 16
    color = np.zeros((nb, ci.height, pitch), np.uint8) if (region and frames) else None
    dframes = np.zeros((nb, di.height, di.width), np.uint16) if (depth and frames) else None
    offset = translation_pose(0.01)
    structures = []
    for c in range(n_chains):
        gc = first_chain + c
        rng = np.random.default_rng([seed, 77, gc])
        q_gt = rng.uniform(-12.0, 12.0, n_links)
        q_start = q_gt + rng.uniform(-joint_deg, joint_deg, n_links)
        root_gt = pose_mul(c_c2w, ground_truth_pose(seed, 100000 + gc, ci, 200.0, 0.6, 0.8))
        root_start = perturb_pose(seed, 100000 + gc, rot_deg, trans_m, root_gt)
        links, constraints = [], []
        for j in range(n_links):
            b = c * n_links + j
            if j == 0:
                gt[b], start[b] = root_gt, root_start
                links.append(LinkSpec(body=b, parent=-1, body2joint=identity_pose(), joint2parent=identity_pose()))
                continue
            gt[b] = pose_mul(pose_mul(gt[b - 1], offset), rotation_pose((1, 0, 0), q_gt[j]))
            start[b] = pose_mul(pose_mul(start[b - 1], offset), rotation_pose((1, 0, 0), q_start[j]))
            if variant == "projected":
                links.append(LinkSpec(body=b, parent=j - 1, body2joint=identity_pose(),
                                      joint2parent=pose_mul(offset, rotation_pose((1, 0, 0), q_start[j])),
                                      free_directions=(1, 0, 0, 0, 0, 0)))
            else:
                links.append(LinkSpec(body=b, parent=0, body2joint=identity_pose(),
                                      joint2parent=pose_mul(pose_inv(start[c * n_links]), start[b])))
                constraints.append(ConstraintSpec(link1=j - 1, link2=j, body12joint1=translation_pose(-0.01),
                                                  body22joint2=identity_pose(), directions=(0, 1, 1, 1, 1, 1), soft=soft))
        structures.append(StructureSpec(links=links, constraints=constraints, tikhonov_rotation=100.0,
                                        tikhonov_translation=1000.0))
        for j in range(n_links):
            b = c * n_links + j
            gb = gc * n_links + j
            if color is not None:
                render_color(ci, pose_mul(c_w2c, gt[b]), seed * 1000003 + 500000 + gb, sigma=color_sigma, out=color[b])
            if dframes is not None:
                render_depth(di, pose_mul(d_w2c, gt[b]), seed * 1000003 + 500000 + gb, depth_scale=0.001, out=dframes[b])
    return Workload(name="c5", n_bodies=nb, region=region, depth=depth, tikhonov_rotation=100.0,
                    tikhonov_translation=1000.0, n_corr_iterations=6, n_update_iterations=2, color_intrinsics=ci,
                    depth_intrinsics=di, color_world2camera=c_w2c, depth_world2camera=d_w2c, depth_scale=0.001,
                    region_model=region_model, depth_model=depth_model, color_frames=color, depth_frames=dframes,
                    gt_body2world=gt, start_body2world=start, seed=seed,
                    notes=dict(n_divides=n_divides, variant=variant, n_links=n_links, n_chains=n_chains, soft=soft,
                               first_body=first_chain * n_links), structures=structures)


def make_multi_camera_workload(n_objects=3, n_lines=200, n_points=200, n_divides=3, seed=0, rot_deg=3.0, trans_m=0.005):
    """n_objects rigid bodies, each observed by TWO colour + depth camera pairs (a stereo-like rig: the second pair is
    the first one moved by 12 cm / 8 degrees). Object i is body i (camera pair A) and body n_objects + i (camera pair
    B) - two modality sets of one physical body, i.e. one m3t::Link with four modalities; structure i is the one-link
    Optimizer that sums them (Link::CalculateGradientAndHessian, link.cpp:184-193)."""
    wl = make_workload("c2", n_bodies=n_objects, n_lines=n_lines, n_points=n_points, n_divides=n_divides, seed=seed,
                       rot_deg=rot_deg, trans_m=trans_m)
    n = n_objects
    ci, di = wl.color_intrinsics, wl.depth_intrinsics
    rig = np.zeros((3, 4), np.float32)
    rig[:, :3] = _rot((0.1, 1.0, 0.05), 8.0)
    rig[:, 3] = (-0.12, 0.01, 0.015)
    c2 = pose_mul(rig, wl.color_world2camera)
    d2 = pose_mul(rig, wl.depth_world2camera)
    color = np.concatenate([wl.color_frames, np.zeros_like(wl.color_frames)])
    depth = np.concatenate([wl.depth_frames, np.zeros_like(wl.depth_frames)])
    for i in range(n):
        render_color(ci, pose_mul(c2, wl.gt_body2world[i]), seed * 1000003 + 700000 + i, out=color[n + i])
        render_depth(di, pose_mul(d2, wl.gt_body2world[i]), seed * 1000003 + 700000 + i, depth_scale=wl.depth_scale, out=depth[n + i])
    wl.n_bodies = 2 * n
    wl.color_frames, wl.depth_frames = color, depth
    wl.gt_body2world = np.concatenate([wl.gt_body2world, wl.gt_body2world])
    wl.start_body2world = np.concatenate([wl.start_body2world, wl.start_body2world])
    wl.color_world2camera_per_body = np.stack([wl.color_world2camera] * n + [c2] * n)
    wl.depth_world2camera_per_body = np.stack([wl.depth_world2camera] * n + [d2] * n)
    wl.structures = [StructureSpec(links=[LinkSpec(body=i, parent=-1, body2joint=identity_pose(), joint2parent=identity_pose(),
                                                   extra_bodies=(n + i,))],
                                   tikhonov_rotation=wl.tikhonov_rotation, tikhonov_translation=wl.tikhonov_translation)
                     for i in range(n)]
    wl.name = "multi_camera"
    return wl


def make_workload(name="c2", n_bodies=None, n_lines=None, n_points=None, n_divides=4, seed=0, rot_deg=3.0,
                  trans_m=0.005, rbot=None, model_points=None, frames=True, color_sigma=10.0, first_body=0,
                  models=None, margin_px=None, z_range=(0.5, 0.7), color_intrinsics=None, depth_intrinsics=None,
                  centers_px=None) -> Workload:
    """Build one of the BASELINE.json workloads (optionally resized) from (seed, global body index).

    first_body: global index of this shard's first body (multi-GPU sharding: rank r of a weak-scaled job
    builds bodies [r*n_bodies, (r+1)*n_bodies)). models: optional (region_model, depth_model) to reuse.
    margin_px: least distance of a body centre from the colour frame's border (default: the longest line half-length
    + the body radius, so that every body sits well inside the frame); z_range: depth range of the body centres in the
    colour camera; color_intrinsics / depth_intrinsics: other cameras (frame sizes) than the presets'. centers_px: one
    (u, v, z) per body that pins the ground-truth centre to colour pixel (u, v) at depth z (z < 0: behind the camera;
    the rotation stays the seeded one)."""
    preset = dict(PRESETS[name])
    if n_bodies is not None:
        preset["n_bodies"] = n_bodies
    if n_lines is not None:
        preset["n_lines"] = n_lines
    if n_points is not None:
        preset["n_points"] = n_points
    if rbot is not None:
        preset["rbot"] = rbot
    nb = preset["n_bodies"]
    rb = preset["rbot"]
    region = depth = None
    if preset["n_lines"] > 0:
        region = RegionSettings(n_lines_max=preset["n_lines"])
        if rb:  # evaluate_rbot_dataset.cpp:25-44,76-83
            region.scales = (5, 2, 2, 1)
            region.standard_deviations = (20.0, 7.0, 3.0, 1.5)
            region.function_amplitude = 0.36
            region.function_slope = 0.0
            region.n_histogram_bins = 32
    if preset["n_points"] > 0:
        depth = DepthSettings(n_points_max=preset["n_points"])
    ci = default_color_intrinsics(rb) if color_intrinsics is None else color_intrinsics.copy()
    di = default_depth_intrinsics() if depth_intrinsics is None else depth_intrinsics.copy()
    if centers_px is not None and len(centers_px) != nb:
        raise ValueError(f"centers_px has {len(centers_px)} entries for {nb} bodies")
    # non-identity camera poses (the reference's fixture has a non-identity depth camera2world as well)
    c_w2c = np.zeros((3, 4), np.float32)
    c_w2c[:, :3] = _rot((0.2, 1.0, 0.1), 4.0)
    c_w2c[:, 3] = (0.01, -0.02, 0.03)
    d_rel = np.zeros((3, 4), np.float32)      # colour-camera -> depth-camera
    d_rel[:, :3] = _rot((1.0, 0.3, -0.2), 0.6)
    d_rel[:, 3] = (-0.015, 0.001, 0.002)
    d_w2c = pose_mul(d_rel, c_w2c)
    c_c2w = pose_inv(c_w2c)

    mp_r = model_points or max(preset["n_lines"], 1)
    mp_d = model_points or max(preset["n_points"], 1)
    if models is not None:
        region_model, depth_model = models
    else:
        region_model = generate_region_model(n_divides, mp_r, 0.8, seed) if region else None
        depth_model = generate_depth_model(n_divides, mp_d, 0.8, seed) if depth else None

    max_scale = max(region.scales) if region else 0
    # longest line half-length + body radius in px (+ slack for the depth camera)
    margin = 19 * max_scale / 2 + 75.0 if margin_px is None else margin_px
    gt = np.zeros((nb, 3, 4), np.float32)
    start = np.zeros((nb, 3, 4), np.float32)
    pitch = (3 * ci.width + 15) // 16 * 16
    color = np.zeros((nb, ci.height, pitch), np.uint8) if (region and frames) else None
    dframes = np.zeros((nb, di.height, di.width), np.uint16) if (depth and frames) else None
    for b in range(nb):
        gb = first_body + b  # global body index: the only thing (besides seed) a body's data depends on
        b2c = ground_truth_pose(seed, gb, ci, margin, z_range[0], z_range[1])
        if centers_px is not None:
            u, v, z = (float(c) for c in centers_px[b])
            b2c[:, 3] = ((u - ci.ppu) / ci.fu * z, (v - ci.ppv) / ci.fv * z, z)
        b2w = pose_mul(c_c2w, b2c)
        gt[b] = b2w
        start[b] = perturb_pose(seed, gb, rot_deg, trans_m, b2w)
        if color is not None:
            render_color(ci, pose_mul(c_w2c, b2w), seed * 1000003 + gb, sigma=color_sigma, out=color[b])
        if dframes is not None:
            render_depth(di, pose_mul(d_w2c, b2w), seed * 1000003 + gb, depth_scale=0.001, out=dframes[b])
    lam = (1000.0, 30000.0)  # optimizer.h:52-53
    return Workload(name=name, n_bodies=nb, region=region, depth=depth, tikhonov_rotation=lam[0],
                    tikhonov_translation=lam[1], n_corr_iterations=7, n_update_iterations=2,
                    color_intrinsics=ci, depth_intrinsics=di, color_world2camera=c_w2c, depth_world2camera=d_w2c,
                    depth_scale=0.001, region_model=region_model, depth_model=depth_model, color_frames=color,
                    depth_frames=dframes, gt_body2world=gt, start_body2world=start, seed=seed,
                    notes=dict(n_divides=n_divides, rot_deg=rot_deg, trans_m=trans_m, rbot=rb, color_sigma=color_sigma,
                               first_body=first_body))


def model_radius(model: Model) -> float:
    """Largest distance of a model point from the body origin, in float32 as m3tb_set_*_model computes it (the radius
    the kernels size their ROIs with; a body closer than twice of it gets no tile)."""
    p = model.points[:, :, :3].astype(np.float32)
    return float(np.sqrt(np.float32((p * p).sum(-1, dtype=np.float32).max())))


def _color_pixel(wl_cameras, camera, u, v, z):
    """(u, v, z) in the colour camera of the point that `camera` ("color" | "depth") sees at pixel (u, v), depth z."""
    ci, di, c_w2c, d_w2c = wl_cameras
    intr = ci if camera == "color" else di
    X = np.array([(u - intr.ppu) / intr.fu * z, (v - intr.ppv) / intr.fv * z, z, 1.0])
    if camera == "depth":
        T = lambda p: np.vstack([np.asarray(p, np.float64), [0, 0, 0, 1]])
        X = T(c_w2c) @ np.linalg.inv(T(d_w2c)) @ X
    return (float(X[0] / X[2] * ci.fu + ci.ppu), float(X[1] / X[2] * ci.fv + ci.ppv), float(X[2]))


EDGE_KINDS = ("border", "depth_border", "near", "far", "out")
EDGE_MODALITIES = ("region+depth", "region16", "region32", "depth")


def _border_placements(w, h, offsets=(20.0, 0.0, -30.0)):
    """Body centres on the four edges (at mid-edge) and the four corners, `offset` px inside the frame (negative:
    outside). Pixel centres are integers: column 0 and column w - 1 are the border columns."""
    out = []
    for d in offsets:
        lo_u, hi_u, lo_v, hi_v = d, w - 1 - d, d, h - 1 - d
        mid_u, mid_v = 0.5 * (w - 1), 0.5 * (h - 1)
        out += [(lo_u, mid_v), (hi_u, mid_v), (mid_u, lo_v), (mid_u, hi_v),
                (lo_u, lo_v), (hi_u, lo_v), (lo_u, hi_v), (hi_u, hi_v)]
    return out


def make_edge_workload(kind, modalities="region+depth", n_divides=2, seed=0, color_intrinsics=None,
                       depth_intrinsics=None, rot_deg=3.0, trans_m=0.005) -> Workload:
    """Deterministic placements where the per-line / per-point validity tests, the ROI and tile sizing and the depth
    search windows meet the frame's edges (the random workloads keep every body well inside the frame):
      border        the four edges and four corners of the colour frame, centre +20 / 0 / -30 px from the border
      depth_border  the same in the depth camera's pixels
      near          centre depth just below and just above twice the model radius (the kernels' no-tile branch)
      far           1.5 - 3 m (few or no lines / points pass min_continuous_distance / the stride)
      out           fully outside the frame on each side, and one body behind the camera
    modalities: "region+depth" (200 lines + 200 points), "region16" / "region32" (200 lines, 16 / 32 histogram bins)
    or "depth" (200 points)."""
    if kind not in EDGE_KINDS or modalities not in EDGE_MODALITIES:
        raise ValueError((kind, modalities))
    n_lines = 0 if modalities == "depth" else 200
    n_points = 200 if modalities in ("region+depth", "depth") else 0
    ci = default_color_intrinsics(False) if color_intrinsics is None else color_intrinsics.copy()
    di = default_depth_intrinsics() if depth_intrinsics is None else depth_intrinsics.copy()
    # cameras and models first (their data does not depend on the placements), then the placements
    probe = make_workload("c2", n_bodies=1, n_lines=n_lines, n_points=n_points, n_divides=n_divides, seed=seed,
                          frames=False, color_intrinsics=ci, depth_intrinsics=di)
    cams = (ci, di, probe.color_world2camera, probe.depth_world2camera)
    models = (probe.region_model, probe.depth_model)
    if kind in ("border", "depth_border"):
        cam = "color" if kind == "border" else "depth"
        intr = ci if cam == "color" else di
        centers = [_color_pixel(cams, cam, u, v, 0.6) for u, v in _border_placements(intr.width, intr.height)]
    elif kind == "near":
        # the depth camera's z decides the depth tile, the colour camera's the colour tile: straddle both
        r = model_radius(probe.depth_model if probe.depth_model is not None else probe.region_model)
        uc, vc = 0.5 * (ci.width - 1), 0.5 * (ci.height - 1)
        centers = [(uc + du, vc + dv, 2.0 * r * f) for f in (0.9, 0.97, 1.03, 1.1) for du, dv in ((0.0, 0.0), (-60.0, 40.0))]
    elif kind == "far":
        centers = [(u, v, z) for z in (1.5, 2.0, 2.5, 3.0) for u, v in ((0.3 * ci.width, 0.4 * ci.height),
                                                                         (0.7 * ci.width, 0.6 * ci.height))]
    else:  # out: a frame width / height beyond each edge (outside the wider-angle depth frame as well), and behind the
        # camera (its centre projects to the middle of the frame)
        w, h = ci.width, ci.height
        centers = [(-w, 0.5 * h, 0.6), (2.0 * w, 0.5 * h, 0.6), (0.5 * w, -h, 0.6), (0.5 * w, 2.0 * h, 0.6),
                   (0.5 * w, 0.5 * h, -0.6)]
    wl = make_workload("c2", n_bodies=len(centers), n_lines=n_lines, n_points=n_points, n_divides=n_divides, seed=seed,
                       rot_deg=rot_deg, trans_m=trans_m, color_intrinsics=ci, depth_intrinsics=di, centers_px=centers,
                       models=models)
    if modalities == "region32":
        wl.region.n_histogram_bins = 32
    wl.name = f"edge_{kind}_{modalities}"
    wl.notes.update(kind=kind, modalities=modalities, centers_px=centers)
    return wl
