"""Reader / writer of M3T's sparse-viewpoint-model .bin files (SURVEY §8 f2).

Format (M3T/src/model.cpp:218-322, region_model.cpp:259-363, depth_model.cpp:215-300; little-endian, x86-64):
    header : char type ('r' | 'd'), int32 version (10 | 9), float sphere_radius, int32 n_divides, int32 n_points,
             float max_radius_depth_offset, float stride_depth_offset, bool use_random_seed, int32 image_size
    body   : size_t path_len, path bytes, float geometry_unit_in_meter, bool counterclockwise, bool enable_culling,
             float maximum_body_diameter, float[16] geometry2body (Eigen column-major 4x4)
    region : size_t n_associated, then 4 x (size_t n, n body blocks)   [fixed, fixed-same-region, movable, movable-same-region]
    depth  : size_t n_occlusion_bodies, n body blocks
    views  : size_t n_views, n_views x ( n_points x DataPoint, float[3] orientation, float contour_length | surface_area )
DataPoint: region 38 floats (center_f_body[3], normal_f_body[3], foreground_distance, background_distance,
           depth_offsets[30]) = 152 B; depth 36 floats (center_f_body[3], normal_f_body[3], depth_offsets[30]) = 144 B.
The points are handed to m3tb_set_region_model / m3tb_set_depth_model exactly as stored (no renormalisation of the
8-bit-decoded depth-model normals, SURVEY App. A.6).
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field

import numpy as np

from .synth import DEPTH_POINT_FLOATS, REGION_POINT_FLOATS, Model


@dataclass
class BodyBlock:
    geometry_path: bytes
    geometry_unit_in_meter: float
    geometry_counterclockwise: bool
    geometry_enable_culling: bool
    maximum_body_diameter: float
    geometry2body: np.ndarray  # [4,4] float32 (row-major view of the stored column-major matrix)


@dataclass
class ModelFile:
    kind: str            # "region" | "depth"
    version: int
    sphere_radius: float
    n_divides: int
    n_points: int
    max_radius_depth_offset: float
    stride_depth_offset: float
    use_random_seed: bool
    image_size: int
    body: BodyBlock
    associated: list = field(default_factory=list)  # region: 4 lists of BodyBlock; depth: 1 list
    model: Model = None


class _Reader:
    def __init__(self, data):
        self.d, self.o = data, 0

    def take(self, fmt):
        v = struct.unpack_from("<" + fmt, self.d, self.o)
        self.o += struct.calcsize("<" + fmt)
        return v if len(v) > 1 else v[0]

    def raw(self, n):
        v = self.d[self.o:self.o + n]
        self.o += n
        return v


def _read_body(r: _Reader) -> BodyBlock:
    n = r.take("Q")
    path = bytes(r.raw(n))
    unit = r.take("f")
    ccw = bool(r.take("B"))
    cull = bool(r.take("B"))
    diam = r.take("f")
    m = np.frombuffer(r.raw(64), "<f4").reshape(4, 4).T.copy()  # stored column-major
    return BodyBlock(path, unit, ccw, cull, diam, m)


def read_model(path) -> ModelFile:
    data = memoryview(open(path, "rb").read())
    r = _Reader(data)
    kind_c = bytes(r.raw(1))
    if kind_c not in (b"r", b"d"):
        raise ValueError(f"{path}: not an M3T model file (type {kind_c!r})")
    kind = "region" if kind_c == b"r" else "depth"
    version = r.take("i")
    if version != (10 if kind == "region" else 9):
        raise ValueError(f"{path}: unsupported {kind} model version {version}")
    sphere_radius, n_divides, n_points = r.take("f"), r.take("i"), r.take("i")
    max_radius, stride = r.take("f"), r.take("f")
    use_random_seed = bool(r.take("B"))
    image_size = r.take("i")
    body = _read_body(r)
    associated = []
    if kind == "region":
        n_assoc = r.take("Q")
        total = 0
        for _ in range(4):
            n = r.take("Q")
            associated.append([_read_body(r) for _ in range(n)])
            total += n
        if total != n_assoc:
            raise ValueError(f"{path}: associated body count mismatch")
    else:
        n = r.take("Q")
        associated.append([_read_body(r) for _ in range(n)])
    n_views = r.take("Q")
    fl = REGION_POINT_FLOATS if kind == "region" else DEPTH_POINT_FLOATS
    rec = n_points * fl * 4 + 16
    if len(data) - r.o != n_views * rec:
        raise ValueError(f"{path}: view block size mismatch ({len(data) - r.o} != {n_views} x {rec})")
    views = np.frombuffer(r.raw(n_views * rec), np.uint8).reshape(n_views, rec)
    points = views[:, :n_points * fl * 4].copy().view("<f4").reshape(n_views, n_points, fl)
    tail = views[:, n_points * fl * 4:].copy().view("<f4").reshape(n_views, 4)
    model = Model(kind, np.ascontiguousarray(tail[:, :3]), np.ascontiguousarray(tail[:, 3]), points,
                  stride_depth_offset=stride, max_radius_depth_offset=max_radius)
    return ModelFile(kind, version, sphere_radius, n_divides, n_points, max_radius, stride, use_random_seed, image_size,
                     body, associated, model)


def _write_body(b: BodyBlock) -> bytes:
    return (struct.pack("<Q", len(b.geometry_path)) + b.geometry_path +
            struct.pack("<fBBf", b.geometry_unit_in_meter, b.geometry_counterclockwise, b.geometry_enable_culling,
                        b.maximum_body_diameter) + np.ascontiguousarray(b.geometry2body.T, "<f4").tobytes())


def write_model(path, mf: ModelFile):
    m = mf.model
    out = [b"r" if mf.kind == "region" else b"d",
           struct.pack("<ifiiffBi", mf.version, mf.sphere_radius, mf.n_divides, mf.n_points,
                       mf.max_radius_depth_offset, mf.stride_depth_offset, mf.use_random_seed, mf.image_size),
           _write_body(mf.body)]
    if mf.kind == "region":
        out.append(struct.pack("<Q", sum(len(g) for g in mf.associated)))
        for g in (mf.associated + [[], [], [], []])[:4]:
            out.append(struct.pack("<Q", len(g)))
            out.extend(_write_body(b) for b in g)
    else:
        g = mf.associated[0] if mf.associated else []
        out.append(struct.pack("<Q", len(g)))
        out.extend(_write_body(b) for b in g)
    out.append(struct.pack("<Q", m.n_views))
    tail = np.concatenate([m.orientations, m.view_scalars[:, None]], 1).astype("<f4")
    for v in range(m.n_views):
        out.append(np.ascontiguousarray(m.points[v], "<f4").tobytes())
        out.append(tail[v].tobytes())
    with open(path, "wb") as f:
        f.write(b"".join(out))


def model_from_synthetic(model: Model, n_divides=4, sphere_radius=0.8, geometry_path=b"triangle.obj") -> ModelFile:
    """Wrap an analytic model (synth.generate_*_model) so that it can be saved in the reference's format."""
    g2b = np.eye(4, dtype=np.float32)
    g2b[2, 3] = -0.006
    body = BodyBlock(geometry_path, 1.0, True, True, 0.0782, g2b)
    kind = model.kind
    return ModelFile(kind, 10 if kind == "region" else 9, sphere_radius, n_divides, model.n_points,
                     model.max_radius_depth_offset, model.stride_depth_offset, False, 2000, body,
                     [[], [], [], []] if kind == "region" else [[]], model)


def model_from_generated(model: Model, params, body: BodyBlock, occlusion_bodies=()) -> ModelFile:
    """Wrap a model read back from the device (capi.Context.get_depth_model / get_region_model) with the parameters it
    was generated with (capi.ModelParams) and the caller's body blocks, so that write_model saves it in the
    reference's format (DepthModel::SaveModel, depth_model.cpp:265-291; RegionModel::SaveModel,
    region_model.cpp:309-345). occlusion_bodies: the depth model's occlusion body blocks, or for a region model the
    four associated groups (fixed, fixed same-region, movable, movable same-region), each in insertion order."""
    if model.kind == "depth":
        return ModelFile("depth", 9, params.sphere_radius, params.n_divides, model.n_points,
                         params.max_radius_depth_offset, params.stride_depth_offset, bool(params.use_random_seed),
                         params.image_size, body, [list(occlusion_bodies)], model)
    groups = [list(g) for g in occlusion_bodies] if len(occlusion_bodies) else [[], [], [], []]
    if len(groups) != 4:
        raise ValueError("a region model has four associated-body groups")
    return ModelFile("region", 10, params.sphere_radius, params.n_divides, model.n_points,
                     params.max_radius_depth_offset, params.stride_depth_offset, bool(params.use_random_seed),
                     params.image_size, body, groups, model)
