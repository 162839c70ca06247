"""CPU restatement of depth-model generation (DESIGN.md §3 "k_model_raster / k_model_points"), operation for
operation in float32 like the kernels built with -fmad=false, so that views, points, surface areas and the debug images
are compared bit for bit. Rasterisation goes through render_reference.raster_keyed; the sampler replays
std::mt19937{7} with numpy's RandomState(7), as tests/golden/reference_rig.py does. Test infrastructure only."""
import ctypes
import ctypes.util

import numpy as np

import render_reference as rr

f32 = np.float32
CLEAR = np.uint64(0xFFFFFFFFFFFFFFFF)
IMAGE_SIZE_SAFETY_BOUNDARY = 20
MAX_OFFSETS = 30

_libm = ctypes.CDLL(ctypes.util.find_library("m"))
for _n in ("asinf", "tanf"):
    getattr(_libm, _n).restype = ctypes.c_float
    getattr(_libm, _n).argtypes = [ctypes.c_float]


def _libm_f(name, x):
    """The C library's float function, as the host code calls it."""
    return f32(getattr(_libm, name)(float(f32(x))))


def _normalized(v):
    n = v[0] * v[0] + v[1] * v[1] + v[2] * v[2]
    if not n > 0:
        return v
    s = np.sqrt(n)
    return np.array([v[0] / s, v[1] / s, v[2] / s], f32)


def _cross(a, b):
    return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]], f32)


def geodesic_poses(n_divides, sphere_radius):
    """Model::GenerateGeodesicPoints / GenerateGeodesicPoses: camera2body [n,3,4] float32 in std::set order."""
    x, z, o = f32(0.525731112119133606), f32(0.850650808352039932), f32(0)
    ico = [(-x, o, z), (x, o, z), (-x, o, -z), (x, o, -z), (o, z, x), (o, z, -x), (o, -z, x), (o, -z, -x), (z, x, o),
           (-z, x, o), (z, -x, o), (-z, -x, o)]
    ids = [(0, 4, 1), (0, 9, 4), (9, 5, 4), (4, 5, 8), (4, 8, 1), (8, 10, 1), (8, 3, 10), (5, 3, 8), (5, 2, 3), (2, 7, 3),
           (7, 10, 3), (7, 6, 10), (7, 11, 6), (11, 0, 6), (0, 1, 6), (6, 1, 10), (9, 0, 11), (9, 11, 2), (9, 2, 5),
           (7, 2, 11)]
    pts = {}  # insertion order kept; equal vectors (== on floats) are inserted once, as in std::set

    def sub(v1, v2, v3, n):
        if n == 0:
            for v in (v1, v2, v3):
                pts.setdefault(tuple(float(c) for c in v), v)
            return
        v12, v13, v23 = _normalized(v1 + v2), _normalized(v1 + v3), _normalized(v2 + v3)
        sub(v1, v12, v13, n - 1); sub(v2, v12, v23, n - 1); sub(v3, v13, v23, n - 1); sub(v12, v13, v23, n - 1)

    for a, b, c in ids:
        sub(np.array(ico[a], f32), np.array(ico[b], f32), np.array(ico[c], f32), n_divides)
    r = f32(sphere_radius)
    poses = []
    for key in sorted(pts):
        p = pts[key]
        c2 = -p
        c0 = np.array([1, 0, 0], f32) if (p[0] == 0 and p[2] == 0) else _normalized(_cross(np.array([0, 1, 0], f32), c2))
        c1 = _cross(c2, c0)
        poses.append(np.stack([c0, c1, c2, p * r], 1))
    return np.array(poses, f32)


def pose_inverse(p):
    """m3tb::PoseInverse (Transform3fA::inverse, 3x3 cofactor inverse) on float32 [3,4]."""
    p = np.asarray(p, f32).reshape(12)
    m = [p[0], p[1], p[2], p[4], p[5], p[6], p[8], p[9], p[10]]

    def cof(i, j):
        return (m[3 * ((i + 1) % 3) + (j + 1) % 3] * m[3 * ((i + 2) % 3) + (j + 2) % 3] -
                m[3 * ((i + 1) % 3) + (j + 2) % 3] * m[3 * ((i + 2) % 3) + (j + 1) % 3])
    c00, c10, c20 = cof(0, 0), cof(1, 0), cof(2, 0)
    det = c00 * m[0] + c10 * m[3] + c20 * m[6]
    invdet = f32(1) / det
    inv = [c00 * invdet, c10 * invdet, c20 * invdet, cof(0, 1) * invdet, cof(1, 1) * invdet, cof(2, 1) * invdet,
           cof(0, 2) * invdet, cof(1, 2) * invdet, cof(2, 2) * invdet]
    o = np.zeros(12, f32)
    for i in range(3):
        o[4 * i:4 * i + 3] = inv[3 * i:3 * i + 3]
        o[4 * i + 3] = (-inv[3 * i]) * p[3] + (-inv[3 * i + 1]) * p[7] + (-inv[3 * i + 2]) * p[11]
    return o


def face_normals(triangles):
    """(p2 - p1).cross(p0 - p1).normalized() per triangle (RendererGeometry::AssembleVertexData)."""
    t = np.asarray(triangles, f32).reshape(-1, 3, 3)
    out = np.zeros((t.shape[0], 3), f32)
    for k in range(t.shape[0]):
        out[k] = _normalized(_cross(t[k, 2] - t[k, 1], t[k, 0] - t[k, 1]))
    return out


class Setup:
    """Model::SetUpRenderer / AddBodiesToRenderer for a body and its occlusion bodies (rr.Geometry each)."""

    def __init__(self, body, occlusion, sphere_radius, image_size):
        self.body, self.occlusion = body, list(occlusion)
        r = f32(sphere_radius)
        self.r, self.S = r, int(image_size)
        rad = HALF_D(body)
        self.z_min, self.z_max = r - rad, r + rad
        zo_min, zo_max = self.z_min, self.z_max
        for g in self.occlusion:
            lo, hi = r - HALF_D(g), r + HALF_D(g)
            zo_min, zo_max = min(lo, zo_min), max(hi, zo_max)
        self.zo_min, self.zo_max = zo_min, zo_max
        self.fu = f32(0.5) * f32(self.S - IMAGE_SIZE_SAFETY_BOUNDARY) / _libm_f("tanf", _libm_f("asinf", rad / r))
        self.pp = f32(self.S) / f32(2)
        a, b = self.z_max, self.z_min
        self.projection_term_a = a * b * f32(65535) / (a - b)
        self.projection_term_b = a * f32(65535) / (a - b)
        self.normals = face_normals(body.triangles)

    def matrices(self, camera2body):
        """Per drawn body of both renderers: M = P * world2camera * geometry2world (16 float32), and the main body's
        rotation block."""
        fS = f32(self.S)
        P00 = f32(2) * self.fu / fS
        P02 = f32(2) * (self.pp + f32(0.5)) / fS - f32(1)
        w2c = pose_inverse(camera2body)
        out = []
        for pr, (lo, hi), bodies in ((0, (self.z_min, self.z_max), [self.body]),
                                     (1, (self.zo_min, self.zo_max), [self.body] + self.occlusion)):
            P22 = (hi + lo) / (hi - lo)
            P23 = f32(-2) * hi * lo / (hi - lo)
            Ms = []
            for g in bodies:
                T = rr.pose_mul(w2c, g.geometry2body)
                M = np.zeros(16, f32)
                for c in range(4):
                    M[c] = P00 * T[c] + P02 * T[8 + c]
                    M[4 + c] = P00 * T[4 + c] + P02 * T[8 + c]
                    M[8 + c] = P22 * T[8 + c]
                    M[12 + c] = T[8 + c]
                M[11] = M[11] + P23
                Ms.append(M)
                if pr == 0:
                    rot = T.reshape(3, 4)[:, :3].copy()
            out.append(Ms)
        return out, rot


def HALF_D(g):
    return f32(0.5) * f32(g.maximum_body_diameter)


def raster(M, triangles, culling, S, draw, zbuf, stats=None):
    """Every triangle of one body through M into zbuf [S,S] uint64 (depth16 << 48 | draw << 32 | triangle):
    rr.raster_keyed, whose `stats` count what it reaches."""
    rr.raster_keyed(M, triangles, culling, S, S, draw, zbuf, stats)


def _unorm8(c):
    return np.rint(np.fmin(np.fmax(c, f32(0)), f32(1)) * f32(255)).astype(np.uint8)


def render_view(st: Setup, camera2body, stats=None):
    """The two z-buffers of one view and its normal (BGRA), depth and silhouette images (stats: see rr.raster_keyed)."""
    S = st.S
    Ms, rot = st.matrices(camera2body)
    z0 = np.full((S, S), CLEAR, np.uint64)
    raster(Ms[0][0], st.body.triangles, st.body.enable_culling, S, 0, z0, stats)
    if st.occlusion:
        zs = np.full((S, S), CLEAR, np.uint64)
        for g, G in enumerate([st.body] + st.occlusion):
            raster(Ms[1][g], G.triangles, G.enable_culling, S, g, zs, stats)
        sil = (zs != CLEAR) & (((zs >> np.uint64(32)) & np.uint64(0xFFFF)) == 0)
    else:
        sil = z0 != CLEAR
    covered = z0 != CLEAR
    tri = (z0 & np.uint64(0xFFFFFFFF)).astype(np.int64)
    n = st.normals[np.where(covered, tri, 0)]
    normal = np.zeros((S, S, 4), np.uint8)
    for r in range(3):
        nc = rot[r, 0] * n[..., 0] + rot[r, 1] * n[..., 1] + rot[r, 2] * n[..., 2]
        normal[..., r] = np.where(covered, _unorm8(f32(0.5) - f32(0.5) * nc), 0)
    normal[..., 3] = np.where(covered, 255, 0)
    depth = (z0 >> np.uint64(48)).astype(np.uint16)
    return dict(normal=normal, depth=depth, silhouette=np.where(sil, 255, 0).astype(np.uint8))


def mt19937_stream(seed=7):
    rs = np.random.RandomState(seed)  # std::mt19937 generator{seed}
    while True:
        for v in rs.randint(0, 2 ** 32, size=64, dtype=np.uint64):
            yield int(v)


def view_points(st: Setup, camera2body, images, n_points, stride_depth_offset, max_radius_depth_offset, seed=7):
    """DepthModel::GeneratePointData + Model::CalculateDepthOffsets for one view -> ([n_points,36] f32, area)."""
    S = st.S
    sil, depth, normal = images["silhouette"], images["depth"], images["normal"]
    px = st.r / st.fu
    area = f32(np.count_nonzero(sil)) * (px * px)
    out = np.zeros((n_points, 36), f32)
    if area == 0:
        return out, area
    n_pix = S * S
    gen = mt19937_stream(seed)
    coords = []
    while len(coords) < n_points:
        idx = next(gen) % n_pix
        x, y = idx // S, idx % S
        if sil[y, x]:
            coords.append((x, y))
    T = np.asarray(camera2body, f32).reshape(3, 4)
    a, b = st.projection_term_a, st.projection_term_b
    stride_m = f32(stride_depth_offset)
    n_values = int(f32(max_radius_depth_offset) / stride_m + f32(1))
    for k, (x, y) in enumerate(coords):
        d16c = depth[y, x]
        dep = a / (b - f32(d16c))
        c = (dep * (f32(x) - st.pp) / st.fu, dep * (f32(y) - st.pp) / st.fu, dep)
        nb = normal[y, x]
        nv = [f32(1) - f32(nb[r]) / f32(127.5) for r in range(3)]
        for r in range(3):
            out[k, r] = T[r, 0] * c[0] + T[r, 1] * c[1] + T[r, 2] * c[2] + T[r, 3]
            out[k, 3 + r] = T[r, 0] * nv[0] + T[r, 1] * nv[1] + T[r, 2] * nv[2]
        out[k, 6:] = depth_offsets(depth, x, y, c[2] / st.fu, stride_m, n_values, a, b)
    return out, area


def depth_offsets(depth, x, y, pixel_to_meter, stride_depth_offset, n_values, a, b, sqrt=np.sqrt):
    """Model::CalculateDepthOffsets. `sqrt` takes the integer squared distance; the reference's std::sqrt(int) works
    in double, the result is stored as a float."""
    S = depth.shape[0]
    stride = f32(stride_depth_offset) / f32(pixel_to_meter)
    max_diameter = f32(2) * f32(n_values) * stride
    image_stride = int(stride + f32(1))
    n_image_strides = int(max_diameter / f32(image_stride) + f32(1))
    image_diameter = n_image_strides * image_stride
    rm = image_diameter // 2
    rp = image_diameter - rm
    v_min, v_max = max(y - rm, 0), min(y + rp, S - 1)
    u_min, u_max = max(x - rm, 0), min(x + rp, S - 1)
    mins = np.full(MAX_OFFSETS, 0xFFFF, np.int64)
    mins[0] = depth[y, x]
    vv, uu = np.meshgrid(np.arange(v_min, v_max + 1, image_stride), np.arange(u_min, u_max + 1, image_stride),
                         indexing="ij")
    dist = sqrt(((uu - x) ** 2 + (vv - y) ** 2).astype(np.float64)).astype(f32)
    i = (dist / stride).astype(np.int64)  # float quotient, truncated (non-negative)
    sel = i < n_values
    np.minimum.at(mins, i[sel], depth[vv[sel], uu[sel]].astype(np.int64))
    dc = a / (b - f32(depth[y, x]))
    out = np.zeros(MAX_OFFSETS, f32)
    m = mins[0]
    out[0] = dc - a / (b - f32(m))
    for i in range(1, MAX_OFFSETS):
        m = min(mins[i], m)
        out[i] = dc - a / (b - f32(m))
    return out


def generate(body, occlusion, sphere_radius=0.8, n_divides=4, n_points=200, max_radius_depth_offset=0.05,
             stride_depth_offset=0.002, image_size=2000, views=None):
    """The whole model: (camera2body [nv,3,4], orientations [nv,3], areas [nv], points [nv,n_points,36]). `views`
    restricts it to some view indices."""
    st = Setup(body, occlusion, sphere_radius, image_size)
    poses = geodesic_poses(n_divides, sphere_radius)
    sel = range(poses.shape[0]) if views is None else views
    pts, areas = [], []
    for v in sel:
        img = render_view(st, poses[v])
        p, a = view_points(st, poses[v], img, n_points, stride_depth_offset, max_radius_depth_offset)
        pts.append(p)
        areas.append(a)
    return poses, poses[:, :, 2].copy(), np.array(areas, f32), np.array(pts, f32).reshape(len(areas), n_points, 36)
