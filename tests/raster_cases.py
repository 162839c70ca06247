"""Adversarial scenes for the device rasterisers and the region contour tracer, shared by the CPU checks
(test_raster_cases.py) and the device comparisons (test_gpu_raster_sweep.py, test_gpu_model_generation_masks.py).

Camera-image scenes use an intrinsics with fu = W / 2, ppu = W / 2 - 0.5 (same for v), so that with identity poses the
full projection has P00 = P11 = 1 and P02 = P12 = 0 exactly and x_w = (X / Z + 1) * W / 2: dyadic X at Z = 1 or 2 put
vertices on pixel centres and edges exactly through them. z_min = 1, z_max = 3 give P22 = 2 and P23 = -3, so a vertex
at Z = 1 has dist = z + w == 0 exactly. Each scene names the reach counters of render_reference (rr.fragments,
rr.clip_polygon, rr.raster_keyed) it is built to reach.

mask_mesh builds a body whose main silhouette at one geodesic view of model generation is a given mask. Test
infrastructure only."""
from dataclasses import dataclass, field
from types import SimpleNamespace

import numpy as np

import model_generation_reference as mg
import region_model_generation_reference as rg
import render_reference as rr

f32 = np.float32
I34 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(f32)
EXACT_Z = (1.0, 3.0)  # z_min, z_max of the exact projection


def exact_intrinsics(W, H):
    return SimpleNamespace(fu=W / 2, fv=H / 2, ppu=W / 2 - 0.5, ppv=H / 2 - 0.5, width=W, height=H)


@dataclass
class Scene:
    name: str
    geometry: dict                     # body -> rr.Geometry
    bodies: list                       # draw order
    z_range: tuple = EXACT_Z
    reaches: tuple = ()                # reach counters the scene must reach at its own size
    size: tuple = (64, 64)
    poses: dict = field(default_factory=dict)

    def pose_map(self):
        return {b: self.poses.get(b, I34) for b in self.geometry}


def _geometry(tri, culling, body_id=1, region_id=1):
    tri = np.ascontiguousarray(tri, f32).reshape(-1, 3, 3)
    v = tri.reshape(-1, 3).astype(np.float64)
    v = v[np.isfinite(v).all(1)]
    diam = float(f32(2.0 * np.linalg.norm(v, axis=1).max())) if len(v) else 1.0
    return rr.Geometry(tri, I34.copy(), diam, culling, body_id, region_id)


def _at(W, H, x, y, Z):
    """Camera-frame point whose window position is (x, y) at depth Z under exact_intrinsics(W, H)."""
    return (Z * (2.0 * x / W - 1.0), Z * (2.0 * y / H - 1.0), Z)


def _grid(W, H, step, Z, x_lo, x_hi, y_lo, y_hi):
    """Cells of a pixel-centre grid, each split into two triangles, the diagonal direction alternating."""
    xs = np.arange(x_lo, x_hi + 1, step) + 0.5
    ys = np.arange(y_lo, y_hi + 1, step) + 0.5
    tri = []
    for a in range(len(ys) - 1):
        for b in range(len(xs) - 1):
            p00, p10 = _at(W, H, xs[b], ys[a], Z), _at(W, H, xs[b + 1], ys[a], Z)
            p01, p11 = _at(W, H, xs[b], ys[a + 1], Z), _at(W, H, xs[b + 1], ys[a + 1], Z)
            tri += [(p00, p10, p11), (p00, p11, p01)] if (a + b) % 2 == 0 else [(p00, p10, p01), (p10, p11, p01)]
    return np.array(tri, f32)


def _fan(W, H, cx, cy, r, Z):
    """Triangles around the pixel centre (cx + 0.5, cy + 0.5) to a square ring of pixel centres at distance r, both
    windings alternating."""
    ring = [(cx + dx, cy - r) for dx in range(-r, r)] + [(cx + r, cy + dy) for dy in range(-r, r)] + \
           [(cx - dx, cy + r) for dx in range(-r, r)] + [(cx - r, cy - dy) for dy in range(-r, r)]
    c = _at(W, H, cx + 0.5, cy + 0.5, Z)
    tri = []
    for k in range(len(ring)):
        a, b = ring[k], ring[(k + 1) % len(ring)]
        pa, pb = _at(W, H, a[0] + 0.5, a[1] + 0.5, Z), _at(W, H, b[0] + 0.5, b[1] + 0.5, Z)
        tri.append((c, pa, pb) if k % 2 == 0 else (c, pb, pa))
    return np.array(tri, f32)


def _both_windings(tri):
    tri = np.asarray(tri, f32)
    return np.concatenate([tri, tri[:, ::-1]])


def tie_scenes(W=64, H=64):
    """Exact-tie scenes: a tessellated grid over and beyond the image (every pixel covered exactly once, horizontal and
    vertical edges on centre rows and columns, diagonals through centres), and a fan around a pixel centre."""
    step = max(4, min(W, H) // 8)
    grid = _grid(W, H, step, 2.0, -6, W + step + 1, -6, H + step + 1)
    fan = _fan(W, H, W // 2, H // 2, 6, 2.0)
    return [
        Scene("grid", {0: _geometry(grid, False, 3, 4)}, [0],
              reaches=("tie_owned", "tie_not_owned", "box_lo_x", "box_hi_x", "box_lo_y", "box_hi_y"), size=(W, H)),
        Scene("fan", {0: _geometry(fan, False, 5, 6)}, [0], reaches=("tie_owned", "tie_not_owned"), size=(W, H)),
    ]


def _near_triangles(W, H):
    """Triangles against the near plane z = 1 (dist = 3 Z - 3) in every inside / outside vertex pattern, with vertices
    exactly on it, partly behind the camera (Z < 0) and cut by the far plane z = 3."""
    def t(*pts):
        return [_at(W, H, x, y, Z) for x, y, Z in pts]
    return np.array([
        t((10.5, 8.5, 2.0), (30.5, 8.5, 2.0), (20.5, 30.5, 2.0)),       # in, in, in
        t((40.5, 4.5, 0.5), (60.5, 20.5, 2.0), (34.5, 40.5, 2.0)),      # one outside: a quad
        t((4.5, 30.5, 0.5), (24.5, 44.5, 0.5), (8.5, 46.5, 2.0)),       # two outside
        t((5.5, 5.5, 0.5), (9.5, 5.5, 0.5), (5.5, 9.5, 0.5)),           # all outside
        t((20.5, 20.5, 1.0), (44.5, 12.5, 2.0), (36.5, 36.5, 2.0)),     # one on the plane
        t((12.5, 22.5, 1.0), (2.5, 40.5, 0.5), (26.5, 42.5, 2.0)),      # on the plane, outside, inside
        t((30.5, 2.5, 1.0), (50.5, 2.5, 1.0), (40.5, 18.5, 2.0)),       # two on the plane
        t((16.5, 16.5, -1.0), (48.5, 30.5, 2.0), (20.5, 44.5, 2.0)),    # one behind the camera
        t((2.5, 2.5, 2.0), (62.5, 10.5, 4.0), (30.5, 46.5, 2.5)),       # cut by the far plane
    ], f32)


def near_scenes(W=64, H=64):
    tri = _both_windings(_near_triangles(W, H))
    return [
        Scene("near_culled", {0: _geometry(tri, True, 7, 8)}, [0],
              reaches=("clip_in_in", "clip_in_out", "clip_out_in", "clip_out_out", "dist_zero", "fan4",
                       "far_reject"), size=(W, H)),
        Scene("near_unculled", {0: _geometry(tri, False, 9, 10)}, [0],
              reaches=("clip_in_out", "clip_out_in", "dist_zero", "fan4", "far_reject"), size=(W, H)),
    ]


def nan_edge_scene(W=64, H=64):
    """z_min = 1e-30: triangles crossing the near plane put a vertex at w of about 1e-30, window coordinates about
    1e30, and the edge products overflow to NaN."""
    tri = np.array([[(-0.3, -0.2, 0.5), (0.4, -0.1, 0.6), (0.1, 0.3, -0.4)],
                    [(-0.2, 0.1, -0.3), (0.3, 0.2, 0.7), (-0.1, -0.3, 0.8)],
                    [(0.05, 0.05, 1e-31), (0.3, -0.2, 0.9), (-0.25, 0.2, 0.9)]], f32)
    return Scene("nan_edges", {0: _geometry(_both_windings(tri), False, 11, 12)}, [0], z_range=(1e-30, 10.0),
                 reaches=("nan_edge", "fan4"), size=(W, H))


def tie_depth_scenes(W=64, H=64):
    """Coplanar overlapping triangles inside one body (ties broken by triangle index) and the same body drawn twice
    (ties broken by draw index)."""
    a = [_at(W, H, x, y, 2.0) for x, y in ((6.3, 5.1), (50.7, 9.9), (20.2, 41.6))]
    b = [_at(W, H, x, y, 2.0) for x, y in ((10.1, 30.3), (58.6, 3.4), (44.9, 44.2))]
    c = [_at(W, H, x, y, 2.0) for x, y in ((3.3, 20.7), (61.1, 24.9), (30.0, 2.2))]
    tri = np.array([a, b, c, a[::-1], b[::-1]], f32)
    g0, g1 = _geometry(tri, False, 13, 14), _geometry(tri, False, 15, 16)
    return [Scene("coplanar", {0: g0}, [0], reaches=("triangle_tie",), size=(W, H)),
            Scene("two_draws", {0: g0, 1: g1}, [1, 0], reaches=("triangle_tie", "draw_tie"), size=(W, H))]


def degenerate_scene(W=64, H=64):
    """Zero-area, collinear, sliver, NaN and inf vertices, both windings, culling on and off, and triangles much larger
    than the image."""
    P = [_at(W, H, x, y, 2.0) for x, y in ((10.5, 10.5), (30.5, 10.5), (50.5, 10.5), (10.5, 30.5))]
    nan, inf = float("nan"), float("inf")
    tri = np.array([
        [P[0], P[0], P[1]],                                    # zero area (a repeated vertex)
        [P[0], P[1], P[2]],                                    # collinear
        [P[0], P[2], _at(W, H, 30.5, 10.5001, 2.0)],           # sliver
        [P[0], (nan, 0.0, 2.0), P[3]],
        [P[0], (inf, 0.0, 2.0), P[3]],
        [(0.0, 0.0, inf), P[1], P[3]],
        [(-inf, -inf, 2.0), P[2], P[3]],
        [_at(W, H, -900, -700, 2.0), _at(W, H, 1500, -600, 2.0), _at(W, H, 300, 1900, 2.0)],   # much larger
        [P[1], P[2], P[3]],
    ], f32)
    return [Scene("degenerate_culled", {0: _geometry(_both_windings(tri), True, 17, 18)}, [0],
                  reaches=("box_lo_x", "box_hi_y"), size=(W, H)),
            Scene("degenerate_unculled", {0: _geometry(_both_windings(tri), False, 19, 20)}, [0],
                  reaches=("box_lo_x", "box_hi_y"), size=(W, H))]


def tile_scene(W=64, H=64):
    """Triangles whose pixel boxes end exactly on 32-pixel tile edges and span several tiles."""
    tri = np.array([[_at(W, H, x, y, 2.0) for x, y in pts] for pts in (
        ((0.5, 0.5), (31.5, 0.5), (0.5, 31.5)),        # box [0, 32) x [0, 32): one tile, ends on its edge
        ((31.5, 31.5), (32.5, 31.5), (31.5, 32.5)),
        ((32.2, 0.7), (63.9, 0.7), (32.2, 31.9)),      # box [32, 64) x [0, 32)
        ((0.7, 33.0), (63.6, 40.0), (10.0, 47.9)),     # over two tiles in x
    )], f32)
    return Scene("tiles", {0: _geometry(_both_windings(tri), True, 21, 22)}, [0],
                 reaches=("tile_end", "multi_tile"), size=(W, H))


def near_plane_fans(W=640, H=480, n=40, seed=1):
    """Large triangles with one vertex exactly on the near plane (Z = 1) and the others at non-dyadic positions, in
    front of it or behind it: the polygon ClipTriangle builds from a vertex with dist == 0 decides the fan order, and
    with it the rounding of every fragment's depth."""
    rng = np.random.default_rng(seed)
    tri = []
    for k in range(n):
        p0 = _at(W, H, rng.uniform(0, W), rng.uniform(0, H), 1.0)
        z1, z2 = rng.uniform(1.1, 2.9), (rng.uniform(1.1, 2.9) if k % 2 else rng.uniform(0.3, 0.9))
        p1 = _at(W, H, rng.uniform(-W, 2 * W), rng.uniform(-H, 2 * H), z1)
        p2 = _at(W, H, rng.uniform(-W, 2 * W), rng.uniform(-H, 2 * H), z2)
        tri.append((p0, p1, p2) if k % 4 < 2 else (p1, p2, p0))
    return Scene("near_plane_fans", {0: _geometry(np.array(tri, f32), False, 23, 24)}, [0],
                 reaches=("dist_zero", "fan4", "clip_out_in", "clip_in_out"), size=(W, H))


def camera_scenes(W=64, H=64):
    """Every camera-image scene at W x H, and the near-plane fans at their own size."""
    return (tie_scenes(W, H) + near_scenes(W, H) + [nan_edge_scene(W, H)] + tie_depth_scenes(W, H) +
            degenerate_scene(W, H) + [tile_scene(W, H), near_plane_fans()])


# image sizes that are not multiples of the 32-pixel tile, and frames 1 pixel wide or high
ODD_SIZES = [(1, 1), (1, 333), (333, 1), (31, 33), (1280, 720)]
FOCUSED_SIZES = [1, 31, 32, 33, 240]


def sized_scenes(W, H):
    """The scenes that make sense at any size: the grid and the fan stretched over the frame, the near-plane and
    degenerate triangles."""
    return [tie_scenes(W, H)[0]] + near_scenes(W, H)[:1] + degenerate_scene(W, H)[1:]


def render_camera(scene, stats=None, z_range=None):
    """fr.render_full of a scene at its size with the exact intrinsics, body ids."""
    import full_renderer_reference as fr
    W, H = scene.size
    z0, z1 = z_range or scene.z_range
    return fr.render_full(exact_intrinsics(W, H), I34, scene.pose_map(), scene.geometry, scene.bodies, z0, z1, "body",
                          stats)


# ---- focused renderers (k_render) -----------------------------------------------------------------------------------

def focused_scene(n_bodies, seed):
    """n_bodies tetrahedra around (0, 0, 0.5) with random poses, some crossing the near plane z = 0.3 and
    some far beyond the image, for k_render's shared-memory z-buffer; ids repeat, so that silhouettes tie."""
    rng = np.random.default_rng(seed)
    base = np.array([[0.02, 0, 0], [-0.01, 0.017, 0], [-0.01, -0.017, 0], [0, 0, 0.03]], f32)
    faces = [(0, 2, 1), (0, 1, 3), (1, 2, 3), (2, 0, 3)]
    geometry, poses = {}, {}
    for b in range(n_bodies):
        s = rng.uniform(0.5, 4.0)
        tri = (base * s)[np.array(faces)]
        geometry[b] = rr.Geometry(np.ascontiguousarray(tri, f32), I34.copy(), float(f32(0.08 * s)), b % 3 != 0,
                                  b % 255 + 1, b % 5 + 1)
        ang = rng.uniform(-np.pi, np.pi, 3)
        R = _rot(ang)
        t = (rng.uniform(-0.15, 0.15), rng.uniform(-0.15, 0.15), rng.uniform(0.25, 0.9))
        poses[b] = np.hstack([R, np.array(t)[:, None]]).astype(f32)
    return geometry, poses


def _rot(ang):
    R = np.eye(3)
    for axis, a in enumerate(ang):
        i, j = [k for k in range(3) if k != axis]
        Q = np.eye(3)
        Q[i, i], Q[i, j], Q[j, i], Q[j, j] = np.cos(a), -np.sin(a), np.sin(a), np.cos(a)
        R = R @ Q
    return R


# ---- masks through model generation ---------------------------------------------------------------------------------

MASK_DIAMETER = 0.2  # fixes the pixel size; quads beyond the body's sphere are clipped in the other views
MASK_INSET = 0.25    # px: quads end this far inside the pixel borders, so each covers exactly its run's centres


def mask_fu(image_size, sphere_radius=0.8):
    return mg.Setup(rr.Geometry(np.zeros((1, 3, 3), f32), I34, MASK_DIAMETER, False), [], sphere_radius,
                    image_size).fu


def mask_mesh(mask, view, n_divides=0, sphere_radius=0.8):
    """A body (culling off) whose main silhouette at geodesic view `view` of model generation is `mask` [S,S]: one quad
    per horizontal run of mask pixels in the plane through the body origin perpendicular to the view axis, inset from
    the pixel borders by MASK_INSET. Pixel (i, j) is seen at x_c / z_c * fu + pp = i (and j), z_c = sphere_radius."""
    mask = np.asarray(mask) != 0
    S = mask.shape[0]
    fu, pp = float(mask_fu(S, sphere_radius)), S / 2.0
    pose = mg.geodesic_poses(n_divides, sphere_radius)[view].astype(np.float64)
    c0, c1 = pose[:, 0], pose[:, 1]
    r = float(f32(sphere_radius))

    def vertex(u, v):
        return c0 * ((u - pp) * r / fu) + c1 * ((v - pp) * r / fu)

    tri = []
    for j in range(S):
        row = np.concatenate([[False], mask[j], [False]])
        d = np.diff(row.astype(np.int8))
        for i0, i1 in zip(np.nonzero(d == 1)[0], np.nonzero(d == -1)[0] - 1):
            lo, hi = i0 - 0.5 + MASK_INSET, i1 + 0.5 - MASK_INSET
            a, b = vertex(lo, j - 0.5 + MASK_INSET), vertex(hi, j - 0.5 + MASK_INSET)
            c, e = vertex(hi, j + 0.5 - MASK_INSET), vertex(lo, j + 0.5 - MASK_INSET)
            tri += [(a, b, c), (a, c, e)]
    if not tri:
        tri = [(vertex(0, 0), vertex(0, 0), vertex(0, 0))]
    return rr.Geometry(np.ascontiguousarray(tri, f32), I34.copy(), MASK_DIAMETER, False)


def _put(mask, shape, x, y):
    h, w = shape.shape
    mask[y:y + h, x:x + w] |= shape.astype(bool)


def contour_blob(n_points, seed=0, box=6):
    """A small 8-connected blob without holes whose single outer contour has exactly n_points points (found by a
    seeded search)."""
    rng = np.random.default_rng(seed)
    for _ in range(200000):
        m = rng.random((box, box)) < rng.uniform(0.3, 0.8)
        pad = np.zeros((box + 2, box + 2), bool)
        pad[1:-1, 1:-1] = m
        cs = rg.find_contours(pad)
        if len(cs) == 1 and len(cs[0]) == n_points:
            return pad
    raise RuntimeError(n_points)


def _line(direction, length):
    dx, dy = direction
    m = np.zeros((length * abs(dy) + 1 if dy else 1, length * abs(dx) + 1 if dx else 1), bool)
    for k in range(length + 1):
        m[k * abs(dy) if dy else 0, k * abs(dx) if dx else 0] = True
    if dx * dy < 0:
        m = m[:, ::-1]
    return m


def _nested(levels):
    n = 4 * levels + 1
    m = np.zeros((n, n), bool)
    for k in range(levels):
        o = 2 * k
        m[o:n - o, o:n - o] = True
        if n - 2 * o - 2 > 0:
            m[o + 1:n - o - 1, o + 1:n - o - 1] = False
    return m


def contour_masks(S):
    """Engineered silhouettes of an S x S generation image (S >= 21): name -> mask."""
    out = {}
    m = np.zeros((S, S), bool)
    for k in range(min(6, S // 4)):
        m[2 + 3 * k, 2 + (5 * k) % (S - 4)] = True
    m[S // 2 - 3:S // 2 + 4, S // 2 - 3:S // 2 + 4] = True
    out["single_pixels"] = m
    m = np.zeros((S, S), bool)
    for k, n in enumerate((14, 15, 16)):
        _put(m, contour_blob(n, seed=n), 1 + 10 * (k % 2), 1 + 10 * (k // 2))
    out["lengths_14_15_16"] = m
    m = np.zeros((S, S), bool)
    L = max(3, min(7, (S - 8) // 6))
    for k, d in enumerate(((1, 0), (1, 1), (0, 1), (-1, 1))):  # the 8 directions: each line runs both ways
        _put(m, _line(d, L), 1 + (k % 2) * (L + 3), 1 + (k // 2) * (L + 3))
    out["lines"] = m
    m = np.zeros((S, S), bool)
    for k in range(min(6, S // 3 - 1)):
        m[2 + 2 * k:4 + 2 * k, 2 + 2 * k:4 + 2 * k] = True     # 2 x 2 blocks joined at their corners only
    m[S - 6, 3:9:2] = True
    m[S - 5, 4:9:2] = True                                     # a row of pixels joined diagonally
    out["diagonal_joins"] = m
    m = np.zeros((S, S), bool)
    m[S // 2 - 3:S // 2 + 4, S // 2 - 3:S // 2 + 4] = True
    m[S // 2, S // 2] = False
    out["ring_1px_hole"] = m
    m = np.zeros((S, S), bool)
    _put(m, _nested(4), (S - 17) // 2, (S - 17) // 2)
    out["nested_4"] = m
    m = np.zeros((S, S), bool)
    for y0, x0 in ((0, 0), (0, S - 5), (S - 5, 0), (S - 5, S - 5)):
        m[y0:y0 + 5, x0:x0 + 5] = True                        # the corners: 16 contour points each
    c = S // 2
    m[0:3, c - 3:c + 4] = m[S - 3:S, c - 3:c + 4] = True       # the edges: 16 contour points each
    m[c - 3:c + 4, 0:3] = m[c - 3:c + 4, S - 3:S] = True
    out["border"] = m
    out["full"] = np.ones((S, S), bool)
    return out


def block_grid(S, n, block=5, gap=1):
    """n x n blocks of block x block pixels with gaps of `gap` from the top-left corner: 4 (block - 1) contour points
    each."""
    m = np.zeros((S, S), bool)
    p = block + gap
    for a in range(n):
        for b in range(n):
            m[a * p:a * p + block, b * p:b * p + block] = True
    return m
