"""CPU restatement of k_render (DESIGN.md §3 "k_render"), operation for operation in float32: every NumPy operation on
float32 values rounds once, like the kernel built with -fmad=false, so images, corner, scale, projection terms and
visible flags are compared bit for bit. Test infrastructure only."""
from dataclasses import dataclass

import numpy as np

f32 = np.float32
FLT_MAX = np.finfo(np.float32).max
FLT_MIN = np.finfo(np.float32).tiny  # std::numeric_limits<float>::min()
HALF = f32(0.5)


@dataclass
class Geometry:
    triangles: np.ndarray        # [n,3,3] float32, geometry frame
    geometry2body: np.ndarray    # [3,4] float32
    maximum_body_diameter: float
    enable_culling: bool = True
    body_id: int = 0
    region_id: int = 0


def pose_mul(a, b):
    """m3tb::PoseMul on float32[12] (row-major 3x4)."""
    a = np.asarray(a, f32).reshape(12)
    b = np.asarray(b, f32).reshape(12)
    o = np.zeros(12, f32)
    for i in range(3):
        for j in range(3):
            o[4 * i + j] = a[4 * i] * b[j] + a[4 * i + 1] * b[4 + j] + a[4 * i + 2] * b[8 + j]
        o[4 * i + 3] = a[4 * i] * b[3] + a[4 * i + 1] * b[7] + a[4 * i + 2] * b[11] + a[4 * i + 3]
    return o


def focus(intr, world2camera, poses, geometry, referenced, image_size, z_min, z_max):
    """FocusedRenderer::CalculateProjectionMatrix (renderer.cpp:348-405) + CalculateProjectionTerms (:567-570)."""
    w = np.asarray(world2camera, f32).reshape(12)
    fu, fv, ppu, ppv = f32(intr.fu), f32(intr.fv), f32(intr.ppu), f32(intr.ppv)
    z_min, z_max = f32(z_min), f32(z_max)
    u_min, u_max, v_min, v_max = FLT_MAX, FLT_MIN, FLT_MAX, FLT_MIN
    visible = []
    for b in referenced:
        rr = HALF * f32(geometry[b].maximum_body_diameter)
        p = np.asarray(poses[b], f32).reshape(12)
        x = w[0] * p[3] + w[1] * p[7] + w[2] * p[11] + w[3]
        y = w[4] * p[3] + w[5] * p[7] + w[6] * p[11] + w[7]
        z = w[8] * p[3] + w[9] * p[7] + w[10] * p[11] + w[11]
        vis = 0
        if not (z < rr * f32(1.5) or z - rr < z_min or z + rr > z_max):
            abs_x, abs_y = np.abs(x), np.abs(y)
            x2, y2, z2, r2, rz = x * x, y * y, z * z, rr * rr, rr * z
            z2_r2 = z2 - r2
            z3_zr2 = z2_r2 * z
            r_u = fu * (abs_x * r2 + rz * np.sqrt(z2_r2 + x2)) / z3_zr2
            r_v = fv * (abs_y * r2 + rz * np.sqrt(z2_r2 + y2)) / z3_zr2
            center_u = x * fu / z + ppu
            center_v = y * fv / z + ppv
            u0, u1, v0, v1 = center_u - r_u, center_u + r_u, center_v - r_v, center_v + r_v
            if not (u0 > f32(intr.width) or u1 < 0 or v0 > f32(intr.height) or v1 < 0):
                u_min = u0 if u0 < u_min else u_min
                u_max = u1 if u_max < u1 else u_max
                v_min = v0 if v0 < v_min else v_min
                v_max = v1 if v_max < v1 else v_max
                vis = 1
        visible.append(vis)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        du, dv = f32(u_max - u_min), f32(v_max - v_min)
        d = (dv if du < dv else du) * f32(1.05)
        S = f32(image_size)
        out = dict(corner_u=HALF * (u_min + u_max - d), corner_v=HALF * (v_min + v_max - d), scale=S / d,
                   projection_term_a=z_max * z_min * f32(65535) / (z_max - z_min),
                   projection_term_b=z_max * f32(65535) / (z_max - z_min), visible=np.array(visible, np.int32))
        ppu_scaled = (ppu - out["corner_u"]) * out["scale"]
        ppv_scaled = (ppv - out["corner_v"]) * out["scale"]
        P = (f32(2) * fu / d, f32(2) * (ppu_scaled + HALF) / S - f32(1), f32(2) * fv / d,
             f32(2) * (ppv_scaled + HALF) / S - f32(1), (z_max + z_min) / (z_max - z_min),
             f32(-2) * z_max * z_min / (z_max - z_min))
    return out, P, any(visible)


def _edge(a, b, px, py):
    fwd = a[0] < b[0] or (a[0] == b[0] and a[1] < b[1])
    s, t = (a, b) if fwd else (b, a)
    e = (t[0] - s[0]) * (py - s[1]) - (t[1] - s[1]) * (px - s[0])
    return e if fwd else -e


def _covers(e, a, b):
    with np.errstate(invalid="ignore", over="ignore"):
        dy, dx = b[1] - a[1], b[0] - a[0]
    owned = dy > 0 or (dy == 0 and dx < 0)
    return (e > 0) | ((e == 0) & owned), owned


def count(stats, key, n=1):
    """Adds n to stats[key] (stats: a dict, or None for no counting)."""
    if stats is not None and n:
        stats[key] = stats.get(key, 0) + int(n)


def fragments(v0, v1, v2, culling, W, H, stats=None, coverage=None):
    """RasterTriangle of one window-space triangle (x, y, z float32 triples) on a W x H image: (rows, columns, depth16
    uint32) of the covered pixel centres in front of the far plane, or None. `stats` counts what the walk reaches:
    tie-rule decisions ('tie_owned' / 'tie_not_owned' edge values exactly 0), 'nan_edge' values, 'q_clamp' (q < 0 kept
    as 0), 'far_reject' (covered, q >= 65535 or NaN), 'box_lo_x' / 'box_hi_x' / 'box_lo_y' / 'box_hi_y' (the pixel
    box clamped to the image on that side; 'q_clamp' is not reached by any known scene: fragments in front of the near
    plane have z >= -0), and for the 32 x 32 screen tiles of k_view_raster 'multi_tile' (a box
    over more than one tile) and 'tile_end' (a box ending on a tile edge)."""
    with np.errstate(invalid="ignore", over="ignore"):
        A = (v1[0] - v0[0]) * (v2[1] - v0[1]) - (v2[0] - v0[0]) * (v1[1] - v0[1])
    if not (A != 0):
        return None
    if culling and A > 0:
        return None
    if A < 0:
        v1, v2 = v2, v1
        A = -A
    fW, fH = f32(W), f32(H)
    with np.errstate(invalid="ignore", over="ignore"):
        x_lo, x_hi = np.ceil(np.fmin(np.fmin(v0[0], v1[0]), v2[0]) - HALF), np.floor(np.fmax(np.fmax(v0[0], v1[0]), v2[0]) - HALF)
        y_lo, y_hi = np.ceil(np.fmin(np.fmin(v0[1], v1[1]), v2[1]) - HALF), np.floor(np.fmax(np.fmax(v0[1], v1[1]), v2[1]) - HALF)
    lo_x = np.fmin(np.fmax(x_lo, f32(0)), fW)
    hi_x = np.fmin(np.fmax(x_hi, f32(-1)), fW - f32(1))
    lo_y = np.fmin(np.fmax(y_lo, f32(0)), fH)
    hi_y = np.fmin(np.fmax(y_hi, f32(-1)), fH - f32(1))
    i0, j0 = int(lo_x), int(lo_y)
    nx, ny = int(hi_x) - i0 + 1, int(hi_y) - j0 + 1
    if nx <= 0 or ny <= 0:
        return None
    count(stats, "box_lo_x", lo_x != x_lo)
    count(stats, "box_hi_x", hi_x != x_hi)
    count(stats, "box_lo_y", lo_y != y_lo)
    count(stats, "box_hi_y", hi_y != y_hi)
    count(stats, "multi_tile", (i0 + nx - 1) // 32 != i0 // 32 or (j0 + ny - 1) // 32 != j0 // 32)
    count(stats, "tile_end", (i0 + nx) % 32 == 0 or (j0 + ny) % 32 == 0)
    jj, ii = np.mgrid[j0:j0 + ny, i0:i0 + nx]
    px = ii.astype(f32) + HALF
    py = jj.astype(f32) + HALF
    with np.errstate(invalid="ignore", over="ignore"):
        e0, e1, e2 = _edge(v1, v2, px, py), _edge(v2, v0, px, py), _edge(v0, v1, px, py)
    inside = np.ones(e0.shape, bool)
    for e, (a, b) in ((e0, (v1, v2)), (e1, (v2, v0)), (e2, (v0, v1))):
        cov, owned = _covers(e, a, b)
        inside &= cov
        count(stats, "tie_owned" if owned else "tie_not_owned", np.count_nonzero(e == 0))
        count(stats, "nan_edge", np.count_nonzero(np.isnan(e)))
    if coverage is not None:
        coverage[jj[inside], ii[inside]] += 1
    with np.errstate(invalid="ignore", over="ignore"):
        z = (e0 * v0[2] + e1 * v1[2] + e2 * v2[2]) / A
        q = np.rint(z * f32(65535))
        keep = inside & (q < f32(65535))
    count(stats, "far_reject", np.count_nonzero(inside & ~keep))
    count(stats, "q_clamp", np.count_nonzero(keep & (q < 0)))
    return jj[keep], ii[keep], np.fmax(q[keep], f32(0)).astype(np.uint32)


def raster_triangle(v0, v1, v2, culling, S, draw_index, zbuf, coverage=None, stats=None):
    """One window-space triangle (x, y, z float32 triples) into zbuf [S,S] uint32 (packed depth16 << 16 | index);
    `stats` also counts 'draw_tie' (a fragment whose depth16 equals that of another draw's at the pixel)."""
    f = fragments(v0, v1, v2, culling, S, S, stats, coverage)
    if f is None:
        return
    ji, ij, d16 = f
    packed = (d16 << np.uint32(16)) | np.uint32(draw_index)
    old = zbuf[ji, ij]
    count(stats, "draw_tie", np.count_nonzero((old != 0xFFFFFFFF) & ((old >> np.uint32(16)) == d16) &
                                              ((old & np.uint32(0xFFFF)) != draw_index)))
    zbuf[ji, ij] = np.minimum(old, packed)


def _intersect(a, da, b, db):
    t = da / (da - db)
    return tuple(a[k] + t * (b[k] - a[k]) for k in range(4))


def clip_polygon(c, d, stats=None):
    """ClipTriangle's Sutherland-Hodgman against the near plane: the polygon (0, 3 or 4 clip-space vertices) of one
    triangle's vertices c and their distances d = z + w. `stats` counts the edge patterns 'clip_in_in' / 'clip_in_out'
    / 'clip_out_in' / 'clip_out_out', 'dist_zero' vertices (exactly on the plane) and 'fan4' (polygons of 4)."""
    poly = []
    for e in range(3):
        e1 = 0 if e == 2 else e + 1
        in0, in1 = d[e] >= 0, d[e1] >= 0
        count(stats, f"clip_{'in' if in0 else 'out'}_{'in' if in1 else 'out'}")
        count(stats, "dist_zero", d[e] == 0)
        if in0:
            poly.append(c[e])
        if in0 != in1:
            poly.append(_intersect(c[e], d[e], c[e1], d[e1]) if in0 else _intersect(c[e1], d[e1], c[e], d[e]))
    count(stats, "fan4", len(poly) == 4)
    return poly


def clip_body(M, triangles):
    """Every triangle of one body through M (16 float32, row-major): clip coordinates [4][n,3] and distances [n,3]."""
    tv = np.asarray(triangles, f32).reshape(-1, 3, 3)
    vx, vy, vz = tv[..., 0], tv[..., 1], tv[..., 2]
    with np.errstate(invalid="ignore", over="ignore"):
        clip = [M[4 * r] * vx + M[4 * r + 1] * vy + M[4 * r + 2] * vz + M[4 * r + 3] for r in range(4)]
        return clip, clip[2] + clip[3]


def window(poly, half_x, half_y):
    """Window mapping of a clip-space polygon onto an image of half sizes half_x, half_y (float32)."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return [((p[0] / p[3] + f32(1)) * half_x, (p[1] / p[3] + f32(1)) * half_y, (p[2] / p[3] + f32(1)) * HALF)
                for p in poly]


def fans(win):
    """The fan of a window-space polygon: (w0, w1, w2) and, for 4 vertices, (w0, w2, w3)."""
    return [(win[0], win[1], win[2])] + ([(win[0], win[2], win[3])] if len(win) == 4 else [])


def raster_keyed(M, triangles, culling, W, H, draw, zbuf, stats=None):
    """Every triangle of one body through M into zbuf [H,W] uint64 (depth16 << 48 | draw << 32 | triangle), as
    k_model_raster and k_view_raster key their z-buffers. `stats` also counts fragments whose depth16 equals the one at
    the pixel: of another triangle of the same draw ('triangle_tie') or of another draw ('draw_tie')."""
    clear = np.uint64(0xFFFFFFFFFFFFFFFF)
    clip, dist = clip_body(M, triangles)
    half_x, half_y = HALF * f32(W), HALF * f32(H)
    for t in range(dist.shape[0]):
        c = [tuple(clip[r][t, k] for r in range(4)) for k in range(3)]
        poly = clip_polygon(c, [dist[t, k] for k in range(3)], stats)
        if len(poly) < 3:
            continue
        tag = (np.uint64(draw) << np.uint64(32)) | np.uint64(t)
        for v0, v1, v2 in fans(window(poly, half_x, half_y)):
            f = fragments(v0, v1, v2, culling, W, H, stats)
            if f is None:
                continue
            j, i, d16 = f
            d16 = d16.astype(np.uint64)
            if stats is not None:
                old = zbuf[j, i]
                tie = (old != clear) & ((old >> np.uint64(48)) == d16)
                same = ((old >> np.uint64(32)) & np.uint64(0xFFFF)) == np.uint64(draw)
                count(stats, "triangle_tie", np.count_nonzero(tie & same & ((old & np.uint64(0xFFFFFFFF)) != t)))
                count(stats, "draw_tie", np.count_nonzero(tie & ~same))
            np.minimum.at(zbuf, (j, i), (d16 << np.uint64(48)) | tag)


def render_focused(intr, world2camera, poses, geometry, geometry_bodies, referenced_bodies, image_size=200, z_min=0.02,
                   z_max=10.0, id_type="body", coverage=False, stats=None):
    """FocusedRenderer::StartRendering as k_render performs it. poses / geometry: {body: [3,4] body2world / Geometry}.
    Returns dict(depth [S,S] u16, silhouette [S,S] u8, corner_u, corner_v, scale, projection_term_a / b, visible
    [n_referenced] int32, coverage [S,S] covered-pixel counter when asked for). `stats`: see fragments, clip_polygon
    and raster_triangle."""
    S = int(image_size)
    out, P, any_visible = focus(intr, world2camera, poses, geometry, referenced_bodies, S, z_min, z_max)
    zbuf = np.full((S, S), 0xFFFFFFFF, np.uint32)
    cov = np.zeros((S, S), np.int32) if coverage else None
    w2c = np.asarray(world2camera, f32).reshape(12)
    half = HALF * f32(S)
    if any_visible:
        for g, b in enumerate(geometry_bodies):
            G = geometry[b]
            T = pose_mul(w2c, pose_mul(poses[b], G.geometry2body))
            M = np.zeros(16, f32)
            for c in range(4):
                M[c] = P[0] * T[c] + P[1] * T[8 + c]
                M[4 + c] = P[2] * T[4 + c] + P[3] * T[8 + c]
                M[8 + c] = P[4] * T[8 + c]
                M[12 + c] = T[8 + c]
            M[11] = M[11] + P[5]
            clip, dist = clip_body(M, G.triangles)
            for t in range(dist.shape[0]):
                c = [tuple(clip[r][t, k] for r in range(4)) for k in range(3)]
                poly = clip_polygon(c, [dist[t, k] for k in range(3)], stats)
                if len(poly) < 3:
                    continue
                for v0, v1, v2 in fans(window(poly, half, half)):
                    raster_triangle(v0, v1, v2, G.enable_culling, S, g, zbuf, cov, stats)
    depth = (zbuf >> np.uint32(16)).astype(np.uint16)
    ids = np.array([geometry[b].region_id if id_type == "region" else geometry[b].body_id for b in geometry_bodies] + [0],
                   np.uint8)
    idx = (zbuf & np.uint32(0xFFFF)).astype(np.int64)
    sil = np.where(depth != 0xFFFF, ids[np.minimum(idx, len(ids) - 1)], 0).astype(np.uint8)
    out.update(depth=depth, silhouette=sil)
    if coverage:
        out["coverage"] = cov
    return out
