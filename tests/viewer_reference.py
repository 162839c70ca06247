"""CPU restatement of the device viewers (DESIGN.md §3 "k_view_setup / k_view_raster / k_view_resolve"): the full
normal renderer over a W x H camera image, the normal bytes, DepthCamera::NormalizedDepthImage and CalculateAlphaBlend,
operation for operation in float32 like the kernels built with -fmad=false, so that normal and viewer images are
compared bit for bit. The triangle walk is render_reference's (edge functions, tie rule, DEPTH_COMPONENT16) with the
model-generation z-buffer key (depth16 << 48 | draw << 32 | triangle). Test infrastructure only."""
from fractions import Fraction

import numpy as np

import model_generation_reference as mg
import render_reference as rr

f32 = np.float32
CLEAR = mg.CLEAR
Z_MIN, Z_MAX = f32(0.02), f32(10.0)  # FullNormalRenderer defaults of the viewers' renderers
HALF = rr.HALF


def projection(intr, z_min=Z_MIN, z_max=Z_MAX):
    """FullRenderer::CalculateProjectionMatrix (renderer.cpp:257-264): P00, P02, P11, P12, P22, P23."""
    W, H = f32(intr.width), f32(intr.height)
    z_min, z_max = f32(z_min), f32(z_max)
    return (f32(2) * f32(intr.fu) / W, f32(2) * (f32(intr.ppu) + HALF) / W - f32(1),
            f32(2) * f32(intr.fv) / H, f32(2) * (f32(intr.ppv) + HALF) / H - f32(1),
            (z_max + z_min) / (z_max - z_min), f32(-2) * z_max * z_min / (z_max - z_min))


def clip_matrix(P, T):
    """P * [T; 0 0 0 1] without the products with P's zero entries (k_render, k_view_setup)."""
    M = np.zeros(16, f32)
    for c in range(4):
        M[c] = P[0] * T[c] + P[1] * T[8 + c]
        M[4 + c] = P[2] * T[4 + c] + P[3] * T[8 + c]
        M[8 + c] = P[4] * T[8 + c]
        M[12 + c] = T[8 + c]
    M[11] = M[11] + P[5]
    return M


def raster_triangle(v0, v1, v2, culling, W, H, tag, zbuf):
    """One window-space triangle into zbuf [H,W] uint64 (rr.raster_triangle with separate x and y limits)."""
    A = (v1[0] - v0[0]) * (v2[1] - v0[1]) - (v2[0] - v0[0]) * (v1[1] - v0[1])
    if not (A != 0):
        return
    if culling and A > 0:
        return
    if A < 0:
        v1, v2 = v2, v1
        A = -A
    fW, fH = f32(W), f32(H)
    lo_x = np.fmin(np.fmax(np.ceil(np.fmin(np.fmin(v0[0], v1[0]), v2[0]) - HALF), f32(0)), fW)
    hi_x = np.fmin(np.fmax(np.floor(np.fmax(np.fmax(v0[0], v1[0]), v2[0]) - HALF), f32(-1)), fW - f32(1))
    lo_y = np.fmin(np.fmax(np.ceil(np.fmin(np.fmin(v0[1], v1[1]), v2[1]) - HALF), f32(0)), fH)
    hi_y = np.fmin(np.fmax(np.floor(np.fmax(np.fmax(v0[1], v1[1]), v2[1]) - HALF), f32(-1)), fH - f32(1))
    i0, j0 = int(lo_x), int(lo_y)
    nx, ny = int(hi_x) - i0 + 1, int(hi_y) - j0 + 1
    if nx <= 0 or ny <= 0:
        return
    jj, ii = np.mgrid[j0:j0 + ny, i0:i0 + nx]
    px = ii.astype(f32) + HALF
    py = jj.astype(f32) + HALF
    e0, e1, e2 = rr._edge(v1, v2, px, py), rr._edge(v2, v0, px, py), rr._edge(v0, v1, px, py)
    inside = rr._covers(e0, v1, v2) & rr._covers(e1, v2, v0) & rr._covers(e2, v0, v1)
    with np.errstate(invalid="ignore", over="ignore"):
        z = (e0 * v0[2] + e1 * v1[2] + e2 * v2[2]) / A
        q = np.rint(z * f32(65535))
        keep = inside & (q < f32(65535))
    d16 = np.fmax(q[keep], f32(0)).astype(np.uint64)
    np.minimum.at(zbuf, (jj[keep], ii[keep]), (d16 << np.uint64(48)) | np.uint64(tag))


def raster(M, triangles, culling, W, H, draw, zbuf):
    """Every triangle of one body through M: near-plane clipping, window mapping onto W x H, fans."""
    tv = np.asarray(triangles, f32).reshape(-1, 3, 3)
    vx, vy, vz = tv[..., 0], tv[..., 1], tv[..., 2]
    clip = [M[4 * r] * vx + M[4 * r + 1] * vy + M[4 * r + 2] * vz + M[4 * r + 3] for r in range(4)]
    dist = clip[2] + clip[3]
    half_x, half_y = HALF * f32(W), HALF * f32(H)
    for t in range(tv.shape[0]):
        c = [tuple(clip[r][t, k] for r in range(4)) for k in range(3)]
        d = [dist[t, k] for k in range(3)]
        poly = []
        for e in range(3):
            e1 = 0 if e == 2 else e + 1
            in0, in1 = d[e] >= 0, d[e1] >= 0
            if in0:
                poly.append(c[e])
            if in0 != in1:
                poly.append(rr._intersect(c[e], d[e], c[e1], d[e1]) if in0 else rr._intersect(c[e1], d[e1], c[e], d[e]))
        if len(poly) < 3:
            continue
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            win = [((p[0] / p[3] + f32(1)) * half_x, (p[1] / p[3] + f32(1)) * half_y, (p[2] / p[3] + f32(1)) * HALF)
                   for p in poly]
        tag = (draw << 32) | t
        raster_triangle(win[0], win[1], win[2], culling, W, H, tag, zbuf)
        if len(win) == 4:
            raster_triangle(win[0], win[2], win[3], culling, W, H, tag, zbuf)


def encode_normals(zbuf, rots, normals):
    """FullNormalRenderer::normal_image(): per pixel 0.5 - 0.5 * Rot * n of the winning triangle as unorm8, GL_BGRA
    order (byte 0 = x), alpha 255; background (0, 0, 0, 0). rots / normals: per draw."""
    H, W = zbuf.shape
    out = np.zeros((H, W, 4), np.uint8)
    covered = zbuf != CLEAR
    draw = ((zbuf >> np.uint64(32)) & np.uint64(0xFFFF)).astype(np.int64)
    tri = (zbuf & np.uint64(0xFFFFFFFF)).astype(np.int64)
    for g, (R, nrm) in enumerate(zip(rots, normals)):
        sel = covered & (draw == g)
        if not sel.any():
            continue
        n = nrm[tri[sel]]
        for r in range(3):
            nc = R[r, 0] * n[:, 0] + R[r, 1] * n[:, 1] + R[r, 2] * n[:, 2]
            out[..., r][sel] = mg._unorm8(f32(0.5) - f32(0.5) * nc)
        out[..., 3][sel] = 255
    return out


def render_normal(intr, world2camera, poses, geometry, bodies, z_min=Z_MIN, z_max=Z_MAX):
    """FullNormalRenderer::StartRendering + FetchNormalImage: (normal [H,W,4] u8, zbuf [H,W] u64). poses /
    geometry: {body: [3,4] body2world / rr.Geometry}; bodies: render_data_bodies order."""
    W, H = int(intr.width), int(intr.height)
    P = projection(intr, z_min, z_max)
    w2c = np.asarray(world2camera, f32).reshape(12)
    zbuf = np.full((H, W), CLEAR, np.uint64)
    rots, normals = [], []
    for g, b in enumerate(bodies):
        G = geometry[b]
        T = rr.pose_mul(w2c, rr.pose_mul(poses[b], G.geometry2body))
        raster(clip_matrix(P, T), G.triangles, G.enable_culling, W, H, g, zbuf)
        rots.append(T.reshape(3, 4)[:, :3].copy())
        normals.append(mg.face_normals(G.triangles))
    return encode_normals(zbuf, rots, normals), zbuf


def char_of(x):
    """char(x) of a float on x86-64 as stored into a uchar: the low byte of the 32-bit truncation; out of the int32
    range (and NaN) cvttss2si gives 0x80000000, whose low byte is 0."""
    x = np.asarray(x, f32)
    with np.errstate(invalid="ignore"):
        ok = (x >= f32(-2147483648.0)) & (x < f32(2147483648.0))
        t = np.where(ok, np.trunc(x), 0).astype(np.int64)
    return (t & 0xFF).astype(np.uint8)


def alpha_blend(camera_bgr, normal, opacity):
    """CalculateAlphaBlend (normal_viewer.cpp:8-44)."""
    alpha_scale = f32(opacity) / f32(255)
    alpha = normal[..., 3].astype(f32) * alpha_scale
    alpha_inv = f32(1) - alpha
    x = camera_bgr.astype(f32) * alpha_inv[..., None] + normal[..., :3].astype(f32) * alpha[..., None]
    return char_of(x)


def _fma_f32(a, x, b):
    """round_f32(a * x + b) with a single rounding, a uint16 array, x and b float32. The product is exact in float64;
    where the float64 sum is not exact (TwoSum error term), the value is recomputed with fractions."""
    p = a.astype(np.float64) * np.float64(x)
    s = p + np.float64(b)
    bb = s - p
    err = (p - (s - bb)) + (np.float64(b) - bb)
    out = s.astype(f32)
    for idx in zip(*np.nonzero(err != 0)):
        exact = Fraction(int(a[idx])) * Fraction(float(x)) + Fraction(float(b))
        lo = f32(float(exact))
        cands = [np.nextafter(lo, f32(-np.inf)), lo, np.nextafter(lo, f32(np.inf))]
        dist = [abs(Fraction(float(c)) - exact) for c in cands]
        best = min(range(3), key=lambda k: (dist[k], int(np.asarray(cands[k], f32).view(np.uint32)) & 1))
        out[idx] = cands[best]
    return out


def normalized_depth(depth_u16, depth_scale, min_depth, max_depth):
    """DepthCamera::NormalizedDepthImage (camera.cpp:108-115): convertTo(CV_8UC1, alpha, beta) as OpenCV 4.13 computes it
    on x86-64 - one fused multiply-add, cvRound (half to even, INT_MIN out of the int range), saturation."""
    ds = f32(depth_scale)
    alpha = f32(255) / ((f32(max_depth) - f32(min_depth)) / ds)
    beta = -(f32(min_depth) / ds) * alpha
    v = _fma_f32(np.asarray(depth_u16, np.uint16), alpha, beta)
    with np.errstate(invalid="ignore"):
        r = np.rint(v)
        ok = (r >= f32(-2147483648.0)) & (r < f32(2147483648.0))
        return np.where(ok, np.clip(np.nan_to_num(r), 0, 255), 0).astype(np.uint8)


def viewer_image(kind, frame, normal, opacity=0.5, depth_scale=0.001, min_depth=0.0, max_depth=1.0):
    """NormalColorViewer (kind "color": frame [H,W,3] BGR8) / NormalDepthViewer ("depth": frame [H,W] u16, GRAY2BGR)."""
    if kind == "color":
        cam = np.asarray(frame, np.uint8)
    else:
        g = normalized_depth(frame, depth_scale, min_depth, max_depth)
        cam = np.repeat(g[..., None], 3, axis=2)
    return alpha_blend(cam, normal, opacity)
