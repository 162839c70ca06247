"""CPU restatement of the device focused normal renderers (FocusedNormalRenderer, m3tb_render_focused_normals;
DESIGN.md §3 "Focused normal renderers"): render_reference's focus (FocusedRenderer::CalculateProjectionMatrix) and
viewer_reference's keyed raster and normal bytes over an S x S image, so that the depth and normal images are compared
bit for bit. Also FocusedNormalRenderer::NormalVector / NormalImageValue and FullDepthRenderer::NormalizedDepthImage.
Test infrastructure only."""
import numpy as np

import model_generation_reference as mg
import render_reference as rr
import viewer_reference as vr

f32 = np.float32


def render_focused_normal(intr, world2camera, poses, geometry, geometry_bodies, referenced_bodies, image_size=200,
                          z_min=0.02, z_max=10.0):
    """FocusedNormalRenderer::StartRendering + FetchDepthImage / FetchNormalImage: dict(depth [S,S] u16 (65535 =
    nothing drawn), normal [S,S,4] u8 (GL_BGRA, background 0), corner_u, corner_v, scale, projection_term_a / b,
    visible). With no referenced body visible nothing is drawn (the projection is not finite)."""
    S = int(image_size)
    out, P, any_visible = rr.focus(intr, world2camera, poses, geometry, referenced_bodies, S, z_min, z_max)
    w2c = np.asarray(world2camera, f32).reshape(12)
    zbuf = np.full((S, S), mg.CLEAR, np.uint64)
    rots, normals = [], []
    if any_visible:
        for g, b in enumerate(geometry_bodies):
            G = geometry[b]
            T = rr.pose_mul(w2c, rr.pose_mul(poses[b], G.geometry2body))
            vr.raster(vr.clip_matrix(P, T), G.triangles, G.enable_culling, S, S, g, zbuf)
            rots.append(T.reshape(3, 4)[:, :3].copy())
            normals.append(mg.face_normals(G.triangles))
    out.update(depth=(zbuf >> np.uint64(48)).astype(np.uint16), normal=vr.encode_normals(zbuf, rots, normals))
    return out


def normal_vector(value):
    """FocusedNormalRenderer::NormalVector(cv::Vec4b) (normal_renderer.cpp:393-398): 1 - byte / 127.5 of bytes 0-2."""
    v = np.asarray(value, np.uint8)[..., :3].astype(f32)
    return f32(1) - v / f32(127.5)


def image_value_index(out, x, y):
    """The focused image pixel (row v, column u) that FocusedNormalRenderer::NormalVector(Point2i) /
    NormalImageValue read for camera pixel (x, y) (normal_renderer.cpp:400-415)."""
    u = int(np.trunc((f32(x) - out["corner_u"]) * out["scale"] + f32(0.5)))
    v = int(np.trunc((f32(y) - out["corner_v"]) * out["scale"] + f32(0.5)))
    return v, u


def normalized_full_depth(depth_u16, projection_term_a, projection_term_b, min_depth, max_depth):
    """FullDepthRenderer::NormalizedDepthImage (renderer.cpp:407-427): uchar(min(max(a / (b - value) - min, 0),
    delta) * 255 / delta) in float32, uchar() the low byte of the 32-bit truncation."""
    delta = f32(max_depth) - f32(min_depth)
    scale = f32(255) / delta
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        depth = f32(projection_term_a) / (f32(projection_term_b) - np.asarray(depth_u16).astype(f32))
        depth = depth - f32(min_depth)
        depth = np.where(depth < f32(0), f32(0), depth).astype(f32)  # std::max(x, 0) = x < 0 ? 0 : x
        depth = np.where(delta < depth, delta, depth).astype(f32)    # std::min(x, delta) = delta < x ? delta : x
        return vr.char_of(depth * scale)
