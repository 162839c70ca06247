"""CPU restatement of the device full renderers (FullBasicDepthRenderer / FullSilhouetteRenderer / FullNormalRenderer,
m3tb_render_full; DESIGN.md §3 "Full renderers"): viewer_reference's full raster with the renderer's own z range, and the
three images k_view_resolve reads out of the z-buffer key (depth16 << 48 | draw << 32 | triangle). Also the scene of the
reference's renderer test (M3T/test/renderer_test.cpp), whose OpenGL images are stored under tests/golden/renderer_test/.
Test infrastructure only."""
import json
import os
from types import SimpleNamespace

import numpy as np

import model_generation_reference as mg
import render_reference as rr
import viewer_reference as vr

f32 = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def render_full(intr, world2camera, poses, geometry, bodies, z_min=0.02, z_max=10.0, id_type="body"):
    """FullRenderer::StartRendering + Fetch{Depth,Silhouette,Normal}Image: dict(depth [H,W] u16 (65535 = nothing drawn),
    silhouette [H,W] u8 (0 = background), normal [H,W,4] u8, projection_term_a / b). poses / geometry: {body: [3,4]
    body2world / rr.Geometry}; bodies: render_data_bodies order."""
    normal, zbuf = vr.render_normal(intr, world2camera, poses, geometry, bodies, z_min, z_max)
    depth = (zbuf >> np.uint64(48)).astype(np.uint16)  # the cleared key reads 65535
    ids = np.array([geometry[b].region_id if id_type == "region" else geometry[b].body_id for b in bodies] + [0],
                   np.uint8)
    draw = ((zbuf >> np.uint64(32)) & np.uint64(0xFFFF)).astype(np.int64)
    sil = np.where(zbuf != mg.CLEAR, ids[np.minimum(draw, len(ids) - 1)], 0).astype(np.uint8)
    z_min, z_max = f32(z_min), f32(z_max)
    return dict(depth=depth, silhouette=sil, normal=normal,
                projection_term_a=z_max * z_min * f32(65535) / (z_max - z_min),
                projection_term_b=z_max * f32(65535) / (z_max - z_min))


def depth_of(out, value):
    """FullDepthRenderer::Depth(ushort) (renderer.cpp:431-433)."""
    return out["projection_term_a"] / (out["projection_term_b"] - f32(value))


def point_vector(out, intr, x, y):
    """FullDepthRenderer::PointVector (renderer.cpp:445-452) at column x, row y."""
    depth = depth_of(out, out["depth"][y, x])
    return np.array([depth * (f32(x) - f32(intr.ppu)) / f32(intr.fu),
                     depth * (f32(y) - f32(intr.ppv)) / f32(intr.fv), depth], f32)


# ---- the scene of renderer_test.cpp (common_test.cpp:9-11,27-29) ----------------------------------------------------

def _inverse(m):
    R, t = m[:3, :3], m[:3, 3]
    return np.hstack([R.T, (-R.T @ t)[:, None]]).astype(f32)


def golden_scene():
    """The bodies, poses and camera of the reference's renderer test: triangle.obj (geometry2body z -0.006, ids 150 /
    150) and schauma (z -0.097, body_id 50, region_id 150), both culled and drawn triangle first; world2camera =
    translation (0.01, 0, 0), 640 x 480, z 0.1 .. 2.0. maximum_body_diameter = 2 max |geometry2body * v| (body.cpp)."""
    with open(os.path.join(GOLDEN, "reference_known_answers.json")) as f:
        ka = json.load(f)["triangle_obj"]
    tri_v = np.array(ka["vertices"], f32)
    tri_f = np.array(ka["faces"], np.int64) - 1
    mesh = np.load(os.path.join(GOLDEN, "schauma_mesh.npz"))
    sch_v, sch_f = mesh["vertices"].astype(f32), mesh["faces"]

    def g2b(dz):
        return np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, dz]], f32)

    def diameter(v, dz):
        return float(f32(2) * np.max(np.linalg.norm((v + np.array([0, 0, dz], f32)).astype(f32), axis=1)))

    geometry = {0: rr.Geometry(tri_v[tri_f], g2b(-0.006), diameter(tri_v, -0.006), True, 150, 150),
                1: rr.Geometry(sch_v[sch_f], g2b(-0.097), diameter(sch_v, -0.097), True, 50, 150)}
    w2b_t = np.array([[0.607676, 0.408914, -0.680823, 0.472944], [0.786584, -0.428213, 0.444880, -0.213009],
                      [-0.109620, -0.805867, -0.581860, 0.346384]], np.float64)
    w2b_s = w2b_t.copy()
    w2b_s[:, 3] = [0.297794, -0.189009, 0.255284]
    poses = {0: _inverse(w2b_t), 1: _inverse(w2b_s)}  # body2world: inverted in float64, then rounded once
    w2c = np.array([[1, 0, 0, 0.01], [0, 1, 0, 0], [0, 0, 1, 0]], f32)
    intr = SimpleNamespace(fu=698.128, fv=698.617, ppu=478.459, ppv=274.426, width=640, height=480)
    return SimpleNamespace(geometry=geometry, poses=poses, world2camera=w2c, intrinsics=intr, bodies=[0, 1],
                           z_min=0.1, z_max=2.0, focused_size=200, focused_referenced=[0])


def load_golden(name):
    """A PNG of tests/golden/renderer_test/ as the reference test loads it (cv::imread, IMREAD_UNCHANGED)."""
    import cv2
    img = cv2.imread(os.path.join(GOLDEN, "renderer_test", name), cv2.IMREAD_UNCHANGED)
    assert img is not None, name
    return img


def wrong_pixels(got, expected):
    """CompareImages (common_test.cpp): pixels where a channel differs by more than 1."""
    d = np.abs(np.asarray(got, np.int64) - np.asarray(expected, np.int64))
    if d.ndim == 3:
        d = d.max(-1)
    return int((d > 1).sum())
