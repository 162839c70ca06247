"""m3tb_get_normalized_depth_image (k_normalized_depth): DepthCamera::NormalizedDepthImage equals cv2's convertTo for
every u16 value and several ranges (tests/golden/normalized_depth.npz), with ties, both saturations and depth 0; it reads
the rectified frame of an undistorted camera and a pinned frame in place; FullDepthRenderer::NormalizedDepthImage
equals its NumPy restatement bit for bit, with the 65535 background and ranges that clamp at both ends; host and
device destinations at any pitch give the same bytes; refusals; one launch per call."""
import os

import numpy as np
import pytest

import focused_normal_reference as fn
import full_renderer_reference as fr
import viewer_reference as vr
from test_gpu_viewers import I34, _intr, _scene

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "normalized_depth.npz")


def _depth_context(capi, ranges, W=256, H=256):
    ctx = capi.Context(0, max_bodies=1, max_cameras=len(ranges), max_models=1)
    for c, (ds, _, _) in enumerate(ranges):
        ctx.set_depth_camera(c, _intr(capi, W, H), I34, float(ds))
    return ctx


def test_camera_equals_opencv_for_every_value(capi):
    d = np.load(GOLDEN)
    values = np.arange(65536, dtype=np.uint16).reshape(256, 256)
    ctx = _depth_context(capi, d["ranges"])
    for c in range(len(d["ranges"])):
        ctx.upload_depth(c, values)
    for c, ((_, lo, hi), exp) in enumerate(zip(d["ranges"], d["images"])):
        n0 = ctx.launch_count
        got = ctx.get_normalized_depth_image("camera", c, float(lo), float(hi), 256, 256)
        assert ctx.launch_count == n0 + 1
        assert np.array_equal(got, exp), (c, np.argwhere(got != exp)[:5])
    ctx.close()


def test_host_and_device_destinations(capi):
    import torch
    rng = np.random.default_rng(5)
    frame = rng.integers(0, 1500, (217, 333), dtype=np.uint16)
    frame[::9, ::4] = 0
    ctx = _depth_context(capi, [(0.001, 0, 0)], 333, 217)
    ctx.upload_depth(0, frame)
    exp = vr.normalized_depth(frame, 0.001, 0.25, 0.9)
    assert np.array_equal(ctx.get_normalized_depth_image("camera", 0, 0.25, 0.9, 333, 217), exp)
    dev = torch.full((217, 333 + 11), 7, dtype=torch.uint8, device="cuda")  # pitched rows, padding left alone
    ctx.get_normalized_depth_image_to("camera", 0, 0.25, 0.9, dev.data_ptr(), dev.stride(0))
    ctx.synchronize()
    got = dev.cpu().numpy()
    assert np.array_equal(got[:, :333], exp) and (got[:, 333:] == 7).all()
    host = np.full((217, 340), 9, np.uint8)  # pitched host rows
    ctx.get_normalized_depth_image_to("camera", 0, 0.25, 0.9, host.ctypes.data, host.strides[0])
    assert np.array_equal(host[:, :333], exp) and (host[:, 333:] == 9).all()
    pinned = torch.zeros((217, 333), dtype=torch.uint8).pin_memory()
    ctx.get_normalized_depth_image_to("camera", 0, 0.25, 0.9, pinned.data_ptr(), 333)
    assert np.array_equal(pinned.numpy(), exp)
    ctx.close()


def test_rectified_and_pinned_frames(capi):
    import torch
    W, H = 320, 240
    intr = _intr(capi, W, H)
    rng = np.random.default_rng(11)
    raw = rng.integers(0, 2000, (H, W), dtype=np.uint16)
    raw[::5, ::7] = 0
    m = capi.undistortion_map(intr, np.array([-0.2, 0.05, 1e-3, -2e-3, 0.0, 0.0, 0.0, 0.0], np.float32), intr)
    ctx = capi.Context(0, max_bodies=1, max_cameras=2, max_models=1)
    for c in range(2):
        ctx.set_depth_camera(c, intr, I34, 0.001)
    ctx.set_camera_undistortion("depth", 0, m, 1, 0)
    ctx.upload_depth(0, raw)
    pin = torch.from_numpy(raw.view(np.uint8).reshape(1, H, 2 * W).copy()).pin_memory()
    ctx.upload_batch_ptr(False, 1, 1, pin.data_ptr(), pin.stride(0), pin.stride(1))
    rectified = ctx.get_camera_image("depth", 0, W, H)
    assert not np.array_equal(rectified, raw)
    for c, frame in ((0, rectified), (1, raw)):
        got = ctx.get_normalized_depth_image("camera", c, 0.2, 1.6, W, H)
        assert np.array_equal(got, vr.normalized_depth(frame, 0.001, 0.2, 1.6)), c
    ctx.synchronize()
    ctx.close()
    del pin


@pytest.mark.parametrize("z_range,depth_range", [((0.1, 2.0), (0.38, 0.46)), ((0.02, 10.0), (0.0, 10.0)),
                                                 ((0.3, 0.8), (0.4, 0.5)), ((0.1, 2.0), (-1.0, 3.0))])
def test_full_renderer_equals_restatement(capi, synth, z_range, depth_range):
    import torch
    intr = _intr(capi, 333, 217)
    geometry, poses, order = _scene(synth, "bodies8", 333)
    ctx = capi.Context(0, max_bodies=8, max_cameras=1, max_models=1)
    ctx.set_color_camera(0, intr, I34)
    ctx.set_poses(np.stack([poses[b] for b in range(8)]))
    for b, g in geometry.items():
        ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling)
    ctx.set_full_renderer(0, "color", 0, order, *z_range)
    ctx.render_full()
    full = ctx.get_full_rendering(0, 333, 217)
    exp = fn.normalized_full_depth(full["depth"], full["projection_term_a"], full["projection_term_b"], *depth_range)
    assert np.array_equal(exp, fn.normalized_full_depth(
        fr.render_full(intr, I34, poses, geometry, order, *z_range)["depth"], full["projection_term_a"],
        full["projection_term_b"], *depth_range))
    n0 = ctx.launch_count
    got = ctx.get_normalized_depth_image("full_renderer", 0, *depth_range, 333, 217)
    assert ctx.launch_count == n0 + 1
    assert np.array_equal(got, exp), np.argwhere(got != exp)[:5]
    assert (full["depth"] == 65535).any() and (full["depth"] != 65535).any()
    dev = torch.zeros((217, 400), dtype=torch.uint8, device="cuda")
    ctx.get_normalized_depth_image_to("full_renderer", 0, *depth_range, dev.data_ptr(), 400)
    ctx.synchronize()
    assert np.array_equal(dev[:, :333].cpu().numpy(), exp)
    if depth_range == (0.38, 0.46):  # the bodies span about 0.35 .. 0.52 m: drawn values on both clamps
        drawn = exp[full["depth"] != 65535]
        assert (drawn == 0).any() and (drawn >= 254).any()
    ctx.close()


def test_refusals(capi, synth):
    intr = _intr(capi, 64, 48)
    ctx = capi.Context(0, max_bodies=1, max_cameras=2, max_models=1)
    L, h = ctx.L, ctx.h
    buf = np.zeros((48, 64), np.uint8)
    f = L.m3tb_get_normalized_depth_image
    p = buf.ctypes.data
    assert f(h, 0, 0, 0.0, 1.0, p, 64) == -1      # depth camera 0 not set
    ctx.set_depth_camera(0, intr, I34, 0.001)
    ctx.set_color_camera(1, intr, I34)
    assert f(h, 0, 0, 0.0, 1.0, p, 64) == -4      # no frame yet
    assert f(h, 0, 1, 0.0, 1.0, p, 64) == -1      # camera 1 is a colour camera
    assert f(h, 0, 2, 0.0, 1.0, p, 64) == -1      # out of range
    ctx.upload_depth(0, np.full((48, 64), 500, np.uint16))
    assert f(h, 0, 0, 1.0, 1.0, p, 64) == -1      # max_depth <= min_depth
    assert f(h, 0, 0, 1.0, 0.5, p, 64) == -1
    assert f(h, 0, 0, float("nan"), 1.0, p, 64) == -1
    assert f(h, 0, 0, 0.0, 1.0, p, 63) == -1      # pitch smaller than a row
    assert f(h, 0, 0, 0.0, 1.0, None, 64) == -1   # no destination
    assert f(h, 2, 0, 0.0, 1.0, p, 64) == -1      # bad source
    assert f(h, 1, 0, 0.0, 1.0, p, 64) == -1      # no full renderer
    assert f(h, 0, 0, 0.0, 1.0, p, 64) == 0
    assert np.array_equal(buf, vr.normalized_depth(np.full((48, 64), 500, np.uint16), 0.001, 0.0, 1.0))
    geometry, poses, order = _scene(synth, "prism", 64)
    ctx.set_poses(np.stack([poses[0]]))
    ctx.set_body_geometry(0, geometry[0].triangles, geometry[0].geometry2body, geometry[0].maximum_body_diameter,
                          geometry[0].enable_culling)
    ctx.set_full_renderer(0, "depth", 0, [0], 0.1, 2.0)
    assert f(h, 1, 0, 0.0, 1.0, p, 64) == -4      # not rendered yet
    ctx.render_full()
    assert f(h, 1, 0, 0.0, 1.0, p, 64) == 0
    ctx.set_depth_camera(0, _intr(capi, 32, 24), I34, 0.001)  # the camera changes size
    assert f(h, 1, 0, 0.0, 1.0, p, 64) == -4
    ctx.close()
