"""Undistortion of raw frames as they are uploaded (m3tb_set_camera_undistortion, k_undistort): the frame a camera holds
(m3tb_get_camera_image) equals the NumPy restatement of cv::remap / image_ += offset bit for bit on every upload path,
tracking on undistorted uploads equals tracking on frames rectified beforehand, cameras without an undistortion launch
what they launched before, and the lifecycle rules of include/m3t_b200.h hold."""
import ctypes as C
import dataclasses
import os
import subprocess

import numpy as np
import pytest

import undistortion_reference as ur
from helpers import assert_lines_bit_equal, assert_points_bit_equal

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EYE = np.eye(4, dtype=np.float32)[:3]


def _intr(synth, w, h, fu, fv, cx, cy):
    return synth.Intrinsics(fu, fv, cx, cy, w, h)


def _golden(synth, name):
    m, c = ur.load_golden_map(name)
    return m, _intr(synth, int(c["width"]), int(c["height"]), c["fu"], c["fv"], c["cx"], c["cy"])


def _pinned(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


def _device(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _upload(ctx, color, cam, frame, how):
    """frame: [H, W, ch] u8 or [H, W] u16 numpy; how: pageable | pinned | device."""
    L = ctx.L
    if how == "pageable":
        f = L.m3tb_upload_color if color else L.m3tb_upload_depth
        ctx._ck(f(ctx.h, cam, frame.ctypes.data, frame.strides[0]))
        return None
    t = _pinned(frame) if how == "pinned" else _device(frame)
    if how == "pinned":
        f = L.m3tb_upload_color if color else L.m3tb_upload_depth
    else:
        f = L.m3tb_upload_color_device if color else L.m3tb_upload_depth_device
    ctx._ck(f(ctx.h, cam, C.c_void_p(t.data_ptr()), t.stride(0) * t.element_size()))
    ctx.synchronize()  # the raw frame must stay unchanged until the stream has passed the upload
    return t


@pytest.mark.parametrize("name", ["color_1280x720", "color_640x480", "odd_333x217"])
@pytest.mark.parametrize("channels", [3, 4])
def test_color_frames_equal_the_restatement(capi, synth, name, channels):
    m, intr = _golden(synth, name)
    H, W = m.shape[:2]
    rng = np.random.default_rng(channels * 1000 + W)
    # cameras 0..3 share the pool (its size is set by camera 0's first frame); 4..6 are private allocations because the
    # pool was made for camera 7's other size first
    ctx = capi.Context(max_cameras=8)
    small = _intr(synth, 64, 48, 60.0, 60.0, 32.0, 24.0)
    for cam in range(8):
        ctx.set_color_camera(cam, intr if cam < 7 else small, EYE)
        if cam < 7:
            ctx.set_camera_undistortion("color", cam, m, channels)
    raws = rng.integers(0, 256, (7, H, W, channels), dtype=np.uint8)
    expect = [ur.undistort_color(r, m) for r in raws]
    for cam, how in enumerate(("pageable", "pinned", "device")):
        _upload(ctx, True, cam, raws[cam], how)
        assert np.array_equal(ctx.get_camera_image("color", cam, W, H), expect[cam]), (name, channels, how)
    ctx.upload_color_batch(0, raws[:4])  # pooled batch, pageable
    for cam in range(4):
        assert np.array_equal(ctx.get_camera_image("color", cam, W, H), expect[cam]), (name, channels, "batch", cam)
    # private allocations: a fresh context whose pool is made by the small camera first
    ctx2 = capi.Context(max_cameras=4)
    ctx2.set_color_camera(0, small, EYE)
    ctx2.upload_color(0, np.zeros((48, 64, 3), np.uint8))
    for cam in (1, 2, 3):
        ctx2.set_color_camera(cam, intr, EYE)
        ctx2.set_camera_undistortion("color", cam, m, channels)
    pin = _pinned(raws[4:7])
    ctx2.upload_batch_ptr(True, 1, 3, pin.data_ptr(), pin.stride(0), pin.stride(1))  # pinned batch, not pooled
    ctx2.synchronize()
    for k in range(3):
        assert np.array_equal(ctx2.get_camera_image("color", 1 + k, W, H), expect[4 + k]), (name, channels, "private", k)
    # into device memory at another pitch
    import torch
    dst = torch.zeros((H, W * 3 + 20), dtype=torch.uint8, device="cuda")
    ctx2.get_camera_image_to("color", 2, dst.data_ptr(), dst.stride(0))
    torch.cuda.synchronize()
    assert np.array_equal(dst[:, :W * 3].cpu().numpy().reshape(H, W, 3), expect[5])
    ctx.close()
    ctx2.close()


@pytest.mark.parametrize("offset", [-37, 0, 37])
def test_depth_frames_equal_the_restatement(capi, synth, offset):
    m, intr = _golden(synth, "depth_640x576")
    H, W = m.shape[:2]
    m[:3] = -1          # entries outside the raw frame (this calibration has none of its own)
    m[:, -2:, 0] = W + 1
    rng = np.random.default_rng(100 + offset)
    raws = rng.integers(0, 65536, (6, H, W), dtype=np.uint16)
    raws[:, ::7, ::5] = 0        # invalid pixels: a positive offset moves them too
    raws[:, 3::11, 2::3] = 65535  # saturation at the top
    raws[:, 5::13, 1::4] = 20     # and at the bottom for a negative offset
    ctx = capi.Context(max_cameras=6)
    for cam in range(6):
        ctx.set_depth_camera(cam, intr, EYE, 0.001)
        ctx.set_camera_undistortion("depth", cam, m, 1, offset)
    expect = [ur.undistort_depth(r, m, offset) for r in raws]
    for cam, how in enumerate(("pageable", "pinned", "device")):
        _upload(ctx, False, cam, raws[cam], how)
        assert np.array_equal(ctx.get_camera_image("depth", cam, W, H), expect[cam]), (offset, how)
    ctx.upload_depth_batch(3, raws[3:6])
    for cam in range(3, 6):
        assert np.array_equal(ctx.get_camera_image("depth", cam, W, H), expect[cam]), (offset, "batch", cam)
    ctx.close()


def _mild_map(capi, synth, intr, seed):
    """A mild rational distortion of camera `intr` (the rectified camera equals the raw one)."""
    rng = np.random.default_rng(seed)
    k = np.array([rng.uniform(-0.06, 0.06), rng.uniform(-0.02, 0.02), rng.uniform(-1e-3, 1e-3), rng.uniform(-1e-3, 1e-3),
                  rng.uniform(-5e-3, 5e-3), rng.uniform(-0.05, 0.05), rng.uniform(-0.02, 0.02), rng.uniform(-5e-3, 5e-3)],
                 np.float32)
    return capi.undistortion_map(intr, k, intr)


def _color_raw(wl):
    W, H = wl.color_intrinsics.width, wl.color_intrinsics.height
    return np.ascontiguousarray(wl.color_frames[:, :, :W * 3]).reshape(wl.n_bodies, H, W, 3)


def _pair(capi, synth, wl, offset=0, channels=3):
    """(A: raw frames through undistortions, B: the restatement's rectified frames through plain uploads, maps)."""
    cm = _mild_map(capi, synth, wl.color_intrinsics, 1)
    dm = _mild_map(capi, synth, wl.depth_intrinsics, 2)
    raw_c = _color_raw(wl)
    if channels == 4:
        raw_c = np.concatenate([raw_c, np.full(raw_c.shape[:3] + (1,), 201, np.uint8)], axis=3)
    raw_d = wl.depth_frames
    wl_b = dataclasses.replace(wl, color_frames=np.stack([ur.undistort_color(f, cm) for f in raw_c]),
                               depth_frames=np.stack([ur.undistort_depth(f, dm, offset) for f in raw_d]))
    b = capi.context_from_workload(wl_b)
    a = capi.context_from_workload(wl, upload_frames=False)
    for cam in range(wl.n_bodies):
        a.set_camera_undistortion("color", cam, cm, channels)
        a.set_camera_undistortion("depth", cam, dm, 1, offset)
    a.upload_color_batch(0, raw_c)
    a.upload_depth_batch(0, raw_d)
    return a, b, wl_b


def _track_and_compare(wl, a, b, steps=2):
    for ctx in (a, b):
        ctx.start_modalities(0)
    for it in range(steps):
        for ctx in (a, b):
            ctx.tracking_step(it, wl.n_corr_iterations, wl.n_update_iterations)
        assert a.last_launch() == b.last_launch()
        for body in range(wl.n_bodies):
            if wl.region:
                assert_lines_bit_equal(a.get_region_lines(body, wl.lines_per_body), b.get_region_lines(body, wl.lines_per_body))
            if wl.depth:
                assert_points_bit_equal(a.get_depth_points(body, wl.points_per_body),
                                        b.get_depth_points(body, wl.points_per_body))
        assert np.array_equal(a.get_poses().view(np.uint32), b.get_poses().view(np.uint32))
        for ctx in (a, b):
            ctx.calculate_results(it)
        for body in range(wl.n_bodies):
            ha, hb = a.get_histograms(body, wl.region.n_histogram_bins), b.get_histograms(body, wl.region.n_histogram_bins)
            assert np.array_equal(ha[0], hb[0]) and np.array_equal(ha[1], hb[1])


@pytest.mark.parametrize("kernel", ["k_track2", "k_track"])
def test_tracking_on_undistorted_uploads_is_unchanged(capi, synth, monkeypatch, kernel):
    if kernel == "k_track":
        monkeypatch.setenv("M3TB_KERNEL", "1")
    wl = synth.make_workload("c2", n_bodies=3, n_divides=2, seed=41)
    a, b, _ = _pair(capi, synth, wl, channels=4)
    W, H = wl.color_intrinsics.width, wl.color_intrinsics.height
    for cam in range(wl.n_bodies):
        assert np.array_equal(a.get_camera_image("color", cam, W, H), b.get_camera_image("color", cam, W, H))
    _track_and_compare(wl, a, b)
    assert a.last_launch()["kernel"] == kernel
    if kernel == "k_track2":
        assert a.last_launch()["tma_mode"] == 1
    a.close()
    b.close()


def test_measured_occlusions_with_a_depth_offset_are_unchanged(capi, synth):
    wl = synth.make_workload("c2", n_bodies=2, n_lines=64, n_points=64, n_divides=2, seed=9)
    synth.fill_depth_offsets(wl.region_model, 9)
    synth.fill_depth_offsets(wl.depth_model, 9)
    for body in range(wl.n_bodies):
        synth.add_occluder(wl, body, side="left" if body % 2 == 0 else "top", seed=9)
    wl.region = dataclasses.replace(wl.region, measure_occlusions=True, n_unoccluded_iterations=0)
    wl.depth = dataclasses.replace(wl.depth, measure_occlusions=True, n_unoccluded_iterations=0)
    a, b, _ = _pair(capi, synth, wl, offset=-25)
    _track_and_compare(wl, a, b)
    assert a.last_launch()["occ"] == 1
    a.close()
    b.close()


def test_viewer_images_are_unchanged(capi, synth):
    wl = synth.make_workload("c2", n_bodies=1, n_divides=2, seed=5)
    a, b, _ = _pair(capi, synth, wl)
    tri = np.array([[[-0.05, -0.05, 0.0], [0.05, -0.05, 0.0], [0.0, 0.05, 0.0]]], np.float32)
    W, H = wl.color_intrinsics.width, wl.color_intrinsics.height
    Wd, Hd = wl.depth_intrinsics.width, wl.depth_intrinsics.height
    out = []
    for ctx in (a, b):
        ctx.set_body_geometry(0, tri)
        ctx.set_viewer(0, "color", 0, [0])
        ctx.set_viewer(1, "depth", 0, [0], min_depth=0.3, max_depth=1.0)
        ctx.update_viewers()
        out.append(ctx.get_viewer_image(0, W, H) + ctx.get_viewer_image(1, Wd, Hd))
    for x, y in zip(*out):
        assert np.array_equal(x, y)
    a.close()
    b.close()


def test_launch_counts(capi, synth):
    """A camera without an undistortion launches what it did before; each upload call to cameras with one adds one
    launch, a batch one for all of them."""
    wl = synth.make_workload("c2", n_bodies=2, n_divides=2, seed=3)
    a, b, wl_b = _pair(capi, synth, wl)
    assert a.launch_count == b.launch_count + 2  # one colour batch, one depth batch
    base_a, base_b = a.launch_count, b.launch_count
    for ctx in (a, b):
        ctx.start_modalities(0)
        ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    assert a.launch_count - base_a == b.launch_count - base_b
    n = a.launch_count
    a.upload_color(0, np.ascontiguousarray(_color_raw(wl)[0]))  # one single upload: one launch
    assert a.launch_count == n + 1
    n = b.launch_count
    b.upload_color(0, np.ascontiguousarray(wl_b.color_frames[0]))  # plain upload: none
    assert b.launch_count == n
    a.close()
    b.close()


def test_lifecycle(capi, synth):
    m, intr = _golden(synth, "color_640x480")
    H, W = m.shape[:2]
    rng = np.random.default_rng(7)
    raw4 = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
    raw3 = np.ascontiguousarray(raw4[..., :3])
    ctx = capi.Context(max_cameras=2)
    ctx.set_color_camera(0, intr, EYE)
    ctx.set_camera_undistortion("color", 0, m, 4)
    ctx.upload_color(0, raw4)
    assert np.array_equal(ctx.get_camera_image("color", 0, W, H), ur.undistort_color(raw4, m))
    # a raw pitch below width * channels is refused
    with pytest.raises(capi.M3TBError):
        ctx._ck(ctx.L.m3tb_upload_color(ctx.h, 0, raw3.ctypes.data, raw3.strides[0]))
    # same size: the undistortion is kept
    ctx.set_color_camera(0, intr, EYE)
    ctx.upload_color(0, raw4)
    assert np.array_equal(ctx.get_camera_image("color", 0, W, H), ur.undistort_color(raw4, m))
    # another size drops it
    small = _intr(synth, 320, 240, 260.0, 260.0, 160.0, 120.0)
    ctx.set_color_camera(0, small, EYE)
    f = np.ascontiguousarray(raw3[:240, :320])
    ctx.upload_color(0, f)
    assert np.array_equal(ctx.get_camera_image("color", 0, 320, 240), f)
    # removing the map: uploads are plain again
    ctx.set_color_camera(1, intr, EYE)
    ctx.set_camera_undistortion("color", 1, m, 3)
    ctx.upload_color(1, raw3)
    assert np.array_equal(ctx.get_camera_image("color", 1, W, H), ur.undistort_color(raw3, m))
    ctx.set_camera_undistortion("color", 1, None, 3)
    ctx.upload_color(1, raw3)
    assert np.array_equal(ctx.get_camera_image("color", 1, W, H), raw3)
    # refusals
    for args in ((m, 2, 0), (m, 3, 5), (m[:, :W // 2], 3, 0)):
        with pytest.raises(capi.M3TBError):
            ctx.set_camera_undistortion("color", 1, *args)
    ctx.close()


def test_allocation_failures_leave_the_context_unchanged(capi, synth):
    m, intr = _golden(synth, "color_640x480")
    H, W = m.shape[:2]
    rng = np.random.default_rng(8)
    raw = rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)
    ctx = capi.Context(max_cameras=1)
    ctx.set_color_camera(0, intr, EYE)
    ctx.upload_color(0, raw[0])  # plain frame, images allocated
    live = capi.debug_resources()
    capi.debug_resources(1)
    with pytest.raises(capi.M3TBError):
        ctx.set_camera_undistortion("color", 0, m, 3)
    capi.debug_resources(0)
    assert capi.debug_resources() == live
    ctx.upload_color(0, raw[1])  # still no undistortion
    assert np.array_equal(ctx.get_camera_image("color", 0, W, H), raw[1])
    ctx.set_camera_undistortion("color", 0, m, 3)
    dev = _device(raw[0])
    ctx._ck(ctx.L.m3tb_upload_color_device(ctx.h, 0, C.c_void_p(dev.data_ptr()), W * 3))  # no staging needed
    before = ctx.get_camera_image("color", 0, W, H)
    assert np.array_equal(before, ur.undistort_color(raw[0], m))
    live = capi.debug_resources()
    capi.debug_resources(1)
    with pytest.raises(capi.M3TBError):
        ctx.upload_color(0, raw[1])  # the first staging allocation fails
    capi.debug_resources(0)
    assert capi.debug_resources() == live
    assert np.array_equal(ctx.get_camera_image("color", 0, W, H), before)
    ctx.upload_color(0, raw[1])
    assert np.array_equal(ctx.get_camera_image("color", 0, W, H), ur.undistort_color(raw[1], m))
    ctx.close()


def test_prefetch_and_detach_with_an_undistorted_camera(capi, synth):
    wl = synth.make_workload("c2", n_bodies=2, n_divides=2, seed=12)
    a, b, _ = _pair(capi, synth, wl)
    raw_c = _color_raw(wl)
    pin_c = _pinned(raw_c)
    for ctx in (a, b):
        ctx.start_modalities(0)
        ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    a.upload_batch_ptr(True, 0, wl.n_bodies, pin_c.data_ptr(), pin_c.stride(0), pin_c.stride(1))
    a.prefetch_frames()   # the undistorted cameras hold no pinned frame: nothing is prefetched
    a.detach_frames()     # and nothing is detached
    pin_c.fill_(3)        # so the caller may reuse the raw buffer
    for ctx in (a, b):
        ctx.tracking_step(1, wl.n_corr_iterations, wl.n_update_iterations)
    assert np.array_equal(a.get_poses().view(np.uint32), b.get_poses().view(np.uint32))
    a.close()
    b.close()


def test_mirror_example_equals_the_python_path(capi, synth, tmp_path):
    """examples/undistortion_selftest.cpp (AzureKinectColorCamera / AzureKinectDepthCamera) on the device."""
    pkg_build = __import__("importlib").import_module("3dobjecttracking_b200._build")
    lib = pkg_build.build_cuda()
    exe = str(tmp_path / "undistortion_selftest")
    csrc = os.path.dirname(lib)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "3dobjecttracking_b200", "host"), os.path.join(ROOT, "examples", "undistortion_selftest.cpp"),
           "-o", exe, "-L", csrc, "-lm3t_b200", "-Wl,-rpath," + csrc]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0, (r.stdout, r.stderr)
    import json
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["device"] == 1, out
    # the same calibration through the Python path
    for kind in ("color", "depth"):
        c = out[kind]
        raw_intr = _intr(synth, c["width"], c["height"], c["fx"], c["fy"], c["cx"], c["cy"])
        rect = _intr(synth, c["width"], c["height"], c["fu"], c["fv"], c["cx"], c["cy"])
        m = capi.undistortion_map(raw_intr, np.array(c["coefficients"], np.float32), rect)
        raw = np.fromfile(str(tmp_path / f"{kind}_raw.bin"), np.uint8 if kind == "color" else np.uint16)
        got = np.fromfile(str(tmp_path / f"{kind}_image.bin"), np.uint8 if kind == "color" else np.uint16)
        if kind == "color":
            raw = raw.reshape(c["height"], c["width"], 4)
            expect = ur.undistort_color(raw, m)
        else:
            raw = raw.reshape(c["height"], c["width"])
            expect = ur.undistort_depth(raw, m, c["depth_value_offset"])
        assert np.array_equal(got.reshape(expect.shape), expect), kind
