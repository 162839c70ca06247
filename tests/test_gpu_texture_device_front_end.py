"""The texture modality's device front end: k_texture_crop (m3tb_texture_crop) against cv2's crops in
tests/golden/texture_crops.npz, from pageable, device, pinned (prefetched) and undistorted frames and on an all-colours
frame; k_texture_features (m3tb_upload_texture_features_device) against the host upload, bit for bit, for ORB, SIFT and
DAISY, on rigid bodies, a kinematic chain and more than one launch's worth of bodies, and its refusals, stale-frame
rule and non-finite flag; the C++ mirror tracking through the device path (examples/texture_device_mirror_tracker.cpp)."""
import json
import os
import subprocess

import numpy as np
import pytest

import texture_crop_reference as cr

pytestmark = pytest.mark.gpu

FIX = np.load(os.path.join(os.path.dirname(__file__), "golden", "texture_crops.npz"))
W2C = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def _load_frame():
    path = os.path.join(os.path.dirname(__file__), "golden", "color_camera_image_200.png")
    try:
        import cv2
        return cv2.imread(path, cv2.IMREAD_COLOR)
    except ImportError:
        from PIL import Image
        rgb = np.asarray(Image.open(path).convert("RGB"))
        return np.ascontiguousarray(rgb[:, :, ::-1])


FIX_FRAME = _load_frame()


def _intr(capi, synth):
    fu, fv, ppu, ppv, w, h = (float(v) for v in FIX["intrinsics"])
    return synth.Intrinsics(fu, fv, ppu, ppv, int(w), int(h))


def _chain(synth):
    """Root with 6 DoF, two revolute children 3 cm apart along x (about z, then about y)."""
    I = synth.identity_pose
    links = [synth.LinkSpec(body=0, parent=-1, body2joint=I(), joint2parent=I()),
             synth.LinkSpec(body=1, parent=0, body2joint=I(), joint2parent=synth.translation_pose(0.03),
                            free_directions=(0, 0, 1, 0, 0, 0)),
             synth.LinkSpec(body=2, parent=1, body2joint=I(), joint2parent=synth.translation_pose(0.03),
                            free_directions=(0, 1, 0, 0, 0, 0))]
    return synth.StructureSpec(links=links, constraints=[], tikhonov_rotation=1000.0, tikhonov_translation=30000.0)


CHAIN_POSES = np.stack([np.hstack([np.eye(3), [[x], [0.0], [0.3]]]) for x in (-0.03, 0.0, 0.03)]).astype(np.float32)


def _scene(capi, synth, bodies=None, descriptor=None, upload=True, poses=None, chain=False, own_geometry=False):
    """One texture body per fixture pose (or the listed ones, or `poses`), depth modality with an empty depth frame;
    chain: the three bodies are the links of _chain; own_geometry: each renderer draws its own body only."""
    descriptor = capi.DESCRIPTOR_ORB if descriptor is None else descriptor
    if poses is None:
        poses = FIX["poses"] if bodies is None else FIX["poses"][list(bodies)]
    n = len(poses)
    intr = _intr(capi, synth)
    ctx = capi.Context(0, max_bodies=n, max_cameras=1, max_models=1)
    ctx.set_color_camera(0, intr, W2C)
    ctx.set_depth_camera(0, intr, W2C, 0.001)
    ctx.upload_depth(0, np.zeros((intr.height, intr.width), np.uint16))
    if upload:
        ctx.upload_color(0, FIX_FRAME)
    tri, diam = synth.prism_triangles()
    assert np.float32(diam) == FIX["diameter"]
    for b in range(n):
        ctx.set_body_geometry(b, tri, W2C, diam, True, body_id=b + 1, region_id=b + 1)
    ctx.generate_depth_model(0, 0, params=capi.model_params(n_divides=1, n_points=40, image_size=200))
    params = capi.texture_params_default()
    params.descriptor_type = descriptor
    params.focused_image_size = int(FIX["focused_image_size"])
    op = capi.OptimizerParams(1000.0, 30000.0)
    for b in range(n):
        ctx.set_body(b, None, capi.depth_params(), op, region_model=0, depth_model=0, color_camera=0, depth_camera=0)
    ctx.set_poses(poses)
    for b in range(n):
        ctx.set_focused_renderer(b, "color", 0, [b] if own_geometry else list(range(n)), [b], 200, id_type="body")
        ctx.set_texture_modality(b, params, 0)
        ctx.attach_renderer(b, "texture_silhouette", b)
    if chain:
        ctx.set_structure(0, _chain(synth))
    return ctx


def _crop(ctx, bodies, cap=(400, 400)):
    import torch
    cw, ch = cap
    out = torch.full((len(bodies), ch, cw), 0xAB, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    roi, scale, size, valid = ctx.texture_crop(bodies, out.data_ptr(), cw, cw * ch, cw, ch)
    ctx.synchronize()
    return out, roi, scale, size, valid


def _check_fixture(out, roi, scale, size, valid, idx):
    host = out.cpu().numpy()
    for k, i in enumerate(idx):
        assert valid[k]
        assert tuple(roi[k]) == tuple(FIX["rois"][i]) and scale[k] == FIX["scales"][i]
        w, h = FIX["sizes"][i]
        assert tuple(size[k]) == (w, h)
        assert np.array_equal(host[k, :h, :w], FIX["crops"][i, :h, :w]), (i, int((host[k, :h, :w] != FIX["crops"][i, :h, :w]).sum()))
        assert (host[k, :, w:] == 0xAB).all() and (host[k, h:, :] == 0xAB).all()  # nothing outside the crop


@pytest.mark.parametrize("source", ["pageable", "device", "pinned"])
def test_crops_equal_cv2(capi, synth, source):
    import torch
    ctx = _scene(capi, synth, upload=source == "pageable")
    n = len(FIX["poses"])
    if source == "device":
        dev = torch.from_numpy(FIX_FRAME).cuda()
        torch.cuda.synchronize()
        ctx._ck(ctx.L.m3tb_upload_color_device(ctx.h, 0, dev.data_ptr(), dev.stride(0)))
    elif source == "pinned":
        pin = torch.from_numpy(FIX_FRAME.copy()).pin_memory()
        pin_d = torch.zeros((FIX_FRAME.shape[0], FIX_FRAME.shape[1] * 2), dtype=torch.uint8).pin_memory()
        ctx.upload_batch_ptr(True, 0, 1, pin.data_ptr(), pin.stride(0) * pin.shape[0], pin.stride(0))
        ctx.upload_batch_ptr(False, 0, 1, pin_d.data_ptr(), pin_d.stride(0) * pin_d.shape[0], pin_d.stride(0))
        before = ctx.launch_count
        ctx.prefetch_frames()  # the ROI ingest runs on the side stream, the frame pool and camera tables swap
        assert ctx.launch_count == before + 1, "the prefetch did not take effect"
    # in a shuffled order, so the output slot follows the list
    order = list(np.random.default_rng(3).permutation(n))
    out, roi, scale, size, valid = _crop(ctx, order)
    _check_fixture(out, roi, scale, size, valid, order)
    focus_roi, focus_scale, _ = ctx.get_texture_focus()
    assert np.array_equal(roi, focus_roi[order]) and np.array_equal(scale, focus_scale[order])
    ctx.close()


def test_crops_of_an_undistorted_frame(capi, synth):
    ctx = _scene(capi, synth, upload=False)
    intr = _intr(capi, synth)
    k = np.array([0.05, -0.01, 5e-4, -5e-4, 2e-3, 0.03, -0.01, 2e-3], np.float32)
    ctx.set_camera_undistortion("color", 0, capi.undistortion_map(intr, k, intr), 3)
    ctx.upload_color(0, FIX_FRAME)
    rectified = ctx.get_camera_image("color", 0, intr.width, intr.height)
    assert not np.array_equal(rectified, FIX_FRAME)
    n = len(FIX["poses"])
    out, roi, scale, size, valid = _crop(ctx, list(range(n)))
    host = out.cpu().numpy()
    for b in range(n):
        w, h = size[b]
        assert np.array_equal(host[b, :h, :w], cr.crop(rectified, roi[b], scale[b]))
    ctx.close()


def test_grey_on_every_colour(capi, synth):
    """A 4097 x 4097 frame holding every BGR triple in its first 4096 x 4096 pixels, and a body so close that its focus
    region is the whole frame at a scale that keeps its size: the crop is the grey conversion of every triple."""
    ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
    intr = synth.Intrinsics(4000.0, 4000.0, 2048.0, 2048.0, 4097, 4097)
    ctx.set_color_camera(0, intr, W2C)
    ctx.set_depth_camera(0, intr, W2C, 0.001)
    ctx.upload_depth(0, np.zeros((intr.height, intr.width), np.uint16))
    v = np.arange(1 << 24, dtype=np.uint32).reshape(4096, 4096)
    frame = np.zeros((4097, 4097, 3), np.uint8)
    frame[:4096, :4096, 0], frame[:4096, :4096, 1], frame[:4096, :4096, 2] = v & 255, (v >> 8) & 255, v >> 16
    ctx.upload_color(0, frame)
    tri, diam = synth.prism_triangles()
    ctx.set_body_geometry(0, tri, W2C, diam, True, body_id=1, region_id=1)
    ctx.generate_depth_model(0, 0, params=capi.model_params(n_divides=1, n_points=40, image_size=200))
    ctx.set_body(0, None, capi.depth_params(), capi.OptimizerParams(1000.0, 30000.0), region_model=0, depth_model=0,
                 color_camera=0, depth_camera=0)
    pose = np.hstack([np.eye(3), [[0.0], [0.0], [0.07]]]).astype(np.float32)
    ctx.set_poses(pose[None])
    params = capi.texture_params_default()
    ctx.set_texture_modality(0, params, 0)
    (roi,), (scale,), _ = ctx.get_texture_focus()
    assert tuple(roi) == (0, 0, 4096, 4096)
    params.focused_image_size = int(round(200 / float(scale)))  # max(2 r_u, 2 r_v), so that the scale is about 1
    ctx.set_texture_modality(0, params, 0)
    (roi,), (scale,), _ = ctx.get_texture_focus()
    assert cr.output_size(4096, 4096, scale) == (4096, 4096), scale
    out, roi, scale, size, valid = _crop(ctx, [0], cap=(4096, 4096))
    assert valid[0] and tuple(size[0]) == (4096, 4096)
    assert np.array_equal(out[0].cpu().numpy(), cr.grey(frame[:4096, :4096]))
    ctx.close()


# ---- k_texture_features -------------------------------------------------------------------------------------------
TRACKED = [0, 1, 4, 9]  # fixture bodies with features on their crops


def _features(kind, b, rng=None):
    """(crop xy [n, 2] float32, descriptors) of fixture body b: ORB, SIFT, or DAISY-like unit vectors of length 104."""
    if kind == "orb":
        n = int(FIX["orb_n"][b])
        return FIX["orb_xy"][b, :n], FIX["orb_desc"][b, :n]
    n = int(FIX["sift_n"][b])
    if kind == "sift":
        return FIX["sift_xy"][b, :n], FIX["sift_desc"][b, :n]
    d = np.random.default_rng(100 + b).random((n, 104)).astype(np.float32)
    return FIX["sift_xy"][b, :n], (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def _device(capi, xy, desc, layout):
    """DeviceFeatures over torch tensors: keypoints interleaved (stride 2) or as the x and y rows of a [2, n] matrix
    (cv::cuda::ORB's GpuMat layout, stride 1); descriptors in rows of a wider pitch than their width."""
    import torch
    n = len(xy)
    if layout == "rows":
        kp = torch.from_numpy(np.ascontiguousarray(xy.T)).cuda()
        x, y, stride = kp.data_ptr(), kp.data_ptr() + kp.stride(0) * 4, 1
    else:
        kp = torch.from_numpy(np.ascontiguousarray(xy)).cuda()
        x, y, stride = kp.data_ptr(), kp.data_ptr() + 4, 2
    width = desc.shape[1]
    padded = np.zeros((max(n, 1), width + 8), desc.dtype)
    padded[:n, :width] = desc
    d = torch.from_numpy(padded).cuda()
    f = capi.DeviceFeatures(n, 0 if desc.dtype == np.uint8 else width, x, y, stride, d.data_ptr(),
                            d.stride(0) * d.element_size())
    return f, (kp, d)


def _descriptor(capi, kind):
    return {"orb": capi.DESCRIPTOR_ORB, "sift": capi.DESCRIPTOR_SIFT, "daisy": capi.DESCRIPTOR_DAISY}[kind]


def _frame_features(capi, ctx_h, ctx_d, kind, layout, keep, sources=TRACKED):
    """One frame's features (body b: those of fixture body sources[b]): host upload into ctx_h, device crop + device
    upload into ctx_d."""
    import torch
    n = len(sources)
    roi, scale, valid = ctx_h.get_texture_focus()
    for b in range(n):
        xy, desc = _features(kind, sources[b])
        ctx_h.upload_texture_features(b, xy, desc, roi[b][0], roi[b][1], scale[b])
    out, droi, dscale, _, dvalid = _crop(ctx_d, list(range(n)))
    assert np.array_equal(droi, roi) and np.array_equal(dscale, scale) and dvalid.all()
    fs = []
    for b in range(n):
        f, tensors = _device(capi, *_features(kind, sources[b]), layout)
        fs.append(f)
        keep.append(tensors)
    torch.cuda.synchronize()
    ctx_d.upload_texture_features_device(list(range(n)), fs)
    keep.append(out)


def _same(a, b):
    return np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


@pytest.mark.parametrize("kind,layout,chain", [("orb", "rows", False), ("orb", "interleaved", False),
                                               ("sift", "interleaved", False), ("daisy", "rows", False),
                                               ("orb", "interleaved", True), ("sift", "rows", True)])
def test_device_upload_equals_host_upload(capi, synth, kind, layout, chain):
    """Rigid bodies at fixture poses, or a textured 3-link chain (k_track + k_structure per update)."""
    sources = [0, 9, 4] if chain else TRACKED
    scene = dict(poses=CHAIN_POSES, chain=True) if chain else dict(bodies=TRACKED)
    ctx_h = _scene(capi, synth, descriptor=_descriptor(capi, kind), **scene)
    ctx_d = _scene(capi, synth, descriptor=_descriptor(capi, kind), **scene)
    if chain:
        assert ctx_h.n_structures() == 1 and ctx_d.n_structures() == 1
    keep = []
    _frame_features(capi, ctx_h, ctx_d, kind, layout, keep, sources)
    ctx_h.start_modalities(0)
    ctx_d.start_modalities(0)
    total = 0
    for b in range(len(sources)):
        kh, kd = ctx_h.get_texture_keyframes(b), ctx_d.get_texture_keyframes(b)
        assert _same(kh["sizes"], kd["sizes"]) and _same(kh["points"], kd["points"])
        assert _same(kh["descriptors"], kd["descriptors"])
        total += int(kh["sizes"].sum())
    assert total > 50
    for it in (1, 2):
        for ctx in (ctx_h, ctx_d):
            ctx.upload_color(0, FIX_FRAME)  # the next frame
        _frame_features(capi, ctx_h, ctx_d, kind, layout, keep, sources)
        for ctx in (ctx_h, ctx_d):
            ctx.texture_correspondences(it, 0)
        points = 0
        for b in range(len(sources)):
            ph = ctx_h.get_texture_points(b)
            assert _same(ph, ctx_d.get_texture_points(b))
            points += len(ph)
        assert points > 20
        gh, Hh = ctx_h.texture_gradient_hessian(it, 0, 0)
        gd, Hd = ctx_d.texture_gradient_hessian(it, 0, 0)
        assert _same(gh, gd) and _same(Hh, Hd)
        for ctx in (ctx_h, ctx_d):
            ctx.tracking_step(it, 2, 2)
            ctx.calculate_results(it)
        assert _same(ctx_h.get_poses(), ctx_d.get_poses())
        for b in range(len(sources)):
            kh, kd = ctx_h.get_texture_keyframes(b), ctx_d.get_texture_keyframes(b)
            assert _same(kh["points"], kd["points"]) and _same(kh["descriptors"], kd["descriptors"])
    assert not ctx_d.get_texture_feature_flags().any()
    ctx_h.close()
    ctx_d.close()


def test_refusals_stale_frames_and_the_non_finite_flag(capi, synth):
    import torch
    ctx = _scene(capi, synth, [0, 1], capi.DESCRIPTOR_SIFT)
    keep = []

    def dev(b, kind="sift", n=None, length=None):
        xy, desc = _features(kind, [0, 1][b])
        if n is not None:
            xy, desc = np.resize(xy, (n, 2)).astype(np.float32), np.resize(desc, (n, desc.shape[1])).astype(desc.dtype)
        if length is not None:
            desc = np.ascontiguousarray(np.resize(desc, (len(desc), length)), np.float32)
        f, t = _device(capi, xy, desc, "interleaved")
        keep.append(t)
        torch.cuda.synchronize()
        return f

    def refused(code, bodies, fs):
        before = ctx.launch_count
        with pytest.raises(capi.M3TBError, match="status %d" % code):
            ctx.upload_texture_features_device(bodies, fs)
        assert ctx.launch_count == before  # nothing launched

    # no crop yet
    refused(-1, [0], [dev(0)])
    _crop(ctx, [0, 1])
    refused(-3, [0], [dev(0, n=513)])
    refused(-1, [0], [dev(0, kind="orb")])      # ORB rows for a SIFT body
    refused(-1, [0], [dev(0, length=104)])      # SIFT is 128 long
    refused(-1, [0, 0], [dev(0), dev(0)])       # listed twice
    refused(-1, [0, 1], [dev(0), dev(1, kind="orb")])     # one refused body: nothing is launched or recorded
    ctx.start_modalities(0)  # so body 0 has no features: no keyframe points
    assert int(ctx.get_texture_keyframes(0)["sizes"].sum()) == 0
    before = ctx.launch_count
    ctx.upload_texture_features_device([0, 1], [dev(0), dev(1)])
    assert ctx.launch_count == before + 1
    # a newer frame makes the crop stale
    ctx.upload_color(0, FIX_FRAME)
    refused(-1, [0], [dev(0)])
    _crop(ctx, [0])
    ctx.upload_texture_features_device([0], [dev(0)])
    refused(-1, [1], [dev(1)])  # body 1 was not cropped on this frame
    # a non-finite value: no features for that body, its flag raised; the other body is unaffected
    _crop(ctx, [0, 1])
    xy, desc = _features("sift", 1)
    desc = desc.copy()
    desc[3, 17] = np.nan
    f1, t = _device(capi, xy, desc, "interleaved")
    keep.append(t)
    torch.cuda.synchronize()
    ctx.upload_texture_features_device([0, 1], [dev(0), f1])
    assert list(ctx.get_texture_feature_flags()) == [False, True]
    ctx.start_modalities(0)
    assert int(ctx.get_texture_keyframes(0)["sizes"].sum()) > 0
    assert int(ctx.get_texture_keyframes(1)["sizes"].sum()) == 0
    # a crop larger than the capacity: refused with nothing launched, the sizes reported, the last crops kept
    _, _, _, sizes, _ = _crop(ctx, [0, 1])
    out = torch.zeros((2, 8, 8), dtype=torch.uint8, device="cuda")
    ids = np.array([0, 1], np.int32)
    roi, scale = np.zeros((2, 4), np.int32), np.zeros(2, np.float32)
    size, valid = np.full((2, 2), -1, np.int32), np.zeros(2, np.int32)
    import ctypes as C
    ip = C.POINTER(C.c_int)
    before = ctx.launch_count
    rc = ctx.L.m3tb_texture_crop(ctx.h, ids.ctypes.data_as(ip), 2, C.c_void_p(out.data_ptr()), 8, 64, 8, 8,
                                 roi.ctypes.data_as(ip), scale.ctypes.data_as(C.POINTER(C.c_float)),
                                 size.ctypes.data_as(ip), valid.ctypes.data_as(ip))
    assert rc == -1 and ctx.launch_count == before
    assert np.array_equal(size, sizes) and valid.all()
    ctx.upload_texture_features_device([0, 1], [dev(0), dev(1)])  # still the crops of this frame
    assert list(ctx.get_texture_feature_flags()) == [False, False]
    # setting the modality again clears the body's flag
    ctx.upload_texture_features_device([1], [f1])
    assert list(ctx.get_texture_feature_flags()) == [False, True]
    params = capi.texture_params_default()
    params.descriptor_type = capi.DESCRIPTOR_SIFT
    ctx.set_texture_modality(1, params, 0)
    assert list(ctx.get_texture_feature_flags()) == [False, False]
    ctx.close()


def test_more_bodies_than_one_launch_takes(capi, synth):
    """131 bodies: k_texture_crop and k_texture_features each split into two launches."""
    n = 131
    src = [b % len(FIX["poses"]) for b in range(n)]
    ctx_h = _scene(capi, synth, poses=FIX["poses"][src], own_geometry=True)
    ctx_d = _scene(capi, synth, poses=FIX["poses"][src], own_geometry=True)
    order = list(np.random.default_rng(7).permutation(n))
    before = ctx_d.launch_count
    out, roi, scale, size, valid = _crop(ctx_d, order)
    assert ctx_d.launch_count == before + 2
    _check_fixture(out, roi, scale, size, valid, [src[b] for b in order])
    del out
    keep = []
    before = ctx_d.launch_count
    _frame_features(capi, ctx_h, ctx_d, "orb", "interleaved", keep, src)
    assert ctx_d.launch_count == before + 4  # two crop and two feature launches
    ctx_h.start_modalities(0)
    ctx_d.start_modalities(0)
    for b in range(n):
        kh, kd = ctx_h.get_texture_keyframes(b), ctx_d.get_texture_keyframes(b)
        assert _same(kh["sizes"], kd["sizes"]) and _same(kh["points"], kd["points"])
        assert _same(kh["descriptors"], kd["descriptors"])
    ctx_h.close()
    ctx_d.close()


@pytest.mark.parametrize("descriptor", ["orb", "sift"])
def test_cpp_mirror_tracks_through_the_device_path(pkg, tmp_path, descriptor):
    """examples/texture_device_mirror_tracker.cpp: a rigid body and a 3-link chain tracked by Tracker::ExecuteTrackingStep
    with features from TextureModality::CropFocusedImages + SetFeatures(const m3tb_device_features&), against the same
    scene through the host SetFeatures; with SIFT, a non-finite descriptor of body 0 drops its features and is reported."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg._build.build_cuda()
    pkg._build.build_synth()
    csrc = os.path.join(root, "3dobjecttracking_b200", "csrc")
    synth_dir = os.path.join(root, "3dobjecttracking_b200", "synth")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "texture_device_mirror_tracker")
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(root, "include"), "-I",
           os.path.join(root, "3dobjecttracking_b200", "host"), "-I", synth_dir, "-I", os.path.join(cuda, "include"),
           os.path.join(root, "examples", "texture_device_mirror_tracker.cpp"), "-o", exe, "-L", csrc, "-L", synth_dir,
           "-L", os.path.join(cuda, "lib64"), "-lm3t_b200", "-lm3t_synth", "-lcudart", "-Wl,-rpath," + csrc,
           "-Wl,-rpath," + synth_dir, "-Wl,-rpath," + os.path.join(cuda, "lib64"), "-fopenmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, "1", "300", descriptor], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    out = json.loads(r.stdout.strip().split("\n")[-1])
    assert min(out["texture_points_host"]) > 20 and out["texture_points_device"] == out["texture_points_host"]
    host, dev = (np.array(out[k], np.float32).reshape(-1, 12) for k in ("host", "device"))
    assert _same(host, dev)
    start, gt = (np.array(out[k], np.float32).reshape(-1, 3, 4) for k in ("start", "gt"))
    assert np.abs(dev.reshape(-1, 3, 4) - gt).max() < np.abs(start - gt).max()
    if descriptor == "sift":
        assert out["features_dropped"] == [1, 0, 0, 0]
        assert out["texture_points_dropped"][0] == 0 and out["texture_points_dropped"][1:] == out["texture_points_host"][1:]
        assert _same(np.array(out["dropped"], np.float32).reshape(-1, 12)[1:], host[1:])  # the chain is untouched
        assert "non-finite texture descriptor" in r.stderr
