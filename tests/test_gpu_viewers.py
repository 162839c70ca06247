"""Device viewers (m3tb_set_viewer / m3tb_update_viewers / m3tb_get_viewer_image, k_view_setup / k_view_raster /
k_view_resolve): normal images and blended viewer images equal the CPU restatement (tests/viewer_reference.py) bit for
bit at several frame sizes, for both viewer kinds and every frame source; viewers render the poses of the last tracking
step and never change what tracking computes; refused and failed calls leave the viewers as they were."""
import numpy as np
import pytest

import render_reference as rr
import viewer_reference as vr

pytestmark = pytest.mark.gpu

I34 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
W2C_DEPTH = np.hstack([np.eye(3), np.array([[-0.02], [0.005], [0.01]])]).astype(np.float32)


def _pose(rot_deg=(0.0, 0.0, 0.0), t=(0.0, 0.0, 0.5)):
    R = np.eye(3)
    for axis, deg in enumerate(rot_deg):
        c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
        i, j = [k for k in range(3) if k != axis]
        Q = np.eye(3)
        Q[i, i], Q[i, j], Q[j, i], Q[j, j] = c, -s, s, c
        R = R @ Q
    return np.hstack([R, np.array(t)[:, None]]).astype(np.float32)


def _intr(capi, W, H):
    return capi.Intrinsics(0.96 * W, 0.955 * W, 0.52 * W - 3.3, 0.47 * H + 2.1, W, H)


def _frame(kind, W, H, seed):
    rng = np.random.default_rng(seed)
    if kind == "color":
        return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    return rng.integers(0, 1300, (H, W), dtype=np.uint16)


def _mesh(synth, mesh, culling=True, n_divides=4):
    if mesh == "prism":
        tri, diam = synth.prism_triangles()
    else:
        tri, diam = synth.icosphere_triangles(0.04, n_divides)
    return rr.Geometry(tri, I34.copy(), diam, culling)


def _expected(kind, intr, w2c, poses, geometry, bodies, frame, opacity, depth_scale, min_depth, max_depth):
    normal, _ = vr.render_normal(intr, w2c, poses, geometry, bodies)
    return vr.viewer_image(kind, frame, normal, opacity, depth_scale, min_depth, max_depth), normal


def _setup(capi, geometry, poses, cams, max_bodies=None):
    """cams: [(kind, intr, w2c, depth_scale)]; camera c of its kind is cams[c]."""
    nb = max_bodies or (max(max(geometry), max(poses)) + 1)
    ctx = capi.Context(0, max_bodies=nb, max_cameras=len(cams), max_models=1)
    for c, (kind, intr, w2c, ds) in enumerate(cams):
        if kind == "color":
            ctx.set_color_camera(c, intr, w2c)
        else:
            ctx.set_depth_camera(c, intr, w2c, ds)
    ctx.set_poses(np.stack([poses.get(b, I34) for b in range(nb)]))
    for b, g in geometry.items():
        ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling)
    return ctx


def _upload(ctx, kind, cam, frame):
    (ctx.upload_color if kind == "color" else ctx.upload_depth)(cam, np.ascontiguousarray(frame))


def _check(ctx, viewer, kind, intr, w2c, poses, geometry, bodies, frame, opacity=0.5, depth_scale=0.001,
           min_depth=0.0, max_depth=1.0):
    img, normal = ctx.get_viewer_image(viewer, intr.width, intr.height)
    exp_img, exp_normal = _expected(kind, intr, w2c, poses, geometry, bodies, frame, opacity, depth_scale, min_depth,
                                    max_depth)
    assert np.array_equal(normal, exp_normal), np.argwhere(np.any(normal != exp_normal, axis=2))[:5]
    assert np.array_equal(img, exp_img), np.argwhere(np.any(img != exp_img, axis=2))[:5]
    return exp_normal


def _scene(synth, scene, W):
    """geometry, poses and draw order of a scene; bodies sit closer to the camera at larger frames"""
    near = 0.35 if W < 1000 else 0.2
    if scene == "prism":
        return {0: _mesh(synth, "prism")}, {0: _pose((25, -30, 10), (0.01, -0.005, near - 0.15))}, [0]
    if scene == "icosphere":
        return {0: _mesh(synth, "icosphere")}, {0: _pose((10, 5, 0), (0.02, 0.01, near))}, [0]
    if scene == "icosphere_nocull":
        g = _mesh(synth, "icosphere", culling=False)
        return {0: g}, {0: _pose((40, 5, 0), (-0.03, 0.01, near))}, [0]
    # 8 overlapping bodies: equal copies at the same pose (equal-depth ties: the body drawn first wins), culling mixed
    rng = np.random.default_rng(W)
    geometry, poses = {}, {}
    for b in range(8):
        geometry[b] = _mesh(synth, "prism" if b % 2 == 0 else "icosphere", culling=b % 3 != 2, n_divides=2)
        poses[b] = _pose(tuple(rng.uniform(-40, 40, 3)), (rng.uniform(-0.06, 0.06), rng.uniform(-0.05, 0.05),
                                                          rng.uniform(near, near + 0.2)))
    poses[2] = poses[0].copy()
    poses[3] = poses[1].copy()
    return geometry, poses, [3, 1, 0, 2, 4, 5, 6, 7]


@pytest.mark.parametrize("size", [(640, 480), (1280, 720), (333, 217)])
@pytest.mark.parametrize("scene", ["prism", "icosphere", "icosphere_nocull", "bodies8"])
@pytest.mark.parametrize("kind", ["color", "depth"])
def test_viewer_bit_exact(capi, synth, kind, scene, size):
    W, H = size
    intr = _intr(capi, W, H)
    w2c = I34 if kind == "color" else W2C_DEPTH
    geometry, poses, bodies = _scene(synth, scene, W)
    ctx = _setup(capi, geometry, poses, [(kind, intr, w2c, 0.00025)])
    frame = _frame(kind, W, H, W + len(bodies))
    _upload(ctx, kind, 0, frame)
    opacity, min_depth, max_depth = (0.5, 0.0, 1.0) if kind == "color" else (0.3, 0.1, 0.4)
    ctx.set_viewer(0, kind, 0, bodies, opacity, min_depth, max_depth)
    n0 = ctx.launch_count
    ctx.update_viewers()
    assert ctx.launch_count == n0 + 3
    normal = _check(ctx, 0, kind, intr, w2c, poses, geometry, bodies, frame, opacity, 0.00025, min_depth, max_depth)
    covered = (normal[..., 3] == 255).mean()
    assert covered > (0.1 if scene != "prism" and W >= 1000 else 0.005)  # large on-screen triangles at 1280x720
    if scene == "bodies8":  # the tie is visible: body 3 is drawn before body 1 at the same pose
        ctx.update_viewers()  # a second update from the cleared z-buffers gives the same bytes
        _check(ctx, 0, kind, intr, w2c, poses, geometry, bodies, frame, opacity, 0.00025, min_depth, max_depth)
    ctx.close()


def test_near_plane_border_and_nothing_visible(capi, synth):
    W, H = 640, 480
    intr = _intr(capi, W, H)
    geometry = {0: _mesh(synth, "icosphere", culling=False, n_divides=3), 1: _mesh(synth, "prism", culling=False),
                2: _mesh(synth, "prism")}
    cases = [  # body 0 crosses the near plane z = 0.02, body 1 is cut by the image border, body 2 is behind the camera
        ({0: _pose(t=(-0.03, 0.0, 0.05)), 1: _pose((0, 30, 0), (0.19, 0.0, 0.4)), 2: _pose(t=(0, 0, -0.5))}, [0, 1, 2]),
        ({0: _pose(t=(0.0, 0.0, -1.0)), 1: _pose(t=(3.0, 0.0, 0.5)), 2: _pose(t=(0, 0, 20.0))}, [0, 1, 2]),
    ]
    frame = _frame("color", W, H, 5)
    for k, (poses, bodies) in enumerate(cases):
        ctx = _setup(capi, geometry, poses, [("color", intr, I34, 0.001)])
        _upload(ctx, "color", 0, frame)
        ctx.set_viewer(0, "color", 0, bodies)
        ctx.update_viewers()
        normal = _check(ctx, 0, "color", intr, I34, poses, geometry, bodies, frame)
        if k == 1:
            assert not normal.any()
        else:  # the near-plane cut of body 0 reaches the top row, body 1 the right border
            assert normal[0, :, 3].any() and normal[:, -1, 3].any()
        ctx.close()


def test_two_viewers_two_cameras_one_update(capi, synth):
    ci, di = _intr(capi, 640, 480), _intr(capi, 333, 217)
    geometry, poses, _ = _scene(synth, "bodies8", 640)
    nb = 8
    ctx = capi.Context(0, max_bodies=nb, max_cameras=2, max_models=1)
    ctx.set_color_camera(1, ci, I34)
    ctx.set_depth_camera(0, di, W2C_DEPTH, 0.001)
    ctx.set_poses(np.stack([poses[b] for b in range(nb)]))
    for b, g in geometry.items():
        ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling)
    fc, fd = _frame("color", 640, 480, 1), _frame("depth", 333, 217, 2)
    _upload(ctx, "color", 1, fc)
    _upload(ctx, "depth", 0, fd)
    ctx.set_viewer(0, "color", 1, [0, 1, 2, 3], 0.7)
    ctx.set_viewer(1, "depth", 0, [7, 6, 5, 4, 3], 0.5, 0.2, 0.6)
    n0 = ctx.launch_count
    ctx.update_viewers()
    assert ctx.launch_count == n0 + 3
    _check(ctx, 0, "color", ci, I34, poses, geometry, [0, 1, 2, 3], fc, 0.7)
    _check(ctx, 1, "depth", di, W2C_DEPTH, poses, geometry, [7, 6, 5, 4, 3], fd, 0.5, 0.001, 0.2, 0.6)
    ctx.close()


def _workload(synth):
    return synth.make_workload("c2", n_bodies=2, n_divides=2, seed=1)


def _pinned(wl):
    import torch
    c = torch.from_numpy(np.ascontiguousarray(wl.color_frames)).pin_memory()
    d = np.ascontiguousarray(wl.depth_frames).view(np.uint8).reshape(wl.n_bodies, wl.depth_intrinsics.height, -1)
    return c, torch.from_numpy(d).pin_memory()


def _workload_context(capi, synth, wl, upload):
    if upload == "full":
        ctx = capi.context_from_workload(wl)
        pin = None
    else:
        ctx = capi.context_from_workload(wl, upload_frames=False)
        pin = _pinned(wl)
        for t, color in ((pin[0], True), (pin[1], False)):
            ctx.upload_batch_ptr(color, 0, wl.n_bodies, t.data_ptr(), t.stride(0), t.stride(1))
        if upload == "prefetch":
            ctx.prefetch_frames()
    g = _mesh(synth, "icosphere", n_divides=3)
    for b in range(wl.n_bodies):
        ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling)
    ctx.set_viewer(0, "color", 0, list(range(wl.n_bodies)), 0.6)
    ctx.set_viewer(1, "depth", 1, list(range(wl.n_bodies))[::-1], 0.5, 0.3, 0.7)
    return ctx, pin, g


def _viewer_bytes(ctx, wl):
    ci, di = wl.color_intrinsics, wl.depth_intrinsics
    return [ctx.get_viewer_image(0, ci.width, ci.height), ctx.get_viewer_image(1, di.width, di.height)]


@pytest.mark.parametrize("upload", ["pinned", "prefetch"])
def test_pinned_and_prefetched_frames_match_pageable(capi, synth, upload):
    wl = _workload(synth)
    ref, _, _ = _workload_context(capi, synth, wl, "full")
    ref.update_viewers()
    exp = _viewer_bytes(ref, wl)
    ref.close()
    ctx, pin, _ = _workload_context(capi, synth, wl, upload)
    ctx.update_viewers()
    got = _viewer_bytes(ctx, wl)
    for (a, b), (c, d) in zip(got, exp):
        assert np.array_equal(a, c) and np.array_equal(b, d)
    ctx.synchronize()
    ctx.close()
    del pin


def test_viewer_renders_the_tracked_poses(capi, synth):
    wl = _workload(synth)
    ctx, _, g = _workload_context(capi, synth, wl, "full")
    ctx.start_modalities(0)
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    ctx.update_viewers()
    poses = {b: p for b, p in enumerate(ctx.get_poses())}
    assert not np.array_equal(poses[0], wl.start_body2world[0].astype(np.float32))
    geometry = {b: g for b in range(wl.n_bodies)}
    W, H = wl.color_intrinsics.width, wl.color_intrinsics.height
    frame = wl.color_frames[0][:, :3 * W].reshape(H, W, 3)
    _check(ctx, 0, "color", wl.color_intrinsics, wl.color_world2camera, poses, geometry, [0, 1], frame, 0.6)
    ctx.close()


def test_tracking_is_unchanged_by_viewer_updates(capi, synth):
    wl = _workload(synth)
    runs = []
    for with_viewers in (False, True):
        ctx, _, _ = _workload_context(capi, synth, wl, "full")
        ctx.start_modalities(0)
        out = []
        for it in range(3):
            ctx.tracking_step(it, wl.n_corr_iterations, wl.n_update_iterations)
            if with_viewers:
                ctx.update_viewers()
            out.append(ctx.get_poses().copy())
            for b in range(wl.n_bodies):
                out.append(np.ascontiguousarray(ctx.get_region_lines(b, 4096)).view(np.uint8).copy())
                out.append(np.ascontiguousarray(ctx.get_depth_points(b, 4096)).view(np.uint8).copy())
        runs.append(out)
        ctx.close()
    for a, b in zip(*runs):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


def test_refusals(capi, synth):
    intr = _intr(capi, 320, 240)
    geometry = {0: _mesh(synth, "prism")}
    ctx = _setup(capi, geometry, {0: _pose()}, [("color", intr, I34, 0.001)], max_bodies=2)
    L, h = ctx.L, ctx.h
    ip = np.array([0], np.int32)
    p = ip.ctypes.data_as(capi.C.POINTER(capi.C.c_int))
    assert L.m3tb_set_viewer(h, 1, 0, 0, p, 1, 0.5, 0.0, 1.0) == -1    # ids are dense
    assert L.m3tb_set_viewer(h, 0, 2, 0, p, 1, 0.5, 0.0, 1.0) == -1    # bad kind
    assert L.m3tb_set_viewer(h, 0, 1, 0, p, 1, 0.5, 0.0, 1.0) == -1    # depth camera 0 is not set
    assert L.m3tb_set_viewer(h, 0, 0, 1, p, 1, 0.5, 0.0, 1.0) == -1    # camera out of range
    bad = np.array([1], np.int32)                                        # body 1 has no geometry
    assert L.m3tb_set_viewer(h, 0, 0, 0, bad.ctypes.data_as(capi.C.POINTER(capi.C.c_int)), 1, 0.5, 0.0, 1.0) == -1
    twice = np.array([0, 0], np.int32)
    assert L.m3tb_set_viewer(h, 0, 0, 0, twice.ctypes.data_as(capi.C.POINTER(capi.C.c_int)), 2, 0.5, 0.0, 1.0) == -1
    assert L.m3tb_get_viewer_image(h, 0, None, 0, None, 0) == -1       # no viewer
    n0 = ctx.launch_count
    assert L.m3tb_update_viewers(h) == 0 and ctx.launch_count == n0    # no viewer: nothing launched
    ctx.set_viewer(0, "color", 0, [0])
    assert L.m3tb_get_viewer_image(h, 0, None, 0, None, 0) == -4       # not updated yet
    assert L.m3tb_update_viewers(h) == -4                                # the camera has no frame
    assert ctx.launch_count == n0
    frame = _frame("color", 320, 240, 1)
    _upload(ctx, "color", 0, frame)
    ctx.update_viewers()
    img = np.zeros((240, 320, 3), np.uint8)
    assert L.m3tb_get_viewer_image(h, 0, img.ctypes.data, 3 * 320 - 1, None, 0) == -1  # pitch below a row
    _check(ctx, 0, "color", intr, I34, {0: _pose()}, geometry, [0], frame)
    ctx.close()


def test_failed_allocations_leave_viewers_as_they_were(capi, synth):
    """Every allocating viewer call refused at each of its resource creations keeps the resource count, and the next
    update is bit-identical to that of a context that never failed."""
    intr, intr2 = _intr(capi, 320, 240), _intr(capi, 200, 150)
    geometry, poses, bodies = _scene(synth, "bodies8", 320)
    frame, frame2 = _frame("color", 320, 240, 3), _frame("color", 200, 150, 4)

    def fresh():
        ctx = _setup(capi, geometry, poses, [("color", intr, I34, 0.001)])
        _upload(ctx, "color", 0, frame)
        return ctx

    def resize(c):  # the camera changes size; its new frame is a private image (made here, not by the viewers)
        c.set_color_camera(0, intr2, I34)
        _upload(c, "color", 0, frame2)

    calls = [  # (name, what precedes the call, the allocating viewer call)
        ("set_viewer", None, lambda c: c.set_viewer(0, "color", 0, bodies, 0.4)),
        ("update_viewers", None, lambda c: c.update_viewers()),
        ("set_viewer_again", None, lambda c: c.set_viewer(1, "color", 0, bodies[:3], 0.9)),
        ("update_after_resize", resize, lambda c: c.update_viewers()),
    ]

    def run(ctx, entries):
        for _, prefix, call in entries:
            if prefix:
                prefix(ctx)
            call(ctx)

    for n_done in range(len(calls)):
        k = 1
        while True:
            ctx = fresh()
            run(ctx, calls[:n_done])
            if calls[n_done][1]:
                calls[n_done][1](ctx)
            ctx.synchronize()
            live = capi.debug_resources(-1)
            capi.debug_resources(k)
            try:
                calls[n_done][2](ctx)
                failed = False
            except capi.M3TBError:
                failed = True
            finally:
                capi.debug_resources(0)
            if not failed:
                ctx.close()
                break
            assert capi.debug_resources(-1) == live, (calls[n_done][0], k)
            # the context goes on: the remaining calls and one more update equal a context that never failed
            calls[n_done][2](ctx)
            run(ctx, calls[n_done + 1:])
            ctx.update_viewers()
            ref = fresh()
            run(ref, calls)
            ref.update_viewers()
            for v in range(2):
                a = ctx.get_viewer_image(v, 200, 150)
                b = ref.get_viewer_image(v, 200, 150)
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (calls[n_done][0], k, v)
            ref.close()
            ctx.close()
            k += 1
        assert k > 1, calls[n_done][0]  # the call creates at least one resource
