"""Device focused normal renderers (m3tb_set_focused_normal_renderer / m3tb_render_focused_normals /
m3tb_get_focused_normal_rendering, k_view_focus + k_view_* with VK_FOCUSED): focus, depth and normal images equal the
CPU restatement (tests/focused_normal_reference.py) bit for bit for one and several bodies, unreferenced occluders,
culling on and off, referenced bodies partly outside the camera or invisible, colour and depth cameras and image sizes
32 to 333; the depth image and focus equal those of a device focused renderer (k_render); reads into device memory
equal host reads; refused and failed calls leave the context as it was; and contexts that render focused normals track
and launch as before."""
import numpy as np
import pytest

import focused_normal_reference as fn
from test_gpu_viewers import I34, W2C_DEPTH, _intr, _mesh, _pose, _scene, _workload

pytestmark = pytest.mark.gpu

FOCUS_KEYS = ("corner_u", "corner_v", "scale", "projection_term_a", "projection_term_b")


def _context(capi, geometry, poses, cams, max_bodies=None):
    """cams: [(kind, intr, w2c)]; colour and depth cameras are numbered separately, in list order."""
    nb = max_bodies or (max(max(geometry), max(poses)) + 1)
    ctx = capi.Context(0, max_bodies=nb, max_cameras=len(cams), max_models=1)
    index = {"color": 0, "depth": 0}
    for kind, intr, w2c in cams:
        if kind == "color":
            ctx.set_color_camera(index[kind], intr, w2c)
        else:
            ctx.set_depth_camera(index[kind], intr, w2c, 0.001)
        index[kind] += 1
    ctx.set_poses(np.stack([poses.get(b, I34) for b in range(nb)]))
    for b, g in geometry.items():
        ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling, g.body_id,
                              g.region_id)
    return ctx


def _scene_mixed(capi, synth):
    """The viewers' eight overlapping bodies (culling mixed, equal copies at equal poses), body 8 (not culled) half
    outside the colour camera's right border, body 9 behind both cameras (never visible)."""
    geometry, poses, order = _scene(synth, "bodies8", 640)
    geometry[8] = _mesh(synth, "icosphere", culling=False, n_divides=3)
    poses[8] = _pose((0, 20, 0), (0.27, 0.0, 0.45))
    geometry[9] = _mesh(synth, "prism")
    poses[9] = _pose(t=(0.0, 0.0, -0.5))
    cams = [("color", _intr(capi, 640, 480), I34), ("depth", _intr(capi, 333, 217), W2C_DEPTH)]
    # (camera kind, image size, z range, geometry bodies, referenced bodies)
    renderers = [("color", 200, (0.02, 10.0), [0], [0]),                 # one body
                 ("color", 32, (0.1, 2.0), order, [0, 1, 4]),            # several bodies, tiny image
                 ("depth", 333, (0.02, 10.0), order + [8], [5]),         # occluders drawn, not referenced; above 240
                 ("color", 200, (0.05, 3.0), [8] + order, [8]),          # referenced body partly outside the camera
                 ("color", 64, (0.02, 10.0), [9, 0, 1], [9]),            # invisible: nothing is drawn
                 ("depth", 200, (0.02, 10.0), [9, 6, 7, 8], [9, 6, 7]),  # one invisible of three
                 ("color", 240, (0.3, 0.45), order, [2, 3])]             # narrow z range: body 2 is not visible
    return geometry, poses, cams, renderers


def _cam(cams, kind):
    return [c for c in cams if c[0] == kind][0]


def _expected(cams, poses, geometry, r):
    kind, S, (z0, z1), bodies, ref = r
    _, intr, w2c = _cam(cams, kind)
    return fn.render_focused_normal(intr, w2c, poses, geometry, bodies, ref, S, z0, z1)


def _check(got, exp, tag):
    assert np.array_equal(got["depth"], exp["depth"]), (tag, np.argwhere(got["depth"] != exp["depth"])[:5])
    assert np.array_equal(got["normal"], exp["normal"]), (tag, np.argwhere(np.any(got["normal"] != exp["normal"], 2))[:5])
    for key in FOCUS_KEYS:
        assert got[key].tobytes() == np.float32(exp[key]).tobytes(), (tag, key, got[key], exp[key])
    assert np.array_equal(got["visible"], exp["visible"]), tag


def test_against_restatement_many_renderers_one_render(capi, synth):
    geometry, poses, cams, renderers = _scene_mixed(capi, synth)
    ctx = _context(capi, geometry, poses, cams)
    for r, (kind, S, (z0, z1), bodies, ref) in enumerate(renderers):
        ctx.set_focused_normal_renderer(r, kind, 0, bodies, ref, S, z0, z1)
    n0 = ctx.launch_count
    ctx.render_focused_normals()
    assert ctx.launch_count == n0 + 4
    for rep in range(2):  # a second render from the cleared z-buffers gives the same bytes
        for r, spec in enumerate(renderers):
            exp = _expected(cams, poses, geometry, spec)
            _check(ctx.get_focused_normal_rendering(r), exp, (rep, r))
            drawn = (exp["depth"] != 65535).mean()
            assert (drawn == 0) == (r == 4), (r, drawn)  # every renderer but the invisible one draws something
        ctx.render_focused_normals()
    exp = [_expected(cams, poses, geometry, spec) for spec in renderers]
    assert list(exp[5]["visible"]) == [0, 1, 1] and list(exp[4]["visible"]) == [0] and list(exp[6]["visible"]) == [0, 1]
    # the partly outside body: its focus reaches beyond the image border
    assert exp[3]["corner_u"] + np.float32(200) / exp[3]["scale"] > 640
    ctx.close()


@pytest.mark.parametrize("size", [32, 200, 240])
@pytest.mark.parametrize("kind", ["color", "depth"])
def test_depth_image_equals_focused_depth_renderer(capi, synth, kind, size):
    """At sizes k_render supports, the depth image and focus equal those of m3tb_set_focused_renderer's renderer."""
    geometry, poses, cams, _ = _scene_mixed(capi, synth)
    ctx = _context(capi, geometry, poses, cams)
    order = [3, 1, 0, 2, 4, 5, 6, 7, 8]
    ref = [0, 5, 7] if kind == "color" else [6, 9]
    ctx.set_focused_normal_renderer(0, kind, 0, order, ref, size, 0.05, 4.0)
    ctx.set_focused_renderer(0, kind, 0, order, ref, size, 0.05, 4.0, "body")
    ctx.render_focused_normals()
    ctx.render()
    got = ctx.get_focused_normal_rendering(0)
    basic = ctx.get_rendering(0)
    assert np.array_equal(got["depth"], basic["depth"])
    assert (got["depth"] != 65535).any()
    for key in FOCUS_KEYS:
        assert got[key].tobytes() == basic[key].tobytes(), key
    assert np.array_equal(got["visible"], basic["visible"])
    _check(got, _expected(cams, poses, geometry, (kind, size, (0.05, 4.0), order, ref)), kind)
    ctx.close()


def test_device_reads_equal_host_reads(capi, synth):
    import torch
    geometry, poses, cams, renderers = _scene_mixed(capi, synth)
    ctx = _context(capi, geometry, poses, cams)
    for r, (kind, S, (z0, z1), bodies, ref) in enumerate(renderers[:3]):
        ctx.set_focused_normal_renderer(r, kind, 0, bodies, ref, S, z0, z1)
    ctx.render_focused_normals()
    for r, (_, S, _, _, _) in enumerate(renderers[:3]):
        host = ctx.get_focused_normal_rendering(r)
        depth = torch.zeros((S, S), dtype=torch.int16, device="cuda")
        normal = torch.zeros((S, S, 4), dtype=torch.uint8, device="cuda")
        focus = ctx.get_focused_normal_rendering_to(r, depth.data_ptr(), normal.data_ptr())
        ctx.synchronize()
        assert np.array_equal(depth.cpu().numpy().view(np.uint16), host["depth"])
        assert np.array_equal(normal.cpu().numpy(), host["normal"])
        for key in FOCUS_KEYS:
            assert focus[key] == host[key]
        pinned = torch.zeros((S, S, 4), dtype=torch.uint8).pin_memory()  # one image only, into pinned host memory
        ctx.get_focused_normal_rendering_to(r, normal_ptr=pinned.data_ptr())
        assert np.array_equal(pinned.numpy(), host["normal"])
    ctx.close()


def test_normal_vector_decoding(capi, synth):
    """FocusedNormalRenderer::NormalVector of the drawn bytes: unit vectors to the accuracy of 8-bit bytes, and the
    background decodes to (1, 1, 1)."""
    geometry, poses, cams, renderers = _scene_mixed(capi, synth)
    ctx = _context(capi, geometry, poses, cams)
    kind, S, (z0, z1), bodies, ref = renderers[0]
    ctx.set_focused_normal_renderer(0, kind, 0, bodies, ref, S, z0, z1)
    ctx.render_focused_normals()
    got = ctx.get_focused_normal_rendering(0)
    drawn = got["normal"][..., 3] == 255
    n = fn.normal_vector(got["normal"][drawn])
    assert drawn.any() and np.allclose(np.linalg.norm(n, axis=1), 1.0, atol=0.02)
    assert np.array_equal(fn.normal_vector(got["normal"][~drawn]), np.ones(((~drawn).sum(), 3), np.float32))
    ctx.close()


def test_refusals(capi, synth):
    intr = _intr(capi, 320, 240)
    geometry = {0: _mesh(synth, "prism")}
    ctx = _context(capi, geometry, {0: _pose()}, [("color", intr, I34)], max_bodies=2)
    L, h = ctx.L, ctx.h
    ip = capi.C.POINTER(capi.C.c_int)
    one = np.array([0], np.int32)
    p = one.ctypes.data_as(ip)
    f = L.m3tb_set_focused_normal_renderer
    assert f(h, 1, 0, 0, 200, 0.1, 2.0, p, 1, p, 1) == -1    # ids are dense
    assert f(h, 0, 2, 0, 200, 0.1, 2.0, p, 1, p, 1) == -1    # bad camera kind
    assert f(h, 0, 1, 0, 200, 0.1, 2.0, p, 1, p, 1) == -1    # depth camera 0 is not set
    assert f(h, 0, 0, 1, 200, 0.1, 2.0, p, 1, p, 1) == -1    # camera out of range
    assert f(h, 0, 0, 0, 0, 0.1, 2.0, p, 1, p, 1) == -1      # image_size must be positive
    assert f(h, 0, 0, 0, 4097, 0.1, 2.0, p, 1, p, 1) == -3   # above 4096
    assert f(h, 0, 0, 0, 200, 0.0, 2.0, p, 1, p, 1) == -1    # z_min must be positive
    assert f(h, 0, 0, 0, 200, 0.5, 0.5, p, 1, p, 1) == -1    # z_max must exceed z_min
    assert f(h, 0, 0, 0, 200, 0.1, 2.0, p, 1, None, 0) == -1  # no referenced body
    assert f(h, 0, 0, 0, 200, 0.1, 2.0, None, 0, p, 1) == -1  # no geometry body
    bad = np.array([1], np.int32)                              # body 1 has no geometry
    assert f(h, 0, 0, 0, 200, 0.1, 2.0, bad.ctypes.data_as(ip), 1, p, 1) == -1
    assert f(h, 0, 0, 0, 200, 0.1, 2.0, p, 1, bad.ctypes.data_as(ip), 1) == -1
    twice = np.array([0, 0], np.int32)
    assert f(h, 0, 0, 0, 200, 0.1, 2.0, twice.ctypes.data_as(ip), 2, p, 1) == -1
    g = L.m3tb_get_focused_normal_rendering
    assert g(h, 0, None, None, None, None, None, None, None, None) == -1  # not set
    n0 = ctx.launch_count
    assert L.m3tb_render_focused_normals(h) == 0 and ctx.launch_count == n0  # none: nothing launched
    ctx.set_focused_normal_renderer(0, "color", 0, [0], [0], 100, 0.1, 2.0)
    assert g(h, 0, None, None, None, None, None, None, None, None) == -4  # not rendered yet
    ctx.render_full()                                                      # other renderers: not this one
    ctx.update_viewers()
    assert g(h, 0, None, None, None, None, None, None, None, None) == -4
    ctx.render_focused_normals()
    assert ctx.launch_count == n0 + 4
    assert g(h, 0, None, None, None, None, None, None, None, None) == 0
    exp = fn.render_focused_normal(intr, I34, {0: _pose()}, geometry, [0], [0], 100, 0.1, 2.0)
    _check(ctx.get_focused_normal_rendering(0), exp, "first")
    ctx.set_focused_normal_renderer(0, "color", 0, [0], [0], 50, 0.2, 1.0)  # replaced: not rendered since
    assert g(h, 0, None, None, None, None, None, None, None, None) == -4
    ctx.render_focused_normals()
    exp = fn.render_focused_normal(intr, I34, {0: _pose()}, geometry, [0], [0], 50, 0.2, 1.0)
    _check(ctx.get_focused_normal_rendering(0), exp, "replaced")
    ctx.close()


def test_resources_and_failed_allocations(capi, synth):
    """Create / set / render / destroy leaks nothing; every allocating call refused at each of its resource creations
    keeps the resource count, and the next render equals that of a context that never failed."""
    intr = _intr(capi, 320, 240)
    geometry, poses, order = _scene(synth, "bodies8", 320)
    live0 = capi.debug_resources(-1)
    ctx = _context(capi, geometry, poses, [("color", intr, I34)])
    ctx.set_focused_normal_renderer(0, "color", 0, order, [0, 1], 300, 0.1, 2.0)
    ctx.render_focused_normals()
    ctx.get_focused_normal_rendering(0)
    ctx.close()
    assert capi.debug_resources(-1) == live0

    def fresh():
        return _context(capi, geometry, poses, [("color", intr, I34)])

    calls = [
        ("set", lambda c: c.set_focused_normal_renderer(0, "color", 0, order, [0, 1], 120, 0.1, 2.0)),
        ("render", lambda c: c.render_focused_normals()),
        ("set_again", lambda c: c.set_focused_normal_renderer(1, "color", 0, order[:3], [2, 3, 4, 5], 250, 0.3, 0.9)),
        ("resize", lambda c: c.set_focused_normal_renderer(0, "color", 0, order, [0, 1], 77, 0.1, 2.0)),
        ("render_again", lambda c: c.render_focused_normals()),
    ]
    for n_done in range(len(calls)):
        k = 1
        while True:
            ctx = fresh()
            for _, call in calls[:n_done]:
                call(ctx)
            ctx.synchronize()
            live = capi.debug_resources(-1)
            capi.debug_resources(k)
            try:
                calls[n_done][1](ctx)
                failed = False
            except capi.M3TBError:
                failed = True
            finally:
                capi.debug_resources(0)
            if not failed:
                ctx.close()
                break
            assert capi.debug_resources(-1) == live, (calls[n_done][0], k)
            for _, call in calls[n_done:]:
                call(ctx)
            ref = fresh()
            for _, call in calls:
                call(ref)
            for r in range(2):
                a, b = ctx.get_focused_normal_rendering(r), ref.get_focused_normal_rendering(r)
                for key in ("depth", "normal", "visible") + FOCUS_KEYS:
                    assert np.array_equal(a[key], b[key]), (calls[n_done][0], k, r, key)
            ref.close()
            ctx.close()
            k += 1
        assert k > 1, calls[n_done][0]


def test_tracking_and_launches_unchanged(capi, synth):
    """A context with focused normal renderers tracks, renders and updates its viewers with the same launches and the
    same results as one without; the focused normal images show the tracked poses."""
    wl = _workload(synth)
    g = _mesh(synth, "icosphere", n_divides=3)
    runs = []
    for with_focused in (False, True):
        ctx = capi.context_from_workload(wl)
        bodies = list(range(wl.n_bodies))
        for b in bodies:
            ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling)
        ctx.set_viewer(0, "color", 0, bodies, 0.6)
        ctx.set_full_renderer(0, "depth", 1, bodies, 0.1, 2.0)
        ctx.set_focused_renderer(0, "color", 0, bodies, [0], 200, 0.02, 10.0, "body")
        if with_focused:
            ctx.set_focused_normal_renderer(0, "color", 0, bodies, [0], 200)
            ctx.set_focused_normal_renderer(1, "depth", 1, bodies[::-1], bodies, 96, 0.1, 2.0)
        ctx.start_modalities(0)
        out = []
        for it in range(3):
            for call in (lambda: ctx.tracking_step(it, wl.n_corr_iterations, wl.n_update_iterations),
                         ctx.render, ctx.render_full, ctx.update_viewers):
                n0 = ctx.launch_count
                call()
                out.append(np.array([ctx.launch_count - n0]))
            out.append(np.frombuffer(str(ctx.last_launch()).encode(), np.uint8))
            if with_focused:
                ctx.render_focused_normals()
            out.append(ctx.get_poses().copy())
            ci = wl.color_intrinsics
            out.extend(ctx.get_viewer_image(0, ci.width, ci.height))
            out.append(ctx.get_rendering(0)["depth"])
            for b in bodies:
                out.append(np.ascontiguousarray(ctx.get_region_lines(b, 4096)).view(np.uint8).copy())
                out.append(np.ascontiguousarray(ctx.get_depth_points(b, 4096)).view(np.uint8).copy())
        if with_focused:
            poses = {b: p for b, p in enumerate(ctx.get_poses())}
            geometry = {b: g for b in poses}
            exp = fn.render_focused_normal(wl.color_intrinsics, wl.color_world2camera, poses, geometry, bodies, [0])
            _check(ctx.get_focused_normal_rendering(0), exp, "tracked")
            assert (exp["depth"] != 65535).any()
        runs.append(out)
        ctx.close()
    assert len(runs[0]) == len(runs[1])
    for a, b in zip(*runs):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
