"""Device full renderers (m3tb_set_full_renderer / m3tb_render_full / m3tb_get_full_rendering, k_view_* with VK_FULL):
depth, silhouette and normal images equal the CPU restatement (tests/full_renderer_reference.py) bit for bit on the
reference's renderer-test scene and on many renderers of mixed cameras, sizes, z ranges and id types rendered together;
the device meets the reference's OpenGL images as the restatement does; reads into device memory equal host reads;
refused and failed calls leave the context as it was; full renders change neither tracking nor the viewers; and the
C++ mirror's classes return the same images."""
import json
import os
import subprocess

import numpy as np
import pytest

import full_renderer_reference as fr
import render_reference as rr
from test_gpu_viewers import I34, W2C_DEPTH, _frame, _intr, _mesh, _pose, _scene, _workload

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def _check(ctx, renderer, intr, w2c, poses, geometry, bodies, z_min, z_max, id_type):
    got = ctx.get_full_rendering(renderer, intr.width, intr.height)
    exp = fr.render_full(intr, w2c, poses, geometry, bodies, z_min, z_max, id_type)
    for key in ("depth", "silhouette", "normal"):
        assert np.array_equal(got[key], exp[key]), (renderer, key, np.argwhere(got[key] != exp[key])[:5])
    for key in ("projection_term_a", "projection_term_b"):
        assert got[key].tobytes() == exp[key].tobytes(), key
    return exp


def _golden_context(capi, s):
    intr = capi.Intrinsics(s.intrinsics.fu, s.intrinsics.fv, s.intrinsics.ppu, s.intrinsics.ppv, 640, 480)
    return _context(capi, s.geometry, s.poses, [("color", intr, s.world2camera)]), intr


def test_golden_scene(capi):
    s = fr.golden_scene()
    ctx, intr = _golden_context(capi, s)
    ctx.set_full_renderer(0, "color", 0, s.bodies, s.z_min, s.z_max, "body")
    n0 = ctx.launch_count
    ctx.render_full()
    assert ctx.launch_count == n0 + 3
    got = _check(ctx, 0, intr, s.world2camera, s.poses, s.geometry, s.bodies, s.z_min, s.z_max, "body")
    assert fr.wrong_pixels(got["silhouette"], fr.load_golden("silhouette_image.png")) == 0
    assert fr.wrong_pixels(got["depth"], fr.load_golden("depth_image.png")) <= 10
    assert fr.wrong_pixels(got["normal"], fr.load_golden("normal_image.png")) == 30  # see test_full_renderer_reference
    # k_render against the focused goldens directly
    ctx.set_focused_renderer(0, "color", 0, s.bodies, s.focused_referenced, s.focused_size, s.z_min, s.z_max, "body")
    ctx.render()
    foc = ctx.get_rendering(0)
    exp = rr.render_focused(intr, s.world2camera, s.poses, s.geometry, s.bodies, s.focused_referenced, s.focused_size,
                            s.z_min, s.z_max, "body")
    assert np.array_equal(foc["depth"], exp["depth"]) and np.array_equal(foc["silhouette"], exp["silhouette"])
    assert fr.wrong_pixels(foc["silhouette"], fr.load_golden("focused_silhouette_image.png")) <= 10
    assert fr.wrong_pixels(foc["depth"], fr.load_golden("focused_depth_image.png")) <= 10
    ctx.close()


def _mixed(capi, synth):
    """Bodies 0-7: the viewers' eight overlapping bodies (equal copies at equal poses tie: the body drawn first wins),
    body 8 crosses the near plane of every z range below, body 9 is cut by the image border; ids differ per body."""
    geometry, poses, order = _scene(synth, "bodies8", 640)
    geometry[8] = _mesh(synth, "icosphere", culling=False, n_divides=3)
    poses[8] = _pose(t=(-0.03, 0.0, 0.05))
    geometry[9] = _mesh(synth, "prism", culling=False)
    poses[9] = _pose((0, 30, 0), (0.19, 0.0, 0.4))
    for b, g in geometry.items():
        g.body_id, g.region_id = 10 + b, 200 + b % 3
    cams = [("color", _intr(capi, 640, 480), I34), ("depth", _intr(capi, 1280, 720), W2C_DEPTH),
            ("color", _intr(capi, 333, 217), W2C_DEPTH), ("depth", _intr(capi, 161, 97), I34)]
    # (camera kind, camera index, z range, id type, bodies)
    renderers = [("color", 0, (0.1, 2.0), "body", order + [8, 9]),
                 ("depth", 0, (0.02, 10.0), "region", [9, 8] + order),
                 ("color", 1, (0.3, 0.45), "body", order),          # the far plane cuts the bodies
                 ("depth", 1, (0.07, 0.6), "region", [8, 0, 1]),
                 ("color", 0, (0.02, 10.0), "region", []),           # draws nothing
                 ("color", 0, (0.35, 3.0), "body", [2, 0, 9])]
    return geometry, poses, cams, renderers


def _cam(cams, kind, index):
    return [c for c in cams if c[0] == kind][index]


def test_many_renderers_one_render(capi, synth):
    geometry, poses, cams, renderers = _mixed(capi, synth)
    ctx = _context(capi, geometry, poses, cams)
    for r, (kind, cam, (z0, z1), idt, bodies) in enumerate(renderers):
        ctx.set_full_renderer(r, kind, cam, bodies, z0, z1, idt)
    n0 = ctx.launch_count
    ctx.render_full()
    assert ctx.launch_count == n0 + 3
    for _ in range(2):  # a second render from the cleared z-buffers gives the same bytes
        for r, (kind, cam, (z0, z1), idt, bodies) in enumerate(renderers):
            _, intr, w2c = _cam(cams, kind, cam)
            exp = _check(ctx, r, intr, w2c, poses, geometry, bodies, z0, z1, idt)
            if bodies:
                assert (exp["silhouette"] != 0).mean() > 0.002, r
        ctx.render_full()
    # the tie is visible: body 3 is drawn before its equal copy body 1 at the same pose, so body 1 never wins
    exp = fr.render_full(_cam(cams, "color", 0)[1], I34, poses, geometry, renderers[0][4], 0.1, 2.0, "body")
    assert (exp["silhouette"] == 13).any() and not (exp["silhouette"] == 11).any()
    ctx.close()


def test_device_reads_equal_host_reads(capi, synth):
    import torch
    geometry, poses, cams, renderers = _mixed(capi, synth)
    ctx = _context(capi, geometry, poses, cams)
    for r, (kind, cam, (z0, z1), idt, bodies) in enumerate(renderers[:2]):
        ctx.set_full_renderer(r, kind, cam, bodies, z0, z1, idt)
    ctx.render_full()
    for r, (kind, cam, _, _, _) in enumerate(renderers[:2]):
        intr = _cam(cams, kind, cam)[1]
        W, H = intr.width, intr.height
        host = ctx.get_full_rendering(r, W, H)
        # pitched device images (rows wider than the image)
        depth = torch.zeros((H, W + 7), dtype=torch.int16, device="cuda")
        sil = torch.zeros((H, W + 13), dtype=torch.uint8, device="cuda")
        normal = torch.zeros((H, W + 3, 4), dtype=torch.uint8, device="cuda")
        terms = ctx.get_full_rendering_to(r, depth.data_ptr(), depth.stride(0) * 2, sil.data_ptr(), sil.stride(0),
                                          normal.data_ptr(), normal.stride(0))
        ctx.synchronize()
        assert np.array_equal(depth[:, :W].cpu().numpy().view(np.uint16), host["depth"])
        assert np.array_equal(sil[:, :W].cpu().numpy(), host["silhouette"])
        assert np.array_equal(normal[:, :W].cpu().numpy(), host["normal"])
        assert terms["projection_term_a"] == host["projection_term_a"]
        # one image only, into pinned host memory
        pinned = torch.zeros((H, W), dtype=torch.uint8).pin_memory()
        ctx.get_full_rendering_to(r, silhouette_ptr=pinned.data_ptr(), silhouette_pitch=W)
        assert np.array_equal(pinned.numpy(), host["silhouette"])
    ctx.close()


def test_refusals(capi, synth):
    intr, intr2 = _intr(capi, 320, 240), _intr(capi, 200, 150)
    geometry = {0: _mesh(synth, "prism")}
    ctx = _context(capi, geometry, {0: _pose()}, [("color", intr, I34)], max_bodies=2)
    L, h = ctx.L, ctx.h
    ip = capi.C.POINTER(capi.C.c_int)
    one = np.array([0], np.int32)
    p = one.ctypes.data_as(ip)
    assert L.m3tb_set_full_renderer(h, 1, 0, 0, 0.1, 2.0, 0, p, 1) == -1   # ids are dense
    assert L.m3tb_set_full_renderer(h, 0, 2, 0, 0.1, 2.0, 0, p, 1) == -1   # bad camera kind
    assert L.m3tb_set_full_renderer(h, 0, 1, 0, 0.1, 2.0, 0, p, 1) == -1   # depth camera 0 is not set
    assert L.m3tb_set_full_renderer(h, 0, 0, 1, 0.1, 2.0, 0, p, 1) == -1   # camera out of range
    assert L.m3tb_set_full_renderer(h, 0, 0, 0, 0.0, 2.0, 0, p, 1) == -1   # z_min must be positive
    assert L.m3tb_set_full_renderer(h, 0, 0, 0, 0.5, 0.5, 0, p, 1) == -1   # z_max must exceed z_min
    assert L.m3tb_set_full_renderer(h, 0, 0, 0, 0.1, 2.0, 2, p, 1) == -1   # bad id type
    bad = np.array([1], np.int32)                                            # body 1 has no geometry
    assert L.m3tb_set_full_renderer(h, 0, 0, 0, 0.1, 2.0, 0, bad.ctypes.data_as(ip), 1) == -1
    twice = np.array([0, 0], np.int32)
    assert L.m3tb_set_full_renderer(h, 0, 0, 0, 0.1, 2.0, 0, twice.ctypes.data_as(ip), 2) == -1
    assert L.m3tb_get_full_rendering(h, 0, None, 0, None, 0, None, 0, None, None) == -1  # no full renderer
    n0 = ctx.launch_count
    assert L.m3tb_render_full(h) == 0 and ctx.launch_count == n0          # none: nothing launched
    ctx.set_full_renderer(0, "color", 0, [0], 0.1, 2.0)
    assert L.m3tb_get_full_rendering(h, 0, None, 0, None, 0, None, 0, None, None) == -4  # not rendered yet
    ctx.update_viewers()                                                    # no viewer: nothing launched
    ctx.render_full()
    assert ctx.launch_count == n0 + 3
    sil = np.zeros((240, 320), np.uint8)
    assert L.m3tb_get_full_rendering(h, 0, None, 0, sil.ctypes.data, 319, None, 0, None, None) == -1  # pitch
    _check(ctx, 0, intr, I34, {0: _pose()}, geometry, [0], 0.1, 2.0, "body")
    ctx.set_color_camera(0, intr2, I34)                                     # the camera changes size
    assert L.m3tb_get_full_rendering(h, 0, None, 0, None, 0, None, 0, None, None) == -4
    ctx.render_full()
    _check(ctx, 0, intr2, I34, {0: _pose()}, geometry, [0], 0.1, 2.0, "body")
    ctx.set_full_renderer(0, "color", 0, [0], 0.2, 1.0, "region")          # replaced: not rendered since
    assert L.m3tb_get_full_rendering(h, 0, None, 0, None, 0, None, 0, None, None) == -4
    ctx.close()


def test_failed_allocations_leave_full_renderers_as_they_were(capi, synth):
    """Every allocating full-renderer call refused at each of its resource creations keeps the resource count, and the
    next render is bit-identical to that of a context that never failed."""
    intr, intr2 = _intr(capi, 320, 240), _intr(capi, 200, 150)
    geometry, poses, bodies = _scene(synth, "bodies8", 320)

    def fresh():
        return _context(capi, geometry, poses, [("color", intr, I34)])

    calls = [  # (name, what precedes the call, the allocating call)
        ("set_full_renderer", None, lambda c: c.set_full_renderer(0, "color", 0, bodies, 0.1, 2.0)),
        ("render_full", None, lambda c: c.render_full()),
        ("set_full_renderer_again", None, lambda c: c.set_full_renderer(1, "color", 0, bodies[:3], 0.3, 0.6, "region")),
        ("render_after_resize", lambda c: c.set_color_camera(0, intr2, I34), lambda c: c.render_full()),
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
            calls[n_done][2](ctx)
            run(ctx, calls[n_done + 1:])
            ctx.render_full()
            ref = fresh()
            run(ref, calls)
            ref.render_full()
            for r in range(2):
                a, b = ctx.get_full_rendering(r, 200, 150), ref.get_full_rendering(r, 200, 150)
                for key in ("depth", "silhouette", "normal"):
                    assert np.array_equal(a[key], b[key]), (calls[n_done][0], k, r, key)
            ref.close()
            ctx.close()
            k += 1
        assert k > 1, calls[n_done][0]


def test_tracking_and_viewers_unchanged_by_full_renders(capi, synth):
    wl = _workload(synth)
    g = _mesh(synth, "icosphere", n_divides=3)
    runs = []
    for with_full in (False, True):
        ctx = capi.context_from_workload(wl)
        for b in range(wl.n_bodies):
            ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling)
        ctx.set_viewer(0, "color", 0, list(range(wl.n_bodies)), 0.6)
        if with_full:
            ctx.set_full_renderer(0, "color", 0, list(range(wl.n_bodies)), 0.1, 2.0)
            ctx.set_full_renderer(1, "depth", 1, list(range(wl.n_bodies))[::-1], 0.02, 10.0, "region")
        ctx.start_modalities(0)
        out = []
        for it in range(3):
            n0 = ctx.launch_count
            ctx.tracking_step(it, wl.n_corr_iterations, wl.n_update_iterations)
            out.append(np.array([ctx.launch_count - n0]))
            if with_full:
                ctx.render_full()
            ctx.update_viewers()
            out.append(ctx.get_poses().copy())
            ci = wl.color_intrinsics
            out.extend(ctx.get_viewer_image(0, ci.width, ci.height))
            for b in range(wl.n_bodies):
                out.append(np.ascontiguousarray(ctx.get_region_lines(b, 4096)).view(np.uint8).copy())
                out.append(np.ascontiguousarray(ctx.get_depth_points(b, 4096)).view(np.uint8).copy())
        if with_full:  # and the full renders show the tracked poses
            poses = {b: p for b, p in enumerate(ctx.get_poses())}
            _check(ctx, 0, wl.color_intrinsics, wl.color_world2camera, poses, {b: g for b in poses},
                   list(range(wl.n_bodies)), 0.1, 2.0, "body")
        runs.append(out)
        ctx.close()
    for a, b in zip(*runs):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


def _build_selftest(pkg, tmp_path):
    pkg._build.build_cuda()
    csrc = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
    exe = str(tmp_path / "full_renderer_selftest")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "3dobjecttracking_b200", "host"), os.path.join(ROOT, "examples", "full_renderer_selftest.cpp"),
           "-o", exe, "-L", csrc, "-lm3t_b200", "-Wl,-rpath," + csrc]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def _floats(a):
    return " ".join(repr(float(x)) for x in np.asarray(a, np.float32).reshape(-1))


@pytest.mark.parametrize("id_type", ["body", "region"])
def test_mirror_classes_return_the_same_images(pkg, tmp_path, id_type):
    s = fr.golden_scene()
    exe = _build_selftest(pkg, tmp_path)
    lines = [str(len(s.bodies))]
    for b in s.bodies:
        G = s.geometry[b]
        path = tmp_path / f"body{b}.f32"
        np.ascontiguousarray(G.triangles, np.float32).tofile(path)
        lines.append(f"{path} {_floats(G.geometry2body)} {float(np.float32(G.maximum_body_diameter))!r} "
                     f"{int(G.enable_culling)} {G.body_id} {G.region_id} {_floats(s.poses[b])}")
    i = s.intrinsics
    lines.append(f"{i.fu!r} {i.fv!r} {i.ppu!r} {i.ppv!r} {i.width} {i.height}")
    lines.append(_floats(s.world2camera))
    lines.append(f"{s.z_min!r} {s.z_max!r} {0 if id_type == 'body' else 1}")
    exp = fr.render_full(i, s.world2camera, s.poses, s.geometry, s.bodies, s.z_min, s.z_max, id_type)
    drawn = np.argwhere(exp["depth"] != 65535)
    points = [(0, 0), (639, 479)] + [(int(x), int(y)) for y, x in drawn[::max(1, len(drawn) // 40)]]
    lines.append(str(len(points)))
    lines += [f"{x} {y}" for x, y in points]
    lines.append(str(tmp_path))
    (tmp_path / "spec.txt").write_text("\n".join(lines) + "\n")
    r = subprocess.run([exe, str(tmp_path / "spec.txt")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    out = json.loads(r.stdout)
    assert out["start_before_setup_fails"] and out["fetch_before_setup_fails"] and out["fetch_before_render_fails"]
    assert out["setup_without_camera_fails"] and out["setup_without_geometry_setup_fails"]
    assert np.array_equal(np.fromfile(tmp_path / "depth.u16", np.uint16).reshape(480, 640), exp["depth"])
    assert np.array_equal(np.fromfile(tmp_path / "silhouette.u8", np.uint8).reshape(480, 640), exp["silhouette"])
    assert np.array_equal(np.fromfile(tmp_path / "normal.u8", np.uint8).reshape(480, 640, 4), exp["normal"])
    assert np.float32(out["projection_terms"][0]) == exp["projection_term_a"]
    assert np.float32(out["projection_terms"][1]) == exp["projection_term_b"]
    for (x, y), p in zip(points, out["points"]):  # renderer.cpp:431-452, bit for bit
        assert p["value"] == exp["depth"][y, x] and p["silhouette"] == exp["silhouette"][y, x]
        assert np.float32(p["depth"]) == np.float32(p["depth_of_value"]) == fr.depth_of(exp, exp["depth"][y, x])
        assert np.array_equal(np.array(p["point"], np.float32), fr.point_vector(exp, i, x, y)), (x, y)
