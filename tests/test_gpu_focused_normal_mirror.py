"""The C++ mirror's FocusedNormalRenderer, the two NormalizedDepthImage methods and ImageColorViewer / ImageDepthViewer
(examples/focused_normal_selftest.cpp, built with plain g++ -std=c++17): images, focus and visible flags equal the CPU
restatements bit for bit; NormalImageValue / NormalVector(Point2i) read the pixel normal_renderer.cpp reads and
NormalVector decodes as tests/focused_normal_reference.py does; the image viewers show the frames the cameras hold; the
reference's structural rules hold."""
import json
import os
import subprocess

import numpy as np
import pytest

import focused_normal_reference as fn
import full_renderer_reference as fr
import viewer_reference as vr

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I34 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def _floats(a):
    return " ".join(repr(float(x)) for x in np.asarray(a, np.float32).reshape(-1))


def test_mirror_focused_normal_renderer_and_image_viewers(pkg, tmp_path):
    pkg._build.build_cuda()
    csrc = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
    exe = str(tmp_path / "focused_normal_selftest")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "3dobjecttracking_b200", "host"),
           os.path.join(ROOT, "examples", "focused_normal_selftest.cpp"), "-o", exe, "-L", csrc, "-lm3t_b200",
           "-Wl,-rpath," + csrc]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]

    s = fr.golden_scene()
    ci = s.intrinsics
    di = type(ci)(fu=300.0, fv=301.0, ppu=161.5, ppv=118.25, width=320, height=240)
    w2c_depth = np.array([[1, 0, 0, -0.02], [0, 1, 0, 0.005], [0, 0, 1, 0.01]], np.float32)
    depth_scale, min_depth, max_depth, S, z_min, z_max = 0.001, 0.2, 0.55, 160, 0.1, 2.0
    referenced = [1, 0]
    rng = np.random.default_rng(3)
    color_frame = rng.integers(0, 256, (ci.height, ci.width, 3), dtype=np.uint8)
    depth_frame = rng.integers(0, 800, (di.height, di.width), dtype=np.uint16)
    depth_frame[::7, ::3] = 0
    color_frame.tofile(tmp_path / "color.u8")
    depth_frame.tofile(tmp_path / "depth.u16")

    exp = fn.render_focused_normal(ci, s.world2camera, s.poses, s.geometry, s.bodies, referenced, S, z_min, z_max)
    # camera pixels whose focused pixel is drawn, and some that are not
    drawn = np.argwhere(exp["depth"] != 65535)
    cam_points = []
    for v, u in drawn[:: max(1, len(drawn) // 30)]:
        x = int(round(float(exp["corner_u"]) + (u + 0.25) / float(exp["scale"])))
        y = int(round(float(exp["corner_v"]) + (v + 0.25) / float(exp["scale"])))
        if fn.image_value_index(exp, x, y)[0] < S and fn.image_value_index(exp, x, y)[1] < S:
            cam_points.append((x, y))
    cx, cy = int(exp["corner_u"]) + 1, int(exp["corner_v"]) + 1
    cam_points.append((cx, cy))
    values = [(k, 255 - k, (7 * k) % 256, 255) for k in range(256)]

    lines = [str(len(s.bodies))]
    for b in s.bodies:
        G = s.geometry[b]
        path = tmp_path / f"body{b}.f32"
        np.ascontiguousarray(G.triangles, np.float32).tofile(path)
        lines.append(f"{path} {_floats(G.geometry2body)} {float(np.float32(G.maximum_body_diameter))!r} "
                     f"{int(G.enable_culling)} {G.body_id} {G.region_id} {_floats(s.poses[b])}")
    lines.append(f"{ci.fu!r} {ci.fv!r} {ci.ppu!r} {ci.ppv!r} {ci.width} {ci.height}")
    lines.append(_floats(s.world2camera))
    lines.append(f"{di.fu!r} {di.fv!r} {di.ppu!r} {di.ppv!r} {di.width} {di.height}")
    lines.append(_floats(w2c_depth))
    lines.append(repr(depth_scale))
    lines.append(f"{tmp_path / 'color.u8'} {tmp_path / 'depth.u16'}")
    lines.append(f"{S} {z_min!r} {z_max!r}")
    lines.append(f"{len(referenced)} " + " ".join(map(str, referenced)))
    lines.append(f"{min_depth!r} {max_depth!r}")
    lines.append(str(len(cam_points)))
    lines += [f"{x} {y}" for x, y in cam_points]
    lines.append(str(len(values)))
    lines += [" ".join(map(str, v)) for v in values]
    lines.append(str(tmp_path))
    (tmp_path / "spec.txt").write_text("\n".join(lines) + "\n")
    r = subprocess.run([exe, str(tmp_path / "spec.txt")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    out = json.loads(r.stdout)
    for key in ("start_before_setup_fails", "fetch_before_setup_fails", "setup_without_referenced_fails",
                "fetch_before_render_fails", "update_before_setup_fails"):
        assert out[key], key

    # the focused normal renderer
    got_depth = np.fromfile(tmp_path / "focused_depth.u16", np.uint16).reshape(S, S)
    got_normal = np.fromfile(tmp_path / "focused_normal.u8", np.uint8).reshape(S, S, 4)
    assert np.array_equal(got_depth, exp["depth"]) and np.array_equal(got_normal, exp["normal"])
    keys = ("corner_u", "corner_v", "scale", "projection_term_a", "projection_term_b")
    for k, key in enumerate(keys):
        assert np.float32(out["focus"][k]) == np.float32(exp[key]), key
    assert out["visible"] == [int(exp["visible"][referenced.index(b)]) for b in s.bodies]
    n_drawn = 0
    for (x, y), p in zip(cam_points, out["points"]):
        v, u = fn.image_value_index(exp, x, y)
        assert p["value"] == list(exp["normal"][v, u]), (x, y)
        assert np.array_equal(np.array(p["normal"], np.float32), fn.normal_vector(exp["normal"][v, u])), (x, y)
        n_drawn += int(exp["normal"][v, u, 3] == 255)
    assert n_drawn > 10
    for value, n in zip(values, out["values"]):
        assert np.array_equal(np.array(n, np.float32), fn.normal_vector(value)), value

    # NormalizedDepthImage of the depth camera and of the full renderer
    exp_camera = vr.normalized_depth(depth_frame, depth_scale, min_depth, max_depth)
    assert np.array_equal(np.fromfile(tmp_path / "camera_normalized.u8", np.uint8).reshape(di.height, di.width),
                          exp_camera)
    full = fr.render_full(ci, s.world2camera, s.poses, s.geometry, s.bodies, z_min, z_max)
    exp_full = fn.normalized_full_depth(full["depth"], full["projection_term_a"], full["projection_term_b"], min_depth,
                                        max_depth)
    assert np.array_equal(np.fromfile(tmp_path / "full_normalized.u8", np.uint8).reshape(ci.height, ci.width), exp_full)
    assert len(np.unique(exp_full)) > 3

    # the image viewers show the frames the cameras hold; the normal viewer was updated with them
    assert np.array_equal(np.fromfile(tmp_path / "image_color_viewer.u8", np.uint8).reshape(ci.height, ci.width, 3),
                          color_frame)
    assert np.array_equal(np.fromfile(tmp_path / "image_depth_viewer.u8", np.uint8).reshape(di.height, di.width),
                          exp_camera)
    normal, _ = vr.render_normal(ci, s.world2camera, s.poses, s.geometry, s.bodies)
    assert np.array_equal(np.fromfile(tmp_path / "normal_viewer.u8", np.uint8).reshape(ci.height, ci.width, 3),
                          vr.viewer_image("color", color_frame, normal, 0.5))
