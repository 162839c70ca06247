"""The C++ mirror's DepthModel::SaveModel (examples/model_save_selftest.cpp) writes the bytes model_io.write_model
writes: for the views of the reference's depth_model_occlusion.bin (no device needed), and on the device for a model
the mirror's DepthModel::GenerateModel made, against the same generation through the Python binding."""
import importlib
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _build(pkg, tmp_path):
    pkg._build.build_cuda()
    csrc = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
    exe = str(tmp_path / "model_save_selftest")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "3dobjecttracking_b200", "host"), os.path.join(ROOT, "examples", "model_save_selftest.cpp"),
           "-o", exe, "-L", csrc, "-lm3t_b200", "-Wl,-rpath," + csrc]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def _spec(mode, out, p, bodies, tail=""):
    """bodies: [(BodyBlock, triangle file or "-")]."""
    lines = [f"{mode} {out}",
             " ".join(repr(float(np.float32(x))) for x in (p.sphere_radius,)) +
             f" {p.n_divides} {p.n_points} {float(np.float32(p.max_radius_depth_offset))!r}"
             f" {float(np.float32(p.stride_depth_offset))!r} {p.image_size}",
             str(len(bodies))]
    for b, tri in bodies:
        g = " ".join(repr(float(x)) for x in np.asarray(b.geometry2body, np.float32)[:3].reshape(12))
        lines.append(f"{b.geometry_path.decode()} {float(np.float32(b.geometry_unit_in_meter))!r} "
                     f"{int(b.geometry_counterclockwise)} {int(b.geometry_enable_culling)} "
                     f"{float(np.float32(b.maximum_body_diameter))!r} {g} {tri}")
    return "\n".join(lines) + "\n" + tail + "\n"


def _run(exe, tmp_path, spec):
    path = tmp_path / "spec.txt"
    path.write_text(spec)
    r = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and '"ok": 1' in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])


def test_mirror_save_model_matches_writer(pkg, tmp_path):
    capi = importlib.import_module("3dobjecttracking_b200.capi")
    model_io = importlib.import_module("3dobjecttracking_b200.model_io")
    exe = _build(pkg, tmp_path)
    src = os.path.join(GOLDEN, "depth_model_occlusion.bin")
    mf = model_io.read_model(src)
    p = capi.model_params(sphere_radius=mf.sphere_radius, n_divides=mf.n_divides, n_points=mf.n_points,
                          max_radius_depth_offset=mf.max_radius_depth_offset,
                          stride_depth_offset=mf.stride_depth_offset, image_size=mf.image_size)
    rec = mf.n_points * 36 * 4 + 16
    offset = os.path.getsize(src) - mf.model.n_views * rec
    out = tmp_path / "mirror.bin"
    bodies = [(mf.body, "-")] + [(b, "-") for b in mf.associated[0]]
    _run(exe, tmp_path, _spec("save", out, p, bodies, f"{src} {offset} {mf.model.n_views}"))
    ref = tmp_path / "writer.bin"
    model_io.write_model(ref, model_io.model_from_generated(mf.model, p, mf.body, mf.associated[0]))
    assert out.read_bytes() == ref.read_bytes() == open(src, "rb").read()


@pytest.mark.gpu
def test_mirror_generate_and_save_matches_binding(pkg, synth, tmp_path):
    capi = importlib.import_module("3dobjecttracking_b200.capi")
    model_io = importlib.import_module("3dobjecttracking_b200.model_io")
    exe = _build(pkg, tmp_path)
    tri, diam = synth.prism_triangles()
    occ_tri, _ = synth.icosphere_triangles(radius=0.02, n_divides=1)
    g2b = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
    occ_g2b = g2b.copy()
    occ_g2b[:, 3] = (0.015, 0.01, 0.0)
    occ_diam = float(np.float32(2.0 * np.linalg.norm(occ_tri.reshape(-1, 3) + occ_g2b[:, 3], axis=1).max()))
    diam = float(np.float32(diam))
    body = model_io.BodyBlock(b"prism.obj", 1.0, True, True, diam, np.vstack([g2b, [0, 0, 0, 1]]))
    occ = model_io.BodyBlock(b"sphere.obj", 1.0, True, True, occ_diam, np.vstack([occ_g2b, [0, 0, 0, 1]]))
    np.ascontiguousarray(tri, np.float32).tofile(tmp_path / "body.f32")
    np.ascontiguousarray(occ_tri, np.float32).tofile(tmp_path / "occ.f32")
    p = capi.model_params(n_divides=1, n_points=20, image_size=200)
    out = tmp_path / "mirror.bin"
    _run(exe, tmp_path, _spec("generate", out, p, [(body, tmp_path / "body.f32"), (occ, tmp_path / "occ.f32")]))
    ctx = capi.Context(0, max_bodies=2, max_cameras=1, max_models=1)
    ctx.set_body_geometry(0, tri, g2b, diam, True)
    ctx.set_body_geometry(1, occ_tri, occ_g2b, occ_diam, True)
    ctx.generate_depth_model(0, 0, [1], p)
    ref = tmp_path / "binding.bin"
    model_io.write_model(ref, model_io.model_from_generated(ctx.get_depth_model(0), p, body, [occ]))
    ctx.close()
    assert out.read_bytes() == ref.read_bytes()
