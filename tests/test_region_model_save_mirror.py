"""The C++ mirror's RegionModel::SaveModel (examples/region_model_save_selftest.cpp) writes the bytes
model_io.write_model writes: for the views of the reference's region_model.bin (no device needed), and on the device
for models the mirror's RegionModel::GenerateModel made, with and without associated bodies, against the same
generation through the Python binding."""
import importlib
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
I34 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def _build(pkg, tmp_path):
    pkg._build.build_cuda()
    csrc = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
    exe = str(tmp_path / "region_model_save_selftest")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "3dobjecttracking_b200", "host"),
           os.path.join(ROOT, "examples", "region_model_save_selftest.cpp"), "-o", exe, "-L", csrc, "-lm3t_b200",
           "-Wl,-rpath," + csrc]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return exe


def _spec(mode, out, p, bodies, tail=""):
    """bodies: [(BodyBlock, movable, same_region, triangle file or "-")]."""
    lines = [f"{mode} {out}",
             f"{float(np.float32(p.sphere_radius))!r} {p.n_divides} {p.n_points}"
             f" {float(np.float32(p.max_radius_depth_offset))!r} {float(np.float32(p.stride_depth_offset))!r}"
             f" {p.image_size}",
             str(len(bodies))]
    for b, movable, same, tri in bodies:
        g = " ".join(repr(float(x)) for x in np.asarray(b.geometry2body, np.float32)[:3].reshape(12))
        lines.append(f"{b.geometry_path.decode()} {float(np.float32(b.geometry_unit_in_meter))!r} "
                     f"{int(b.geometry_counterclockwise)} {int(b.geometry_enable_culling)} "
                     f"{float(np.float32(b.maximum_body_diameter))!r} {g} {movable} {same} {tri}")
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
    src = os.path.join(GOLDEN, "region_model.bin")
    mf = model_io.read_model(src)
    p = capi.model_params(sphere_radius=mf.sphere_radius, n_divides=mf.n_divides, n_points=mf.n_points,
                          max_radius_depth_offset=mf.max_radius_depth_offset,
                          stride_depth_offset=mf.stride_depth_offset, image_size=mf.image_size)
    rec = mf.n_points * 38 * 4 + 16
    offset = os.path.getsize(src) - mf.model.n_views * rec
    out = tmp_path / "mirror.bin"
    _run(exe, tmp_path, _spec("save", out, p, [(mf.body, 0, 0, "-")], f"{src} {offset} {mf.model.n_views}"))
    ref = tmp_path / "writer.bin"
    model_io.write_model(ref, model_io.model_from_generated(mf.model, p, mf.body, mf.associated))
    assert out.read_bytes() == ref.read_bytes() == open(src, "rb").read()


def _block(model_io, name, tri, g2b):
    diam = float(np.float32(2.0 * np.linalg.norm(tri.reshape(-1, 3) + g2b[:, 3], axis=1).max()))
    return model_io.BodyBlock(name, 1.0, True, True, diam, np.vstack([g2b, [0, 0, 0, 1]]).astype(np.float32))


@pytest.mark.gpu
@pytest.mark.parametrize("kinds", [(), ((1, 0), (0, 0), (1, 1), (0, 1), (0, 0))])
def test_mirror_generate_and_save_matches_binding(pkg, synth, tmp_path, kinds):
    """kinds: (movable, same_region) of each associated body, in insertion order (the groups interleave)."""
    capi = importlib.import_module("3dobjecttracking_b200.capi")
    model_io = importlib.import_module("3dobjecttracking_b200.model_io")
    exe = _build(pkg, tmp_path)
    tri, _ = synth.prism_triangles()
    small, _ = synth.icosphere_triangles(radius=0.012, n_divides=1)
    blocks = [_block(model_io, b"prism.obj", tri, I34)]
    tris = [tri]
    for k, _ in enumerate(kinds):
        g2b = I34.copy()
        g2b[:, 3] = 0.03 * np.array([np.cos(k), np.sin(k), 0.3 * (k % 2) - 0.15], np.float32)
        blocks.append(_block(model_io, f"b{k}.obj".encode(), small, g2b))
        tris.append(small)
    for k, t in enumerate(tris):
        np.ascontiguousarray(t, np.float32).tofile(tmp_path / f"t{k}.f32")
    p = capi.model_params(n_divides=1, n_points=20, image_size=200)
    out = tmp_path / "mirror.bin"
    spec_bodies = [(blocks[0], 0, 0, tmp_path / "t0.f32")] + [
        (blocks[1 + k], m, s, tmp_path / f"t{1 + k}.f32") for k, (m, s) in enumerate(kinds)]
    _run(exe, tmp_path, _spec("generate", out, p, spec_bodies))
    ctx = capi.Context(0, max_bodies=len(blocks), max_cameras=1, max_models=1)
    for k, (b, t) in enumerate(zip(blocks, tris)):
        ctx.set_body_geometry(k, t, b.geometry2body[:3], b.maximum_body_diameter, True)
    ctx.generate_region_model(0, 0, [(1 + k, m, s) for k, (m, s) in enumerate(kinds)], p)
    groups = [[], [], [], []]
    for k, (m, s) in enumerate(kinds):
        groups[2 * m + s].append(blocks[1 + k])
    ref = tmp_path / "binding.bin"
    model_io.write_model(ref, model_io.model_from_generated(ctx.get_region_model(0), p, blocks[0], groups))
    ctx.close()
    assert out.read_bytes() == ref.read_bytes()
