"""CPU checks of depth-model generation: the host port of the geodesic views against the reference's own model file,
and the restatement (tests/model_generation_reference.py) against closed forms on the prism."""
import importlib
import os

import numpy as np
import pytest

import model_generation_reference as mg
import render_reference as rr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
f32 = np.float32


@pytest.fixture(scope="module")
def capi():
    return importlib.import_module("3dobjecttracking_b200.capi")


def test_geodesic_views_match_reference_model(capi):
    model_io = importlib.import_module("3dobjecttracking_b200.model_io")
    for fname in ("depth_model.bin", "depth_model_occlusion.bin"):
        mf = model_io.read_model(os.path.join(GOLDEN, fname))
        poses = capi.model_views(capi.model_params(n_divides=mf.n_divides, sphere_radius=mf.sphere_radius))
        assert poses.shape[0] == mf.model.n_views
        assert np.abs(poses[:, :, 2] - mf.model.orientations).max() <= 1e-7
        # the restatement builds the same poses bit for bit
        assert np.array_equal(mg.geodesic_poses(mf.n_divides, mf.sphere_radius).view(np.uint32), poses.view(np.uint32))


@pytest.mark.parametrize("n", range(5))
def test_geodesic_view_count(capi, n):
    poses = capi.model_views(capi.model_params(n_divides=n))
    assert poses.shape[0] == 10 * 4 ** n + 2
    R = poses[:, :, :3].astype(np.float64)
    assert np.abs(np.einsum("nij,nik->njk", R, R) - np.eye(3)).max() < 1e-6   # rotations
    assert np.allclose(poses[:, :, 3], -0.8 * poses[:, :, 2], atol=1e-6)        # looking at the body origin


def _prism(synth_mod):
    tri, diam = synth_mod.prism_triangles()
    return rr.Geometry(tri, np.hstack([np.eye(3), np.zeros((3, 1))]).astype(f32), diam, True)


@pytest.fixture(scope="module")
def synth_mod():
    return importlib.import_module("3dobjecttracking_b200.synth")


TOP = np.array([[1, 0, 0, 0], [0, -1, 0, 0], [0, 0, -1, 0.8]], f32)  # camera on +z looking at the top face


def _top_view(synth_mod, S=400, n_points=60):
    st = mg.Setup(_prism(synth_mod), [], 0.8, S)
    img = mg.render_view(st, TOP)
    pts, area = mg.view_points(st, TOP, img, n_points, 0.002, 0.05)
    return st, img, pts, area


def test_top_view_closed_forms(synth_mod):
    st, img, pts, area = _top_view(synth_mod)
    a, b = np.float64(st.projection_term_a), np.float64(st.projection_term_b)
    d16 = np.float64(img["depth"][img["depth"] != 0xFFFF])
    step = (a / (b - d16 - 1) - a / (b - d16)).max()
    # every centre lies on the top face (z = +0.006) within one depth step, inside the triangle's footprint
    assert np.abs(pts[:, 2] - 0.006).max() <= step
    # decoded normals equal the face normal (0, 0, 1) within one 8-bit step
    assert np.abs(pts[:, 3:6] - [0, 0, 1]).max() <= 1 / 127.5
    # surface area = projected area of the prism's triangle, within the pixels along its edges
    v = synth_mod.PRISM_VERTICES[synth_mod.PRISM_VERTICES[:, 2] > 0][:, :2].astype(np.float64)
    tri_area = 0.5 * abs((v[1, 0] - v[0, 0]) * (v[2, 1] - v[0, 1]) - (v[2, 0] - v[0, 0]) * (v[1, 1] - v[0, 1]))
    z = 0.8 - 0.006
    px = float(st.r / st.fu) ** 2          # square(sphere_radius / fu): one pixel's area as the model counts it
    pixels_exact = tri_area * (float(st.fu) / z) ** 2
    perimeter = sum(np.linalg.norm(v[i] - v[(i + 1) % 3]) for i in range(3)) * float(st.fu) / z
    assert abs(float(area) / px - pixels_exact) <= perimeter
    # a fronto-parallel face: every depth offset is zero up to one depth step
    assert np.abs(pts[:, 6:]).max() <= step


def test_oblique_views_closed_forms(synth_mod):
    """Geodesic views that see the prism's side faces: every sampled centre lies on a face whose normal equals its
    decoded normal (rotated to the body frame) within one 8-bit step; off the plane by at most one depth step plus the
    pixel-centre offset of PointVector (integer pixel coordinates, sampled at pixel centres)."""
    tri = np.asarray(synth_mod.prism_triangles()[0], np.float64).reshape(-1, 3, 3)
    normals = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    normals /= np.linalg.norm(normals, axis=1, keepdims=True)
    normals *= np.sign(np.einsum("ij,ij->i", normals, tri.mean(1)))[:, None]  # outward (the prism holds the origin)
    st = mg.Setup(_prism(synth_mod), [], 0.8, 300)
    a, b = np.float64(st.projection_term_a), np.float64(st.projection_term_b)
    poses = mg.geodesic_poses(0, 0.8)
    side = 0
    for pose in poses:
        img = mg.render_view(st, pose)
        pts, area = mg.view_points(st, pose, img, 40, 0.002, 0.05)
        assert area > 0
        R, t = pose[:, :3].astype(np.float64), pose[:, 3].astype(np.float64)
        for p in pts.astype(np.float64):
            c_cam = R.T @ (p[:3] - t)
            d16 = (b - a / c_cam[2])
            step = a / (b - d16 - 1) - a / (b - d16)
            tol = step + 0.75 * c_cam[2] / float(st.fu)
            same = np.abs(normals - p[3:6]).max(1) <= 1 / 127.5
            assert same.any(), p[3:6]
            dist = np.abs(np.einsum("ij,ij->i", normals[same], p[:3] - tri[same, 0]))
            assert dist.min() <= tol, (dist.min(), tol)
            side += int(abs(normals[same][0, 2]) < 0.5)
    assert side > 40  # the side faces are covered, not only the caps


def test_step_depth_offsets():
    """A step of height h at 10 px from the centre: offsets are 0 below the step's slot and h from it on."""
    S, a, b = 200, f32(0.6 * 1.0 * 65535 / 0.4), f32(1.0 * 65535 / 0.4)   # z range 0.6 .. 1.0
    depth_of = lambda d16: a / (b - f32(d16))
    depth = np.full((S, S), 40000, np.uint16)
    depth[:, 110:] = 30000  # nearer
    x = y = 100
    pixel_to_meter = f32(1e-3)  # stride 2 px, image_stride 3
    off = mg.depth_offsets(depth, x, y, pixel_to_meter, f32(0.002), 26, a, b)
    h = depth_of(40000) - depth_of(30000)
    stride = f32(0.002) / pixel_to_meter
    first = None
    rm = (int(f32(2) * f32(26) * stride / f32(3) + f32(1)) * 3) // 2
    for u in range(x - rm, x + rm + 1, 3):   # the nearest sampled column on the step
        if u >= 110:
            first = int(f32(np.sqrt(np.float64((u - x) ** 2))) / stride)
            break
    assert np.all(off[:first] == 0)
    assert np.all(off[first:] == h)


def test_offset_distance_is_stored_as_float():
    """std::sqrt(int) runs in double, the result is stored in a float and divided in float. For this pixel_to_meter
    the sampled pixel at (du, dv) = (-49, -28) falls in slot 20 that way; kept in double the quotient would put it in
    slot 19. A nearer depth there must therefore show up from slot 20 on."""
    S, a, b = 300, f32(0.6 * 1.0 * 65535 / 0.4), f32(1.0 * 65535 / 0.4)
    pixel_to_meter = f32(0.0007087699486874044)
    stride = f32(0.002) / pixel_to_meter
    n = 49 * 49 + 28 * 28
    d = np.sqrt(np.float64(n))
    assert int(f32(d) / stride) == 20 and int(d / np.float64(stride)) == 19
    assert f32(d) == np.sqrt(f32(n))  # sqrtf gives the same float: the double rounding of sqrt is innocuous
    depth = np.full((S, S), 40000, np.uint16)
    x = y = 150
    depth[y - 28, x - 49] = 30000
    off = mg.depth_offsets(depth, x, y, pixel_to_meter, f32(0.002), 26, a, b)
    h = a / (b - f32(40000)) - a / (b - f32(30000))
    assert np.all(off[:20] == 0) and np.all(off[20:] == h)


def test_occluder_hides_and_ties_go_to_the_body(synth_mod):
    body = _prism(synth_mod)
    twin = rr.Geometry(body.triangles, body.geometry2body, body.maximum_body_diameter, True)
    st = mg.Setup(body, [twin], 0.8, 200)
    img = mg.render_view(st, TOP)
    assert np.array_equal(img["silhouette"] != 0, img["depth"] != 0xFFFF)  # equal depths: the body drawn first wins
    tri, _ = synth_mod.icosphere_triangles(radius=0.02, n_divides=1)
    g2b = np.hstack([np.eye(3), [[0.0], [0.0], [0.03]]]).astype(f32)  # between the camera and the top face
    st = mg.Setup(body, [rr.Geometry(tri, g2b, 0.1, True)], 0.8, 200)
    img2 = mg.render_view(st, TOP)
    assert np.array_equal(img2["depth"], img["depth"])  # the main renderer draws the body alone
    assert 0 < np.count_nonzero(img2["silhouette"]) < np.count_nonzero(img["silhouette"])


def test_generated_model_file_round_trip(capi, tmp_path):
    """model_io.model_from_generated + write_model give the reference's file layout: wrapping the views of the
    reference's own depth_model.bin with its parameters and body block writes the same bytes."""
    model_io = importlib.import_module("3dobjecttracking_b200.model_io")
    path = os.path.join(GOLDEN, "depth_model.bin")
    mf = model_io.read_model(path)
    p = capi.model_params(sphere_radius=mf.sphere_radius, n_divides=mf.n_divides, n_points=mf.n_points,
                          max_radius_depth_offset=mf.max_radius_depth_offset,
                          stride_depth_offset=mf.stride_depth_offset, image_size=mf.image_size)
    out = tmp_path / "generated.bin"
    model_io.write_model(out, model_io.model_from_generated(mf.model, p, mf.body, mf.associated[0]))
    assert out.read_bytes() == open(path, "rb").read()
