"""CPU checks of the region-model generation restatement (tests/region_model_generation_reference.py): its border
following equals cv2.findContours(RETR_LIST, CHAIN_APPROX_NONE) point for point and in order, and the sampling loop
gives up after 101 consecutive rejections as RegionModel::GeneratePointData does."""
import os
import sys
import types

import numpy as np
import pytest

import region_model_generation_reference as rg

cv2 = pytest.importorskip("cv2")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
if GOLDEN not in sys.path:
    sys.path.insert(0, GOLDEN)


def _cv2(mask):
    contours, _ = cv2.findContours(np.ascontiguousarray(mask, np.uint8), cv2.RETR_LIST, cv2.CHAIN_APPROX_NONE)
    return [c.reshape(-1, 2) for c in contours]


def _same(mask):
    exp, got = _cv2(mask), rg.find_contours(mask)
    assert len(exp) == len(got)
    for a, b in zip(exp, got):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("size", [1, 2, 3, 5, 8, 17, 40, 96])
@pytest.mark.parametrize("fill", [0.2, 0.5, 0.8])
def test_random_masks(size, fill):
    rng = np.random.RandomState(size * 10 + int(fill * 10))
    for _ in range(6):
        w = max(1, size + rng.randint(-1, 3))
        _same((rng.rand(size, w) < fill).astype(np.uint8) * 255)


def test_nested_holes():
    m = np.zeros((30, 30), np.uint8)
    for k, v in enumerate((1, 0, 1, 0, 1, 0)):
        m[2 + 2 * k:28 - 2 * k, 2 + 2 * k:28 - 2 * k] = v
    _same(m)


def test_thin_lines_and_diagonal_joins():
    m = np.zeros((24, 24), np.uint8)
    m[3, 2:20] = 1                          # 1-px horizontal line
    m[5:20, 4] = 1                          # 1-px vertical line
    for k in range(10):
        m[8 + k, 8 + k] = 1                 # diagonal-only joins
        m[8 + k, 20 - k] = 1
    m[20, 20] = 1                           # single pixels
    m[22, 2] = 1
    _same(m)


def test_shapes_touching_every_edge():
    m = np.zeros((16, 20), np.uint8)
    m[0, :] = 1
    m[:, 0] = 1
    m[-1, 5:] = 1
    m[3:12, -1] = 1
    m[6:9, 6:9] = 1
    _same(m)
    _same(np.ones((7, 9), np.uint8))


def test_exhausted_tries_zero_the_view():
    """A 1-px line whose only valid points are its two tips: at a tip the contour folds back, the chord between the
    ends of the +-3 segment is 0, every draw is rejected, and after 101 rejections contour_length is 0 and no point is
    produced."""
    S = 40
    main = np.zeros((S, S), np.uint8)
    main[20, 10:30] = rg.MAIN_BODY_ID
    occ = np.full((S, S), rg.MAIN_BODY_ID, np.uint8)
    occ[20, 10] = occ[20, 29] = 0
    st = types.SimpleNamespace(S=S, r=np.float32(0.8), fu=np.float32(50), pp=np.float32(20),
                               projection_term_a=np.float32(1000), projection_term_b=np.float32(70000))
    depth = np.full((S, S), 1000, np.uint16)
    c2b = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
    pts, length, contours = rg.view_points(st, c2b, {"main": main, "occlusion": occ}, depth, 4, 0.002, 0.05)
    assert len(contours) == 1 and len(contours[0]) == 38
    assert length == 0 and not pts.any()
    # without the occlusion every contour point is valid and most segments are straight: the view is kept
    pts, length, _ = rg.view_points(st, c2b, {"main": main}, depth, 4, 0.002, 0.05)
    assert length == np.float32(38) * (st.r / st.fu) and pts[:, 2].all()


def _rig_setup(f, pp, depth_m):
    """A restatement setup on the reference rig's 2000 px render: its focal length and principal point, a depth16
    image of its ray-cast depth in a projection whose range holds every depth of the view."""
    import reference_rig as rig
    fin = np.isfinite(depth_m)
    lo, hi = np.float32(depth_m[fin].min() - 0.01), np.float32(depth_m[fin].max() + 0.01)
    a = hi * lo * np.float32(65535) / (hi - lo)
    b = hi * np.float32(65535) / (hi - lo)
    d16 = np.full(depth_m.shape, 65535, np.uint16)
    d16[fin] = np.rint(b - a / depth_m[fin].astype(np.float32)).astype(np.uint16)
    return types.SimpleNamespace(S=rig.IMAGE_SIZE, r=np.float32(rig.SPHERE_RADIUS), fu=np.float32(f), pp=np.float32(pp),
                                 projection_term_a=a, projection_term_b=b), d16


def test_triangle_views_match_the_rig():
    """On the triangle's template views that tests/golden/reference_rig.py renders (exact ray cast, cv2 contours,
    float64 arithmetic), the restatement samples the same contour points, and gives the same normals, centres and
    foreground / background distances up to depth quantisation and float32 rounding."""
    import reference_rig as rig
    r = rig.rig()
    for w2c in (r["color_w2c"], r["depth_w2c"]):
        _, _, c2b, _ = rig.closest_view_pose(w2c @ r["body2world"])
        exp, exp_length = rig.region_view_points(c2b)
        mask, depth_m, _, f, pp = rig.render(c2b)
        st, d16 = _rig_setup(f, pp, depth_m)
        got, length, contours = rg.view_points(st, c2b[:3].astype(np.float32), {"main": mask}, d16, rig.N_POINTS,
                                               0.002, 0.05)
        assert [len(c) for c in contours] == [len(c) for c in rig.cv2.findContours(
            mask, rig.cv2.RETR_LIST, rig.cv2.CHAIN_APPROX_NONE)[0] if len(c) >= rg.MIN_CONTOUR_LENGTH]
        assert abs(float(length) / float(exp_length) - 1) < 1e-6
        assert np.abs(got[:, 3:6] - exp[:, 3:6]).max() < 1e-6                 # the same centres and segments
        assert np.abs(got[:, 0:3] - exp[:, 0:3]).max() < 2e-5                 # depth16 quantisation
        assert np.array_equal(got[:, 7] == rg.FLT_MAX, exp[:, 7] == rg.FLT_MAX)
        # the rig walks the line in float64, the reference in float32: a few walks end one pixel apart
        pixel_to_meter = depth_m[np.isfinite(depth_m)].max() / f
        fg_err = np.abs(got[:, 6] - exp[:, 6])
        assert (fg_err <= 1.5 * pixel_to_meter).all(), fg_err.max() / pixel_to_meter
        assert (np.abs(got[:, 6] / exp[:, 6] - 1) < 1e-5).mean() >= 0.95


def _top_view():
    """camera2body of a camera 0.8 m above the prism on its axis, looking down -z (Model::GenerateGeodesicPoses form)."""
    p = np.array([0.0, 0.0, 1.0], np.float32)
    c2 = -p
    c0 = np.cross([0.0, 1.0, 0.0], c2).astype(np.float32)
    c0 /= np.linalg.norm(c0)
    c1 = np.cross(c2, c0).astype(np.float32)
    return np.stack([c0, c1, c2, p * np.float32(0.8)], 1).astype(np.float32)


def test_prism_top_view_closed_forms():
    """From above, the prism's silhouette is the triangle of its top face. Contour length = its 8-connected pixel
    perimeter, normals = the outward unit normals of its edges, foreground distance = the chord across the triangle
    along the normal, background = FLT_MAX (nothing else is drawn)."""
    import importlib
    import render_reference as rr
    synth = importlib.import_module("3dobjecttracking_b200.synth")
    tri, diam = synth.prism_triangles()
    I34 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
    body = rr.Geometry(tri, I34, diam, True)
    S = 400
    st = rg.Setup(body, ((), (), (), ()), 0.8, S)
    pose = _top_view()
    sils, depth = st.render(pose)
    n = 60
    pts, length, contours = rg.view_points(st, pose, sils, depth, n, 0.002, 0.05)
    # the top face (z = 0.006) in pixel coordinates: column = fu * x_c / z_c + pp, with camera x = -body x, y = body y
    top = synth.PRISM_VERTICES[1::2]
    zc = 0.8 - 0.006
    uv = np.stack([float(st.fu) * -top[:, 0] / zc + float(st.pp), float(st.fu) * top[:, 1] / zc + float(st.pp)], 1)
    edges = [(uv[i], uv[(i + 1) % 3]) for i in range(3)]
    centroid = uv.mean(0)
    steps = sum(max(abs(q[0] - p[0]), abs(q[1] - p[1])) for p, q in edges)  # 8-connected perimeter in pixels
    px = float(st.r / st.fu)
    assert abs(float(length) / px - steps) <= 6, (float(length) / px, steps)
    assert (pts[:, 7] == rg.FLT_MAX).all()
    flat = np.concatenate(contours)
    for k in range(n):
        nb = pts[k, 3:6]  # body frame; the camera looks down -z, so the normal lies in the xy plane
        assert abs(nb[2]) < 1e-6 and abs(np.linalg.norm(nb) - 1) < 1e-6
        nc = np.array([-nb[0], nb[1]])  # image direction of the normal
        c = pts[k, 0:3]
        cu = np.array([float(st.fu) * -c[0] / zc + float(st.pp), float(st.fu) * c[1] / zc + float(st.pp)])
        d_edge = [abs((q - p)[0] * (cu - p)[1] - (q - p)[1] * (cu - p)[0]) / np.linalg.norm(q - p) for p, q in edges]
        e = int(np.argmin(d_edge))
        if min(np.linalg.norm(cu - v) for v in uv) < 6:
            continue  # the +-3 segment bends round a corner
        p, q = edges[e]
        t = (q - p) / np.linalg.norm(q - p)
        out = np.array([t[1], -t[0]])
        if np.dot(out, p - centroid) < 0:
            out = -out
        assert np.dot(nc, out) > np.cos(np.radians(6)), (k, nc, out)
        # chord: from the point along -normal to the far side of the triangle
        best = np.inf
        for j, (a, b) in enumerate(edges):
            if j == e:
                continue
            m = np.array([[-nc[0], a[0] - b[0]], [-nc[1], a[1] - b[1]]])
            s_, w = np.linalg.solve(m, a - cu)
            if s_ > 0 and -1e-6 <= w <= 1 + 1e-6:
                best = min(best, s_)
        chord_px = float(pts[k, 6]) / (zc / float(st.fu))
        assert abs(chord_px - best) <= 3, (k, chord_px, best)
    assert len(flat) == int(round(float(length) / px))
