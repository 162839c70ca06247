"""The CPU restatement of k_render (tests/render_reference.py) against closed forms: the exact silhouette and ray-cast
depth of the prism, single coverage of shared edges, culling on a closed mesh, and the focus terms of
FocusedRenderer::CalculateProjectionMatrix (renderer.cpp:348-405) evaluated independently in float64."""
import numpy as np
import pytest

import render_reference as rr

INTR = type("Intr", (), dict(fu=614.0, fv=614.5, ppu=321.3, ppv=238.9, width=640, height=480))()
W2C = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def _pose(rot_deg=(20.0, -35.0, 10.0), t=(0.03, -0.02, 0.5)):
    R = np.eye(3)
    for axis, deg in enumerate(rot_deg):
        c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
        i, j = [k for k in range(3) if k != axis]
        Q = np.eye(3)
        Q[i, i], Q[i, j], Q[j, i], Q[j, j] = c, -s, s, c
        R = R @ Q
    return np.hstack([R, np.array(t)[:, None]]).astype(np.float32)


def _geometry(synth, culling=True):
    tri, diam = synth.prism_triangles()
    return rr.Geometry(tri, W2C.copy(), diam, culling, body_id=3, region_id=9)


def _pixel_rays(out, S):
    """Camera pixel coordinates of the focused image's pixel centres: corner + (i, j) / scale."""
    j, i = np.mgrid[0:S, 0:S].astype(np.float64)
    return float(out["corner_u"]) + i / float(out["scale"]), float(out["corner_v"]) + j / float(out["scale"])


def test_prism_coverage_is_the_projected_silhouette_and_depth_is_the_ray_cast(synth):
    S = 200
    pose = _pose()
    geo = {0: _geometry(synth)}
    out = rr.render_focused(INTR, W2C, {0: pose}, geo, [0], [0], S)
    u, v = _pixel_rays(out, S)
    P = pose.astype(np.float64)
    verts = synth.PRISM_VERTICES @ P[:, :3].T + P[:, 3]
    # exact silhouette: the convex hull of the projected vertices (the prism is convex)
    pu, pv = INTR.fu * verts[:, 0] / verts[:, 2] + INTR.ppu, INTR.fv * verts[:, 1] / verts[:, 2] + INTR.ppv
    pts = np.stack([pu, pv], 1)
    c = pts.mean(0)
    hull = pts[np.argsort(np.arctan2(pts[:, 1] - c[1], pts[:, 0] - c[0]))]
    def turn(p, q, s):
        return (q[0] - p[0]) * (s[1] - q[1]) - (q[1] - p[1]) * (s[0] - q[0])
    keep = [k for k in range(len(hull)) if turn(hull[k - 1], hull[k], hull[(k + 1) % len(hull)]) > 1e-12]
    hull = hull[keep]
    dist = np.full(u.shape, np.inf)
    inside = np.ones(u.shape, bool)
    for k in range(len(hull)):
        a, b = hull[k], hull[(k + 1) % len(hull)]
        e = ((b[0] - a[0]) * (v - a[1]) - (b[1] - a[1]) * (u - a[0])) / np.hypot(*(b - a))
        inside &= e > 0
        dist = np.minimum(dist, np.abs(e))
    sure = dist * float(out["scale"]) > 1e-3  # farther than 1/1000 pixel from the outline
    covered = out["silhouette"] > 0
    assert covered.sum() > 2000
    assert np.array_equal(covered[sure], inside[sure])
    assert set(np.unique(out["silhouette"])) == {0, 3}
    # depth: the nearest face hit by the ray through the pixel centre
    x, y = (u - INTR.ppu) / INTR.fu, (v - INTR.ppv) / INTR.fv
    z_exact = np.full(u.shape, np.inf)
    for f in synth.PRISM_FACES:
        A, B, C = verts[f]
        n = np.cross(B - A, C - A)
        den = n[0] * x + n[1] * y + n[2]
        with np.errstate(divide="ignore", invalid="ignore"):
            z = (n @ A) / den
            X = np.stack([x * z, y * z, z], -1)
            bary = [np.einsum("...k,k->...", np.cross(Q - P0, X - P0), n) for P0, Q in ((A, B), (B, C), (C, A))]
        hit = (bary[0] >= 0) & (bary[1] >= 0) & (bary[2] >= 0) & (z > 0)
        z_exact = np.where(hit & (z < z_exact), z, z_exact)
    a, b = float(out["projection_term_a"]), float(out["projection_term_b"])
    expected = b - a / z_exact[covered & sure]
    assert np.abs(out["depth"][covered & sure].astype(np.float64) - expected).max() <= 1.0
    assert np.all(out["depth"][~covered] == 65535)


def test_shared_edge_covers_every_pixel_once():
    # a square facing the camera split along its diagonal, both halves drawn: no pixel twice, no hole inside
    s = 0.03
    quad = np.array([[-s, -s, 0], [s, -s, 0], [s, s, 0], [-s, s, 0]], np.float32)
    tri = np.stack([quad[[0, 1, 2]], quad[[0, 2, 3]]])
    g = rr.Geometry(tri, W2C.copy(), float(np.float32(2 * s * np.sqrt(2))), enable_culling=False)
    for pose in (_pose((0, 0, 0), (0.0, 0.0, 0.5)), _pose((0, 0, 45), (0.01, 0.0, 0.4)), _pose((10, 5, 30), (0, 0, 0.6))):
        out = rr.render_focused(INTR, W2C, {0: pose}, {0: g}, [0], [0], 64, coverage=True)
        cov = out["coverage"]
        assert cov.max() == 1
        # no hole: the covered pixels are exactly the centres inside the projected square (away from its outline)
        u, v = _pixel_rays(out, 64)
        P = pose.astype(np.float64)
        corners = quad.astype(np.float64) @ P[:, :3].T + P[:, 3]
        cu, cv = INTR.fu * corners[:, 0] / corners[:, 2] + INTR.ppu, INTR.fv * corners[:, 1] / corners[:, 2] + INTR.ppv
        e = [(cu[(k + 1) % 4] - cu[k]) * (v - cv[k]) - (cv[(k + 1) % 4] - cv[k]) * (u - cu[k]) for k in range(4)]
        inside = np.all([x > 0 for x in e], 0) | np.all([x < 0 for x in e], 0)
        sure = np.min([np.abs(x) / np.hypot(cu[(k + 1) % 4] - cu[k], cv[(k + 1) % 4] - cv[k]) for k, x in enumerate(e)], 0)
        sure = sure * float(out["scale"]) > 1e-3
        assert inside.sum() > 100 and np.array_equal((cov == 1)[sure], inside[sure])
        covered = cov == 1
        # no holes: every row's covered run is contiguous
        for row in covered:
            idx = np.flatnonzero(row)
            if idx.size:
                assert idx[-1] - idx[0] + 1 == idx.size


def test_culling_keeps_the_silhouette_of_a_closed_mesh(synth):
    tri, diam = synth.icosphere_triangles(0.04, 2)
    pose = _pose((0, 30, 0), (0.02, 0.01, 0.45))
    on = rr.render_focused(INTR, W2C, {0: pose}, {0: rr.Geometry(tri, W2C.copy(), diam, True, 1, 1)}, [0], [0], 96)
    off = rr.render_focused(INTR, W2C, {0: pose}, {0: rr.Geometry(tri, W2C.copy(), diam, False, 1, 1)}, [0], [0], 96)
    assert (on["silhouette"] > 0).sum() > 3000
    assert np.array_equal(on["silhouette"], off["silhouette"])
    assert np.array_equal(on["depth"], off["depth"])
    # reversed winding with culling on: only the far side survives (deeper everywhere it is drawn)
    back = rr.render_focused(INTR, W2C, {0: pose}, {0: rr.Geometry(tri[:, [0, 2, 1]], W2C.copy(), diam, True, 1, 1)}, [0], [0], 96)
    both = (back["silhouette"] > 0) & (on["silhouette"] > 0)
    assert both.sum() > 3000 and np.all(back["depth"][both] > on["depth"][both])


def _focus64(intr, centers, radii, S, z_min, z_max):
    """renderer.cpp:348-405 in float64, skipping as written."""
    u_min, u_max, v_min, v_max = np.finfo(np.float32).max, np.finfo(np.float32).tiny, np.finfo(np.float32).max, np.finfo(np.float32).tiny
    vis = []
    for (x, y, z), r in zip(centers, radii):
        if z < r * 1.5 or z - r < z_min or z + r > z_max:
            vis.append(0)
            continue
        z2_r2 = z * z - r * r
        r_u = intr.fu * (abs(x) * r * r + r * z * np.sqrt(z2_r2 + x * x)) / (z2_r2 * z)
        r_v = intr.fv * (abs(y) * r * r + r * z * np.sqrt(z2_r2 + y * y)) / (z2_r2 * z)
        cu, cv = x * intr.fu / z + intr.ppu, y * intr.fv / z + intr.ppv
        if cu - r_u > intr.width or cu + r_u < 0 or cv - r_v > intr.height or cv + r_v < 0:
            vis.append(0)
            continue
        u_min, u_max = min(u_min, cu - r_u), max(u_max, cu + r_u)
        v_min, v_max = min(v_min, cv - r_v), max(v_max, cv + r_v)
        vis.append(1)
    d = max(u_max - u_min, v_max - v_min) * 1.05
    return 0.5 * (u_min + u_max - d), 0.5 * (v_min + v_max - d), S / d, vis


def test_focus_terms_and_skip_rules(synth):
    tri, diam = synth.prism_triangles()
    r = 0.5 * diam
    centers = [(0.02, 0.01, 0.5),        # visible
               (-0.05, 0.03, 0.7),       # visible
               (0.0, 0.0, 1.2 * r),      # z < 1.5 r
               (0.0, 0.0, 0.02 + 0.5 * r),  # z - r < z_min (and not z < 1.5 r: z_min is raised below)
               (0.0, 0.0, 9.99),         # z + r > z_max
               (2.0, 0.0, 0.5)]          # off the image
    poses = {b: np.hstack([np.eye(3), np.array(c)[:, None]]).astype(np.float32) for b, c in enumerate(centers)}
    geo = {b: rr.Geometry(tri, W2C.copy(), diam) for b in poses}
    z_min, z_max = 0.1, 10.0
    centers[3] = (0.0, 0.0, z_min + 0.5 * r)
    poses[3][2, 3] = np.float32(centers[3][2])
    out, _, any_visible = rr.focus(INTR, W2C, poses, geo, list(poses), 200, z_min, z_max)
    cu, cv, sc, vis = _focus64(INTR, [tuple(map(float, poses[b][:, 3])) for b in poses], [float(np.float32(0.5) * np.float32(diam))] * 6, 200, z_min, z_max)
    assert any_visible and list(out["visible"]) == vis == [1, 1, 0, 0, 0, 0]
    assert abs(float(out["corner_u"]) - cu) < 1e-3 and abs(float(out["corner_v"]) - cv) < 1e-3
    assert abs(float(out["scale"]) / sc - 1.0) < 1e-5
    assert float(out["projection_term_a"]) == pytest.approx(z_max * z_min * 65535 / (z_max - z_min), rel=1e-6)
    assert float(out["projection_term_b"]) == pytest.approx(z_max * 65535 / (z_max - z_min), rel=1e-6)
    # no visible body: the limits stay at float max / float min, so the corner is +inf and the scale -0
    hidden = {b: poses[b] for b in (2, 3, 4, 5)}
    out, _, any_visible = rr.focus(INTR, W2C, hidden, geo, list(hidden), 200, z_min, z_max)
    assert not any_visible and list(out["visible"]) == [0, 0, 0, 0]
    assert np.isinf(out["corner_u"]) and out["corner_u"] > 0 and out["scale"] == 0 and np.signbit(out["scale"])
    img = rr.render_focused(INTR, W2C, hidden, geo, list(hidden), list(hidden), 32, z_min, z_max)
    assert np.all(img["depth"] == 65535) and np.all(img["silhouette"] == 0)
