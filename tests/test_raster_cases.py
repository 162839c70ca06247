"""The adversarial raster scenes of raster_cases.py on the CPU: each reaches the branches it is built for (the reach
counters of render_reference), the focused and the keyed triangle walks agree on them, coverage on the exact-tie scenes
equals an exact (fractions.Fraction) evaluation of the edge functions with the top-left rule, and the mask meshes of
model generation render their masks."""
from fractions import Fraction

import numpy as np
import pytest

import model_generation_reference as mg
import raster_cases as rc
import region_model_generation_reference as rg
import render_reference as rr
import viewer_reference as vr

f32 = np.float32
SCENES = {s.name: s for s in rc.camera_scenes()}


@pytest.mark.parametrize("name", list(SCENES))
def test_scene_reaches_what_it_is_built_for(name):
    scene = SCENES[name]
    stats = {}
    rc.render_camera(scene, stats)
    missing = [k for k in scene.reaches if not stats.get(k)]
    assert not missing, (missing, stats)


def _walks(scene, W, H):
    """The scene through rr.raster_keyed (k_view / k_model key) and through rr.raster_triangle (k_render key) with the
    same clip matrices."""
    intr = rc.exact_intrinsics(W, H)
    P = vr.projection(intr, *scene.z_range)
    keyed = np.full((H, W), np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    packed = np.full((H, W), 0xFFFFFFFF, np.uint32)
    poses = scene.pose_map()
    for g, b in enumerate(scene.bodies):
        G = scene.geometry[b]
        M = vr.clip_matrix(P, rr.pose_mul(rc.I34, rr.pose_mul(poses[b], G.geometry2body)))
        rr.raster_keyed(M, G.triangles, G.enable_culling, W, H, g, keyed)
        clip, dist = rr.clip_body(M, G.triangles)
        for t in range(dist.shape[0]):
            poly = rr.clip_polygon([tuple(clip[r][t, k] for r in range(4)) for k in range(3)], list(dist[t]))
            if len(poly) < 3:
                continue
            for v0, v1, v2 in rr.fans(rr.window(poly, rr.HALF * f32(W), rr.HALF * f32(H))):
                assert W == H
                rr.raster_triangle(v0, v1, v2, G.enable_culling, W, g, packed)
    return keyed, packed


@pytest.mark.parametrize("name", list(SCENES))
def test_focused_and_keyed_walks_agree(name):
    scene = SCENES[name]
    keyed, packed = _walks(scene, 48, 48)
    assert np.array_equal((keyed >> np.uint64(48)).astype(np.uint32), packed >> np.uint32(16))
    drawn = packed != 0xFFFFFFFF
    assert np.array_equal(((keyed >> np.uint64(32)) & np.uint64(0xFFFF))[drawn].astype(np.uint32),
                          (packed & np.uint32(0xFFFF))[drawn])
    # and the camera-image restatements (full renderer, viewer normal) are this walk
    out = rc.render_camera(rc.Scene(scene.name, scene.geometry, scene.bodies, scene.z_range, size=(48, 48)))
    assert np.array_equal(out["depth"], (keyed >> np.uint64(48)).astype(np.uint16))


def _exact_coverage(tri, W, H):
    """Coverage count of window-space triangles by exact arithmetic: a pixel centre is covered when every edge
    function of the positively oriented triangle is positive, or zero on a top edge (horizontal, running towards -x)
    or a left edge (running towards +y in window coordinates)."""
    cov = np.zeros((H, W), np.int32)
    for v in tri:
        p = [(Fraction(float(x)), Fraction(float(y))) for x, y, _ in v]
        A = (p[1][0] - p[0][0]) * (p[2][1] - p[0][1]) - (p[2][0] - p[0][0]) * (p[1][1] - p[0][1])
        if A == 0:
            continue
        if A < 0:
            p = [p[0], p[2], p[1]]
        xs = [q[0] for q in p]
        ys = [q[1] for q in p]
        for j in range(max(0, int(min(ys)) - 1), min(H, int(max(ys)) + 2)):
            for i in range(max(0, int(min(xs)) - 1), min(W, int(max(xs)) + 2)):
                c = (Fraction(2 * i + 1, 2), Fraction(2 * j + 1, 2))
                ok = True
                for a, b in ((p[1], p[2]), (p[2], p[0]), (p[0], p[1])):
                    e = (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])
                    top_left = b[1] > a[1] or (b[1] == a[1] and b[0] < a[0])
                    ok &= e > 0 or (e == 0 and top_left)
                cov[j, i] += ok
    return cov


@pytest.mark.parametrize("name", ["grid", "fan"])
def test_exact_ties_follow_the_top_left_rule(name):
    scene = SCENES[name]
    W, H = scene.size
    P = vr.projection(rc.exact_intrinsics(W, H), *scene.z_range)
    G = scene.geometry[0]
    M = vr.clip_matrix(P, rr.pose_mul(rc.I34, G.geometry2body))
    clip, dist = rr.clip_body(M, G.triangles)
    cov = np.zeros((H, W), np.int32)
    wins, stats = [], {}
    for t in range(dist.shape[0]):
        poly = rr.clip_polygon([tuple(clip[r][t, k] for r in range(4)) for k in range(3)], list(dist[t]))
        win = rr.window(poly, rr.HALF * f32(W), rr.HALF * f32(H))
        assert all(float(x) % 1 == 0.5 and float(y) % 1 == 0.5 for x, y, _ in win)  # vertices on pixel centres
        wins.append(win)
        rr.fragments(win[0], win[1], win[2], False, W, H, stats, cov)
    assert np.array_equal(cov, _exact_coverage(wins, W, H))
    assert stats["tie_owned"] > 100 and stats["tie_not_owned"] > 100, stats
    if name == "grid":  # the tessellation covers every pixel of the image exactly once
        assert (cov == 1).all()
    else:
        assert cov.max() == 1 and cov.sum() == 12 * 12


def test_odd_sizes_keep_the_grid_watertight():
    for W, H in rc.ODD_SIZES[:-1]:
        assert (rc.render_camera(rc.sized_scenes(W, H)[0])["silhouette"] != 0).all(), (W, H)


MASK_SIZES = [21, 33, 63, 97, 256]


@pytest.mark.parametrize("S", MASK_SIZES)
def test_mask_meshes_render_their_masks(S):
    for name, mask in rc.contour_masks(S).items():
        view = 3
        body = rc.mask_mesh(mask, view)
        st = mg.Setup(body, [], 0.8, S)
        img = mg.render_view(st, mg.geodesic_poses(0, 0.8)[view])
        assert np.array_equal(img["silhouette"] != 0, mask), (S, name)


def test_contour_masks_reach_what_they_are_built_for():
    masks = rc.contour_masks(33)
    lengths = [len(c) for c in rg.find_contours(masks["lengths_14_15_16"])]
    assert sorted(lengths) == [14, 15, 16]
    assert sorted(len(c) for c in rg.valid_contours(np.where(masks["lengths_14_15_16"], 255, 0))) == [15, 16]
    for c in rg.find_contours(masks["lines"]):  # 1-px lines: every contour visits pixels twice
        assert len({tuple(p) for p in c}) < len(c)
    assert len(rg.find_contours(masks["nested_4"])) == 8 and len(rg.find_contours(masks["ring_1px_hole"])) == 2
    assert any(len(c) == 1 for c in rg.find_contours(masks["single_pixels"]))
    # diagonal-only joins are one 8-connected component
    assert len(rg.find_contours(masks["diagonal_joins"])) == 2
    S = 200
    over, under = rc.block_grid(S, 33), rc.block_grid(S, 28)
    assert sum(len(c) for c in rg.find_contours(over)) > 64 * S >= sum(len(c) for c in rg.find_contours(under))


def test_region_restatement_reads_off_image_neighbours_as_background():
    """Contour points on the image border have neighbours outside it, which read as background: no wrap-around to the
    opposite border and no read past the last row."""
    S = 21
    body = rc.mask_mesh(rc.contour_masks(S)["border"], 3)
    st = rg.Setup(body, ((), (), (), ()), 0.8, S)
    sils, depth = st.render(mg.geodesic_poses(0, 0.8)[3])
    main = sils["main"].copy()
    _, length, contours = rg.view_points(st, mg.geodesic_poses(0, 0.8)[3], sils, depth, 8, 0.002, 0.05)
    assert len(contours) == 8 and length == np.float32(8 * 16) * (st.r / st.fu)
    main[S // 2, S // 2] = rg.DIFFERENT_BODY_ID  # a fixed body far from every border changes nothing
    assert rg.view_points(st, mg.geodesic_poses(0, 0.8)[3], dict(main=main), depth, 8, 0.002, 0.05)[1] == length
