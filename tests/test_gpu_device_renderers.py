"""Device renderers (k_render, m3tb_set_body_geometry / m3tb_set_focused_renderer / m3tb_attach_renderer / m3tb_render):
the focused depth and silhouette images, corner, scale, projection terms and visible flags equal the CPU restatement
(tests/render_reference.py) bit for bit; modalities fed by device renderers give the same records, histograms and poses
as the same context fed those images through m3tb_upload_*_rendering; contexts without attached renderers launch what
they launched before."""
import copy

import numpy as np
import pytest

import render_reference as rr
from helpers import assert_lines_bit_equal, assert_points_bit_equal

pytestmark = pytest.mark.gpu

W2C = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
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


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def _render_and_compare(capi, synth, geometry, poses, renderers, n_cams=1):
    """geometry / poses: {body: Geometry / [3,4]}; renderers: [dict(kind, cam, geometry, referenced, size, z_min, z_max,
    id_type)]. Renders on the device and compares every renderer with the CPU restatement."""
    intr = synth.default_color_intrinsics()
    max_bodies = max(poses) + 1
    ctx = capi.Context(0, max_bodies=max_bodies, max_cameras=n_cams, max_models=1)
    for c in range(n_cams):
        ctx.set_color_camera(c, intr, W2C)
        ctx.set_depth_camera(c, intr, W2C_DEPTH, 0.001)
    all_poses = np.stack([poses.get(b, W2C) for b in range(max_bodies)])
    ctx.set_poses(all_poses)
    for b, g in geometry.items():
        ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling, g.body_id,
                              g.region_id)
    for k, r in enumerate(renderers):
        ctx.set_focused_renderer(k, r.get("kind", "color"), r.get("cam", 0), r["geometry"], r["referenced"],
                                 r.get("size", 200), r.get("z_min", 0.02), r.get("z_max", 10.0), r.get("id_type", "body"))
    n0 = ctx.launch_count
    ctx.render()
    assert ctx.launch_count == n0 + 1
    results = []
    for k, r in enumerate(renderers):
        got = ctx.get_rendering(k)
        w2c = W2C if r.get("kind", "color") == "color" else W2C_DEPTH
        exp = rr.render_focused(intr, w2c, poses, geometry, r["geometry"], r["referenced"], r.get("size", 200),
                                r.get("z_min", 0.02), r.get("z_max", 10.0), r.get("id_type", "body"))
        for key in ("corner_u", "corner_v", "scale", "projection_term_a", "projection_term_b"):
            assert _bits(got[key]) == _bits(exp[key]), (k, key, got[key], exp[key])
        assert np.array_equal(got["visible"], exp["visible"]), k
        assert np.array_equal(got["depth"], exp["depth"]), (k, np.argwhere(got["depth"] != exp["depth"])[:5])
        assert np.array_equal(got["silhouette"], exp["silhouette"]), k
        results.append(exp)
    ctx.close()
    return results


def _prism(synth, body_id=1, region_id=1, culling=True):
    tri, diam = synth.prism_triangles()
    return rr.Geometry(tri, W2C.copy(), diam, culling, body_id, region_id)


@pytest.mark.parametrize("mesh", ["prism", "icosphere"])
@pytest.mark.parametrize("kind", ["color", "depth"])
def test_single_body_bit_exact(capi, synth, mesh, kind):
    if mesh == "prism":
        g = _prism(synth, 5, 9)
    else:
        tri, diam = synth.icosphere_triangles()
        g = rr.Geometry(tri, W2C.copy(), diam, True, 5, 9)
    res = _render_and_compare(capi, synth, {0: g}, {0: _pose((25, -30, 10), (0.03, -0.02, 0.5))},
                              [dict(kind=kind, geometry=[0], referenced=[0], id_type="region")])
    assert (res[0]["silhouette"] == 9).sum() > 2000


@pytest.mark.parametrize("n", [1, 8, 128])
def test_many_renderers_bit_exact(capi, synth, n):
    rng = np.random.default_rng(n)
    poses = {b: _pose(tuple(rng.uniform(-60, 60, 3)), (rng.uniform(-0.2, 0.2), rng.uniform(-0.15, 0.15), rng.uniform(0.3, 1.2)))
             for b in range(n)}
    geometry = {b: _prism(synth, b % 255 + 1, b % 7 + 1) for b in range(n)}
    renderers = [dict(kind="color" if b % 2 == 0 else "depth", cam=b % 4, geometry=[b], referenced=[b],
                      id_type="body" if b % 3 else "region") for b in range(n)]
    _render_and_compare(capi, synth, geometry, poses, renderers, n_cams=4)


def test_multi_body_occlusion_and_equal_depth_ties(capi, synth):
    tri, diam = synth.icosphere_triangles(0.03, 2)
    geometry = {0: _prism(synth, 1, 11), 1: rr.Geometry(tri, W2C.copy(), diam, True, 2, 12), 2: _prism(synth, 3, 13),
                3: _prism(synth, 4, 14, culling=False)}
    p0 = _pose((10, 20, 0), (0.0, 0.0, 0.5))
    poses = {0: p0, 1: _pose(t=(0.025, 0.01, 0.47)), 2: p0.copy(), 3: _pose((0, 180, 0), (-0.03, 0.0, 0.52))}
    res = _render_and_compare(capi, synth, geometry, poses, [
        dict(geometry=[0, 1, 2, 3], referenced=[0]),
        dict(geometry=[2, 1, 0, 3], referenced=[0, 1], id_type="region"),
        dict(geometry=[3, 0], referenced=[3, 0])])
    ids = set(np.unique(res[0]["silhouette"]))
    assert {1, 2, 4} <= ids and 3 not in ids     # the sphere occludes part of the prism; the first of two equal bodies wins
    assert 13 in set(np.unique(res[1]["silhouette"])) and 11 not in set(np.unique(res[1]["silhouette"]))


def test_near_plane_and_off_image(capi, synth):
    geometry = {0: _prism(synth, 1, 1), 1: _prism(synth, 2, 2, culling=False), 2: _prism(synth, 3, 3)}
    # body 1 straddles the near plane z_min = 0.3 inside the focused square; body 2 is cut by the focused image border
    poses = {0: _pose((5, 0, 0), (0.0, 0.0, 0.6)), 1: _pose((0, 70, 0), (0.0, 0.0, 0.3)),
             2: _pose((0, 0, 30), (0.05, 0.0, 0.6))}
    res = _render_and_compare(capi, synth, geometry, poses, [
        dict(geometry=[0, 1, 2], referenced=[0], z_min=0.3),
        dict(geometry=[0, 1, 2], referenced=[0], z_min=0.02)])
    assert 2 in set(np.unique(res[0]["silhouette"])) and 3 in set(np.unique(res[0]["silhouette"]))
    assert not np.array_equal(res[0]["silhouette"], res[1]["silhouette"])   # the clip removed part of body 1
    # a referenced body partly outside the camera image is still focused on; one entirely outside is not
    poses = {0: _pose(t=(-0.27, 0.0, 0.5)), 1: _pose(t=(1.0, 0.0, 0.5))}
    res = _render_and_compare(capi, synth, {0: _prism(synth), 1: _prism(synth)}, poses,
                              [dict(geometry=[0, 1], referenced=[0, 1])])
    assert list(res[0]["visible"]) == [1, 0]


@pytest.mark.parametrize("size", [8, 64, 128, 200, 240])
def test_image_sizes(capi, synth, size):
    _render_and_compare(capi, synth, {0: _prism(synth, 1, 1)}, {0: _pose((30, 10, 0), (0.01, 0.0, 0.4))},
                        [dict(geometry=[0], referenced=[0], size=size)])


def test_no_visible_body_leaves_the_images_cleared(capi, synth):
    res = _render_and_compare(capi, synth, {0: _prism(synth)}, {0: _pose(t=(0.0, 0.0, 0.01))},
                              [dict(geometry=[0], referenced=[0], size=32)])
    assert np.all(res[0]["depth"] == 65535) and np.all(res[0]["silhouette"] == 0)


def test_argument_errors(capi, synth):
    wl = synth.make_workload("c2", n_bodies=2, n_divides=2, seed=1)
    wl.region, wl.depth = copy.copy(wl.region), copy.copy(wl.depth)
    ctx = capi.context_from_workload(wl)
    tri, diam = synth.prism_triangles()
    E = capi.M3TBError
    with pytest.raises(E):
        ctx.set_body_geometry(2, tri)                       # body out of range
    with pytest.raises(E):
        ctx.set_body_geometry(0, tri, body_id=256)          # ids are uint8
    with pytest.raises(E):
        ctx.set_body_geometry(0, tri[:0], None, diam)       # no triangles
    ctx.set_body_geometry(0, tri, body_id=1, region_id=7)
    with pytest.raises(E):
        ctx.set_focused_renderer(0, "color", 0, [1], [1])   # body 1 has no geometry
    with pytest.raises(E):
        ctx.set_focused_renderer(1, "color", 0, [0], [0])   # ids are dense
    with pytest.raises(E):
        ctx.set_focused_renderer(0, "color", 5, [0], [0])   # no such camera
    with pytest.raises(E):
        ctx.set_focused_renderer(0, "color", 0, [0], [0], z_min=0.0)
    with pytest.raises(E, match="status -3"):
        ctx.set_focused_renderer(0, "color", 0, [0], [0], image_size=241)
    with pytest.raises(E):
        ctx.render()                                        # no renderer yet
    ctx.set_body_geometry(1, tri, body_id=2, region_id=7)
    ctx.set_focused_renderer(0, "color", 0, [0, 1], [0], id_type="body")
    ctx.set_focused_renderer(1, "depth", 0, [0], [0], id_type="body")
    ctx.set_focused_renderer(2, "color", 1, [1], [1], id_type="region")
    with pytest.raises(E):
        ctx.get_rendering(0)                                # not rendered yet
    with pytest.raises(E):
        ctx.attach_renderer(0, "region_silhouette", 0)      # region checking needs id_type REGION
    with pytest.raises(E):
        ctx.attach_renderer(0, "region_depth", 1)           # depth camera for the region modality
    with pytest.raises(E):
        ctx.attach_renderer(0, "region_depth", 2)           # camera 1 is body 1's camera, and body 0 is not referenced
    with pytest.raises(E):
        ctx.attach_renderer(1, "region_depth", 0)           # renderer 0 does not reference body 1
    with pytest.raises(E):
        ctx.attach_renderer(0, "region_depth", 7)           # no such renderer
    ctx.attach_renderer(0, "region_depth", 0)
    ctx.attach_renderer(0, "depth_silhouette", 1)
    r = synth.Rendering(np.zeros((200, 200), np.uint16), 0.0, 0.0, 1.0, 1.0, 1.0)
    with pytest.raises(E):
        ctx.upload_rendering(0, "region_depth", r)          # the slot is fed by a device renderer
    with pytest.raises(E):
        ctx.set_focused_renderer(0, "color", 0, [0], [0])   # attached: detach first
    ctx.attach_renderer(0, "region_depth", -1)
    ctx.upload_rendering(0, "region_depth", r)
    ctx.render()
    assert ctx.get_rendering(0)["depth"].shape == (200, 200)
    ctx.close()


# ---- the modalities fed by device renderers --------------------------------------------------------------------------
REGION_ID = 7


def _workload(synth):
    wl = synth.make_workload("c2", n_bodies=5, n_divides=3, seed=19)
    synth.fill_depth_offsets(wl.region_model)
    synth.fill_depth_offsets(wl.depth_model)
    wl.region, wl.depth = copy.copy(wl.region), copy.copy(wl.depth)
    wl.region.model_occlusions = wl.region.use_region_checking = True
    wl.depth.model_occlusions = wl.depth.use_silhouette_checking = True
    wl.region.n_unoccluded_iterations = wl.depth.n_unoccluded_iterations = 0
    return wl


def _scene(synth, wl):
    """One renderer per camera: body b's colour camera draws bodies b and its neighbour (region ids), its depth camera
    the same (body ids)."""
    tri, diam = synth.prism_triangles()
    geometry = {b: rr.Geometry(tri, W2C.copy(), diam, True, b + 1, REGION_ID) for b in range(wl.n_bodies)}
    renderers = []
    for b in range(wl.n_bodies):
        draw = [b, (b + 1) % wl.n_bodies]
        renderers.append(dict(kind="color", cam=b, geometry=draw, referenced=[b], id_type="region", body=b))
        renderers.append(dict(kind="depth", cam=b, geometry=draw, referenced=[b], id_type="body", body=b))
    return geometry, renderers


def _device_context(capi, synth, wl):
    ctx = capi.context_from_workload(wl)
    geometry, renderers = _scene(synth, wl)
    for b, g in geometry.items():
        ctx.set_body_geometry(b, g.triangles, None, g.maximum_body_diameter, True, g.body_id, g.region_id)
    for k, r in enumerate(renderers):
        ctx.set_focused_renderer(k, r["kind"], r["cam"], r["geometry"], r["referenced"], id_type=r["id_type"])
        m = "region" if r["kind"] == "color" else "depth"
        ctx.attach_renderer(r["body"], f"{m}_depth", k)
        ctx.attach_renderer(r["body"], f"{m}_silhouette", k)
    return ctx


def _upload_reference_images(ctx, synth, wl, poses):
    """What the device renderers produce at `poses`, restated on the CPU and handed over as uploaded images."""
    geometry, renderers = _scene(synth, wl)
    pd = {b: poses[b] for b in range(wl.n_bodies)}
    for r in renderers:
        m = "region" if r["kind"] == "color" else "depth"
        intr = wl.color_intrinsics if m == "region" else wl.depth_intrinsics
        w2c = wl.color_world2camera if m == "region" else wl.depth_world2camera
        o = rr.render_focused(intr, w2c, pd, geometry, r["geometry"], r["referenced"], id_type=r["id_type"])
        common = (float(o["corner_u"]), float(o["corner_v"]), float(o["scale"]))
        vis = bool(o["visible"][0])
        ctx.upload_rendering(r["body"], f"{m}_depth", synth.Rendering(o["depth"], *common, float(o["projection_term_a"]),
                                                                     float(o["projection_term_b"]), 0, vis))
        sid = REGION_ID if m == "region" else r["body"] + 1
        ctx.upload_rendering(r["body"], f"{m}_silhouette", synth.Rendering(o["silhouette"], *common, 0.0, 0.0, sid, vis))


def _assert_histograms_equal(a, b, wl):
    nb = wl.region.n_histogram_bins
    for body in range(wl.n_bodies):
        for x, y in zip(a.get_histograms(body, nb), b.get_histograms(body, nb)):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), body


def test_device_renderers_feed_the_modalities_like_uploaded_images(capi, synth):
    wl = _workload(synth)
    dev = _device_context(capi, synth, wl)
    up = capi.context_from_workload(wl)
    _upload_reference_images(up, synth, wl, wl.start_body2world)
    free = copy.deepcopy(wl)  # the same workload without the renderer-image checks
    free.region.model_occlusions = free.region.use_region_checking = False
    free.depth.model_occlusions = free.depth.use_silhouette_checking = False
    base = capi.context_from_workload(free)
    dev.start_modalities(0)
    up.start_modalities(0)
    _assert_histograms_equal(dev, up, wl)
    base.start_modalities(0)
    base.corr_iteration(0, 0, wl.n_update_iterations)
    rejected = 0
    for corr in range(wl.n_corr_iterations):
        _upload_reference_images(up, synth, wl, up.get_poses())
        dev.corr_iteration(0, corr, wl.n_update_iterations)
        up.corr_iteration(0, corr, wl.n_update_iterations)
        for b in range(wl.n_bodies):
            assert dev.get_closest_views(b) == up.get_closest_views(b)
            assert_lines_bit_equal(dev.get_region_lines(b, wl.lines_per_body), up.get_region_lines(b, wl.lines_per_body))
            assert_points_bit_equal(dev.get_depth_points(b, wl.points_per_body), up.get_depth_points(b, wl.points_per_body))
            if corr == 0:  # same start pose as the run without checks: what the checks removed
                rejected += int(base.get_region_lines(b, wl.lines_per_body)["valid"].sum() -
                                dev.get_region_lines(b, wl.lines_per_body)["valid"].sum())
                rejected += int(base.get_depth_points(b, wl.points_per_body)["valid"].sum() -
                                dev.get_depth_points(b, wl.points_per_body)["valid"].sum())
        assert np.array_equal(dev.get_poses().view(np.uint32), up.get_poses().view(np.uint32)), corr
    assert rejected > 50, rejected  # the device renderings really switched lines / points off
    _upload_reference_images(up, synth, wl, up.get_poses())
    dev.calculate_results(0)
    up.calculate_results(0)
    _assert_histograms_equal(dev, up, wl)
    assert dev.last_launch()["occ"] == 1
    for c in (dev, up, base):
        c.close()


def test_tracking_step_renders_before_every_correspondence_iteration(capi, synth):
    wl = _workload(synth)
    n_corr, n_upd = wl.n_corr_iterations, wl.n_update_iterations
    fused, stepwise, plain = _device_context(capi, synth, wl), _device_context(capi, synth, wl), capi.context_from_workload(wl)
    for c in (fused, stepwise, plain):
        c.start_modalities(0)
    for corr in range(n_corr - 1):
        stepwise.corr_iteration(0, corr, n_upd)
    before_last = stepwise.get_poses()
    stepwise.corr_iteration(0, n_corr - 1, n_upd)
    n_fused, n_plain = fused.launch_count, plain.launch_count
    fused.tracking_step(0, n_corr, n_upd)
    plain.tracking_step(0, n_corr, n_upd)
    # one k_render + one k_track per correspondence iteration instead of one fused launch
    assert fused.launch_count - n_fused == (plain.launch_count - n_plain) - 1 + 2 * n_corr
    assert np.array_equal(fused.get_poses().view(np.uint32), stepwise.get_poses().view(np.uint32))
    # what the renderers hold is the rendering at the pose the last correspondence iteration started from
    geometry, renderers = _scene(synth, wl)
    pd = {b: before_last[b] for b in range(wl.n_bodies)}
    for k, r in enumerate(renderers):
        intr = wl.color_intrinsics if r["kind"] == "color" else wl.depth_intrinsics
        w2c = wl.color_world2camera if r["kind"] == "color" else wl.depth_world2camera
        exp = rr.render_focused(intr, w2c, pd, geometry, r["geometry"], r["referenced"], id_type=r["id_type"])
        got = fused.get_rendering(k)
        assert np.array_equal(got["depth"], exp["depth"]) and np.array_equal(got["silhouette"], exp["silhouette"]), k
        assert _bits(got["scale"]) == _bits(exp["scale"]), k
    for c in (fused, stepwise, plain):
        c.close()


def test_contexts_without_attached_renderers_launch_as_before(capi, synth):
    wl = synth.make_workload("c2", n_bodies=4, n_divides=2, seed=3)
    plain = capi.context_from_workload(wl)
    with_geometry = capi.context_from_workload(wl)
    tri, diam = synth.prism_triangles()
    for b in range(wl.n_bodies):
        with_geometry.set_body_geometry(b, tri, None, diam)
    with_geometry.set_focused_renderer(0, "color", 0, [0], [0])   # set up, never attached
    stats = []
    for ctx in (plain, with_geometry):
        ctx.start_modalities(0)
        n0 = ctx.launch_count
        ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
        n1 = ctx.launch_count
        ctx.calculate_results(0)
        stats.append((n1 - n0, ctx.launch_count - n1, ctx.last_launch(), ctx.get_poses().tobytes()))
    assert stats[0] == stats[1]
    assert stats[0][2]["kernel"] == "k_track2"
    plain.close()
    with_geometry.close()
