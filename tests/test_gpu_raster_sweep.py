"""The device rasterisers on the adversarial scenes of raster_cases.py, bit for bit against their restatements: full
renderers (several renderers of mixed sizes in one m3tb_render_full) and viewers of both kinds (k_view_setup /
k_view_raster / k_view_resolve) on exact edge ties, near- and far-plane cuts, vertices on the near plane, NaN edge
values, degenerate and non-finite vertices, triangle- and draw-index depth ties, tile-edge boxes and frames 1 pixel
wide or high; k_render at focused sizes 1 to 240 with a few hundred geometry bodies; k_model_raster through
debug_render_model_view on non-finite and clipped geometry."""
import numpy as np
import pytest

import full_renderer_reference as fr
import model_generation_reference as mg
import raster_cases as rc
from test_gpu_device_renderers import _render_and_compare
from test_gpu_viewers import _check as _check_viewer, _frame, _setup, _upload

pytestmark = pytest.mark.gpu

I34 = rc.I34
SCENES = {s.name: s for s in rc.camera_scenes()}


def _intr(capi, W, H):
    i = rc.exact_intrinsics(W, H)
    return capi.Intrinsics(i.fu, i.fv, i.ppu, i.ppv, W, H)


def _full_context(capi, geometry, poses, sizes):
    """One colour camera per size, in order."""
    nb = max(geometry) + 1
    ctx = capi.Context(0, max_bodies=nb, max_cameras=len(sizes), max_models=1)
    for c, (W, H) in enumerate(sizes):
        ctx.set_color_camera(c, _intr(capi, W, H), I34)
    ctx.set_poses(np.stack([poses.get(b, I34) for b in range(nb)]))
    for b, g in geometry.items():
        ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling, g.body_id,
                              g.region_id)
    return ctx


def _compare_full(ctx, capi, r, size, scene, z_range, id_type):
    W, H = size
    got = ctx.get_full_rendering(r, W, H)
    exp = fr.render_full(rc.exact_intrinsics(W, H), I34, scene.pose_map(), scene.geometry, scene.bodies, *z_range,
                         id_type)
    for key in ("depth", "silhouette", "normal"):
        assert np.array_equal(got[key], exp[key]), (scene.name, size, key, np.argwhere(got[key] != exp[key])[:5])
    return exp


@pytest.mark.parametrize("name", list(SCENES))
def test_full_renderers_on_adversarial_scenes(capi, name):
    """The scene at its own exact frame and at frames of other sizes, z ranges and id types, in one render."""
    scene = SCENES[name]
    sizes = [scene.size, (31, 33), (1, 64), (64, 1)]
    ctx = _full_context(capi, scene.geometry, scene.pose_map(), sizes)
    renderers = [(0, scene.z_range, "body"), (1, scene.z_range, "region"), (2, scene.z_range, "body"),
                 (3, scene.z_range, "region"), (0, (0.02, 10.0), "region")]
    for r, (cam, (z0, z1), idt) in enumerate(renderers):
        ctx.set_full_renderer(r, "color", cam, scene.bodies, z0, z1, idt)
    ctx.render_full()
    for r, (cam, z, idt) in enumerate(renderers):
        exp = _compare_full(ctx, capi, r, sizes[cam], scene, z, idt)
        if r == 0 and scene.name not in ("nan_edges",):
            assert (exp["silhouette"] != 0).any(), name
    ctx.close()


@pytest.mark.parametrize("size", rc.ODD_SIZES)
def test_full_renderers_at_odd_sizes(capi, size):
    scenes = rc.sized_scenes(*size)
    geometry, bodies = {}, []
    for k, s in enumerate(scenes):  # every scene's body in one context, one renderer per scene
        geometry[k] = s.geometry[0]
        bodies.append(k)
    ctx = _full_context(capi, geometry, {}, [size])
    for k, s in enumerate(scenes):
        ctx.set_full_renderer(k, "color", 0, [k], *s.z_range, "body")
    ctx.set_full_renderer(len(scenes), "color", 0, bodies, *rc.EXACT_Z, "body")
    ctx.render_full()
    for k, s in enumerate(scenes):
        _compare_full(ctx, capi, k, size, s, s.z_range, "body")
    _compare_full(ctx, capi, len(scenes), size, rc.Scene("all", geometry, bodies), rc.EXACT_Z, "body")
    ctx.close()


@pytest.mark.parametrize("kind", ["color", "depth"])
def test_viewers_on_adversarial_scenes(capi, kind):
    """One viewer per scene (the viewers' own z range 0.02 .. 10), all updated together."""
    names = ["grid", "fan", "near_culled", "near_unculled", "two_draws", "degenerate_culled", "tiles"]
    geometry, order = {}, {}
    for n in names:
        s = SCENES[n]
        order[n] = []
        for b in s.bodies:
            geometry[len(geometry)] = s.geometry[b]
            order[n].append(len(geometry) - 1)
    W, H = 64, 64
    intr = _intr(capi, W, H)
    ctx = _setup(capi, geometry, {b: I34 for b in geometry}, [(kind, intr, I34, 0.001)])
    frame = _frame(kind, W, H, 5)
    _upload(ctx, kind, 0, frame)
    for v, n in enumerate(names):
        ctx.set_viewer(v, kind, 0, order[n], 0.7)
    ctx.update_viewers()
    for v, n in enumerate(names):
        _check_viewer(ctx, v, kind, intr, I34, {b: I34 for b in geometry}, geometry, order[n], frame, 0.7)
    ctx.close()


# ---- k_render ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("size", rc.FOCUSED_SIZES)
def test_focused_renderers_many_bodies(capi, synth, size):
    geometry, poses = rc.focused_scene(300, size)
    n = len(geometry)
    renderers = [dict(geometry=list(range(n)), referenced=[0, 1, 2], size=size, z_min=0.3),
                 dict(geometry=list(range(n))[::-1], referenced=[5], size=size, id_type="region"),
                 dict(kind="depth", geometry=list(range(0, n, 7)), referenced=[7, 14], size=size, z_min=1e-30)]
    _render_and_compare(capi, synth, geometry, poses, renderers)


def test_focused_renderers_on_adversarial_geometry(capi, synth):
    """The near-plane, NaN-edge and degenerate bodies of the camera scenes (camera frame, identity poses) drawn into
    the focused square of a small referenced body, at z_min 1e-30 and 1."""
    geometry, poses = rc.focused_scene(1, 3)
    poses[0] = np.hstack([np.eye(3), np.array([[0.0], [0.0], [1.5]])]).astype(np.float32)
    for n in ("near_culled", "near_unculled", "nan_edges", "degenerate_culled", "degenerate_unculled", "two_draws"):
        for b in SCENES[n].bodies:
            geometry[len(geometry)] = SCENES[n].geometry[b]
    draw = list(range(len(geometry)))
    poses.update({b: I34 for b in draw[1:]})
    renderers = [dict(geometry=draw, referenced=[0], size=s, z_min=z, z_max=10.0)
                 for s in (33, 240) for z in (1e-30, 1.0)]
    _render_and_compare(capi, synth, geometry, poses, renderers)


# ---- k_model_raster ---------------------------------------------------------------------------------------------------

def test_model_raster_on_adversarial_geometry(capi):
    """A mask mesh larger than the body's sphere (clipped by the near and far planes in the other views) with NaN,
    inf, zero-area and sliver triangles and a copy of part of itself (triangle-index ties), through every view."""
    S = 97
    body = rc.mask_mesh(rc.contour_masks(S)["full"], 3)
    extra = np.array([[(0, 0, 0), (0, 0, 0), (0.01, 0, 0)], [(0, 0, 0), (float("nan"), 0, 0), (0, 0.01, 0)],
                      [(0, 0, 0), (float("inf"), 0, 0), (0, 0.01, 0)], [(0, 0, 0), (0.05, 0, 0), (0.1, 1e-7, 0)]],
                     np.float32)
    tri = np.concatenate([body.triangles, extra, body.triangles[::5]])
    g = mg.rr.Geometry(tri, I34.copy(), body.maximum_body_diameter, False)
    ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
    ctx.set_body_geometry(0, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling)
    p = capi.model_params(n_divides=0, n_points=1, image_size=S)
    st = mg.Setup(g, [], 0.8, S)
    poses = mg.geodesic_poses(0, 0.8)
    stats = {}
    for v in range(len(poses)):
        img = ctx.debug_render_model_view(0, v, (), p)
        exp = mg.render_view(st, poses[v], stats)
        for k in ("normal", "depth", "silhouette"):
            assert np.array_equal(img[k], exp[k]), (v, k, np.argwhere(img[k] != exp[k])[:5])
    ctx.close()
    for k in ("fan4", "clip_in_out", "clip_out_in", "clip_out_out", "triangle_tie", "far_reject"):
        assert stats.get(k, 0) > 0, (k, stats)
