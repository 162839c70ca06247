"""Model generation on engineered silhouettes (raster_cases.mask_mesh): k_region_contours / k_region_points and
k_model_points bit for bit against their restatements on single pixels, contours of 14, 15 and 16 points (around the
drop threshold), 1-px lines that fold back, diagonal-only joins, holes, nested levels, blobs on the image border and the
full image; k_region_contours at 4096 and 8192 px on the device's own silhouettes; generation runs over more than one
view batch; and the contour-buffer overflow, which fails with M3TB_ERR_UNSUPPORTED and leaves the model as it was."""
import ctypes as C

import numpy as np
import pytest

import model_generation_reference as mg
import raster_cases as rc
import region_model_generation_reference as rg
import render_reference as rr

pytestmark = pytest.mark.gpu

I34 = rc.I34
VIEW = 3  # the geodesic view (n_divides 0) the masks are seen from
EMPTY = ((), (), (), ())


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _context(capi, bodies):
    ctx = capi.Context(0, max_bodies=len(bodies), max_cameras=1, max_models=2)
    for b, g in enumerate(bodies):
        ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling)
    return ctx


def _assert_region_model(got, exp):
    _, ori, lengths, pts = exp
    assert np.array_equal(_bits(got.orientations), _bits(ori))
    assert np.array_equal(_bits(got.view_scalars), _bits(lengths)), (got.view_scalars, lengths)
    bad = np.nonzero((_bits(got.points) != _bits(pts)).any(-1))
    assert np.array_equal(_bits(got.points), _bits(pts)), (bad[0][:5], bad[1][:5])


@pytest.mark.parametrize("S", [21, 33, 63, 97, 256])
def test_region_contours_on_engineered_masks(capi, S):
    masks = rc.contour_masks(S)
    for name, mask in masks.items():
        body = rc.mask_mesh(mask, VIEW)
        ctx = _context(capi, [body])
        p = capi.model_params(n_divides=0, n_points=24, image_size=S)
        ctx.generate_region_model(0, 0, (), p)
        _assert_region_model(ctx.get_region_model(0), rg.generate(body, EMPTY, n_divides=0, n_points=24, image_size=S))
        img = ctx.debug_region_model_view(0, VIEW, (), p)
        assert np.array_equal(img["silhouettes"][0] == rg.MAIN_BODY_ID, mask), name
        exp = rg.valid_contours(np.where(mask, rg.MAIN_BODY_ID, 0))
        assert [len(c) for c in img["contours"]] == [len(c) for c in exp], name
        for a, b in zip(img["contours"], exp):
            assert np.array_equal(a, b), name
        if name == "lengths_14_15_16":  # the 15-point contour is kept, the 14-point one dropped
            assert sorted(len(c) for c in exp) == [15, 16]
        ctx.close()


@pytest.mark.parametrize("S", [21, 63])
def test_depth_points_on_a_few_pixels(capi, S):
    """k_model_points' rejection sampling on silhouettes of 1, 2 and 3 pixels, and depth offsets with image_stride 1
    at n_values 30."""
    for n_pix in (1, 2, 3):
        mask = np.zeros((S, S), bool)
        mask[S // 2, S // 2:S // 2 + n_pix] = True
        body = rc.mask_mesh(mask, VIEW)
        ctx = _context(capi, [body])
        p = capi.model_params(n_divides=0, n_points=16, image_size=S, stride_depth_offset=0.0001,
                              max_radius_depth_offset=0.0029)
        st = mg.Setup(body, [], 0.8, S)
        assert int(np.float32(p.max_radius_depth_offset) / np.float32(p.stride_depth_offset) + np.float32(1)) == 30
        ptm = np.float32(0.8) / st.fu  # image_stride = int(stride / pixel_to_meter + 1) = 1
        assert int(np.float32(p.stride_depth_offset) / ptm + np.float32(1)) == 1
        ctx.generate_depth_model(0, 0, (), p)
        got = ctx.get_depth_model(0)
        _, ori, areas, pts = mg.generate(body, [], n_divides=0, n_points=16, image_size=S, stride_depth_offset=0.0001,
                                         max_radius_depth_offset=0.0029)
        assert np.array_equal(_bits(got.view_scalars), _bits(areas))
        assert np.array_equal(_bits(got.points), _bits(pts))
        assert np.count_nonzero(mg.render_view(st, mg.geodesic_poses(0, 0.8)[VIEW])["silhouette"]) == n_pix
        ctx.close()


@pytest.mark.parametrize("S", [4096, 8192])
def test_region_contours_at_large_sizes(capi, synth, S):
    """Without a CPU raster: the restatement's contours and points from the device's own silhouettes and depth."""
    tri, _ = synth.icosphere_triangles(radius=0.04, n_divides=3)
    body = rr.Geometry(tri, I34.copy(), 0.08, True)
    ctx = _context(capi, [body])
    p = capi.model_params(n_divides=0, n_points=12, image_size=S)
    ctx.generate_region_model(0, 0, (), p)
    got = ctx.get_region_model(0)
    st = rg.Setup(body, EMPTY, 0.8, S)
    poses = mg.geodesic_poses(0, 0.8)
    for v in (0, 7):
        img = ctx.debug_region_model_view(0, v, (), p)
        sils = {"main": img["silhouettes"][0]}
        pts, length, contours = rg.view_points(st, poses[v], sils, img["depth"], 12, 0.002, 0.05)
        assert sum(len(c) for c in contours) > 2 * S
        assert [len(c) for c in img["contours"]] == [len(c) for c in contours], v
        for a, b in zip(img["contours"], contours):
            assert np.array_equal(a, b), v
        assert _bits(got.view_scalars[v]) == _bits(length), v
        assert np.array_equal(_bits(got.points[v]), _bits(pts)), v
    ctx.close()


def test_depth_generation_over_two_batches(capi, synth):
    """2000 px, n_divides 1: 42 views in batches of 33; every view's points equal the restatement's sampler on the
    view's debug images."""
    tri, diam = synth.prism_triangles()
    body = rr.Geometry(tri, I34.copy(), diam, True)
    ctx = _context(capi, [body])
    p = capi.model_params(n_divides=1, n_points=10, image_size=2000)
    ctx.generate_depth_model(0, 0, (), p)
    got = ctx.get_depth_model(0)
    st = mg.Setup(body, [], 0.8, 2000)
    poses = mg.geodesic_poses(1, 0.8)
    assert len(poses) == 42
    for v in range(len(poses)):
        img = ctx.debug_render_model_view(0, v, (), p)
        pts, area = mg.view_points(st, poses[v], img, 10, 0.002, 0.05)
        assert _bits(got.view_scalars[v]) == _bits(area), v
        assert np.array_equal(_bits(got.points[v]), _bits(pts)), v
    ctx.close()


def test_region_generation_over_two_batches(capi, synth):
    """Five renderers (a movable and a same-region associated body) at 1000 px, n_divides 1: 42 views in batches of
    25; every view's points equal the restatement on the view's debug images."""
    tri, diam = synth.prism_triangles()
    body = rr.Geometry(tri, I34.copy(), diam, True)
    small, _ = synth.icosphere_triangles(radius=0.012, n_divides=1)
    mov = rr.Geometry(small + np.float32([-0.02, 0.0, 0.02]), I34.copy(), 0.1, True)
    same = rr.Geometry(small + np.float32([0.0, 0.03, 0.0]), I34.copy(), 0.1, True)
    ctx = _context(capi, [body, mov, same])
    triples = [(1, 1, 0), (2, 0, 1)]
    p = capi.model_params(n_divides=1, n_points=10, image_size=1000)
    ctx.generate_region_model(0, 0, triples, p)
    got = ctx.get_region_model(0)
    st = rg.Setup(body, ((), [same], [mov], ()), 0.8, 1000)
    assert list(st.renderers) == ["main", "same_region", "occlusion", "foreground", "background"]
    poses = mg.geodesic_poses(1, 0.8)
    for v in range(len(poses)):
        img = ctx.debug_region_model_view(0, v, triples, p)
        sils = dict(zip(st.renderers, img["silhouettes"]))
        pts, length, _ = rg.view_points(st, poses[v], sils, img["depth"], 10, 0.002, 0.05)
        assert _bits(got.view_scalars[v]) == _bits(length), v
        assert np.array_equal(_bits(got.points[v]), _bits(pts)), v
    assert (got.view_scalars > 0).all()
    ctx.close()


def test_contour_overflow_leaves_the_model(capi):
    """33 x 33 blocks of 5 x 5 px at 200 px have 17424 contour points, above the 64 x 200 the tracer keeps: both the
    generation and the debug view fail with M3TB_ERR_UNSUPPORTED, the model reads back as before, and the same context
    then generates the next model; 28 x 28 blocks (12544 points) fit and match the restatement."""
    S = 200
    good = rc.mask_mesh(rc.contour_masks(S)["nested_4"], VIEW)
    over = rc.mask_mesh(rc.block_grid(S, 33), VIEW)
    under = rc.mask_mesh(rc.block_grid(S, 28), VIEW)
    ctx = _context(capi, [good, over, under])
    p = capi.model_params(n_divides=0, n_points=16, image_size=S)
    ctx.generate_region_model(0, 0, (), p)
    before = ctx.get_region_model(0)
    assert (before.view_scalars > 0).any()
    a = capi.associated_bodies(())
    assert ctx.L.m3tb_generate_region_model(ctx.h, 0, 1, a.ctypes.data, 0, C.byref(p)) == -3
    with pytest.raises(capi.M3TBError, match="status -3"):
        ctx.debug_region_model_view(1, VIEW, (), p)
    after = ctx.get_region_model(0)
    assert np.array_equal(_bits(after.points), _bits(before.points))
    assert np.array_equal(_bits(after.view_scalars), _bits(before.view_scalars))
    assert np.array_equal(_bits(after.orientations), _bits(before.orientations))
    ctx.generate_region_model(0, 2, (), p)
    exp = rg.generate(under, EMPTY, n_divides=0, n_points=16, image_size=S)
    _assert_region_model(ctx.get_region_model(0), exp)
    img = ctx.debug_region_model_view(2, VIEW, (), p)
    assert sum(len(c) for c in img["contours"]) == 28 * 28 * 16 <= 64 * S
    ctx.close()
