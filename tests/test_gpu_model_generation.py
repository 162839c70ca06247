"""Depth-model generation on the device (m3tb_generate_depth_model, k_model_raster / k_model_points): views, points,
surface areas and the debug images equal the CPU restatement (tests/model_generation_reference.py) bit for bit; the
reference's own OpenGL-generated models of schauma are reproduced up to rasteriser differences; a generated model
tracks exactly like the same arrays uploaded; refused calls leave the model as it was."""
import copy
import importlib
import json
import os

import numpy as np
import pytest

import model_generation_reference as mg
import render_reference as rr
from helpers import per_iteration_parity

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
I34 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def _g2b(t):
    g = I34.copy()
    g[:, 3] = t
    return g


def _bodies(synth, mesh, culling):
    if mesh == "prism":
        tri, diam = synth.prism_triangles()
    else:
        tri, diam = synth.icosphere_triangles(radius=0.04, n_divides=2)
    return rr.Geometry(tri, I34.copy(), diam, culling)


def _occluder(synth, kind):
    if kind is None:
        return []
    if kind == "tie":  # the body itself again: every depth ties, the body drawn first must win
        return None
    tri, _ = synth.icosphere_triangles(radius=0.02, n_divides=1)
    g2b = _g2b((0.015, 0.01, 0.0))
    v = tri.reshape(-1, 3) + g2b[:, 3]
    return [rr.Geometry(tri, g2b, 2.0 * float(np.linalg.norm(v, axis=1).max()), True)]


def _set_geometry(ctx, b, g):
    ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling)


CASES = [  # mesh, culling, occluder, image_size, n_divides, n_points
    ("prism", True, None, 200, 1, 100),
    ("prism", False, "icosphere", 64, 0, 1),
    ("prism", True, "tie", 200, 0, 37),
    ("icosphere", True, None, 500, 0, 200),
    ("icosphere", False, "icosphere", 200, 0, 20),
    ("prism", True, "icosphere", 64, 2, 5),
]


@pytest.mark.parametrize("mesh,culling,occ,size,n_divides,n_points", CASES)
def test_generation_bit_exact(capi, synth, mesh, culling, occ, size, n_divides, n_points):
    body = _bodies(synth, mesh, culling)
    occl = _occluder(synth, occ)
    if occl is None:
        occl = [rr.Geometry(body.triangles, body.geometry2body, body.maximum_body_diameter, culling)]
    ctx = capi.Context(0, max_bodies=1 + len(occl), max_cameras=1, max_models=1)
    for b, g in enumerate([body] + occl):
        _set_geometry(ctx, b, g)
    occ_ids = list(range(1, 1 + len(occl)))
    p = capi.model_params(n_divides=n_divides, n_points=n_points, image_size=size)
    ctx.generate_depth_model(0, 0, occ_ids, p)
    got = ctx.get_depth_model(0)
    poses, ori, areas, pts = mg.generate(body, occl, n_divides=n_divides, n_points=n_points, image_size=size)
    assert np.array_equal(_bits(got.orientations), _bits(ori))
    assert np.array_equal(_bits(got.view_scalars), _bits(areas)), np.nonzero(_bits(got.view_scalars) != _bits(areas))
    bad = np.nonzero((_bits(got.points) != _bits(pts)).any(-1))
    assert np.array_equal(_bits(got.points), _bits(pts)), (bad[0][:5], bad[1][:5])
    assert (areas > 0).all()
    st = mg.Setup(body, occl, 0.8, size)
    for v in sorted({0, poses.shape[0] // 2, poses.shape[0] - 1}):
        img = ctx.debug_render_model_view(0, v, occ_ids, p)
        exp = mg.render_view(st, poses[v])
        for k in ("normal", "depth", "silhouette"):
            assert np.array_equal(img[k], exp[k]), (v, k, np.argwhere(img[k] != exp[k])[:5])
        if occ == "tie":  # the occluder's copy never wins a tie
            assert np.array_equal(img["silhouette"] != 0, img["depth"] != 0xFFFF)
    ctx.close()


def test_empty_silhouette_gives_zero_points(capi, synth):
    """An occluder that hides the body from every view (a sphere around it): surface area 0, zero-filled points."""
    body = _bodies(synth, "prism", True)
    tri, _ = synth.icosphere_triangles(radius=0.06, n_divides=2)
    shell = rr.Geometry(tri, I34.copy(), 0.12, True)
    ctx = capi.Context(0, max_bodies=2, max_cameras=1, max_models=1)
    _set_geometry(ctx, 0, body)
    _set_geometry(ctx, 1, shell)
    ctx.generate_depth_model(0, 0, [1], capi.model_params(n_divides=0, n_points=8, image_size=100))
    m = ctx.get_depth_model(0)
    assert (m.view_scalars == 0).all() and (m.points == 0).all()
    ctx.close()


def _schauma(mf):
    mesh = np.load(os.path.join(GOLDEN, "schauma_mesh.npz"))
    tri = mesh["vertices"][mesh["faces"]]
    return tri, mf.body.geometry2body[:3].astype(np.float32), np.float32(mf.body.maximum_body_diameter)


def _match(points, ref, tol_center, tol_normal):
    dc = np.linalg.norm(points[..., 0:3] - ref[..., 0:3], axis=-1)
    dn = np.abs(points[..., 3:6] - ref[..., 3:6]).max(-1)
    return (dc <= tol_center) & (dn <= tol_normal)


# Known answer of the reference's OpenGL generator. The two rasterisers decide some silhouette-edge pixels differently,
# which shifts the remaining draws of that view, so only a fraction of the points must match. Measured on an H100
# (DESIGN.md §6): 99.5 % (depth_model.bin) and 99.2 % (depth_model_occlusion.bin) of the points match, the matched
# centres are mostly bit-identical, the worst matched normal component is one 8-bit step off, surface areas are within
# 1.0e-4 relative; the sampler started from seed 8 matches 0 %.
TOL_CENTER = 2e-5          # m: about six depth steps at 0.4 m
TOL_NORMAL = 1.01 / 127.5  # one step of the 8-bit normal
MIN_MATCH = {"depth_model.bin": 0.95, "depth_model_occlusion.bin": 0.95}
MAX_AREA_REL = 1e-3


@pytest.mark.parametrize("fname", ["depth_model.bin", "depth_model_occlusion.bin"])
def test_reference_known_answer(capi, fname):
    model_io = importlib.import_module("3dobjecttracking_b200.model_io")
    mf = model_io.read_model(os.path.join(GOLDEN, fname))
    tri, g2b, diam = _schauma(mf)
    ctx = capi.Context(0, max_bodies=2, max_cameras=1, max_models=1)
    ctx.set_body_geometry(0, tri, g2b, float(diam), mf.body.geometry_enable_culling)
    occ = []
    for k, ob in enumerate(mf.associated[0]):
        KA = json.load(open(os.path.join(GOLDEN, "reference_known_answers.json")))["triangle_obj"]
        v = np.array(KA["vertices"], np.float32)
        f = np.array(KA["faces"], np.int64) - 1
        ctx.set_body_geometry(1 + k, v[f], ob.geometry2body[:3].astype(np.float32), float(ob.maximum_body_diameter),
                              ob.geometry_enable_culling)
        occ.append(1 + k)
    p = capi.model_params(sphere_radius=mf.sphere_radius, n_divides=mf.n_divides, n_points=mf.n_points,
                          max_radius_depth_offset=mf.max_radius_depth_offset,
                          stride_depth_offset=mf.stride_depth_offset, image_size=mf.image_size)
    ctx.generate_depth_model(0, 0, occ, p)
    got = ctx.get_depth_model(0)
    ref = mf.model
    assert got.n_views == ref.n_views and got.n_points == ref.n_points
    assert np.abs(got.orientations - ref.orientations).max() <= 1e-7
    area_rel = float(np.abs(got.view_scalars / ref.view_scalars - 1).max())
    match = _match(got.points, ref.points, TOL_CENTER, TOL_NORMAL)
    # negative control: the same sampler started from seed 8 on the device's own images
    body = rr.Geometry(tri, g2b, diam, mf.body.geometry_enable_culling)
    st = mg.Setup(body, [rr.Geometry(np.zeros((1, 3, 3), np.float32), I34, d, True)
                         for d in [ob.maximum_body_diameter for ob in mf.associated[0]]], mf.sphere_radius, mf.image_size)
    poses = mg.geodesic_poses(mf.n_divides, mf.sphere_radius)
    seed7, seed8 = [], []
    for v in range(got.n_views):
        img = ctx.debug_render_model_view(0, v, occ, p)
        for seed, out in ((7, seed7), (8, seed8)):
            pts, _ = mg.view_points(st, poses[v], img, mf.n_points, mf.stride_depth_offset, mf.max_radius_depth_offset,
                                    seed=seed)
            out.append(pts)
    seed7, seed8 = np.array(seed7), np.array(seed8)
    assert np.array_equal(_bits(seed7), _bits(got.points))  # the restated sampler on the device images
    neg = _match(seed8, ref.points, TOL_CENTER, TOL_NORMAL)
    rec = dict(file=fname, match=float(match.mean()), seed8_match=float(neg.mean()), area_rel_max=area_rel,
               center_err_median=float(np.median(np.linalg.norm(got.points[..., :3] - ref.points[..., :3], axis=-1))),
               normal_err_matched_max=float(np.abs(got.points[..., 3:6] - ref.points[..., 3:6]).max(-1)[match].max()))
    print("[model-ka]", rec)
    out = os.environ.get("M3TB_MODEL_KA_RECORD")
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(rec) + "\n")
    ctx.close()
    assert area_rel <= MAX_AREA_REL, rec
    assert match.mean() >= MIN_MATCH[fname], rec
    assert neg.mean() < MIN_MATCH[fname], rec


GEN = dict(n_divides=2, n_points=100, image_size=500)


def _generate_in(ctx, synth, capi):
    """Generates depth model 0 of ctx on the device from the prism mesh (geometry on body slot 0)."""
    tri, diam = synth.prism_triangles()
    ctx.set_body_geometry(0, tri, I34, diam, True)
    ctx.generate_depth_model(0, 0, (), capi.model_params(**GEN))


def _workloads(synth, capi):
    """(analytic, uploaded): the same depth-only workload, once with synth's analytic depth model and once with the
    model the device generates from the prism mesh (read back, to be uploaded)."""
    analytic = synth.make_workload("c2", n_bodies=2, n_lines=0, n_points=100, n_divides=2)
    ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
    _generate_in(ctx, synth, capi)
    generated = ctx.get_depth_model(0)
    ctx.close()
    uploaded = copy.copy(analytic)
    uploaded.depth_model = generated
    assert generated.points.shape != analytic.depth_model.points.shape or \
        not np.array_equal(generated.points, analytic.depth_model.points)
    return analytic, uploaded


def _generated_context(synth, capi, analytic):
    """A context built with the analytic model whose depth model is then replaced by m3tb_generate_depth_model alone."""
    ctx = capi.context_from_workload(analytic)
    _generate_in(ctx, synth, capi)
    return ctx


def _step(ctx, wl):
    ctx.set_poses(wl.start_body2world)
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    poses = ctx.get_poses()
    ctx.close()
    return poses


def test_generated_model_tracks_like_uploaded(capi, synth):
    analytic, uploaded = _workloads(synth, capi)
    p_uploaded = _step(capi.context_from_workload(uploaded), uploaded)
    p_generated = _step(_generated_context(synth, capi, analytic), uploaded)
    p_analytic = _step(capi.context_from_workload(analytic), analytic)
    assert np.array_equal(_bits(p_uploaded), _bits(p_generated))
    assert not np.array_equal(_bits(p_analytic), _bits(p_generated))  # the model in use matters to the poses


def test_generated_model_oracle_parity(capi, synth, oracle):
    analytic, uploaded = _workloads(synth, capi)
    per_iteration_parity(capi, oracle, uploaded, "generated_depth_model", ctx=_generated_context(synth, capi, analytic))


def test_refusals_leave_the_model(capi, synth):
    tri, diam = synth.prism_triangles()
    ctx = capi.Context(0, max_bodies=3, max_cameras=1, max_models=1)
    ctx.set_body_geometry(0, tri, I34, diam, True)
    big, _ = synth.icosphere_triangles(radius=0.5, n_divides=0)
    ctx.set_body_geometry(2, big, I34, 1.4, True)  # z_min = 0.8 - 0.7 < 0.2 * 0.8
    good = capi.model_params(n_divides=0, n_points=4, image_size=64)
    ctx.generate_depth_model(0, 0, (), good)
    before = ctx.get_depth_model(0)
    L = ctx.L

    def status(model_id=0, body=0, occ=(), **kw):
        fields = {k: getattr(good, k) for k, _ in capi.ModelParams._fields_}
        fields.update(kw)
        p = capi.ModelParams(**fields)
        o = np.ascontiguousarray(occ, np.int32)
        import ctypes as C
        return L.m3tb_generate_depth_model(ctx.h, model_id, body, o.ctypes.data_as(C.POINTER(C.c_int)), o.size,
                                           C.byref(p))
    assert status(use_random_seed=1) == -3      # M3TB_ERR_UNSUPPORTED
    assert status(max_radius_depth_offset=0.1, stride_depth_offset=0.002) == -1   # 51 offsets > 30
    assert status(sphere_radius=0.04) == -1      # z_min < 0.2 * sphere_radius
    assert status(occ=(2,)) == -1                 # an occlusion body's z_min
    assert status(body=1) == -1                   # no geometry
    assert status(occ=(1,)) == -1
    assert status(model_id=1) == -1               # ids out of range
    assert status(body=5) == -1
    assert status(occ=(0,)) == -1                 # the body itself
    after = ctx.get_depth_model(0)
    assert np.array_equal(_bits(after.points), _bits(before.points))
    assert np.array_equal(_bits(after.view_scalars), _bits(before.view_scalars))
    ctx.close()
