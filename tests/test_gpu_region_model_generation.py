"""Region-model generation on the device (m3tb_generate_region_model, k_model_raster / k_region_contours /
k_region_points): views, contour lengths, points, the debug silhouettes and contour lists equal the CPU restatement
(tests/region_model_generation_reference.py) bit for bit; the reference's own OpenGL-generated model of schauma is
reproduced up to rasteriser differences; a generated model tracks exactly like the same arrays uploaded; refused calls
leave the model as it was."""
import ctypes as C
import importlib
import json
import os

import numpy as np
import pytest

import model_generation_reference as mg
import region_model_generation_reference as rg
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


def _box(synth, lo, hi):
    """Triangles of an axis-aligned box, counter-clockwise seen from outside."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    c = 0.5 * (lo + hi)
    v = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])]) - c
    f = [(0, 1, 3), (0, 3, 2), (4, 6, 7), (4, 7, 5), (0, 4, 5), (0, 5, 1), (2, 3, 7), (2, 7, 6), (0, 2, 6), (0, 6, 4),
         (1, 5, 7), (1, 7, 3)]
    return synth._outward(v, f) + c.astype(np.float32)


def _geometry(tri, culling, g2b=None):
    g2b = I34.copy() if g2b is None else g2b
    v = tri.reshape(-1, 3) + g2b[:, 3]
    return rr.Geometry(np.ascontiguousarray(tri, np.float32), g2b, float(np.float32(2.0 * np.linalg.norm(v, axis=1).max())),
                       culling)


def _mesh(synth, name, culling):
    if name == "prism":
        tri, diam = synth.prism_triangles()
        return rr.Geometry(tri, I34.copy(), diam, culling)
    if name == "icosphere":
        tri, diam = synth.icosphere_triangles(radius=0.04, n_divides=2)
        return rr.Geometry(tri, I34.copy(), diam, culling)
    if name == "frame":  # a square frame: its silhouette has a hole from the front and the back
        a, b, d = 0.04, 0.02, 0.01
        parts = [_box(synth, (-a, -a, -d), (a, -b, d)), _box(synth, (-a, b, -d), (a, a, d)),
                 _box(synth, (-a, -b, -d), (-b, b, d)), _box(synth, (b, -b, -d), (a, b, d))]
        return _geometry(np.concatenate(parts), culling)
    if name == "two":  # two components
        tri, _ = synth.icosphere_triangles(radius=0.015, n_divides=1)
        return _geometry(np.concatenate([tri + np.float32([0.025, 0, 0]), tri - np.float32([0.025, 0, 0])]), culling)
    raise ValueError(name)


def _associated(synth, kinds):
    """(geometries, triples) for associated bodies of the given kinds ("fixed", "fixed_sr", "movable", "movable_sr"),
    small spheres around the body placed so that they are in front of its contour in some views and behind in others."""
    tri, _ = synth.icosphere_triangles(radius=0.012, n_divides=1)
    offsets = {"fixed": (0.03, 0.0, 0.0), "fixed_sr": (0.0, 0.03, 0.0), "movable": (-0.02, 0.0, 0.02),
               "movable_sr": (0.0, -0.025, -0.01)}
    flags = {"fixed": (0, 0), "fixed_sr": (0, 1), "movable": (1, 0), "movable_sr": (1, 1)}
    geoms, triples = [], []
    for k, kind in enumerate(kinds):
        geoms.append(_geometry(tri, True, _g2b(offsets[kind])))
        triples.append((1 + k, *flags[kind]))
    return geoms, triples


def _groups(geoms, triples):
    out = ([], [], [], [])
    for g, (_, movable, same) in zip(geoms, triples):
        out[2 * movable + same].append(g)
    return out


def _set_geometry(ctx, b, g):
    ctx.set_body_geometry(b, g.triangles, g.geometry2body, g.maximum_body_diameter, g.enable_culling)


CASES = [  # mesh, culling, associated kinds, image_size, n_divides, n_points
    ("prism", True, (), 200, 0, 50),
    ("icosphere", True, (), 500, 0, 20),
    ("frame", True, (), 200, 1, 30),
    ("two", False, (), 64, 2, 10),
    ("prism", True, ("fixed",), 200, 0, 30),
    ("prism", True, ("fixed_sr",), 200, 0, 30),
    ("prism", True, ("movable",), 200, 0, 30),
    ("prism", True, ("movable_sr",), 200, 0, 30),
    ("icosphere", False, ("fixed", "movable", "fixed_sr", "movable_sr", "fixed"), 128, 1, 20),
]


@pytest.mark.parametrize("mesh,culling,kinds,size,n_divides,n_points", CASES)
def test_generation_bit_exact(capi, synth, mesh, culling, kinds, size, n_divides, n_points):
    body = _mesh(synth, mesh, culling)
    geoms, triples = _associated(synth, kinds)
    ctx = capi.Context(0, max_bodies=1 + len(geoms), max_cameras=1, max_models=1)
    for b, g in enumerate([body] + geoms):
        _set_geometry(ctx, b, g)
    p = capi.model_params(n_divides=n_divides, n_points=n_points, image_size=size)
    ctx.generate_region_model(0, 0, triples, p)
    got = ctx.get_region_model(0)
    groups = _groups(geoms, triples)
    stats = {}
    poses, ori, lengths, pts = rg.generate(body, groups, n_divides=n_divides, n_points=n_points, image_size=size,
                                           stats=stats)
    # every validity rule the case's associated bodies bring in rejects contour points, and a fixed body also lies
    # behind kept contour points, so each kernel branch decides some points of the comparison
    rules = {"fixed": ("fixed_depth", "fixed_kept"), "fixed_sr": ("same_region",), "movable": ("occlusion",),
             "movable_sr": ("same_region",)}
    for kind in kinds:
        for rule in rules[kind]:
            assert stats.get(rule, 0) > 0, (kind, rule, stats)
    assert np.array_equal(_bits(got.orientations), _bits(ori))
    assert np.array_equal(_bits(got.view_scalars), _bits(lengths)), np.nonzero(_bits(got.view_scalars) != _bits(lengths))
    bad = np.nonzero((_bits(got.points) != _bits(pts)).any(-1))
    assert np.array_equal(_bits(got.points), _bits(pts)), (bad[0][:5], bad[1][:5])
    assert (lengths > 0).any()
    st = rg.Setup(body, groups, 0.8, size)
    for v in sorted({0, poses.shape[0] // 2, poses.shape[0] - 1}):
        img = ctx.debug_region_model_view(0, v, triples, p)
        sils, depth = st.render(poses[v])
        assert img["silhouettes"].shape[0] == len(sils)
        for k, name in enumerate(sils):
            assert np.array_equal(img["silhouettes"][k], sils[name]), (v, name)
        assert np.array_equal(img["depth"], depth), v
        exp = rg.valid_contours(sils["main"])
        assert len(img["contours"]) == len(exp), v
        for a, b in zip(img["contours"], exp):
            assert np.array_equal(a, b), v
    ctx.close()


def test_hidden_body_gives_zero_contour_length(capi, synth):
    """A movable shell around the body hides every contour point: contour_length 0, zero-filled points."""
    body = _mesh(synth, "prism", True)
    tri, _ = synth.icosphere_triangles(radius=0.06, n_divides=2)
    shell = rr.Geometry(tri, I34.copy(), 0.12, True)
    ctx = capi.Context(0, max_bodies=2, max_cameras=1, max_models=1)
    _set_geometry(ctx, 0, body)
    _set_geometry(ctx, 1, shell)
    ctx.generate_region_model(0, 0, [(1, 1, 0)], capi.model_params(n_divides=0, n_points=8, image_size=100))
    m = ctx.get_region_model(0)
    assert (m.view_scalars == 0).all() and (m.points == 0).all()
    ctx.close()


def _schauma(mf):
    mesh = np.load(os.path.join(GOLDEN, "schauma_mesh.npz"))
    tri = mesh["vertices"][mesh["faces"]]
    return tri, mf.body.geometry2body[:3].astype(np.float32), np.float32(mf.body.maximum_body_diameter)


TOL_CENTER = 2e-5   # m: about six depth steps at 0.4 m
TOL_NORMAL = 1e-3
TOL_DISTANCE = 2e-4  # m: about one pixel at 0.4 m and 500 px
# Measured on an H100 (DESIGN.md §6): 96.7 % of the points match, contour lengths are within 9.9e-4 relative, the
# sampler started from seed 8 matches 0 %. The two rasterisers decide some silhouette-edge pixels differently.
MIN_MATCH = 0.9
MAX_LENGTH_REL = 5e-3


def _match(points, ref):
    dc = np.linalg.norm(points[..., 0:3] - ref[..., 0:3], axis=-1)
    dn = np.abs(points[..., 3:6] - ref[..., 3:6]).max(-1)
    dfg = np.abs(points[..., 6] - ref[..., 6])
    bg_same = (points[..., 7] == ref[..., 7]) | (np.abs(points[..., 7] - ref[..., 7]) <= TOL_DISTANCE)
    return (dc <= TOL_CENTER) & (dn <= TOL_NORMAL) & (dfg <= TOL_DISTANCE) & bg_same


def test_reference_known_answer(capi):
    """region_model.bin was made by the reference's OpenGL + OpenCV generator (schauma, 162 views x 10 points)."""
    model_io = importlib.import_module("3dobjecttracking_b200.model_io")
    mf = model_io.read_model(os.path.join(GOLDEN, "region_model.bin"))
    tri, g2b, diam = _schauma(mf)
    ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
    ctx.set_body_geometry(0, tri, g2b, float(diam), mf.body.geometry_enable_culling)
    p = capi.model_params(sphere_radius=mf.sphere_radius, n_divides=mf.n_divides, n_points=mf.n_points,
                          max_radius_depth_offset=mf.max_radius_depth_offset,
                          stride_depth_offset=mf.stride_depth_offset, image_size=mf.image_size)
    ctx.generate_region_model(0, 0, (), p)
    got = ctx.get_region_model(0)
    ref = mf.model
    assert got.n_views == ref.n_views and got.n_points == ref.n_points
    assert np.abs(got.orientations - ref.orientations).max() <= 1e-7
    length_rel = float(np.abs(got.view_scalars / ref.view_scalars - 1).max())
    match = _match(got.points, ref.points)
    # negative control: the restated sampler from seed 8 on the device's own images of every view
    body = rr.Geometry(tri, g2b, diam, mf.body.geometry_enable_culling)
    st = rg.Setup(body, ((), (), (), ()), mf.sphere_radius, mf.image_size)
    poses = mg.geodesic_poses(mf.n_divides, mf.sphere_radius)
    seed8 = []
    for v in range(got.n_views):
        img = ctx.debug_region_model_view(0, v, (), p)
        pts, _, _ = rg.view_points(st, poses[v], {"main": img["silhouettes"][0]}, img["depth"], mf.n_points,
                                   mf.stride_depth_offset, mf.max_radius_depth_offset, seed=8)
        seed8.append(pts)
    neg = _match(np.array(seed8), ref.points)
    rec = dict(file="region_model.bin", match=float(match.mean()), seed8_match=float(neg.mean()),
               length_rel_max=length_rel, length_rel_median=float(np.median(np.abs(got.view_scalars / ref.view_scalars - 1))),
               center_match=float((np.linalg.norm(got.points[..., :3] - ref.points[..., :3], axis=-1) <= TOL_CENTER).mean()),
               bg_flt_max_agree=float(((got.points[..., 7] == np.finfo(np.float32).max) ==
                                       (ref.points[..., 7] == np.finfo(np.float32).max)).mean()))
    print("[region-model-ka]", rec)
    out = os.environ.get("M3TB_MODEL_KA_RECORD")
    if out:
        with open(out, "a") as f:
            f.write(json.dumps(rec) + "\n")
    ctx.close()
    assert length_rel <= MAX_LENGTH_REL, rec
    assert match.mean() >= MIN_MATCH, rec
    assert neg.mean() < MIN_MATCH, rec


GEN = dict(n_divides=2, n_points=100, image_size=500)


def _generated(synth, capi):
    ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
    tri, diam = synth.prism_triangles()
    ctx.set_body_geometry(0, tri, I34, diam, True)
    ctx.generate_region_model(0, 0, (), capi.model_params(**GEN))
    m = ctx.get_region_model(0)
    ctx.close()
    return m


def _workloads(synth, capi):
    import copy
    analytic = synth.make_workload("c2", n_bodies=2, n_lines=100, n_divides=2)
    uploaded = copy.copy(analytic)
    uploaded.region_model = _generated(synth, capi)
    return analytic, uploaded


def _generated_context(synth, capi, analytic):
    ctx = capi.context_from_workload(analytic)
    tri, diam = synth.prism_triangles()
    ctx.set_body_geometry(0, tri, I34, diam, True)
    ctx.generate_region_model(0, 0, (), capi.model_params(**GEN))
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
    assert not np.array_equal(_bits(p_analytic), _bits(p_generated))


def test_generated_model_oracle_parity(capi, synth, oracle):
    analytic, uploaded = _workloads(synth, capi)
    per_iteration_parity(capi, oracle, uploaded, "generated_region_model", ctx=_generated_context(synth, capi, analytic))


def test_save_matches_model_io(capi, synth, tmp_path):
    """model_io.write_model(model_from_generated(...)) of a generated model reads back as generated, with associated
    body blocks in their groups."""
    model_io = importlib.import_module("3dobjecttracking_b200.model_io")
    body = _mesh(synth, "prism", True)
    geoms, triples = _associated(synth, ("movable", "fixed"))
    ctx = capi.Context(0, max_bodies=3, max_cameras=1, max_models=1)
    for b, g in enumerate([body] + geoms):
        _set_geometry(ctx, b, g)
    p = capi.model_params(n_divides=0, n_points=5, image_size=100)
    ctx.generate_region_model(0, 0, triples, p)
    m = ctx.get_region_model(0)
    ctx.close()

    def block(g, name):
        g2b = np.eye(4, dtype=np.float32)
        g2b[:3] = g.geometry2body
        return model_io.BodyBlock(name, 1.0, True, bool(g.enable_culling), g.maximum_body_diameter, g2b)
    groups = [[], [], [block(geoms[0], b"m.obj")], []]
    groups[0].append(block(geoms[1], b"f.obj"))
    path = str(tmp_path / "r.bin")
    model_io.write_model(path, model_io.model_from_generated(m, p, block(body, b"b.obj"), groups))
    back = model_io.read_model(path)
    assert back.kind == "region" and [len(g) for g in back.associated] == [1, 0, 1, 0]
    assert np.array_equal(_bits(back.model.points), _bits(m.points))
    assert np.array_equal(_bits(back.model.view_scalars), _bits(m.view_scalars))


def test_refusals_leave_the_model(capi, synth):
    tri, diam = synth.prism_triangles()
    ctx = capi.Context(0, max_bodies=4, max_cameras=1, max_models=1)
    ctx.set_body_geometry(0, tri, I34, diam, True)
    ctx.set_body_geometry(3, tri, I34, diam, True)
    big, _ = synth.icosphere_triangles(radius=0.5, n_divides=0)
    ctx.set_body_geometry(2, big, I34, 1.4, True)  # z_min = 0.8 - 0.7 < 0.2 * 0.8
    good = capi.model_params(n_divides=0, n_points=4, image_size=64)
    ctx.generate_region_model(0, 0, (), good)
    before = ctx.get_region_model(0)
    L = ctx.L

    def status(model_id=0, body=0, assoc=(), **kw):
        fields = {k: getattr(good, k) for k, _ in capi.ModelParams._fields_}
        fields.update(kw)
        p = capi.ModelParams(**fields)
        a = capi.associated_bodies(assoc)
        return L.m3tb_generate_region_model(ctx.h, model_id, body, a.ctypes.data, len(a), C.byref(p))
    assert status(use_random_seed=1) == -3      # M3TB_ERR_UNSUPPORTED
    assert status(max_radius_depth_offset=0.1, stride_depth_offset=0.002) == -1   # 51 offsets > 30
    assert status(sphere_radius=0.04) == -1      # z_min < 0.2 * sphere_radius
    for kind in ((0, 0), (0, 1), (1, 0), (1, 1)):
        assert status(assoc=[(2, *kind)]) == -1  # an associated body's z_min, in every renderer kind
    assert status(body=1) == -1                   # no geometry
    assert status(assoc=[(1, 0, 0)]) == -1
    assert status(model_id=1) == -1               # ids out of range
    assert status(body=5) == -1
    assert status(assoc=[(0, 1, 0)]) == -1        # the body itself
    assert status(assoc=[(3, 0, 0), (3, 1, 1)]) == -1   # listed twice
    after = ctx.get_region_model(0)
    assert np.array_equal(_bits(after.points), _bits(before.points))
    assert np.array_equal(_bits(after.view_scalars), _bits(before.view_scalars))
    ctx.close()


def test_exhausted_tries_on_the_device(capi, synth):
    """A needle seen side-on renders as a 1-px line whose contour folds back at its tips. A movable box hides all of it
    but the tips, where the chord of every +-3 segment is at most 2 px: every draw is rejected, and after 101
    rejections the device gives contour_length 0 and zero points, like the restatement."""
    w = 0.0001
    needle = _geometry(_box(synth, (-0.03, -w, -w), (0.03, w, w)), True)
    cover = _geometry(_box(synth, (-0.0296, -0.004, -0.004), (0.0296, 0.004, 0.004)), True)
    ctx = capi.Context(0, max_bodies=2, max_cameras=1, max_models=1)
    _set_geometry(ctx, 0, needle)
    _set_geometry(ctx, 1, cover)
    p = capi.model_params(n_divides=0, n_points=4, image_size=200)
    ctx.generate_region_model(0, 0, [(1, 1, 0)], p)
    got = ctx.get_region_model(0)
    stats = {}
    _, _, lengths, pts = rg.generate(needle, ((), (), [cover], ()), n_divides=0, n_points=4, image_size=200, stats=stats)
    ctx.close()
    assert stats.get("exhausted", 0) > 0, stats
    assert np.array_equal(_bits(got.view_scalars), _bits(lengths))
    assert np.array_equal(_bits(got.points), _bits(pts))


def test_tracker_known_answer_from_the_mesh(capi, synth, oracle):
    """TrackerTest.OptimizePoseMatrix with both models generated on the device from the triangle's mesh at the
    reference test's defaults (sphere radius 0.8, 4 divides, 200 points, 2000 px): start, tracking_step(0, 7, 2),
    results. The pose must be within the reference's bound of triangle_pose.txt; dt / dR against the replay on the
    resampled views (triangle_tracker_views.npz) are reported."""
    import sys
    sys.path.insert(0, GOLDEN)
    import reference_rig as rr_rig
    import test_reference_goldens as T
    from replay import ReferenceReplay
    ka = rr_rig.KA
    v = np.array(ka["triangle_obj"]["vertices"], np.float32)
    f = np.array(ka["triangle_obj"]["faces"], np.int64) - 1
    g2b = _g2b(np.array(ka["triangle_obj"]["geometry2body_translation"], np.float32))
    body = _geometry(v[f], True, g2b)
    rig = rr_rig.rig()
    ctx = capi.Context(0, 1, 1, 1)
    _set_geometry(ctx, 0, body)
    p = capi.model_params(sphere_radius=0.8, n_divides=4, n_points=200, image_size=2000)
    ctx.generate_region_model(0, 0, (), p)
    ctx.generate_depth_model(0, 0, (), p)
    cc, dc = ka["color_camera"], ka["depth_camera"]
    ctx.set_color_camera(0, synth.Intrinsics(cc["fu"], cc["fv"], cc["ppu"], cc["ppv"], cc["width"], cc["height"]),
                         rig["color_w2c"][:3])
    ctx.set_depth_camera(0, synth.Intrinsics(dc["fu"], dc["fv"], dc["ppu"], dc["ppv"], dc["width"], dc["height"]),
                         rig["depth_w2c"][:3], dc["depth_scale"])
    ctx.upload_color(0, rig["color"].reshape(540, -1))
    ctx.upload_depth(0, rig["depth"])
    rp, dp = capi.region_params(), capi.depth_params()
    rp.measure_occlusions = 1
    dp.measure_occlusions = 1
    ctx.set_body(0, rp, dp, capi.OptimizerParams(1000.0, 30000.0), 0, 0, 0, 0)
    ctx.set_poses(rig["body2world"][:3].astype(np.float32))
    ctx.start_modalities(0)
    ctx.tracking_step(0, 7, 2)
    ctx.calculate_results(0)
    pose = np.eye(4)
    pose[:3] = ctx.get_poses()[0]
    ctx.close()
    z = np.load(os.path.join(GOLDEN, "triangle_tracker_views.npz"))
    views = {k: {int(i): (z[f"{k}_points"][n], float(z[f"{k}_scalars"][n])) for n, i in enumerate(z[f"{k}_ids"])}
             for k in ("region", "depth")}
    rep = ReferenceReplay(oracle, views)
    assert rep.run("tracker", mirror=False) == []
    replay = rep.pose().astype(np.float64)
    golden = T._mat(ka, "tracker_triangle_pose")
    rec = dict(dt_vs_replay=float(np.linalg.norm(pose[:3, 3] - replay[:3, 3])),
               dR_vs_replay=float(np.abs(pose[:3, :3] - replay[:3, :3]).max()),
               dt_vs_golden=float(np.linalg.norm(pose[:3, 3] - golden[:3, 3])),
               dR_vs_golden=float(np.abs(pose[:3, :3] - golden[:3, :3]).max()))
    print("[tracker-from-mesh]", rec)
    out = os.environ.get("M3TB_MODEL_KA_RECORD")
    if out:
        with open(out, "a") as fo:
            fo.write(json.dumps(rec) + "\n")
    assert rec["dt_vs_golden"] < 1.0e-3, rec
