"""The device's occlusion, region and silhouette checks (SURVEY row f4) across the parameters they accept. Every case
holds k_track<OCC> to three bars: the valid flags equal the restatement's (tests/occlusion_reference.py), the records are
bit-exact against the mirror oracle, and StartModalities / CalculateResults histograms are bit-exact; the pose after
every correspondence iteration stays within 1e-5 of the mirror oracle. Each case asserts the restatement stats it was
built to reach, so that a case which stops exercising its edge fails."""
import copy

import numpy as np
import pytest

import occlusion_reference as ref
from helpers import assert_lines_bit_equal, assert_points_bit_equal, pose_error
from test_occlusion_reference import checks_off, nan_and_behind_workload, rendered_workload
from test_oracle_occlusion import occluded_workload

pytestmark = pytest.mark.gpu


def _set(wl, **kw):
    """Sets each parameter on both modalities; a "depth_only_" prefix sets it on the depth modality alone."""
    for k, v in kw.items():
        mods = (wl.depth,) if k.startswith("depth_only_") else (wl.region, wl.depth)
        k = k.removeprefix("depth_only_")
        for m in mods:
            if m is not None and hasattr(m, k):
                setattr(m, k, v)
    return wl


def run_case(capi, oracle, wl, iterations=(0, 3), corrs=(0, 2), first_iteration=0):
    """Runs the three bars and returns the restatement's stats over every check it made."""
    stats = ref.new_stats()
    ctx = capi.context_from_workload(wl)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    base = oracle.OracleTracker(checks_off(wl), rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    for b in range(wl.n_bodies):
        orc.bodies[b].first_iteration = base.bodies[b].first_iteration = first_iteration
    orc.start_modalities(first_iteration)
    ctx.start_modalities(first_iteration)
    nb = wl.region.n_histogram_bins if wl.region else 0

    def histograms_equal(tag):
        for b in range(wl.n_bodies if wl.region else 0):
            hf, hb = ctx.get_histograms(b, nb)
            assert np.array_equal(hf.view(np.uint32), orc.hist_f[b].view(np.uint32)), (tag, b)
            assert np.array_equal(hb.view(np.uint32), orc.hist_b[b].view(np.uint32)), (tag, b)
    histograms_equal("start")
    for iteration in iterations:
        for corr in corrs:
            poses = orc.get_poses()
            ctx.set_poses(poses)
            if wl.region:
                ctx.region_correspondences(iteration, corr)
            if wl.depth:
                ctx.depth_correspondences(iteration, corr)
            for b in range(wl.n_bodies):
                if wl.region:
                    n, view = orc.region_correspondences(b, iteration, corr)
                    base.region_correspondences(b, iteration, corr)
                    lines = ctx.get_region_lines(b, wl.lines_per_body)
                    assert ctx.get_closest_views(b)[0] == view
                    assert_lines_bit_equal(lines, orc.lines[b][:n])
                    pred = ref.region_valid(wl, b, poses[b], view, n, base.lines[b]["valid"], iteration,
                                            first_iteration, corr, stats)
                    assert np.array_equal(pred, lines["valid"] != 0), (iteration, corr, b)
                if wl.depth:
                    m, view = orc.depth_correspondences(b, iteration, corr)
                    base.depth_correspondences(b, iteration, corr)
                    pts = ctx.get_depth_points(b, wl.points_per_body)
                    assert ctx.get_closest_views(b)[1] == view
                    assert_points_bit_equal(pts, orc.points[b][:m])
                    pred = ref.depth_valid(wl, b, poses[b], view, m, base.points[b]["valid"], iteration,
                                           first_iteration, stats)
                    assert np.array_equal(pred, pts["valid"] != 0), (iteration, corr, b)
    launch = ctx.last_launch()
    assert launch["kernel"] == "k_track" and launch["occ"] == 1, launch
    iteration = iterations[-1]
    for corr in range(wl.n_corr_iterations):
        ctx.set_poses(orc.get_poses())
        ctx.corr_iteration(iteration, corr, wl.n_update_iterations)
        orc.tracking_step(iteration, n_corr=corr + 1, corr_begin=corr)
        dt, dr = pose_error(ctx.get_poses(), orc.get_poses())
        assert dt.max() < 1e-5 and dr.max() < 1e-5, (corr, dt, dr)
    ctx.calculate_results(iteration)
    orc.calculate_results(iteration)
    histograms_equal("results")
    ctx.close()
    return stats


ID_1_5_STRIDES = int(np.float32(0.003) / np.float32(0.002) + np.float32(0.5))   # the +0.5 rounding edge
MEASURED = {
    "radius_0": (dict(measured_occlusion_radius=0.0), lambda s: s["windows"] > 0 and s["stride_above_1"] == 0),
    "radius_0.001": (dict(measured_occlusion_radius=0.001), lambda s: s["stride_above_1"] == 0 and s["occluded"] > 0),
    "radius_0.05": (dict(measured_occlusion_radius=0.05), lambda s: s["stride_above_1"] > 0),
    "radius_0.2": (dict(measured_occlusion_radius=0.2), lambda s: s["stride_above_1"] > 0),
    "threshold_-0.05": (dict(measured_occlusion_threshold=-0.05), lambda s: s["occluded"] > 0),
    "threshold_0": (dict(measured_occlusion_threshold=0.0), lambda s: s["occluded"] > 0),
    "threshold_above_z": (dict(measured_occlusion_threshold=10.0), lambda s: s["wrapped_bounds"] > 0),
    "offset_radius_0": (dict(measured_depth_offset_radius=0.0), lambda s: s["offset_ids"] == {0}),
    "offset_radius_1.5_strides": (dict(measured_depth_offset_radius=0.003),
                                  lambda s: s["offset_ids"] == {ID_1_5_STRIDES}),
    "offset_radius_max": (dict(measured_depth_offset_radius=0.05), lambda s: s["offset_ids"] == {25}),
    "depth_scaling": (dict(use_depth_scaling=True, considered_distances=(0.08, 0.04, 0.02),
                           depth_only_measured_depth_offset_radius=0.09), lambda s: s["top_ids"] > 0),
}


@pytest.mark.parametrize("case", list(MEASURED))
def test_measured(capi, oracle, case):
    kw, expect = MEASURED[case]
    wl = _set(occluded_workload(n_bodies=3), **kw)
    st = run_case(capi, oracle, wl)
    assert expect(st), st


@pytest.mark.parametrize("depth_scale", [0.001, 0.0001])
def test_measured_depth_scale_and_invalid_pixels(capi, oracle, depth_scale):
    wl = occluded_workload(n_bodies=3)
    if depth_scale != wl.depth_scale:
        k = wl.depth_scale / depth_scale
        wl.depth_frames = np.clip(wl.depth_frames.astype(np.float64) * k, 0, 65535).astype(np.uint16)
        wl.depth_scale = depth_scale
    wl.depth_frames[:, ::7, ::5] = 0            # invalid pixels inside the windows
    st = run_case(capi, oracle, wl)
    assert st["zero_pixels"] > 0 and st["occluded"] > 0, st


@pytest.mark.parametrize("n_unoccluded", [0, 1, 3])
@pytest.mark.parametrize("first_iteration", [0, 2])
def test_unoccluded_iterations_gate(capi, oracle, n_unoccluded, first_iteration):
    wl = _set(occluded_workload(n_bodies=2), n_unoccluded_iterations=n_unoccluded)
    st = run_case(capi, oracle, wl, iterations=tuple(range(first_iteration, first_iteration + 5)), corrs=(0,),
                  first_iteration=first_iteration)
    # iterations first_iteration .. +4: passes without occlusion handling exactly while fewer than n_unoccluded have run
    assert st["unhandled_passes"] == 2 * 2 * n_unoccluded and st["handled_passes"] == 2 * 2 * (5 - n_unoccluded), st


@pytest.mark.parametrize("above", [0, 1])
def test_fallback_at_the_survivor_count(capi, oracle, above):
    """min_n_unoccluded_lines / _points at exactly the survivor count (no second pass) and one above."""
    wl = occluded_workload(n_bodies=1)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    n, _ = orc.region_correspondences(0, 0, 0)
    m, _ = orc.depth_correspondences(0, 0, 0)
    wl = _set(wl, min_n_unoccluded_lines=int(orc.lines[0]["valid"][:n].sum()) + above,
              min_n_unoccluded_points=int(orc.points[0]["valid"][:m].sum()) + above)
    st = run_case(capi, oracle, wl, iterations=(0,), corrs=(0,))
    assert (st["fallbacks"] > 0) == bool(above), st


RENDERED = {
    "default": (dict(), lambda s: s["region_id_mismatch"] > 0 and s["occluded"] > 0 and s["offset_ids"] == {5}),
    "modeled_radius_threshold": (dict(modeled_occlusion_radius=0.05, modeled_occlusion_threshold=-0.05,
                                      modeled_depth_offset_radius=0.0),
                                 lambda s: s["clipped_left"] > 0 and s["clipped_bottom"] > 0 and s["offset_ids"] == {0}),
    "modeled_offset_max": (dict(modeled_depth_offset_radius=0.05), lambda s: s["offset_ids"] == {25}),
    "size_50": (dict(image_size=50), lambda s: s["occluded"] > 0 and s["walk_outside"] > 0),
    "size_400": (dict(image_size=400), lambda s: s["occluded"] > 0 and s["walk_outside"] > 0),
    "continuous_0": (dict(min_continuous_distance=0.0), lambda s: s["region_id_mismatch"] > 0 and s["walk_outside"] == 0),
    "continuous_8": (dict(min_continuous_distance=8.0), lambda s: s["walk_outside"] > 21),
    "continuous_30": (dict(min_continuous_distance=30.0), lambda s: s["walk_outside"] > 43),
    "large_window": (dict(modeled_occlusion_radius=0.2), lambda s: s["clipped_left"] > 0 and s["all_background"] > 0),
}


@pytest.mark.parametrize("case", list(RENDERED))
def test_renderer_checks(capi, oracle, synth, case):
    kw, expect = RENDERED[case]
    wl = rendered_workload(synth, n_bodies=3, **kw)
    st = run_case(capi, oracle, wl, iterations=(0,), corrs=(0, 3))
    assert expect(st), st


def test_mixed_batch(capi, oracle, synth):
    """Measured and modeled occlusions, region and silhouette checks in one launch, with a second occluder and a
    fallback on some bodies. Every body shares one parameter set (the synthetic workloads carry one per modality)."""
    wl = rendered_workload(synth, n_bodies=4)
    synth.add_occluder(wl, 2, side="top", seed=19)
    wl = _set(wl, measure_occlusions=True, measured_occlusion_radius=0.02, min_n_unoccluded_lines=60)
    st = run_case(capi, oracle, wl, iterations=(0,), corrs=(0, 2))
    assert st["windows"] > 0 and st["region_id_mismatch"] > 0


# ---- after the fixes -------------------------------------------------------------------------------------------------
def _nan_equal_records(gpu, ref_):
    assert np.array_equal(gpu["valid"], ref_["valid"])
    for f in ("center_u", "center_v"):
        a, b = np.asarray(gpu[f]), np.asarray(ref_[f])
        assert np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)]), f


@pytest.mark.parametrize("kind", ["nan_pose", "behind_depth_camera"])
def test_scans_that_would_not_end(capi, oracle, synth, kind):
    """A NaN-pose body (measured occlusions, region and depth) and region lines behind the depth camera reach windows
    whose stride the reference computes as 0. The launch returns, the NaN body keeps no item, and everything else
    matches the oracle."""
    wl = nan_and_behind_workload(synth, kind)
    ctx = capi.context_from_workload(wl)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    orc.start_modalities(0)
    ctx.start_modalities(0)
    ctx.set_poses(wl.start_body2world)
    ctx.region_correspondences(0, 0)
    if wl.depth:
        ctx.depth_correspondences(0, 0)
    ctx.synchronize()
    for b in range(wl.n_bodies):
        n, _ = orc.region_correspondences(b, 0, 0)
        lines = ctx.get_region_lines(b, wl.lines_per_body)
        if kind == "nan_pose" and b == 1:
            _nan_equal_records(lines, orc.lines[b][:n])
            assert not lines["valid"].any()
            m, _ = orc.depth_correspondences(b, 0, 0)
            assert not ctx.get_depth_points(b, wl.points_per_body)["valid"].any()
            continue
        assert_lines_bit_equal(lines, orc.lines[b][:n])
        assert lines["valid"].sum() > 0
        if wl.depth:
            m, _ = orc.depth_correspondences(b, 0, 0)
            assert_points_bit_equal(ctx.get_depth_points(b, wl.points_per_body), orc.points[b][:m])
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    ctx.calculate_results(0)
    ctx.synchronize()
    good = [b for b in range(wl.n_bodies) if not (kind == "nan_pose" and b == 1)]
    orc.tracking_step(0)
    dt, dr = pose_error(ctx.get_poses()[good], orc.get_poses()[good])
    assert dt.max() < 1e-5 and dr.max() < 1e-5, (dt, dr)
    ctx.close()


def test_region_offset_id_30_is_refused(capi, synth):
    """max_radius / stride in [29.5, 30): a radius at the maximum would select entry 30 of a 30-entry table."""
    wl = occluded_workload(n_bodies=1, region_only=True)
    wl.region_model.stride_depth_offset, wl.region_model.max_radius_depth_offset = 0.001, 0.0297
    for key, radius in (("measured_depth_offset_radius", 0.0297), ("modeled_depth_offset_radius", 0.0297)):
        w = copy.deepcopy(wl)
        setattr(w.region, key, radius)
        w.region.model_occlusions = key.startswith("modeled")
        ctx = capi.context_from_workload(w)
        before = ctx.launch_count
        with pytest.raises(capi.M3TBError, match=r"status -1: .*rounds past the model's 30 depth offsets"):
            ctx.region_correspondences(0, 0)
        with pytest.raises(capi.M3TBError, match=r"status -1: .*rounds past the model's 30 depth offsets"):
            ctx.start_modalities(0)
        assert ctx.launch_count == before
        ctx.close()
    w = copy.deepcopy(wl)
    w.region.measured_depth_offset_radius = 0.0294   # id 29
    ctx = capi.context_from_workload(w)
    ctx.region_correspondences(0, 0)
    ctx.close()


@pytest.mark.parametrize("stride,max_radius", [(0.0, 0.05), (-0.002, 0.05), (float("nan"), 0.05), (float("inf"), 0.05),
                                               (0.002, float("nan")), (0.002, -0.01), (0.002, float("inf")),
                                               (0.001, 0.04)])
def test_bad_model_parameters_are_refused(capi, stride, max_radius):
    wl = occluded_workload(n_bodies=2)
    ctx = capi.context_from_workload(wl)
    ctx.start_modalities(0)
    ctx.region_correspondences(0, 0)
    ctx.depth_correspondences(0, 0)
    before = [(ctx.get_region_lines(b, wl.lines_per_body), ctx.get_depth_points(b, wl.points_per_body))
              for b in range(wl.n_bodies)]
    for setter, m in ((ctx.set_region_model, wl.region_model), (ctx.set_depth_model, wl.depth_model)):
        bad = copy.copy(m)
        bad.stride_depth_offset, bad.max_radius_depth_offset = stride, max_radius
        with pytest.raises(capi.M3TBError, match=r"status -1: bad model depth-offset parameters"):
            setter(0, bad)
    ctx.region_correspondences(0, 0)
    ctx.depth_correspondences(0, 0)
    for b in range(wl.n_bodies):
        assert_lines_bit_equal(ctx.get_region_lines(b, wl.lines_per_body), before[b][0])
        assert_points_bit_equal(ctx.get_depth_points(b, wl.points_per_body), before[b][1])
    ctx.close()


def test_texture_points_behind_the_depth_camera(capi, synth):
    """A texture body with measured and modeled occlusions whose reconstructed points lie in front of the colour camera
    and behind the depth camera, which is turned half round: a measured radius of 0.001 m gives diameters in (-5, 0) px
    (the reference's stride 0), 0.01 m negative strides. k_texture_keyframe returns, the measured check removes no
    point on a frame whose every pixel lies in front of them, and the keyframe equals the restatement's."""
    import test_gpu_texture as rigid
    import texture_reference as tr
    ctx, _, _ = rigid._scene(capi, synth)
    tri, diam = synth.prism_triangles()
    ctx.set_body_geometry(1, tri, rigid.W2C, diam, True, body_id=2, region_id=2)
    ctx.set_poses(np.stack([rigid._pose(), rigid._pose(t=(0.045, 0.0, 0.42))]))
    ctx.set_focused_renderer(1, "color", 0, [0, 1], [0], 64, id_type="body")
    ctx.attach_renderer(0, "texture_depth", 1)
    d_w2c = np.array([[-1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, 0]], np.float32)
    ctx.set_depth_camera(0, synth.default_color_intrinsics(), d_w2c, 0.001)
    frame = np.full((480, 640), 100, np.uint16)   # 0.1 m everywhere
    ctx.upload_depth(0, frame)
    pose = ctx.get_poses()[0]
    b2c, b2d = rigid._b2c(pose), tr.pose_mul(d_w2c, pose)
    roi, scale, _ = ctx.get_texture_focus()
    crop, desc = rigid._features(np.random.default_rng(91), roi[0], scale[0], 300)
    fu = np.float32(rigid.INTR["fu"])
    for radius in (0.001, 0.01):
        p = capi.texture_params_default()
        p.measure_occlusions, p.measured_occlusion_radius, p.measured_occlusion_threshold = 1, radius, 0.03
        p.model_occlusions, p.modeled_occlusion_radius, p.modeled_occlusion_threshold = 1, 0.01, 0.03
        ctx.set_texture_modality(0, p, 0)
        xy = rigid._upload(ctx, 0, crop, desc, roi[0], scale[0])
        ctx.start_modalities(0)
        modeled = dict(rendering=ctx.get_rendering(1), intr=rigid.INTR, b2c=b2c, radius=0.01, threshold=0.03)
        measured = dict(image=frame, intr=rigid.INTR, depth_scale=0.001, b2d=b2d, radius=radius, threshold=0.03)
        rend = ctx.get_rendering(0)
        idx, pts = tr.reconstruct(xy, rend, rigid.INTR, tr.pose_inverse(b2c), 1, measured=measured, modeled=modeled)
        idx_modeled, _ = tr.reconstruct(xy, rend, rigid.INTR, tr.pose_inverse(b2c), 1, modeled=modeled)
        kf = ctx.get_texture_keyframes(0)
        assert list(kf["sizes"]) == [len(idx)], radius
        assert np.array_equal(kf["points"].view(np.uint32), pts.view(np.uint32)), radius
        assert np.array_equal(kf["descriptors"], desc[idx])
        assert len(idx) > 20 and np.array_equal(idx, idx_modeled)
        diameters = [np.float32(2) * np.float32(radius) * (fu / tr.apply(b2d, X)[2]) for X in pts]
        strides = [int(d / np.float32(5) + np.float32(1)) for d in diameters]
        assert all(s == 0 for s in strides) if radius == 0.001 else all(s < 0 for s in strides), (radius, strides[:5])
    ctx.close()
