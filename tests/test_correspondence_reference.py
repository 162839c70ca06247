"""The region line's segment probabilities and the depth point's correspondence search restated from the reference
(tests/correspondence_reference.py): the restatement against the oracle line by line and point by point at the
parameter settings the device is held to, closed forms on hand-made frames, and the proof obligation of the depth
search's reciprocal screen."""
import dataclasses

import numpy as np
import pytest

import correspondence_reference as ref
from test_gpu_parameter_space import SETTINGS

f32 = np.float32
LINE_FIELDS = ("center_f_body", "center_u", "center_v", "normal_u", "normal_v")
LINE_FIELDS_VALID = ("delta_r", "normal_component_to_scale", "distribution", "mean", "measured_variance")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def assert_lines_equal(got, want, tag):
    assert np.array_equal(got["valid"], want["valid"]), (tag, np.nonzero(got["valid"] != want["valid"]))
    for f in LINE_FIELDS:
        assert np.array_equal(_bits(got[f]), _bits(want[f])), (tag, f)
    v = want["valid"] != 0
    for f in LINE_FIELDS_VALID:
        assert np.array_equal(_bits(got[f][v]), _bits(want[f][v])), (tag, f)


def assert_points_equal(got, want, tag):
    assert np.array_equal(got["valid"], want["valid"]), (tag, np.nonzero(got["valid"] != want["valid"]))
    for f in ("center_f_body", "normal_f_body"):
        assert np.array_equal(_bits(got[f]), _bits(want[f])), (tag, f)
    v = want["valid"] != 0
    f = "correspondence_center_f_camera"
    assert np.array_equal(_bits(got[f][v]), _bits(want[f][v])), (tag, f)


def rel_to_max(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def compare_with_oracle(oracle, wl, corrs=None, opts=(0,), stats=None, histograms=None):
    """Records of every body at each correspondence iteration in `corrs` equal the oracle's (mirror mode, after
    StartModalities, or with `histograms` (hf, hb) for every body), and g / H within 1e-6 of max|H|. Returns the
    stats."""
    st = ref.new_stats() if stats is None else stats
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    orc.start_modalities(0)
    for b in range(wl.n_bodies if histograms is not None else 0):
        orc.hist_f[b], orc.hist_b[b] = histograms
    poses = orc.get_poses()
    corrs = range(wl.n_corr_iterations) if corrs is None else corrs
    for corr in corrs:
        for b in range(wl.n_bodies):
            tag = (corr, b)
            if wl.region:
                n, view = orc.region_correspondences(b, 0, corr)
                lines = ref.region_lines(wl, b, poses[b], view, n, orc.hist_f[b], orc.hist_b[b], corr, st,
                                         oracle.REGION_LINE_DTYPE)
                assert_lines_equal(lines, orc.lines[b][:n], tag)
                for opt in opts:
                    og, oH = orc.region_gradient_hessian(b, corr, opt)
                    g, H = ref.region_gradient_hessian(wl, b, poses[b], lines, corr, opt, st)
                    if not np.isfinite(oH).all():
                        assert np.array_equal(np.isnan(H), np.isnan(oH)), tag
                    elif np.abs(oH).max() > 0:
                        assert rel_to_max(H, oH) < 1e-6 and rel_to_max(g, og) < 1e-6 * max(1.0, np.abs(oH).max() /
                                                                                           max(np.abs(og).max(), 1e-30)), tag
            if wl.depth:
                m, view = orc.depth_correspondences(b, 0, corr)
                pts = ref.depth_points(wl, b, poses[b], view, m, corr, st, oracle.DEPTH_POINT_DTYPE)
                assert_points_equal(pts, orc.points[b][:m], tag)
                og, oH = orc.depth_gradient_hessian(b, corr)
                g, H = ref.depth_gradient_hessian(wl, b, poses[b], pts, corr)
                if np.abs(oH).max() > 0:
                    assert rel_to_max(H, oH) < 1e-6, tag
                    assert np.abs(g.astype(np.float64) - og).max() <= 1e-6 * max(np.abs(og).max(), np.abs(oH).max()), tag
    assert st["screen_misses"] == 0, st
    return st


@pytest.fixture(scope="module")
def base(synth):
    return synth.make_workload("c2", n_bodies=2, n_divides=2, seed=3)


def _variant(base, region=None, depth=None):
    return dataclasses.replace(base, region=dataclasses.replace(base.region, **(region or {})),
                               depth=dataclasses.replace(base.depth, **(depth or {})))


# ---- against the oracle ----------------------------------------------------------------------------------------------
EXTRA = {
    "default": ({}, {}),
    "depth_scaling": ({}, dict(use_depth_scaling=True, considered_distances=(0.08, 0.04, 0.02))),
    "amplitude_0.5_slope_0": (dict(function_amplitude=0.5, function_slope=0.0), {}),
    "n_global_0": (dict(n_global_iterations=0), {}),
}
CASES = {**{k: v[:2] for k, v in SETTINGS.items()}, **EXTRA}


@pytest.mark.parametrize("name", list(CASES))
def test_equals_oracle(oracle, base, name):
    region, depth = CASES[name]
    wl = _variant(base, region, depth)
    opts = (0, 1) if name != "n_global_0" else (0,)
    st = compare_with_oracle(oracle, wl, corrs=(0, 3, wl.n_corr_iterations - 1) if name != "scales8" else None, opts=opts)
    assert st["valid_lines"] > 0 and st["valid_points"] > 0, st
    assert st["horizontal"] > 0 and st["vertical"] > 0 and st["forward"] > 0 and st["reverse"] > 0, st


@pytest.mark.parametrize("n_global", [1, 0])
def test_zero_area_keeps_a_nan_variance(oracle, base, n_global):
    """function_amplitude 0.5, function_slope 0 (lookup values 0 / 1) and colours that are all foreground-only: every
    distribution entry multiplies a 0 background term, so the area is 0, the distribution NaN and std::max(NaN, min)
    keeps the NaN variance; global and local gradients."""
    wl = _variant(base, dict(function_amplitude=0.5, function_slope=0.0, n_global_iterations=n_global))
    n3 = wl.region.n_histogram_bins ** 3
    st = compare_with_oracle(oracle, wl, corrs=(0, 3), histograms=(np.full(n3, 1.0 / n3, f32), np.zeros(n3, f32)))
    assert st["zero_areas"] > 0 and st["nan_variances"] == st["zero_areas"], st


# ---- the decision scenes (tests/correspondence_cases.py) -----------------------------------------------------------------
@pytest.mark.parametrize("scales", [(6, 4, 2, 1), (12, 8, 7, 5, 3)])
def test_decision_scene_equals_oracle(oracle, synth, scales):
    """Every line and point of the hand-made scene equals the oracle's at every scale of the schedule, and so do g / H,
    also at poses shifted so that the local-mode gradient reads the distribution's edges; the scene reaches every
    counter it was built for."""
    import correspondence_cases as cases
    st = ref.new_stats()
    for wl in cases.decision_scenes(synth, scales):
        _decision_scene(oracle, wl, st, cases)
    assert cases.reached(st) == [], st


def _decision_scene(oracle, wl, st, cases):
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    orc.hist_f[0], orc.hist_b[0] = cases.histograms(wl.region.n_histogram_bins)
    pose = wl.start_body2world[0]
    for corr in range(wl.n_corr_iterations):
        n, view = orc.region_correspondences(0, 0, corr)
        lines = ref.region_lines(wl, 0, pose, view, n, orc.hist_f[0], orc.hist_b[0], corr, st, oracle.REGION_LINE_DTYPE)
        assert_lines_equal(lines, orc.lines[0][:n], corr)
        m, view = orc.depth_correspondences(0, 0, corr)
        pts = ref.depth_points(wl, 0, pose, view, m, corr, st, oracle.DEPTH_POINT_DTYPE)
        assert_points_equal(pts, orc.points[0][:m], corr)
        for dx in [0.0] + cases.gh_shifts(wl, corr):
            shifted = pose.copy()
            shifted[0, 3] += f32(dx)
            orc.set_poses(shifted[None])
            for opt in (0, 1):
                og, oH = orc.region_gradient_hessian(0, corr, opt)
                g, H = ref.region_gradient_hessian(wl, 0, shifted, lines, corr, opt, st)
                assert rel_to_max(H, oH) < 1e-6 and rel_to_max(g, og) < 1e-6 * max(1.0, np.abs(oH).max() /
                                                                                   max(np.abs(og).max(), 1e-30))
            orc.set_poses(pose[None])


# ---- closed forms on hand-made frames ---------------------------------------------------------------------------------
def _line_case(synth, nu, nv, cu, cv, scale=1, amplitude=0.43, slope=0.5, width=200, height=160):
    """One region line through (cu, cv) with image normal (nu, nv): a model point on the optical axis plane at z = 1,
    identity camera and pose, fu = fv = 100."""
    intr = synth.Intrinsics(100.0, 100.0, 0.0, 0.0, width, height)
    region = synth.RegionSettings(n_lines_max=1, scales=(scale,), standard_deviations=(1.0,),
                                  function_amplitude=amplitude, function_slope=slope, min_continuous_distance=0.0)
    point = np.zeros(38, f32)
    point[0:3] = (cu / 100.0, cv / 100.0, 1.0)
    point[3:6] = (nu, nv, 0.0)
    point[6:8] = (1.0, 1.0)
    model = synth.Model("region", np.zeros((1, 3), f32), np.zeros(1, f32), point.reshape(1, 1, 38))
    eye = np.eye(4, dtype=f32)[:3]
    wl = synth.Workload(name="line", n_bodies=1, region=region, depth=None, tikhonov_rotation=1.0,
                        tikhonov_translation=1.0, n_corr_iterations=1, n_update_iterations=1, color_intrinsics=intr,
                        depth_intrinsics=intr, color_world2camera=eye, depth_world2camera=eye, depth_scale=0.001,
                        region_model=model, depth_model=None, color_frames=np.zeros((1, height, 3 * width), np.uint8),
                        depth_frames=None, gt_body2world=eye[None], start_body2world=eye[None])
    return wl


def _run_line(oracle, wl, hist_f, hist_b, st):
    """The restatement's line, after checking it equal to the oracle's on the same frame and histograms."""
    L = ref.region_lines(wl, 0, wl.start_body2world[0], 0, 1, hist_f, hist_b, 0, st, oracle.REGION_LINE_DTYPE)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    orc.hist_f[0], orc.hist_b[0] = hist_f, hist_b
    assert orc.region_correspondences(0, 0, 0) == (1, 0)
    assert_lines_equal(L, orc.lines[0][:1], "oracle")
    return L[0]


def _run_point(oracle, wl, st):
    P = ref.depth_points(wl, 0, wl.start_body2world[0], 0, 1, 0, st, oracle.DEPTH_POINT_DTYPE)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    assert orc.depth_correspondences(0, 0, 0) == (1, 0)
    assert_points_equal(P, orc.points[0][:1], "oracle")
    return P[0]


def test_constant_probability_line_is_uniform(oracle, synth):
    """Every pixel with the same colour probabilities: every distribution entry equal, mean 0, variance 143 / 12."""
    wl = _line_case(synth, 1.0, 0.0, 100.0, 80.0)
    n3 = 16 ** 3
    st = ref.new_stats()
    L = _run_line(oracle, wl, np.full(n3, 0.3, f32), np.full(n3, 0.7, f32), st)
    assert L["valid"] and st["horizontal"] == 1 and st["forward"] == 1
    assert np.all(L["distribution"] == L["distribution"][0])
    assert abs(float(L["mean"])) < 1e-5 and abs(float(L["measured_variance"]) - 143.0 / 12.0) < 1e-4


def test_two_colour_stripe_reaches_the_segment_fallback(oracle, synth):
    """Scale 2: a stripe of two colours that each occur in only one histogram, so each 2-pixel segment multiplies a
    (1, 0) and a (0, 1) probability: both products are 0 and the segment takes 0.5 / 0.5."""
    wl = _line_case(synth, 1.0, 0.0, 100.0, 80.0, scale=2)
    img = wl.color_frames[0]
    img[:, 0::6] = 255          # even columns: colour (255, 255, 255); odd columns: black
    img[:, 1::6] = 255
    img[:, 2::6] = 255
    n3 = 16 ** 3
    hf, hb = np.zeros(n3, f32), np.zeros(n3, f32)
    hf[n3 - 1] = 1.0            # white only in the foreground histogram
    hb[0] = 1.0                 # black only in the background histogram
    st = ref.new_stats()
    L = _run_line(oracle, wl, hf, hb, st)
    assert L["valid"] and st["segment_fallbacks"] == ref.K_SEGMENTS
    assert np.all(L["distribution"] == L["distribution"][0])


@pytest.mark.parametrize("cu,expect", [(50.5, 0.5), (51.5, 0.5), (8.5, -0.5), (50.25, -0.25)])
def test_delta_r_halves_round_away_from_zero(oracle, synth, cu, expect):
    """delta_r = (round(c - 9) + 9 - c) / n at scale 1 (line_length_minus_1_half = 9). c - 9 = 41.5 and 42.5 (both
    parities) round up and -0.5 rounds down, away from zero; rounding to even would give 0.5 / -0.5 / 0.5."""
    wl = _line_case(synth, 1.0, 0.0, cu, 80.0)
    st = ref.new_stats()
    L = _run_line(oracle, wl, np.full(16 ** 3, 0.5, f32), np.full(16 ** 3, 0.5, f32), st)
    assert L["valid"] and L["delta_r"] == f32(expect)
    assert st["delta_r_ties"] == (1 if cu % 1 == 0.5 else 0)


def test_equal_normal_components_take_the_vertical_branch(oracle, synth):
    s = f32(np.sqrt(f32(0.5)))
    wl = _line_case(synth, float(s), float(s), 100.25, 80.0)   # delta_r and the walk differ between the branches
    st = ref.new_stats()
    L = _run_line(oracle, wl, np.full(16 ** 3, 0.5, f32), np.full(16 ** 3, 0.5, f32), st)
    assert L["valid"] and st["ties_nu_nv"] == 1 and st["vertical"] == 1 and st["horizontal"] == 0
    assert L["normal_component_to_scale"] == abs(L["normal_v"])


@pytest.mark.parametrize("cv,key,valid", [(0.25, "rejected_end_lo", 0), (1.0, "end_at_1", 1),
                                          (158.0, "end_at_minor_m2", 1), (158.6, "rejected_end_hi", 0)])
def test_minor_axis_margins(oracle, synth, cv, key, valid):
    """A horizontal line (step 0) on rows 0, 1, 158 (= height - 2) and 159: int(minor_f_end) must lie in
    [1, height - 2], so rows 0 and 159 are refused although the centre is on the image."""
    wl = _line_case(synth, 1.0, 0.0, 100.0, cv)
    st = ref.new_stats()
    L = _run_line(oracle, wl, np.full(16 ** 3, 0.5, f32), np.full(16 ** 3, 0.5, f32), st)
    assert L["valid"] == valid and st[key] == 1, st


def _depth_case(synth, raw_frame, point_xyz, considered=0.05, stride_length=0.005, depth_scale=0.001):
    h, w = raw_frame.shape
    intr = synth.Intrinsics(100.0, 100.0, w / 2.0, h / 2.0, w, h)
    depth = synth.DepthSettings(n_points_max=1, stride_length=stride_length, considered_distances=(considered,),
                                standard_deviations=(0.05,))
    point = np.zeros(36, f32)
    point[0:3] = point_xyz
    point[3:6] = (0.0, 0.0, -1.0)
    model = synth.Model("depth", np.zeros((1, 3), f32), np.zeros(1, f32), point.reshape(1, 1, 36))
    eye = np.eye(4, dtype=f32)[:3]
    return synth.Workload(name="point", n_bodies=1, region=None, depth=depth, tikhonov_rotation=1.0,
                          tikhonov_translation=1.0, n_corr_iterations=1, n_update_iterations=1, color_intrinsics=intr,
                          depth_intrinsics=intr, color_world2camera=eye, depth_world2camera=eye,
                          depth_scale=depth_scale, region_model=None, depth_model=model, color_frames=None,
                          depth_frames=raw_frame[None], gt_body2world=eye[None], start_body2world=eye[None])


def test_equidistant_samples_take_the_first_in_row_major_order(oracle, synth):
    """A flat frame with a point on the optical axis just in front of it: the two samples left and right of the axis
    at the same distance; the first (left) one wins."""
    frame = np.zeros((40, 40), np.uint16)
    frame[20, 19] = frame[20, 21] = 1000      # 1 m, one pixel either side of the principal point (20, 20)
    wl = _depth_case(synth, frame, (0.0, 0.0, 0.99), stride_length=0.0025)   # 20 strides: every pixel
    st = ref.new_stats()
    P = _run_point(oracle, wl, st)
    assert P["valid"] and st["equal_ties"] == 1 and st["stride_1"] == 1
    assert np.array_equal(P["correspondence_center_f_camera"], np.array([-0.01, 0.0, 1.0], f32))


def test_considered_distance_above_the_depth_admits_raw_0(oracle, synth):
    """considered distance 0.05 m > z = 0.03 m: min_depth_value = std::min(0, negative) < 0, so raw 0 passes the
    depth test and is taken when it is the closest sample (0 m depth at the principal point is 0.03 m away)."""
    frame = np.full((40, 40), 65535, np.uint16)
    frame[20, 20] = 0
    wl = _depth_case(synth, frame, (0.0, 0.0, 0.03), stride_length=0.0001)   # stride 1 over the whole frame
    st = ref.new_stats()
    P = _run_point(oracle, wl, st)
    assert P["valid"] and st["raw0_admitted"] > 0
    assert np.array_equal(P["correspondence_center_f_camera"], np.zeros(3, f32))


# ---- the depth search's screen ----------------------------------------------------------------------------------------
def _screen_misses(depth_scale, use_depth_scaling, parent, n=400_000, seed=0):
    """Samples near the worst case: for a point and a sample inside its considered distance, best is set to the
    smallest float above the sample's exact d2, so the strict test d2 < best just accepts it. Returns how many such
    samples the screen rejects."""
    rng = np.random.default_rng(seed)

    class It:
        pass
    it = It()
    it.fu, it.fv, it.ppu, it.ppv = f32(365.0), f32(365.0), f32(320.5), f32(288.25)
    it.depth_scale = f32(depth_scale)
    z_max = 65535 * depth_scale
    z = rng.uniform(0.05, z_max, n).astype(f32)
    d = rng.uniform(0.0, 1.0, n).astype(f32)                  # considered distance parameter, up to 1 m
    cd = (d * z).astype(f32) if use_depth_scaling else d
    u_c = rng.uniform(0, 640, n).astype(f32)
    v_c = rng.uniform(0, 576, n).astype(f32)
    x = ((u_c - it.ppu) * z / it.fu).astype(f32)
    y = ((v_c - it.ppv) * z / it.fv).astype(f32)
    r_px = np.minimum(cd * it.fu / z, 640).astype(np.float64)
    u = np.clip(np.round(u_c + rng.uniform(-1, 1, n) * r_px), 0, 639)
    v = np.clip(np.round(v_c + rng.uniform(-1, 1, n) * r_px), 0, 575)
    raw = np.clip(np.round((z + rng.uniform(-1, 1, n).astype(f32) * cd) / it.depth_scale), 1, 65535)
    _, _, _, d2 = ref.exact_distance2(u, v, raw, x, y, z, it)
    keep = d2 < cd * cd
    best = np.nextafter(d2, f32(np.inf)).astype(f32)
    bound = None if parent else ref.screen_bound(x, y)
    ok = ref.screen_passes(u, v, raw, x, y, z, best, it, bound)
    return int((keep & ~ok).sum()), int(keep.sum())


@pytest.mark.parametrize("use_depth_scaling", [False, True])
@pytest.mark.parametrize("depth_scale", [1e-4, 1e-3, 1e-2])
def test_screen_never_rejects_an_accepted_sample(depth_scale, use_depth_scaling):
    misses, n = _screen_misses(depth_scale, use_depth_scaling, parent=False)
    assert n > 100_000 and misses == 0, (misses, n)


def test_fixed_margin_screen_rejected_accepted_samples():
    """The earlier screen (a fixed 1e-6 m^2 margin) fails the same proof obligation at far depths."""
    misses, _ = _screen_misses(1e-3, True, parent=True)
    assert misses > 0
