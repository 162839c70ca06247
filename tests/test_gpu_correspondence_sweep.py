"""The device's region lines and depth points held to the restatement of the reference (tests/correspondence_reference.py)
at the places where their integer and tie decisions sit: every k_track2 form (512 / 1024 threads, LUT in shared and
global memory), every scale specialisation of the walk and the generic one, the walk and the depth search on and off the
shared-memory tile, k_track on the same cases, far and off-axis bodies with depth scaling and a coarse depth scale, a
NaN-pose body, and step-function / near-degenerate function lookups in global and local mode.

Each case compares, at every correspondence iteration it runs: the closest views with the mirror oracle's; the per-line
and per-point records of the fine-grained calls and of the fused launch with the restatement's, bit for bit (a NaN
equals a NaN); g / H of the fine-grained calls within 1e-5 of max|H|. It asserts the restatement counters it was built
to reach and the launch it means to exercise (m3tb_debug_last_launch). The pose the fused launch solves stays within
1e-5 of the mirror oracle's, which holds the fused g / H.

The hand-made scenes of tests/correspondence_cases.py put lines and points on the decisions themselves (ties, margins,
truncations, raw bounds, clipped windows, segment fallbacks, the local gradient's distribution edges) and run through
every launch form; the synthetic workloads add volume, far bodies and degenerate lookups."""
import dataclasses

import numpy as np
import pytest

import correspondence_cases as cases
import correspondence_reference as ref
from helpers import pose_error

pytestmark = pytest.mark.gpu

f32 = np.float32
_ENV = ("M3TB_TMA", "M3TB_TMA_MAXW", "M3TB_NO_TILES", "M3TB_NO_ROI_INGEST", "M3TB_KERNEL")
LINE_FIELDS = ("center_f_body", "center_u", "center_v", "normal_u", "normal_v")
LINE_FIELDS_VALID = ("delta_r", "normal_component_to_scale", "distribution", "mean", "measured_variance")


@pytest.fixture(autouse=True)
def _default_staging(monkeypatch):
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)


def _same(a, b):
    """Bit equality of float32 arrays, any NaN equal to any NaN (the device's and the host's NaN payloads differ)."""
    a, b = np.ascontiguousarray(a, f32), np.ascontiguousarray(b, f32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def assert_lines(got, want, tag):
    assert np.array_equal(got["valid"], want["valid"]), (tag, np.nonzero(got["valid"] != want["valid"]))
    for f in LINE_FIELDS:
        assert _same(got[f], want[f]), (tag, f)
    v = want["valid"] != 0
    for f in LINE_FIELDS_VALID:
        assert _same(got[f][v], want[f][v]), (tag, f)


def assert_points(got, want, tag):
    assert np.array_equal(got["valid"], want["valid"]), (tag, np.nonzero(got["valid"] != want["valid"]))
    for f in ("center_f_body", "normal_f_body"):
        assert _same(got[f], want[f]), (tag, f)
    v = want["valid"] != 0
    assert _same(got["correspondence_center_f_camera"][v], want["correspondence_center_f_camera"][v]), tag


def assert_gh(g, H, rg, rH, tag):
    if not (np.isfinite(rH).all() and np.isfinite(rg).all()):
        assert np.array_equal(np.isnan(H), np.isnan(rH)) and np.array_equal(np.isnan(g), np.isnan(rg)), tag
        return
    scale = max(np.abs(rH).max(), 1e-30)
    assert np.abs(H.astype(np.float64) - rH).max() <= 1e-5 * scale, tag
    assert np.abs(g.astype(np.float64) - rg).max() <= 1e-5 * max(scale, np.abs(rg).max()), tag


def sweep(capi, oracle, wl, corrs=None, opts=(0,), histograms=None, reset=False, shifts=None):
    """Runs the comparisons of the module docstring; returns (restatement stats, launch of the fused calls).
    histograms: (hf, hb) that replace every body's histograms after StartModalities, on the device and the oracle.
    reset: every correspondence iteration starts from the start poses (hand-made scenes keep their exact projection).
    shifts(wl, corr): camera-x offsets of the pose at which the region g / H are evaluated as well."""
    st = ref.new_stats()
    ctx = capi.context_from_workload(wl)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    orc.start_modalities(0)
    ctx.start_modalities(0)
    nb = wl.region.n_histogram_bins if wl.region else 0
    if histograms is not None:
        for b in range(wl.n_bodies):
            ctx.set_histograms(b, *histograms)
            orc.hist_f[b], orc.hist_b[b] = histograms
    corrs = range(wl.n_corr_iterations) if corrs is None else corrs
    launch = None
    for corr in corrs:
        if reset:
            orc.set_poses(wl.start_body2world)
        poses = orc.get_poses()
        want_l, want_p = {}, {}
        ctx.set_poses(poses)
        if wl.region:
            ctx.region_correspondences(0, corr)
        if wl.depth:
            ctx.depth_correspondences(0, corr)
        for b in range(wl.n_bodies):
            tag = (corr, b)
            if wl.region:
                n, view = orc.region_correspondences(b, 0, corr)
                assert ctx.get_closest_views(b)[0] == view, tag
                hf, hb = ctx.get_histograms(b, nb)
                want_l[b] = ref.region_lines(wl, b, poses[b], view, n, hf, hb, corr, st, oracle.REGION_LINE_DTYPE)
                assert_lines(ctx.get_region_lines(b, wl.lines_per_body)[:n], want_l[b], ("fine",) + tag)
            if wl.depth:
                m, view = orc.depth_correspondences(b, 0, corr)
                assert ctx.get_closest_views(b)[1] == view, tag
                want_p[b] = ref.depth_points(wl, b, poses[b], view, m, corr, st, oracle.DEPTH_POINT_DTYPE)
                assert_points(ctx.get_depth_points(b, wl.points_per_body)[:m], want_p[b], ("fine",) + tag)
        for opt in opts:
            if wl.region:
                g, H = ctx.region_gradient_hessian(0, corr, opt)
                for b in range(wl.n_bodies):
                    rg, rH = ref.region_gradient_hessian(wl, b, poses[b], want_l[b], corr, opt, st)
                    assert_gh(g[b], H[b], rg, rH, ("region", corr, opt, b))
            if wl.depth:
                g, H = ctx.depth_gradient_hessian(0, corr, opt)
                for b in range(wl.n_bodies):
                    rg, rH = ref.depth_gradient_hessian(wl, b, poses[b], want_p[b], corr)
                    assert_gh(g[b], H[b], rg, rH, ("depth", corr, opt, b))
        for dx in (shifts(wl, corr) if shifts and wl.region else ()):
            shifted = poses.copy()
            shifted[:, 0, 3] += f32(dx)
            ctx.set_poses(shifted)
            for opt in opts:
                g, H = ctx.region_gradient_hessian(0, corr, opt)
                for b in range(wl.n_bodies):
                    rg, rH = ref.region_gradient_hessian(wl, b, shifted[b], want_l[b], corr, opt, st)
                    assert_gh(g[b], H[b], rg, rH, ("region shifted", dx, corr, opt, b))
        ctx.set_poses(poses)
        ctx.corr_iteration(0, corr, wl.n_update_iterations)   # the fused launch: its records are the same lines / points
        launch = launch or ctx.last_launch()
        for b in range(wl.n_bodies):
            if wl.region:
                assert_lines(ctx.get_region_lines(b, wl.lines_per_body)[:len(want_l[b])], want_l[b], ("fused", corr, b))
            if wl.depth:
                assert_points(ctx.get_depth_points(b, wl.points_per_body)[:len(want_p[b])], want_p[b], ("fused", corr, b))
        with np.errstate(invalid="ignore", over="ignore"):
            orc.tracking_step(0, n_corr=corr + 1, corr_begin=corr)
        # the fused launch keeps its g / H to itself: they are held through the pose it solves from them, against the
        # mirror oracle's step (whose g / H equal the restatement's, test_correspondence_reference.py)
        gpu, want = ctx.get_poses(), orc.get_poses()
        fin = np.isfinite(want).all(axis=(1, 2))
        assert np.array_equal(np.isfinite(gpu).all(axis=(1, 2)), fin), ("fused pose", corr)
        if fin.any():
            dt, dr = pose_error(gpu[fin], want[fin])
            assert dt.max() < 1e-5 and dr.max() < 1e-5, ("fused pose", corr, dt, dr)
    ctx.close()
    assert st["screen_misses"] == 0, st
    return st, launch


# ---- the cases --------------------------------------------------------------------------------------------------------
def _bins(wl, bins):
    return dataclasses.replace(wl, region=dataclasses.replace(wl.region, n_histogram_bins=bins))


def base_workload(synth, **kw):
    return synth.make_workload("c2", n_bodies=4, n_divides=2, seed=3, **kw)


def far_workload(synth, depth_scale, use_depth_scaling, considered):
    """Bodies 3-60 m away (off axis: anywhere in the frame) with depth frames re-quantised to depth_scale."""
    wl = synth.make_workload("c2", n_bodies=4, n_divides=2, seed=5, z_range=(3.0, 60.0), margin_px=40.0)
    k = wl.depth_scale / depth_scale
    wl.depth_frames = np.clip(np.round(wl.depth_frames.astype(np.float64) * k), 0, 65535).astype(np.uint16)
    wl.depth_scale = depth_scale
    wl.depth = dataclasses.replace(wl.depth, use_depth_scaling=use_depth_scaling, considered_distances=considered)
    wl.region = dataclasses.replace(wl.region, min_continuous_distance=0.0)
    return wl


def _track2(threads, lut_smem):
    return lambda L: L["kernel"] == "k_track2" and L["threads"] == threads and L["lut_smem"] == lut_smem


WALK = lambda s: s["horizontal"] > 0 and s["vertical"] > 0 and s["forward"] > 0 and s["reverse"] > 0
SEARCH = lambda s: s["stride_above_1"] > 0 and s["valid_points"] > 0
GENERIC_SCALES = dict(scales=(12, 8, 7, 5, 3, 6, 2, 1), standard_deviations=(15.0, 5.0))

CASES = {
    # id: (workload builder, environment, launch check, reach check, options)
    "track2_1024_lut_shared": (lambda s: base_workload(s), {}, _track2(1024, 1),
                               lambda s: WALK(s) and SEARCH(s), {}),
    "track2_1024_lut_global": (lambda s: _bins(base_workload(s), 32), {}, _track2(1024, 0),
                               lambda s: WALK(s) and SEARCH(s), {}),
    "track2_512_lut_shared": (lambda s: dataclasses.replace(base_workload(s), depth=None), {}, _track2(512, 1), WALK, {}),
    "track2_512_lut_global": (lambda s: dataclasses.replace(_bins(base_workload(s), 32), depth=None), {},
                              _track2(512, 0), WALK, {}),
    "track2_generic_scales": (lambda s: dataclasses.replace(base_workload(s), region=dataclasses.replace(
        base_workload(s).region, **GENERIC_SCALES)), {}, _track2(1024, 1), WALK, {}),
    # no tiles: every line takes WalkSlow / GatherSlow and every point DepthSearchSlow on the cases above
    "track2_no_tiles": (lambda s: base_workload(s), {"M3TB_NO_TILES": "1"}, _track2(1024, 1), SEARCH, {}),
    "track2_generic_no_tiles": (lambda s: dataclasses.replace(base_workload(s), region=dataclasses.replace(
        base_workload(s).region, **GENERIC_SCALES)), {"M3TB_NO_TILES": "1"}, _track2(1024, 1), WALK, {}),
    "k_track": (lambda s: base_workload(s), {"M3TB_KERNEL": "1"}, lambda L: L["kernel"] == "k_track",
                lambda s: WALK(s) and SEARCH(s), {}),
    "k_track_generic_scales": (lambda s: dataclasses.replace(base_workload(s), region=dataclasses.replace(
        base_workload(s).region, **GENERIC_SCALES)), {"M3TB_KERNEL": "1"}, lambda L: L["kernel"] == "k_track", WALK, {}),
    "far_depth_scaling_1e-2": (lambda s: far_workload(s, 1e-2, True, (0.5, 0.1, 0.02)), {}, _track2(1024, 1),
                               lambda s: s["valid_points"] > 0 and s["clipped_left"] + s["clipped_top"] > 0, {}),
    "far_1e-3": (lambda s: far_workload(s, 1e-3, False, (0.5, 0.1, 0.02)), {}, _track2(1024, 1),
                 lambda s: s["valid_points"] > 0 and s["stride_1"] > 0, {}),
    "far_k_track": (lambda s: far_workload(s, 1e-2, True, (0.5, 0.1, 0.02)), {"M3TB_KERNEL": "1"},
                    lambda L: L["kernel"] == "k_track", lambda s: s["valid_points"] > 0 and s["clipped_top"] > 0, {}),
}


@pytest.mark.parametrize("case", list(CASES))
def test_sweep(capi, oracle, synth, monkeypatch, case):
    build, env, launch_ok, reach, kw = CASES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    st, launch = sweep(capi, oracle, build(synth), **kw)
    assert launch_ok(launch), launch
    assert reach(st), st


DECISIONS = {
    # id: (scene options, environment, launch check)
    "1024_lut_shared": (dict(), {}, _track2(1024, 1)),
    "1024_lut_global": (dict(n_bins=32), {}, _track2(1024, 0)),
    "512_region_lut_shared": (dict(depth=False), {}, _track2(512, 1)),
    "512_region_lut_global": (dict(depth=False, n_bins=32), {}, _track2(512, 0)),
    "512_depth": (dict(region=False), {}, lambda L: L["kernel"] == "k_track2" and L["threads"] == 512),
    "1024_generic_scales": (dict(scales=(12, 8, 7, 5, 3)), {}, _track2(1024, 1)),
    "1024_no_tiles": (dict(), {"M3TB_NO_TILES": "1"}, _track2(1024, 1)),
    "1024_generic_no_tiles": (dict(scales=(12, 8, 7, 5, 3)), {"M3TB_NO_TILES": "1"}, _track2(1024, 1)),
    "k_track": (dict(), {"M3TB_KERNEL": "1"}, lambda L: L["kernel"] == "k_track"),
    "k_track_generic_scales": (dict(scales=(12, 8, 7, 5, 3)), {"M3TB_KERNEL": "1"}, lambda L: L["kernel"] == "k_track"),
}


@pytest.mark.parametrize("case", list(DECISIONS))
def test_decision_scene(capi, oracle, synth, monkeypatch, case):
    """The hand-made scenes on one launch form: every line and point at every scale of the schedule, g / H also at poses
    shifted so that the local gradient reads the distribution's edges; every counter the scenes were built for. The
    compact body's lines and windows take the tile paths (WalkFast, the screened depth search) where they fit, the
    border body's the out-of-tile ones (WalkSlow / GatherSlow, DepthSearchSlow)."""
    kw, env, launch_ok = DECISIONS[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    total = ref.new_stats()
    for wl in cases.decision_scenes(synth, **kw):
        hist = cases.histograms(wl.region.n_histogram_bins) if wl.region else None
        st, launch = sweep(capi, oracle, wl, opts=(0, 1), histograms=hist, reset=True, shifts=cases.gh_shifts)
        assert launch_ok(launch), launch
        for k in total:
            total[k] += st[k]
    assert cases.reached(total, region=wl.region is not None, depth=wl.depth is not None) == [], total


@pytest.mark.parametrize("env", [{}, {"M3TB_NO_TILES": "1"}, {"M3TB_KERNEL": "1"}], ids=["tiles", "no_tiles", "k_track"])
def test_screen_scene(capi, oracle, synth, monkeypatch, env):
    """Points 20-40 m away whose closest sample the earlier fixed-margin screen rejected (tests/correspondence_cases.
    py::screen_scene): the device takes it, as the restatement and the oracle do, on the tile path, DepthSearchSlow and
    k_track."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    st, launch = sweep(capi, oracle, cases.screen_scene(synth), reset=True)
    assert st["parent_screen_misses"] == st["valid_points"] == 6, st
    assert launch["kernel"] == ("k_track" if "M3TB_KERNEL" in env else "k_track2"), launch


def _one_colour_histograms(nb, foreground):
    """Histograms in which every colour is foreground-only (or background-only): every LUT entry is (1, 0) / (0, 1)."""
    n3 = nb ** 3
    full, empty = np.full(n3, 1.0 / n3, f32), np.zeros(n3, f32)
    return (full, empty) if foreground else (empty, full)


@pytest.mark.parametrize("mode", ["global", "local"])
@pytest.mark.parametrize("lookup", ["zero_areas", "subnormal_areas"])
def test_degenerate_lookups(capi, oracle, synth, lookup, mode):
    """function_amplitude 0.5 with function_slope 0: lookup values 0 / 1, so each distribution entry is the product of
    four foreground and four background segment probabilities. On foreground-only colours every entry is 0, the area
    is 0 and the variance NaN, which std::max keeps. With a colour probability of 1e-10 / 1 every entry is about
    1e-40: at scale 1 the area is subnormal, at the larger scales the segment products underflow to zero entries.
    Global (n_global_iterations 1) and local (0) gradients."""
    wl = base_workload(synth)
    wl.region = dataclasses.replace(wl.region, function_amplitude=0.5, function_slope=0.0,
                                    n_global_iterations=1 if mode == "global" else 0)
    n3 = wl.region.n_histogram_bins ** 3
    hist = (_one_colour_histograms(wl.region.n_histogram_bins, True) if lookup == "zero_areas" else
            (np.full(n3, 1e-10 / n3, f32), np.full(n3, 1.0 / n3, f32)))
    st, launch = sweep(capi, oracle, wl, corrs=(0, 3), opts=(0,), histograms=hist)
    assert _track2(1024, 1)(launch), launch
    assert st["zero_areas"] > 0 and st["nan_variances"] > 0 and st["zero_entries"] > 0, st
    if lookup == "subnormal_areas":
        assert st["subnormal_areas"] > 0, st


def test_nan_pose_body_on_k_track2(capi, oracle, synth):
    """Body 1 with a NaN pose in a k_track2 batch: its lines and points are invalid and the other bodies' records and
    g / H equal the restatement's."""
    wl = base_workload(synth)
    wl.start_body2world = wl.start_body2world.copy()
    wl.start_body2world[1] = np.nan
    st, launch = sweep(capi, oracle, wl, corrs=(0,))
    assert _track2(1024, 1)(launch), launch
    assert st["valid_lines"] > 0 and st["valid_points"] > 0, st


@pytest.mark.parametrize("d,stride", [(0.0, 0.005), (-0.01, 0.005), (float("nan"), 0.005), (float("inf"), 0.005),
                                      (0.0024, 0.005), (0.05, 1e-12)])
def test_unusable_considered_distances_are_refused(capi, synth, d, stride):
    """A considered distance that is not finite, not positive, below half the stride length (0.005 m: 0.0024 gives
    int(0.48 + 0.5) = 0 strides) or 2^31 strides or more (a 1e-12 m stride) is refused before anything of the body
    changes: its histograms stay as they were."""
    wl = base_workload(synth)
    ctx = capi.context_from_workload(wl)
    nb = wl.region.n_histogram_bins
    hf, hb = np.arange(nb ** 3, dtype=f32), np.arange(nb ** 3, dtype=f32)[::-1].copy()
    ctx.set_histograms(0, hf, hb)
    depth = dataclasses.replace(wl.depth, considered_distances=(0.05, d), stride_length=stride)
    with pytest.raises(capi.M3TBError, match="considered distances"):
        ctx.set_body(0, capi.region_params(wl.region), capi.depth_params(depth),
                     capi.OptimizerParams(wl.tikhonov_rotation, wl.tikhonov_translation))
    gf, gb = ctx.get_histograms(0, nb)
    assert np.array_equal(gf, hf) and np.array_equal(gb, hb)
    ctx.close()
