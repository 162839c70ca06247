"""The occlusion / region / silhouette checks of the region and depth modalities (SURVEY row f4) restated from the
reference (tests/occlusion_reference.py): the restatement against the oracle at several parameter settings, closed
forms on hand-made frames, and the two defects the restatement pins: scans whose stride would be 0, and a region
depth-offset id of 30."""
import copy
import ctypes as C

import numpy as np
import pytest

import occlusion_reference as ref
from test_oracle_occlusion import occluded_workload

f32 = np.float32


def checks_off(wl):
    base = copy.deepcopy(wl)
    if base.region:
        base.region.measure_occlusions = base.region.model_occlusions = base.region.use_region_checking = False
    if base.depth:
        base.depth.measure_occlusions = base.depth.model_occlusions = base.depth.use_silhouette_checking = False
    return base


def oracle_counts(oracle, orc, b, handle):
    """Per-bin pixel counts of AddLinePixelColorsToTempHistograms from the oracle."""
    L = orc.L
    L.orc_region_add_line_pixels_occ.argtypes = [C.POINTER(oracle.RegionParams), C.POINTER(oracle.Model),
                                                 C.POINTER(oracle.ColorFrame), C.POINTER(oracle.DepthFrame), C.c_int,
                                                 oracle.fp, C.c_int, oracle.fp, oracle.fp]
    nb = orc.wl.region.n_histogram_bins
    mf, mb = np.zeros(nb ** 3, np.float32), np.zeros(nb ** 3, np.float32)
    B = orc.bodies[b]
    L.orc_region_add_line_pixels_occ(B.region, B.region_model, B.color, B.region_occlusion_frame, int(handle),
                                     B.body2world, orc.rotation_mode, oracle.ptr(mf), oracle.ptr(mb))
    return mf.astype(np.int64), mb.astype(np.int64)


def compare_with_oracle(oracle, wl, iterations=(0, 3), corrs=(0, 2), stats=None):
    """The restatement's valid flags and histogram counts equal the oracle's for every body, line and point."""
    stats = ref.new_stats() if stats is None else stats
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    base = oracle.OracleTracker(checks_off(wl), rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    poses = orc.get_poses()
    n_checked = 0
    for b in range(wl.n_bodies):
        if wl.region:
            view = oracle.lib().orc_closest_view(C.byref(orc.rm), oracle.ptr(oracle.f32(
                ref.pose_mul(ref._camera(wl, b, "color")[1], poses[b]))), orc.rotation_mode)
            n = min(wl.region.n_lines_max, wl.region_model.n_points)
            for handle in (False, True):
                cf, cb = ref.histogram_counts(wl, b, poses[b], view, n, handle, stats)
                of, ob = oracle_counts(oracle, orc, b, handle)
                assert np.array_equal(cf, of) and np.array_equal(cb, ob), (b, handle)
    for iteration in iterations:
        for corr in corrs:
            for b in range(wl.n_bodies):
                if wl.region:
                    n, view = orc.region_correspondences(b, iteration, corr)
                    n0, view0 = base.region_correspondences(b, iteration, corr)
                    assert (n, view) == (n0, view0)
                    pred = ref.region_valid(wl, b, poses[b], view, n, base.lines[b]["valid"], iteration, 0, corr, stats)
                    got = orc.lines[b]["valid"][:n] != 0
                    assert np.array_equal(pred, got), (b, iteration, corr, np.nonzero(pred != got))
                    n_checked += n
                if wl.depth:
                    m, view = orc.depth_correspondences(b, iteration, corr)
                    m0, view0 = base.depth_correspondences(b, iteration, corr)
                    assert (m, view) == (m0, view0)
                    pred = ref.depth_valid(wl, b, poses[b], view, m, base.points[b]["valid"], iteration, 0, stats)
                    got = orc.points[b]["valid"][:m] != 0
                    assert np.array_equal(pred, got), (b, iteration, corr, np.nonzero(pred != got))
                    n_checked += m
    assert n_checked > 0
    return stats


def rendered_workload(synth, n_bodies=3, seed=19, **kw):
    wl = synth.make_workload("c2", n_bodies=n_bodies, n_divides=3, seed=seed)
    synth.fill_depth_offsets(wl.region_model, seed)
    synth.fill_depth_offsets(wl.depth_model, seed)
    synth.add_renderings(wl, occluder_bodies=(1,), image_size=kw.pop("image_size", 200))
    wl.region.model_occlusions = wl.region.use_region_checking = True
    wl.depth.model_occlusions = wl.depth.use_silhouette_checking = True
    wl.region.n_unoccluded_iterations = wl.depth.n_unoccluded_iterations = 0
    for k, v in kw.items():
        for m in (wl.region, wl.depth):
            if hasattr(m, k):
                setattr(m, k, v)
    return wl


# ---- against the oracle ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [
    dict(),
    dict(measured_occlusion_radius=0.0),
    dict(measured_occlusion_radius=0.05, measured_occlusion_threshold=-0.05),
    dict(measured_occlusion_threshold=10.0),                     # above z: the bound wraps
    dict(measured_depth_offset_radius=0.05),                     # max_radius: id 25
    dict(n_unoccluded_iterations=3),
    dict(min_n_unoccluded_lines=150, min_n_unoccluded_points=190),
], ids=lambda kw: ",".join(f"{k}={v}" for k, v in kw.items()) or "default")
def test_measured_equals_oracle(oracle, kw):
    wl = occluded_workload(n_bodies=2, **kw)
    for k, v in kw.items():
        if hasattr(wl.depth, k):
            setattr(wl.depth, k, v)
    st = compare_with_oracle(oracle, wl)
    assert st["windows"] > 0
    if kw.get("measured_occlusion_threshold") == 10.0:
        assert st["wrapped_bounds"] > 0
    if kw.get("measured_occlusion_radius") == 0.05:
        assert st["stride_above_1"] > 0
    if "min_n_unoccluded_lines" in kw:
        assert st["fallbacks"] > 0


def test_depth_scaling_equals_oracle(oracle):
    wl = occluded_workload(n_bodies=2)
    wl.depth.use_depth_scaling = True
    wl.depth.considered_distances = (0.08, 0.04, 0.02)
    wl.depth.measured_depth_offset_radius = 0.09            # * z > max_radius: ids at the top of the table
    compare_with_oracle(oracle, wl)


@pytest.mark.parametrize("kw", [
    dict(),
    dict(min_continuous_distance=0.0),
    dict(min_continuous_distance=8.0),
    dict(min_continuous_distance=30.0),
    dict(modeled_occlusion_radius=0.05, modeled_occlusion_threshold=-0.05, modeled_depth_offset_radius=0.0),
    dict(image_size=50),
    dict(image_size=400),
], ids=lambda kw: ",".join(f"{k}={v}" for k, v in kw.items()) or "default")
def test_renderer_checks_equal_oracle(oracle, synth, kw):
    wl = rendered_workload(synth, **kw)
    st = compare_with_oracle(oracle, wl, iterations=(0,), corrs=(0, 3))
    assert st["windows"] > 0 and st["region_id_mismatch"] > 0


# ---- closed forms on hand-made frames --------------------------------------------------------------------------------
def test_window_closed_forms():
    img = np.zeros((40, 60), np.uint16)
    # diameter 10: stride int(10 / 5 + 1) = 3, n_strides int(10 / 3 + 0.5) = 3, rounded radius 4.5, so the window is
    # [16, 25] x [16, 25] in steps of 3
    st = ref.new_stats()
    assert ref.window_unoccluded(img, 20.0, 20.0, 10.0, 1000.0, st)
    assert st["stride_above_1"] == 1
    img[19, 22] = 500                      # on the stride grid: occludes
    assert not ref.window_unoccluded(img, 20.0, 20.0, 10.0, 1000.0)
    img[19, 22] = 0
    img[20, 22] = 500                      # one row off the grid: not seen
    assert ref.window_unoccluded(img, 20.0, 20.0, 10.0, 1000.0)
    img[20, 22] = 0
    img[16, 16] = 1000                     # equal to the bound: not in front of it
    assert ref.window_unoccluded(img, 20.0, 20.0, 10.0, 1000.0)
    assert ref.window_unoccluded(img, 20.0, 20.0, 10.0, 1000.9)      # ushort(1000.9) truncates to 1000 ...
    assert not ref.window_unoccluded(img, 20.0, 20.0, 10.0, 1001.0)  # ... 1001 puts the pixel in front
    # a window clipped at the left / top border: [0, 3, ...] from u_min = int(1 - 4.5 + 0.5) = -3 -> 0
    st = ref.new_stats()
    img[:] = 0
    img[0, 0] = 5
    assert not ref.window_unoccluded(img, 1.0, 1.0, 9.0, 6.0, st)
    assert st["clipped_left"] == 1 and st["clipped_top"] == 1
    # a centre far outside the image: an empty window, unoccluded
    st = ref.new_stats()
    img[:] = 1
    assert ref.window_unoccluded(img, 500.0, 20.0, 10.0, 1000.0, st)
    assert st["empty_windows"] == 1 and st["clipped_right"] == 1
    # a threshold above z: (z - offset - threshold) / scale < 0 wraps modulo 2^16 (ushort)
    st = ref.new_stats()
    img[:] = 0
    img[20, 20] = 60000
    assert not ref.window_unoccluded(img, 20.0, 20.0, 0.0, -100.0, st)   # 2^16 - 100 = 65436 > 60000
    assert st["wrapped_bounds"] == 1
    # radius 0: a single pixel, stride 1
    img[:] = 0
    img[20, 21] = 1
    assert ref.window_unoccluded(img, 20.0, 20.0, 0.0, 1000.0)
    assert not ref.window_unoccluded(img, 21.0, 20.0, 0.0, 1000.0)


def test_modeled_closed_forms(synth):
    S = 20
    a, b = 2.0, 3.0   # depth = a / (b - value)
    img = np.full((S, S), 65535, np.uint16)
    r = synth.Rendering(img, 100.0, 100.0, 2.0, a, b, 0, True)
    st = ref.new_stats()
    # all background: min value 65535, depth a / (b - 65535) < 0, never above an allowed depth > 0 ...
    assert not ref.modeled_window_unoccluded(r, 105.0, 105.0, 4.0, 0.5, st)
    assert st["all_background"] == 1
    # ... and above a negative allowed depth
    assert ref.modeled_window_unoccluded(r, 105.0, 105.0, 4.0, -1.0)
    img[10, 10] = 1   # depth 2 / (3 - 1) = 1
    assert ref.modeled_window_unoccluded(r, 105.0, 105.0, 0.0, 0.999)
    assert not ref.modeled_window_unoccluded(r, 105.0, 105.0, 0.0, 1.0)   # min_depth > allowed is strict
    # a window clipped at the focused image's edge: centre at focused (19.5, 19.5), diameter 4
    st = ref.new_stats()
    img[:] = 65535
    img[19, 19] = 1
    assert not ref.modeled_window_unoccluded(r, 109.75, 109.75, 4.0, 1.0, st)
    assert st["clipped_right"] == 1 and st["clipped_bottom"] == 1


def test_region_and_silhouette_closed_forms(synth):
    S = 16
    sil = np.zeros((S, S), np.uint8)
    sil[:, :8] = 7
    r = synth.Rendering(sil, 0.0, 0.0, 1.0, 0.0, 0.0, 7, True)
    # a contour at u = 8 with the normal pointing to +u (foreground on the -u side): sufficient for a short
    # min_continuous_distance, not when the foreground walk leaves the focused image
    assert ref.dynamic_line_region_sufficient(r, 3.0, 1.0, 7.5, 8.0, 1.0, 0.0)
    assert not ref.dynamic_line_region_sufficient(r, 30.0, 1.0, 7.5, 8.0, 1.0, 0.0)
    # a normal pointing the wrong way: the foreground sample is background
    st = ref.new_stats()
    assert not ref.dynamic_line_region_sufficient(r, 3.0, 1.0, 7.5, 8.0, -1.0, 0.0, st)
    assert st["region_id_mismatch"] == 1
    # region ids 0 and 255
    for rid in (0, 255):
        s2 = np.where(sil == 7, rid, 255 - rid).astype(np.uint8)
        r2 = synth.Rendering(s2, 0.0, 0.0, 1.0, 0.0, 0.0, rid, True)
        assert ref.dynamic_line_region_sufficient(r2, 3.0, 1.0, 7.5, 8.0, 1.0, 0.0)
    # silhouette checking: the pixel at the focused image's last row / column is inside, one further is outside
    sil[:] = 7
    assert ref.point_on_valid_silhouette(r, S - 1, S - 1)
    assert not ref.point_on_valid_silhouette(r, S, 0)
    assert ref.point_on_valid_silhouette(r, -1, 0)          # int(-1 + 0.5) truncates to 0 ...
    assert not ref.point_on_valid_silhouette(r, -2, 0)      # ... int(-1.5) to -1
    sil[3, 4] = 8
    st = ref.new_stats()
    assert not ref.point_on_valid_silhouette(r, 4, 3, st) and st["region_id_mismatch"] == 1
    # DynamicRegionDistance, max_considered_line_length 10, unconsidered 0.5: stride 2, i_start int(1.5 / 2 + 1) = 1,
    # offset 2.5. From the focused centre u = 5.5 the foreground walk samples u = 3 (own region), u = 1 (background):
    # length_f = 2 * 2 = 4. The background walk samples u = 8, 10 (background), then u = 12, the own region again, at
    # i = 3 > i_start: the reference writes the FOREGROUND length, 2 * 3 = 6 (:1218), and leaves length_b as it was.
    sil[:] = 0
    sil[:, 2:6] = 7
    sil[:, 12:] = 7
    lf, lb = ref.dynamic_region_distance(r, f32(10.0), f32(0.5), f32(5.0), f32(8.0), f32(1.0), f32(0.0), f32(10), f32(10))
    assert (lf, lb) == (f32(6), f32(10))
    sil[:, 12:] = 0   # without the second stretch of own region the foreground length stays 4
    lf, lb = ref.dynamic_region_distance(r, f32(10.0), f32(0.5), f32(5.0), f32(8.0), f32(1.0), f32(0.0), f32(10), f32(10))
    assert (lf, lb) == (f32(4), f32(10))


def test_depth_offset_ids():
    class M:
        stride_depth_offset, max_radius_depth_offset = 0.002, 0.05
    st = ref.new_stats()
    assert ref.region_offset_id(0.0, M, st) == 0
    assert ref.region_offset_id(0.003, M, st) == 2              # (1 + 0.5) * stride rounds up
    assert ref.region_offset_id(0.05, M, st) == 25
    assert ref.region_offset_id(0.0501, M, st) is None          # above max_radius
    assert ref.depth_offset_id(0.1, 1.0, False, 0.002, st) == 29   # past the table: the last entry
    assert st["top_ids"] == 1
    assert ref.depth_offset_id(0.01, 2.0, True, 0.002) == 10


# ---- the defects -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("diameter", [float("nan"), -0.5, -4.9, float("inf")])
def test_scan_of_nonfinite_or_negative_diameter(diameter, synth):
    """A NaN diameter or one in (-5, 0) gives the reference's scans a stride of 0: a loop that never ends. Under the
    new rule such a window (and an infinite one) scans nothing and counts as unoccluded."""
    img = np.full((40, 60), 100, np.uint16)
    rend = synth.Rendering(np.zeros((20, 20), np.uint16), 0.0, 0.0, 1.0, 1.0, 2.0, 0, True)
    if not np.isinf(diameter):
        st = ref.new_stats()
        ref.window_unoccluded(img, 20.0, 20.0, diameter, 1000.0, st, parent_rule=True)
        ref.modeled_window_unoccluded(rend, 10.0, 10.0, diameter, 0.0, st, parent_rule=True)
        assert st["stride0_scans"] == 2
    st = ref.new_stats()
    assert ref.window_unoccluded(img, 20.0, 20.0, diameter, 1000.0, st)
    assert ref.modeled_window_unoccluded(rend, 10.0, 10.0, diameter, 0.0, st)
    assert st["stride0_scans"] == 0 and st["windows"] == 0


def nan_and_behind_workload(synth, kind):
    wl = occluded_workload(n_bodies=2)
    wl.region.measured_occlusion_radius = wl.depth.measured_occlusion_radius = 0.001   # |diameter| < 5 px
    if kind == "nan_pose":
        wl.start_body2world = wl.start_body2world.copy()
        wl.start_body2world[1, 0, 3] = np.nan
    else:  # the depth camera turned half round about its y axis: every region line lies behind it
        wl.depth_world2camera = synth.pose_mul(synth.rotation_pose((0.0, 1.0, 0.0), 180.0), wl.depth_world2camera)
        wl.depth = None
        wl.depth_model = None
    return wl


@pytest.mark.parametrize("kind", ["nan_pose", "behind_depth_camera"])
def test_stride0_scans_reached_from_a_workload(oracle, synth, kind):
    """The parent's guards let a NaN line, or a region line behind the depth camera, reach a scan of stride 0; the new
    guards drop the NaN items before any check and scan nothing for the lines behind the depth camera."""
    wl = nan_and_behind_workload(synth, kind)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    base = oracle.OracleTracker(checks_off(wl), rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    b = 1 if kind == "nan_pose" else 0
    poses = orc.get_poses()
    n, view = base.region_correspondences(b, 0, 0)
    geometric = np.ones(n, bool)   # every line offered to the checks
    st = ref.new_stats()
    ref.region_valid(wl, b, poses[b], view, n, geometric, 0, 0, 0, st, parent_rule=True)
    assert st["stride0_scans"] > 0
    st = ref.new_stats()
    pred = ref.region_valid(wl, b, poses[b], view, n, base.lines[b]["valid"], 0, 0, 0, st)
    assert st["stride0_scans"] == 0
    n1, _ = orc.region_correspondences(b, 0, 0)
    assert np.array_equal(pred, orc.lines[b]["valid"][:n1] != 0)
    if kind == "nan_pose":
        assert not pred.any()
    else:   # nothing is measured as occluded: the lines are those of the run without checks
        assert pred.sum() > 0 and np.array_equal(pred, base.lines[b]["valid"][:n] != 0)


def test_region_offset_id_30_is_refused():
    """max_radius / stride in [29.5, 30) passes the reference's radius test, and a radius near the maximum rounds to
    id 30, one past the 30-entry table."""
    class M:
        stride_depth_offset, max_radius_depth_offset = 0.001, 0.0297
    assert int(f32(M.max_radius_depth_offset) / f32(M.stride_depth_offset) + f32(1)) == 30   # accepted table size
    assert ref.region_offset_id(0.0297, M, parent_rule=True) == 30
    st = ref.new_stats()
    assert ref.region_offset_id(0.0297, M, st) is None and st["refused_ids"] == 1
    assert ref.region_offset_id(0.0294, M) == 29


def test_texture_scan_behind_the_depth_camera():
    """The texture modality's scans: a point in front of the colour camera but behind an independently placed depth
    camera gives a measured diameter in (-5, 0) px, whose stride the reference computes as 0; a non-finite pose gives a
    NaN modeled diameter. Both windows scan nothing and count as unoccluded, even on frames full of occluders."""
    import texture_reference as tr
    intr = dict(fu=600.0, fv=600.0, ppu=320.0, ppv=240.0, width=640, height=480)
    b2d = np.array([-1, 0, 0, 0, 0, 1, 0, 0, 0, 0, -1, -0.5], f32)   # the point 0.5 m behind the depth camera
    X = np.array([0.0, 0.0, 0.0], f32)
    z = tr.apply(b2d, X)[2]
    diameter = f32(2) * f32(0.001) * (f32(intr["fu"]) / z)
    assert -5 < diameter < 0 and int(diameter / f32(5) + f32(1)) == 0   # the stride the scan would step by
    m = dict(image=np.full((480, 640), 100, np.uint16), intr=intr, depth_scale=0.001, b2d=b2d, radius=0.001,
             threshold=0.03)
    assert tr.unoccluded_measured(X, m)
    rendering = dict(depth=np.ones((64, 64), np.uint16), corner_u=0.0, corner_v=0.0, scale=1.0,
                     projection_term_a=1.0, projection_term_b=2.0)
    b2c = np.full(12, np.nan, f32)
    assert tr.unoccluded_modeled(X, dict(rendering=rendering, intr=intr, b2c=b2c, radius=0.01, threshold=0.03))
