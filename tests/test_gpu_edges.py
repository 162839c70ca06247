"""GPU parity where the kernels meet the frame's edges, at other frame sizes, in mixed batches and across every staging
path (synth.make_edge_workload places bodies on the borders and corners, straddling the no-tile depth, far away and
out of view; the random workloads of the other tests keep every body well inside a 640x480 frame).

Bars: per-line / per-point records and closest views bit-exact against the GPU-mirror oracle, g / H <= 1e-5 of max|H|,
poses <= 1e-5 against the mirror oracle and <= 1e-4 against the reference-faithful one after every correspondence
iteration (helpers.per_iteration_parity); histograms of StartModalities and CalculateResults bit-exact. Staging switches
(tile modes, tile width cap, no tiles, full / pinned-ROI / pinned-whole uploads) must not change a single bit; k_track
vs k_track2 only sums in another order, so there each kernel is held to the oracle instead. Every test asserts the
kernel variant it means to exercise (m3tb_debug_last_launch).
"""
import dataclasses

import numpy as np
import pytest

from helpers import TOL, assert_lines_bit_equal, assert_points_bit_equal, per_iteration_parity, pose_error, record

pytestmark = pytest.mark.gpu

# per kind: least fraction of line / point slots (over all bodies and iterations) that must be valid. The depth camera
# sees a wider field than the colour camera, so depth_border bodies lie outside the colour frame: their lines are all
# invalid (an out-of-view case for the region modality), their points straddle the depth frame's border.
FLOORS = {"border": (0.1, 0.5), "depth_border": (0.0, 0.2), "near": (0.5, 0.5), "far": (0.2, 0.5), "out": (0.0, 0.0)}
# the kernel variant each modality set must run (k_track2: 1024 threads with both modalities, else 512)
LAUNCH = {"region+depth": dict(kernel="k_track2", threads=1024, lut_smem=1),
          "region16": dict(kernel="k_track2", threads=512, lut_smem=1),
          "region32": dict(kernel="k_track2", threads=512, lut_smem=0),
          "depth": dict(kernel="k_track2", threads=512)}


def _sizes(synth):
    """(name, colour intrinsics, depth intrinsics, kernel the default staging runs)."""
    I = synth.Intrinsics
    return [
        ("1280x720_848x480", I(912.0, 912.5, 640.3, 359.6, 1280, 720), I(424.6, 424.9, 425.2, 241.1, 848, 480), "k_track2"),
        # width a multiple of 4 (bin-index image) but not of 16: the pooled pitch is padded, packed pinned rows are not
        ("644x480_640x480", I(614.0, 614.5, 322.8, 238.9, 644, 480), synth.default_depth_intrinsics(), "k_track2"),
        # width not a multiple of 4: no bin-index image, TMA staging unusable -> k_track
        ("642x481_637x479", I(614.0, 614.5, 320.6, 240.3, 642, 481), I(385.7, 385.9, 318.4, 239.2, 637, 479), "k_track"),
        ("320x240_320x240", I(307.0, 307.3, 160.4, 119.7, 320, 240), I(192.9, 193.0, 161.1, 120.8, 320, 240), "k_track2"),
    ]


def _pinned(wl):
    """Pinned host copies of the frames with TIGHTLY packed rows (pitch 3 W / 2 W: not 16-byte aligned in general)."""
    import torch
    W, H = wl.color_intrinsics.width, wl.color_intrinsics.height
    out = {}
    if wl.region:
        out["color"] = torch.from_numpy(np.ascontiguousarray(wl.color_frames[:, :, :3 * W])).pin_memory()
        assert out["color"].stride(1) == 3 * W
    if wl.depth:
        d = np.ascontiguousarray(wl.depth_frames).view(np.uint8).reshape(wl.n_bodies, wl.depth_intrinsics.height, -1)
        out["depth"] = torch.from_numpy(d).pin_memory()
    return out


def _context(capi, wl, upload):
    """upload: "full" (pageable copy of the padded frames) or "pinned" (packed pinned frames, ROI ingest)."""
    if upload == "full":
        return capi.context_from_workload(wl), None
    ctx = capi.context_from_workload(wl, upload_frames=False)
    pin = _pinned(wl)
    if "color" in pin:
        ctx.upload_batch_ptr(True, 0, wl.n_bodies, pin["color"].data_ptr(), pin["color"].stride(0), pin["color"].stride(1))
    if "depth" in pin:
        ctx.upload_batch_ptr(False, 0, wl.n_bodies, pin["depth"].data_ptr(), pin["depth"].stride(0), pin["depth"].stride(1))
    return ctx, pin  # the caller keeps `pin` alive while the context reads it


def _histograms_exact(capi, oracle, wl, name, uniform=False):
    """StartModalities and CalculateResults histograms bit-exact against the oracle (uniform: the oracle's fallback for
    a body without a single valid line pixel, 1 / n_bins^3 everywhere)."""
    nb = wl.region.n_histogram_bins
    ctx = capi.context_from_workload(wl)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    for stage in ("start", "results"):
        if stage == "start":
            orc.start_modalities(0)
            ctx.start_modalities(0)
        else:
            orc.calculate_results(0)
            ctx.calculate_results(0)
        for b in range(wl.n_bodies):
            hf, hb = ctx.get_histograms(b, nb)
            assert np.array_equal(hf.view(np.uint32), orc.hist_f[b].view(np.uint32)), (name, stage, b)
            assert np.array_equal(hb.view(np.uint32), orc.hist_b[b].view(np.uint32)), (name, stage, b)
            if uniform:
                u = np.float32(1.0) / np.float32(nb ** 3)
                assert (hf == u).all() and (hb == u).all(), (name, stage, b)
    ctx.close()


@pytest.mark.parametrize("modalities", ["region+depth", "region16", "region32", "depth"])
@pytest.mark.parametrize("kind", ["border", "depth_border", "near", "far", "out"])
def test_edge_parity(capi, oracle, synth, kind, modalities):
    wl = synth.make_edge_workload(kind, modalities, n_divides=2, seed=3)
    fl, fp = FLOORS[kind]
    rec = per_iteration_parity(capi, oracle, wl, f"edge_{kind}_{modalities}", min_valid_lines=fl, min_valid_points=fp,
                               expect_launch=LAUNCH[modalities])
    if kind == "out":
        assert rec["valid_lines"] == 0 and rec["valid_points"] == 0, rec
    if wl.region:
        _histograms_exact(capi, oracle, wl, f"edge_{kind}_{modalities}", uniform=kind == "out")


@pytest.mark.parametrize("upload", ["full", "pinned"])
@pytest.mark.parametrize("size", range(4))
def test_frame_sizes(capi, oracle, synth, size, upload):
    """Other frame sizes, bodies on the borders and corners, full and pinned (packed-pitch) uploads."""
    name, ci, di, kernel = _sizes(synth)[size]
    wl = synth.make_edge_workload("border", "region+depth", n_divides=2, seed=5, color_intrinsics=ci, depth_intrinsics=di)
    ctx, pin = _context(capi, wl, upload)
    per_iteration_parity(capi, oracle, wl, f"frame_{name}_{upload}", min_valid_lines=0.1, min_valid_points=0.5,
                         ctx=ctx, expect_launch=dict(kernel=kernel, threads=1024 if kernel == "k_track2" else 256))
    del pin
    _histograms_exact(capi, oracle, wl, f"frame_{name}")


@pytest.mark.parametrize("which", ["border", "642x481", "near"])
def test_k_track_fallback_parity(capi, oracle, synth, monkeypatch, which):
    """M3TB_KERNEL=1 sends the same batches to k_track: its records are bit-exact against the oracle as well and its
    poses meet the same bars (its sums are ordered differently from k_track2's, so the two are not compared bit for bit)."""
    monkeypatch.setenv("M3TB_KERNEL", "1")
    if which == "642x481":
        _, ci, di, _ = _sizes(synth)[2]
        wl = synth.make_edge_workload("border", "region+depth", n_divides=2, seed=5, color_intrinsics=ci, depth_intrinsics=di)
        floors = (0.1, 0.5)
    else:
        wl = synth.make_edge_workload(which, "region+depth", n_divides=2, seed=3)
        floors = FLOORS[which]
    per_iteration_parity(capi, oracle, wl, f"k_track_{which}", min_valid_lines=floors[0], min_valid_points=floors[1],
                         expect_launch=dict(kernel="k_track", threads=256, items_per_thread=1))


@pytest.mark.parametrize("upload", ["full", "pinned"])
def test_legacy_staging_without_bin_image_parity(capi, oracle, synth, monkeypatch, upload):
    """642 px wide frames have no bin-index image; with legacy staging (M3TB_TMA=0) k_track2 still takes the batch and
    bins the colour tile from the BGR frame itself. Held to the oracle like every other path."""
    monkeypatch.setenv("M3TB_TMA", "0")
    _, ci, di, _ = _sizes(synth)[2]
    wl = synth.make_edge_workload("border", "region+depth", n_divides=2, seed=5, color_intrinsics=ci, depth_intrinsics=di)
    ctx, pin = _context(capi, wl, upload)
    per_iteration_parity(capi, oracle, wl, f"legacy_staging_642x481_{upload}", min_valid_lines=0.1, min_valid_points=0.5,
                         ctx=ctx, expect_launch=dict(kernel="k_track2", threads=1024, tma_mode=0, tiles=1))
    del pin


# ---- staging equivalence ----------------------------------------------------------------------------------------------
STAGINGS = [  # (name, environment, upload)
    ("tma1_full", {}, "full"),
    ("tma0_full", {"M3TB_TMA": "0"}, "full"),
    ("tma2_full", {"M3TB_TMA": "2"}, "full"),
    ("tma1_maxw64", {"M3TB_TMA_MAXW": "64"}, "full"),
    ("tma1_maxw256", {"M3TB_TMA_MAXW": "256"}, "full"),
    ("no_tiles", {"M3TB_NO_TILES": "1"}, "full"),
    ("tma1_pinned", {}, "pinned"),
    ("tma0_pinned", {"M3TB_TMA": "0"}, "pinned"),
    ("tma2_pinned_maxw64", {"M3TB_TMA": "2", "M3TB_TMA_MAXW": "64"}, "pinned"),
    ("pinned_no_roi_ingest", {"M3TB_NO_ROI_INGEST": "1"}, "pinned"),
]
_ENV = ("M3TB_TMA", "M3TB_TMA_MAXW", "M3TB_NO_TILES", "M3TB_NO_ROI_INGEST", "M3TB_KERNEL")


def _staged_run(capi, wl, monkeypatch, env, upload):
    """StartModalities, a tracking step, CalculateResults and a second step; every output of the path."""
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ctx, pin = _context(capi, wl, upload)
    ctx.start_modalities(0)
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    launch = ctx.last_launch()
    ctx.calculate_results(0)
    ctx.tracking_step(1, wl.n_corr_iterations, wl.n_update_iterations)
    out = dict(poses=ctx.get_poses())
    for b in range(wl.n_bodies):
        if wl.region:
            out[f"lines{b}"] = ctx.get_region_lines(b, wl.lines_per_body)
            hf, hb = ctx.get_histograms(b, wl.region.n_histogram_bins)
            out[f"hist{b}"] = np.concatenate([hf, hb])
        if wl.depth:
            out[f"points{b}"] = ctx.get_depth_points(b, wl.points_per_body)
    ctx.close()
    del pin
    return out, launch


@pytest.mark.parametrize("which", ["border", "border_region8", "border_region32", "border_region64", "642x481",
                                   "1280x720", "644x480"])
def test_staging_paths_are_bit_identical(capi, synth, monkeypatch, which):
    if which == "border":
        wl = synth.make_edge_workload("border", "region+depth", n_divides=2, seed=7)
    elif which.startswith("border_region"):
        wl = synth.make_edge_workload("border", "region16", n_divides=2, seed=7)
        wl.region.n_histogram_bins = int(which[len("border_region"):])
    else:
        _, ci, di, _ = next(s for s in _sizes(synth) if s[0].startswith(which))
        wl = synth.make_edge_workload("border", "region+depth", n_divides=2, seed=7, color_intrinsics=ci,
                                      depth_intrinsics=di)
    base = {}   # per kernel: k_track and k_track2 sum in different orders, bit identity holds within each
    launches = {}
    for name, env, upload in STAGINGS:
        out, launch = _staged_run(capi, wl, monkeypatch, env, upload)
        launches[name] = launch
        # the switch must have taken effect where k_track2 runs
        if launch["kernel"] == "k_track2":
            assert launch["tma_mode"] == int(env.get("M3TB_TMA", "1")), (name, launch)
            assert launch["tiles"] == (0 if env.get("M3TB_NO_TILES") == "1" else 1), (name, launch)
        if launch["kernel"] not in base:
            base[launch["kernel"]] = (name, out)
            continue
        ref_name, ref = base[launch["kernel"]]
        for k, v in ref.items():
            assert np.array_equal(np.ascontiguousarray(out[k]).view(np.uint8), np.ascontiguousarray(v).view(np.uint8)), \
                (which, name, ref_name, k)
    record(f"staging_{which}", bodies=wl.n_bodies, configs=len(STAGINGS), launches=launches)
    # 642 wide: no bin-index image, so the TMA modes fall back to k_track; legacy staging (mode 0) needs none
    if which == "642x481":
        assert launches["tma1_full"]["kernel"] == "k_track" and launches["tma0_full"]["kernel"] == "k_track2", launches
    elif which == "border_region64":
        # 64-bin indices do not fit the u16 colour tile of either kernel: k_track without tiles on every staging path
        assert all(l["kernel"] == "k_track" and l["tiles"] == 0 for l in launches.values()), launches
    else:
        assert all(l["kernel"] == "k_track2" for l in launches.values()), launches


# ---- mixed batches ----------------------------------------------------------------------------------------------------
def _mixed(synth, variant):
    """Bodies 3k: region only, 3k+1: depth only, 3k+2: both, all in one context. variant "one_set": one region
    parameter set; "two_sets": the region-only bodies use another function amplitude (another function lookup);
    "bins": the region-only bodies use 32 histogram bins, the two-modality bodies 16; "bins8": the region-only bodies
    use 8 bins, so both table sizes sit in shared memory."""
    wl = synth.make_workload("c2", n_bodies=9, n_divides=2, seed=13, margin_px=60.0, z_range=(0.45, 0.8))
    region_only = dataclasses.replace(wl.region)
    if variant == "two_sets":
        region_only.function_amplitude = 0.36
    elif variant == "bins":
        region_only.n_histogram_bins = 32
    elif variant == "bins8":
        region_only.n_histogram_bins = 8
    kinds = [("region", "depth", "both")[b % 3] for b in range(wl.n_bodies)]
    copies = {"region": dataclasses.replace(wl, region=region_only, depth=None),
              "depth": dataclasses.replace(wl, region=None),
              "both": wl}
    return wl, kinds, copies


@pytest.mark.parametrize("variant,kernel", [("one_set", "k_track2"), ("two_sets", "k_track"), ("bins", "k_track"),
                                            ("bins8", "k_track")])
def test_mixed_batch(capi, oracle, synth, variant, kernel):
    wl, kinds, copies = _mixed(synth, variant)
    nb = wl.n_bodies
    ctx = capi.Context(0, max_bodies=nb, max_cameras=nb, max_models=1)
    ctx.set_region_model(0, wl.region_model)
    ctx.set_depth_model(0, wl.depth_model)
    for b in range(nb):
        ctx.set_color_camera(b, wl.color_intrinsics, wl.color_world2camera)
        ctx.set_depth_camera(b, wl.depth_intrinsics, wl.depth_world2camera, wl.depth_scale)
    ctx.upload_color_batch(0, wl.color_frames)
    ctx.upload_depth_batch(0, wl.depth_frames)
    op = capi.OptimizerParams(wl.tikhonov_rotation, wl.tikhonov_translation)
    for b in range(nb):
        c = copies[kinds[b]]
        ctx.set_body(b, capi.region_params(c.region) if c.region else None,
                     capi.depth_params(c.depth) if c.depth else None, op, 0, 0, b, b)
    ctx.set_poses(wl.start_body2world)
    mirrors = {k: oracle.OracleTracker(c, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
               for k, c in copies.items()}
    faithfuls = {k: oracle.OracleTracker(c, rotation_mode=oracle.ROTATION_POLAR, exp_mode=oracle.EXP_PADE)
                 for k, c in copies.items()}
    for o in list(mirrors.values()) + list(faithfuls.values()):
        o.start_modalities(0)
    ctx.start_modalities(0)
    for b in range(nb):
        c = copies[kinds[b]]
        if c.region:
            hf, hb = ctx.get_histograms(b, c.region.n_histogram_bins)
            m = mirrors[kinds[b]]
            assert np.array_equal(hf.view(np.uint32), m.hist_f[b].view(np.uint32)), (variant, b)
            assert np.array_equal(hb.view(np.uint32), m.hist_b[b].view(np.uint32)), (variant, b)
    worst = dict(mirror_m=0.0, mirror_rad=0.0, faithful_m=0.0, faithful_rad=0.0)
    valid_lines = valid_points = mode_splits = 0
    launch = None
    for corr in range(wl.n_corr_iterations):
        start = np.stack([mirrors[kinds[b]].get_poses()[b] for b in range(nb)])
        for k in copies:
            mirrors[k].set_poses(start)
            faithfuls[k].set_poses(start)
        ctx.set_poses(start)
        ctx.corr_iteration(0, corr, wl.n_update_iterations)
        launch = launch or ctx.last_launch()
        gpu = ctx.get_poses()
        same_views = np.ones(nb, bool)
        for b in range(nb):
            c, m, f = copies[kinds[b]], mirrors[kinds[b]], faithfuls[kinds[b]]
            if c.region:
                n, view = m.region_correspondences(b, 0, corr)
                same_views[b] &= f.region_correspondences(b, 0, corr)[1] == view
                assert ctx.get_closest_views(b)[0] == view, (variant, corr, b)
                lines = ctx.get_region_lines(b, wl.lines_per_body)
                assert_lines_bit_equal(lines, m.lines[b][:n])
                valid_lines += int((lines["valid"] != 0).sum())
            if c.depth:
                n, view = m.depth_correspondences(b, 0, corr)
                same_views[b] &= f.depth_correspondences(b, 0, corr)[1] == view
                assert ctx.get_closest_views(b)[1] == view, (variant, corr, b)
                pts = ctx.get_depth_points(b, wl.points_per_body)
                assert_points_bit_equal(pts, m.points[b][:n])
                valid_points += int((pts["valid"] != 0).sum())
        for k in copies:
            mirrors[k].tracking_step(0, n_corr=corr + 1, corr_begin=corr)
            faithfuls[k].tracking_step(0, n_corr=corr + 1, corr_begin=corr)
        mp = np.stack([mirrors[kinds[b]].get_poses()[b] for b in range(nb)])
        fpz = np.stack([faithfuls[kinds[b]].get_poses()[b] for b in range(nb)])
        dt, dr = pose_error(gpu, mp)
        worst["mirror_m"], worst["mirror_rad"] = max(worst["mirror_m"], dt.max()), max(worst["mirror_rad"], dr.max())
        st, sr = pose_error(mp, fpz)
        comparable = same_views & (st < TOL) & (sr < TOL)   # see helpers.per_iteration_parity
        mode_splits += int((~comparable).sum())
        dt, dr = pose_error(gpu, fpz)
        if comparable.any():
            worst["faithful_m"] = max(worst["faithful_m"], dt[comparable].max())
            worst["faithful_rad"] = max(worst["faithful_rad"], dr[comparable].max())
    ctx.close()
    record(f"mixed_{variant}", bodies=nb, valid_lines=valid_lines, valid_points=valid_points,
           oracle_mode_splits=mode_splits, launch=launch, **{k: float(f"{v:.3e}") for k, v in worst.items()})
    assert launch["kernel"] == kernel, launch
    if kernel == "k_track2":
        assert launch["threads"] == 1024, launch
    if variant == "bins8":
        assert launch["lut_smem"] == 1, launch
    assert valid_lines > 0.3 * wl.lines_per_body * (2 * nb // 3) * wl.n_corr_iterations, valid_lines
    assert valid_points > 0.3 * wl.points_per_body * (2 * nb // 3) * wl.n_corr_iterations, valid_points
    assert mode_splits <= max(1, 0.05 * nb * wl.n_corr_iterations), mode_splits
    assert worst["mirror_m"] < 1e-5 and worst["mirror_rad"] < 1e-5, worst
    assert worst["faithful_m"] < TOL and worst["faithful_rad"] < TOL, worst
