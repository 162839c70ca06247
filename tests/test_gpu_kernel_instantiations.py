"""GPU parity along the instantiation axis: every compiled k_track2<T, LUT_SMEM> and k_track<T, K, LUT_SMEM, OCC> runs
in at least one case here, and every case asserts the exact variant it runs (m3tb_debug_last_launch: kernel,
threads, items per thread, LUT in shared memory, occlusion variant), so that a routing change cannot make a case
vacuous. COVERAGE maps each variant to its cases; test_kernel_instantiation_inventory.py holds it equal to what the
sources instantiate, so an instantiation without a case (or a row for one that does not exist) fails on any machine.

LaunchTrack picks the variant from max(n_lines_max, n_points_max) (<= 256: 256 threads x 1 item, <= 512: 512 x 1,
<= 1024: 512 x 2, <= 2048: 512 x 4; k_track2 takes <= 512 items), whether every region body has <= 16 histogram bins
(LUT in shared memory), whether any body measures occlusions or reads renderer images (OCC) and whether a body
carries both modalities (k_track2 at 1024 threads).

Bars as in test_gpu_edges / test_gpu_parameter_space (helpers.per_iteration_parity): closest views and per-line /
per-point records bit-exact against the mirror oracle, g within 1e-4 and H within 1e-5 of max|H|, poses within 1e-5 of
the mirror oracle (5e-5 at 4 items per thread: 4096 summands, as in test_gpu_bench_shape.test_many_items_per_thread)
and within 1e-4 of the reference-faithful oracle after every correspondence iteration; StartModalities /
CalculateResults histograms bit-exact wherever a region modality exists.
"""
import dataclasses

import numpy as np
import pytest

from helpers import (TOL, assert_lines_bit_equal, assert_points_bit_equal, per_iteration_parity, pose_error, record,
                     rel_to_max)

pytestmark = pytest.mark.gpu

_ENV = ("M3TB_TMA", "M3TB_TMA_MAXW", "M3TB_NO_TILES", "M3TB_NO_ROI_INGEST", "M3TB_KERNEL")

# ---- the cases ----------------------------------------------------------------------------------------------------------
# A. k_track2 with two-modality bodies: bins -> (bins, upload, environment)
TWO_MODALITIES = {"16_full": (16, "full", {}), "32_full": (32, "full", {}), "32_tma0": (32, "full", {"M3TB_TMA": "0"}),
                  "32_pinned": (32, "pinned", {})}
# B. k_track2 at 512 threads: region-only and depth-only bodies in one batch
ONE_MODALITY_BINS = (16, 32)
# C. k_track without occlusion handling: id -> (items per modality, bins, M3TB_KERNEL=1, bodies)
K_TRACK = {"200_16_kernel1": (200, 16, True, 4), "300_16_kernel1": (300, 16, True, 4), "1024_16": (1024, 16, False, 3),
           "2048_16": (2048, 16, False, 3), "200_64": (200, 64, False, 4), "300_64": (300, 64, False, 4),
           "300_32_kernel1": (300, 32, True, 4), "600_32": (600, 32, False, 3), "1500_32": (1500, 32, False, 3)}
# D. k_track with measured occlusions: n_lines = n_points, bins
OCCLUSION = [(n, bins) for n in (200, 300, 600, 1500) for bins in (16, 32)]

CASES = ([f"test_track2_two_modalities[{k}]" for k in TWO_MODALITIES] + ["test_track2_two_modalities_border_32_bins"] +
         [f"test_track2_one_modality_per_body[{b}]" for b in ONE_MODALITY_BINS] +
         [f"test_k_track[{k}]" for k in K_TRACK] +
         [f"test_k_track_measured_occlusion[{n}_{b}]" for n, b in OCCLUSION] +
         ["test_k_track_occlusion_fallback_600", "test_k_track_renderer_checks_600"])

# (kernel, threads, items_per_thread, lut_smem, occ) as m3tb_debug_last_launch reports it -> the cases that launch it.
COVERAGE = {
    ("k_track2", 1024, 1, 1, 0): ["test_track2_two_modalities[16_full]"],
    ("k_track2", 1024, 1, 0, 0): ["test_track2_two_modalities[32_full]", "test_track2_two_modalities[32_tma0]",
                                  "test_track2_two_modalities[32_pinned]", "test_track2_two_modalities_border_32_bins"],
    ("k_track2", 512, 1, 1, 0): ["test_track2_one_modality_per_body[16]"],
    ("k_track2", 512, 1, 0, 0): ["test_track2_one_modality_per_body[32]"],
    ("k_track", 256, 1, 1, 0): ["test_k_track[200_16_kernel1]"],
    ("k_track", 512, 1, 1, 0): ["test_k_track[300_16_kernel1]"],
    ("k_track", 512, 2, 1, 0): ["test_k_track[1024_16]"],
    ("k_track", 512, 4, 1, 0): ["test_k_track[2048_16]"],
    ("k_track", 256, 1, 0, 0): ["test_k_track[200_64]"],
    ("k_track", 512, 1, 0, 0): ["test_k_track[300_64]", "test_k_track[300_32_kernel1]"],
    ("k_track", 512, 2, 0, 0): ["test_k_track[600_32]"],
    ("k_track", 512, 4, 0, 0): ["test_k_track[1500_32]"],
    ("k_track", 256, 1, 1, 1): ["test_k_track_measured_occlusion[200_16]"],
    ("k_track", 512, 1, 1, 1): ["test_k_track_measured_occlusion[300_16]"],
    ("k_track", 512, 2, 1, 1): ["test_k_track_measured_occlusion[600_16]", "test_k_track_renderer_checks_600"],
    ("k_track", 512, 4, 1, 1): ["test_k_track_measured_occlusion[1500_16]"],
    ("k_track", 256, 1, 0, 1): ["test_k_track_measured_occlusion[200_32]"],
    ("k_track", 512, 1, 0, 1): ["test_k_track_measured_occlusion[300_32]"],
    ("k_track", 512, 2, 0, 1): ["test_k_track_measured_occlusion[600_32]", "test_k_track_occlusion_fallback_600"],
    ("k_track", 512, 4, 0, 1): ["test_k_track_measured_occlusion[1500_32]"],
}
_FIELDS = ("kernel", "threads", "items_per_thread", "lut_smem", "occ")


def _expected(case):
    """The COVERAGE row that lists `case` (the pytest node name)."""
    rows = [v for v, cases in COVERAGE.items() if case in cases]
    assert len(rows) == 1, (case, rows)
    return rows[0]


def _check_launch(case, launch):
    """The launch of `case` is its COVERAGE row; recorded either way."""
    got = tuple(launch[k] for k in _FIELDS)
    record(f"variant {case}", variant=list(got), launch=launch)
    assert got == _expected(case), (case, launch)


# ---- fixtures / shared steps --------------------------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _default_staging(monkeypatch):
    """Every case starts from the default staging; the ones that need a switch set it themselves."""
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)


@pytest.fixture
def case(request):
    return request.node.name


def _context(capi, wl, upload):
    from test_gpu_edges import _context as edges_context   # full copy, or packed pinned frames with ROI ingest
    return edges_context(capi, wl, upload)


def _histograms_exact(capi, oracle, wl, name, upload="full"):
    """StartModalities and CalculateResults histograms bit-exact against the mirror oracle."""
    nb = wl.region.n_histogram_bins
    ctx, pin = _context(capi, wl, upload)
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
    ctx.close()
    del pin


def _parity(capi, oracle, wl, case, upload="full", **floors):
    """helpers.per_iteration_parity with the launch of the case's COVERAGE row, then the histograms."""
    expect = _expected(case)
    ctx, pin = _context(capi, wl, upload)
    rec = per_iteration_parity(capi, oracle, wl, case, ctx=ctx, mirror_tol=5e-5 if expect[2] == 4 else 1e-5,
                               expect_launch=dict(zip(_FIELDS, expect)), **floors)
    del pin
    _check_launch(case, rec["launch"])
    if wl.region:
        _histograms_exact(capi, oracle, wl, case, upload)
    return rec


def _with_bins(wl, bins):
    return dataclasses.replace(wl, region=dataclasses.replace(wl.region, n_histogram_bins=bins))


# ---- A. k_track2<1024, *>: two-modality bodies ----------------------------------------------------------------------
@pytest.mark.parametrize("which", list(TWO_MODALITIES))
def test_track2_two_modalities(capi, oracle, synth, monkeypatch, case, which):
    """c2, 4 bodies, region + depth. At 32 bins the LUT of k_track2's 1024-thread warp roles sits in global memory;
    default (TMA) staging, legacy staging (the kernel bins the colour tile itself) and packed-pitch pinned uploads."""
    bins, upload, env = TWO_MODALITIES[which]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    wl = _with_bins(synth.make_workload("c2", n_bodies=4, n_divides=2, seed=3), bins)
    rec = _parity(capi, oracle, wl, case, upload)
    # the staging switch took effect: ROI tiles, staged by TMA unless M3TB_TMA=0
    assert (rec["launch"]["tiles"], rec["launch"]["tma_mode"]) == (1, int(env.get("M3TB_TMA", "1"))), rec["launch"]


def test_track2_two_modalities_border_32_bins(capi, oracle, synth, case):
    """Bodies on the borders and corners of the frame (partial tiles, lines leaving the frame) at 32 bins."""
    wl = _with_bins(synth.make_edge_workload("border", "region+depth", n_divides=2, seed=3), 32)
    _parity(capi, oracle, wl, case, min_valid_lines=0.1, min_valid_points=0.5)


# ---- B. k_track2<512, *>: no body carries both modalities ----------------------------------------------------------
@pytest.mark.parametrize("bins", ONE_MODALITY_BINS)
def test_track2_one_modality_per_body(capi, oracle, synth, case, bins):
    """Region-only and depth-only bodies in one batch (bodies 2k / 2k + 1), built like test_gpu_edges._mixed: k_track2
    runs its 512-thread form, the LUT in shared memory at 16 bins and in global memory at 32."""
    wl = synth.make_workload("c2", n_bodies=4, n_divides=2, seed=13, margin_px=60.0, z_range=(0.45, 0.8))
    kinds = [("region", "depth")[b % 2] for b in range(wl.n_bodies)]
    copies = {"region": dataclasses.replace(wl, region=dataclasses.replace(wl.region, n_histogram_bins=bins), depth=None),
              "depth": dataclasses.replace(wl, region=None)}
    nb, nl, npnt = wl.n_bodies, wl.lines_per_body, wl.points_per_body
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
    region_bodies = [b for b in range(nb) if kinds[b] == "region"]

    def histograms_exact(stage):
        for b in region_bodies:
            hf, hb = ctx.get_histograms(b, bins)
            m = mirrors["region"]
            assert np.array_equal(hf.view(np.uint32), m.hist_f[b].view(np.uint32)), (case, stage, b)
            assert np.array_equal(hb.view(np.uint32), m.hist_b[b].view(np.uint32)), (case, stage, b)

    for o in list(mirrors.values()) + list(faithfuls.values()):
        o.start_modalities(0)
    ctx.start_modalities(0)
    histograms_exact("start")
    worst = dict(mirror_m=0.0, mirror_rad=0.0, faithful_m=0.0, faithful_rad=0.0, H=0.0, g=0.0)
    valid_lines = valid_points = mode_splits = 0
    launch = None
    for corr in range(wl.n_corr_iterations):
        start = np.stack([mirrors[kinds[b]].get_poses()[b] for b in range(nb)])
        for k in copies:
            mirrors[k].set_poses(start)
            faithfuls[k].set_poses(start)
        if corr in (0, wl.n_corr_iterations - 1):   # g / H of the fine-grained calls
            ctx.set_poses(start)
            ctx.region_correspondences(0, corr)
            g_r, H_r = ctx.region_gradient_hessian(0, corr, 0)
            ctx.depth_correspondences(0, corr)
            g_d, H_d = ctx.depth_gradient_hessian(0, corr, 0)
            for b in range(nb):
                m = mirrors[kinds[b]]
                if kinds[b] == "region":
                    m.region_correspondences(b, 0, corr)
                    og, oH = m.region_gradient_hessian(b, corr, 0)
                    g, H = g_r[b], H_r[b]
                else:
                    m.depth_correspondences(b, 0, corr)
                    og, oH = m.depth_gradient_hessian(b, corr)
                    g, H = g_d[b], H_d[b]
                worst["H"] = max(worst["H"], rel_to_max(H, oH))
                worst["g"] = max(worst["g"], rel_to_max(g, og))
        ctx.set_poses(start)
        ctx.corr_iteration(0, corr, wl.n_update_iterations)
        launch = launch or ctx.last_launch()
        gpu = ctx.get_poses()
        assert np.isfinite(gpu).all(), (case, corr)
        same_views = np.ones(nb, bool)
        for b in range(nb):
            m, f = mirrors[kinds[b]], faithfuls[kinds[b]]
            if kinds[b] == "region":
                n, view = m.region_correspondences(b, 0, corr)
                same_views[b] &= f.region_correspondences(b, 0, corr)[1] == view
                assert ctx.get_closest_views(b)[0] == view, (case, corr, b)
                lines = ctx.get_region_lines(b, nl)
                assert_lines_bit_equal(lines, m.lines[b][:n])
                valid_lines += int((lines["valid"] != 0).sum())
            else:
                n, view = m.depth_correspondences(b, 0, corr)
                same_views[b] &= f.depth_correspondences(b, 0, corr)[1] == view
                assert ctx.get_closest_views(b)[1] == view, (case, corr, b)
                pts = ctx.get_depth_points(b, npnt)
                assert_points_bit_equal(pts, m.points[b][:n])
                valid_points += int((pts["valid"] != 0).sum())
        for k in copies:
            mirrors[k].tracking_step(0, n_corr=corr + 1, corr_begin=corr)
            faithfuls[k].tracking_step(0, n_corr=corr + 1, corr_begin=corr)
        mp = np.stack([mirrors[kinds[b]].get_poses()[b] for b in range(nb)])
        fp = np.stack([faithfuls[kinds[b]].get_poses()[b] for b in range(nb)])
        dt, dr = pose_error(gpu, mp)
        worst["mirror_m"], worst["mirror_rad"] = max(worst["mirror_m"], dt.max()), max(worst["mirror_rad"], dr.max())
        st, sr = pose_error(mp, fp)
        comparable = same_views & (st < TOL) & (sr < TOL)   # see helpers.per_iteration_parity
        mode_splits += int((~comparable).sum())
        dt, dr = pose_error(gpu, fp)
        if comparable.any():
            worst["faithful_m"] = max(worst["faithful_m"], dt[comparable].max())
            worst["faithful_rad"] = max(worst["faithful_rad"], dr[comparable].max())
    # CalculateResults from the mirror's poses on both sides
    poses = np.stack([mirrors[kinds[b]].get_poses()[b] for b in range(nb)])
    ctx.set_poses(poses)
    mirrors["region"].set_poses(poses)
    mirrors["region"].calculate_results(0)
    ctx.calculate_results(0)
    histograms_exact("results")
    ctx.close()
    record(case, bodies=nb, valid_lines=valid_lines, valid_points=valid_points, oracle_mode_splits=mode_splits,
           launch=launch, **{k: float(f"{v:.3e}") for k, v in worst.items()})
    _check_launch(case, launch)
    n_iter = wl.n_corr_iterations * (nb // 2)
    assert valid_lines > 0.3 * nl * n_iter and valid_points > 0.3 * npnt * n_iter, (valid_lines, valid_points)
    assert mode_splits <= max(1, 0.05 * nb * wl.n_corr_iterations), mode_splits
    assert worst["H"] < 1e-5 and worst["g"] < 1e-4, worst
    assert worst["mirror_m"] < 1e-5 and worst["mirror_rad"] < 1e-5, worst
    assert worst["faithful_m"] < TOL and worst["faithful_rad"] < TOL, worst


# ---- C. k_track without occlusion handling ------------------------------------------------------------------------
@pytest.mark.parametrize("which", list(K_TRACK))
def test_k_track(capi, oracle, synth, monkeypatch, case, which):
    """Region + depth bodies on k_track: above 512 items (2 and 4 per thread; 2048 fills every slot of the 512 x 4
    mapping, 1500 leaves the last item of most threads empty), at 64 bins (no k_track2: 18-bit bin indices), or sent
    there by M3TB_KERNEL=1."""
    n, bins, kernel1, nb = K_TRACK[which]
    if kernel1:
        monkeypatch.setenv("M3TB_KERNEL", "1")
    wl = _with_bins(synth.make_workload("c2", n_bodies=nb, n_lines=n, n_points=n, n_divides=2, seed=31), bins)
    _parity(capi, oracle, wl, case)


# ---- D. k_track with occlusion handling -----------------------------------------------------------------------------
def _occluded(synth, n, bins, n_bodies=4, seed=9, **kw):
    """test_oracle_occlusion.occluded_workload at n lines and n points per body and n_divides 2: synthetic depth offsets
    on both models, an occluder in front of every body (left / top), measured occlusions from the first iteration."""
    wl = synth.make_workload("c2", n_bodies=n_bodies, n_lines=n, n_points=n, n_divides=2, seed=seed)
    synth.fill_depth_offsets(wl.region_model, seed)
    synth.fill_depth_offsets(wl.depth_model, seed)
    for b in range(n_bodies):
        synth.add_occluder(wl, b, side="left" if b % 2 == 0 else "top", seed=seed)
    wl.region = dataclasses.replace(wl.region, n_histogram_bins=bins, measure_occlusions=True, n_unoccluded_iterations=0,
                                    min_n_unoccluded_lines=kw.get("min_n_unoccluded_lines", 0))
    wl.depth = dataclasses.replace(wl.depth, measure_occlusions=True, n_unoccluded_iterations=0,
                                   min_n_unoccluded_points=kw.get("min_n_unoccluded_points", 0))
    return wl


def _started(oracle, wl, hist_from=None):
    """A mirror oracle after StartModalities(0) at the start poses; hist_from: another started oracle whose histograms
    it takes over (so that line validity differs only where the occlusion handling decides it)."""
    o = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    o.start_modalities(0)
    if hist_from is not None:
        o.hist_f[...] = hist_from.hist_f
        o.hist_b[...] = hist_from.hist_b
    return o


def _first_records(o, b):
    """Lines and points of body b in correspondence iteration 0 of iteration 0 (copies)."""
    n, _ = o.region_correspondences(b, 0, 0)
    m, _ = o.depth_correspondences(b, 0, 0)
    return o.lines[b][:n].copy(), o.points[b][:m].copy()


def _without_checks(wl):
    return dataclasses.replace(
        wl, region=dataclasses.replace(wl.region, measure_occlusions=False, model_occlusions=False,
                                       use_region_checking=False, min_n_unoccluded_lines=0),
        depth=dataclasses.replace(wl.depth, measure_occlusions=False, model_occlusions=False,
                                  use_silhouette_checking=False, min_n_unoccluded_points=0))


def _dropped(oracle, wl):
    """(lines, points) that the checks drop in the first correspondence iteration, against the same workload without
    them and with the same histograms; the checks may only drop, never add."""
    occ = _started(oracle, wl)
    plain = _started(oracle, _without_checks(wl), hist_from=occ)
    dl = dp = 0
    for b in range(wl.n_bodies):
        (l1, p1), (l0, p0) = _first_records(occ, b), _first_records(plain, b)
        assert len(l1) == len(l0) and len(p1) == len(p0)
        assert not (l1["valid"].astype(bool) & ~l0["valid"].astype(bool)).any(), b
        assert not (p1["valid"].astype(bool) & ~p0["valid"].astype(bool)).any(), b
        dl += int(l0["valid"].sum() - l1["valid"].sum())
        dp += int(p0["valid"].sum() - p1["valid"].sum())
    return dl, dp


OCC_FLOORS = dict(min_valid_lines=0.2, min_valid_points=0.1)


@pytest.mark.parametrize("n,bins", OCCLUSION, ids=[f"{n}_{b}" for n, b in OCCLUSION])
def test_k_track_measured_occlusion(capi, oracle, synth, case, n, bins):
    """Measured occlusions (the depth-window scans of every region line and depth point) at every thread <-> item
    mapping, with the LUT in shared and in global memory."""
    wl = _occluded(synth, n, bins)
    dl, dp = _dropped(oracle, wl)
    record(f"dropped {case}", lines=dl, points=dp)
    assert dl > 0 and dp > 0, (dl, dp)
    _parity(capi, oracle, wl, case, **OCC_FLOORS)


def test_k_track_occlusion_fallback_600(capi, oracle, synth, case):
    """min_n_unoccluded_lines / points at 75 % of the 600 items: too few survive the occlusion pass, so the kernel
    counts the survivors over all K = 2 items of every thread and recomputes every line / point without occlusion
    handling. The oracle's records of that second pass must equal a run without occlusion handling (same histograms),
    and the GPU's must equal the oracle's."""
    n = 600
    wl = _occluded(synth, n, 32, min_n_unoccluded_lines=3 * n // 4, min_n_unoccluded_points=3 * n // 4)
    fallback = _started(oracle, wl)
    occ_only = _started(oracle, dataclasses.replace(wl, region=dataclasses.replace(wl.region, min_n_unoccluded_lines=0),
                                                    depth=dataclasses.replace(wl.depth, min_n_unoccluded_points=0)),
                        hist_from=fallback)
    plain = _started(oracle, _without_checks(wl), hist_from=fallback)
    fell_back = [0, 0]
    for b in range(wl.n_bodies):
        (lf, pf), (lo, po), (lp, pp) = (_first_records(o, b) for o in (fallback, occ_only, plain))
        if lo["valid"].sum() < wl.region.min_n_unoccluded_lines:
            assert_lines_bit_equal(lf, lp)
            fell_back[0] += 1
        else:
            assert_lines_bit_equal(lf, lo)
        if po["valid"].sum() < wl.depth.min_n_unoccluded_points:
            assert_points_bit_equal(pf, pp)
            fell_back[1] += 1
        else:
            assert_points_bit_equal(pf, po)
    record(f"fallback {case}", bodies_fell_back_lines=fell_back[0], bodies_fell_back_points=fell_back[1])
    assert fell_back[0] > 0 and fell_back[1] > 0, fell_back
    _parity(capi, oracle, wl, case, **OCC_FLOORS)


def test_k_track_renderer_checks_600(capi, oracle, synth, case):
    """Modeled occlusions, region checking and silhouette checking on renderer images (test_gpu_renderings' "all") at
    600 items: 2 per thread in the OCC variant."""
    wl = synth.make_workload("c2", n_bodies=4, n_lines=600, n_points=600, n_divides=2, seed=19)
    synth.fill_depth_offsets(wl.region_model)
    synth.fill_depth_offsets(wl.depth_model)
    synth.add_renderings(wl, occluder_bodies=(1, 3))
    wl.region = dataclasses.replace(wl.region, model_occlusions=True, use_region_checking=True, n_unoccluded_iterations=0)
    wl.depth = dataclasses.replace(wl.depth, model_occlusions=True, use_silhouette_checking=True, n_unoccluded_iterations=0)
    dl, dp = _dropped(oracle, wl)
    record(f"dropped {case}", lines=dl, points=dp)
    assert dl > 0 and dp > 0, (dl, dp)
    # region checking against start-pose renderings keeps few lines: 2081 of 16800 line slots (12 %) on an H100
    _parity(capi, oracle, wl, case, min_valid_lines=0.1, min_valid_points=0.3)
