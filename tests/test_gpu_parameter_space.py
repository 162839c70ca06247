"""GPU parity across the parameter space m3tb_set_body accepts, beyond the defaults the other tests run: every histogram
resolution (it decides whether the LUT sits in shared memory, whether there is a colour tile and which kernel runs),
resolution changes on a live context, the update schedule (n_update_iterations x n_global_iterations), long scale
schedules, line lengths, learning rates and the depth modality's stride and distance schedules.

Bars as in test_gpu_edges: helpers.per_iteration_parity (closest views and per-line / per-point records bit-exact
against the mirror oracle, g / H within 1e-5, poses within 1e-5 of the mirror oracle and 1e-4 of the reference-faithful
one, valid-line / valid-point floors); StartModalities / CalculateResults histograms bit-exact wherever a region modality
exists; and the kernel variant each case means to run (m3tb_debug_last_launch), so that a routing change cannot make a
case vacuous.
"""
import dataclasses

import numpy as np
import pytest

from helpers import per_iteration_parity, record

pytestmark = pytest.mark.gpu

_ENV = ("M3TB_TMA", "M3TB_TMA_MAXW", "M3TB_NO_TILES", "M3TB_NO_ROI_INGEST", "M3TB_KERNEL")


@pytest.fixture(autouse=True)
def _default_staging(monkeypatch):
    """Every case starts from the default staging; the ones that need a switch set it themselves."""
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)


@pytest.fixture(scope="module")
def base(synth):
    """c2, 4 bodies, n_divides 2, seed 3: 200 lines + 200 points, 16 bins, 2 updates, 1 global iteration."""
    return synth.make_workload("c2", n_bodies=4, n_divides=2, seed=3)


def _variant(base, modalities="region+depth", region=None, depth=None, **fields):
    """A copy of `base` with other region / depth settings (base itself is never modified). modalities: "region+depth"
    or "region" (the depth frames stay, but no depth camera is set up)."""
    r = dataclasses.replace(base.region, **(region or {}))
    d = dataclasses.replace(base.depth, **(depth or {})) if modalities == "region+depth" else None
    return dataclasses.replace(base, region=r, depth=d, **fields)


def _pinned(wl):
    """Pinned host copies of the frames (the padded colour pitch of the workload, packed depth rows)."""
    import torch
    out = {"color": torch.from_numpy(wl.color_frames).pin_memory()}
    if wl.depth:
        d = np.ascontiguousarray(wl.depth_frames).view(np.uint8).reshape(wl.n_bodies, wl.depth_intrinsics.height, -1)
        out["depth"] = torch.from_numpy(d).pin_memory()
    return out


def _context(capi, wl, upload="full"):
    """upload: "full" (pageable copy), "pinned" (ROI ingest at the first consumer launch) or "prefetch" (pinned, ingested
    by m3tb_prefetch_frames into the alternate buffers). Returns (context, pinned frames the caller keeps alive)."""
    if upload == "full":
        return capi.context_from_workload(wl), None
    ctx = capi.context_from_workload(wl, upload_frames=False)
    pin = _pinned(wl)
    for key, color in (("color", True), ("depth", False)):
        if key in pin:
            t = pin[key]
            ctx.upload_batch_ptr(color, 0, wl.n_bodies, t.data_ptr(), t.stride(0), t.stride(1))
    if upload == "prefetch":
        ctx.prefetch_frames()
    return ctx, pin


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


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


def _parity(capi, oracle, wl, name, expect_launch, upload="full", **floors):
    ctx, pin = _context(capi, wl, upload)
    rec = per_iteration_parity(capi, oracle, wl, name, ctx=ctx, expect_launch=expect_launch, **floors)
    del pin
    _histograms_exact(capi, oracle, wl, name, upload)
    return rec


def _default_launch(wl):
    """The variant the default staging runs for a rigid batch of one resolution (DESIGN §2-3, INTEGRATION §5):
    the LUT sits in shared memory up to 16 bins; k_track2 takes <= 32 bins (1024 threads with both modalities, else 512)
    and stages tiles; 64-bin indices do not fit the u16 colour tile, so k_track runs without tiles."""
    bins = wl.region.n_histogram_bins
    if bins > 32:
        return dict(kernel="k_track", threads=256, items_per_thread=1, lut_smem=0, tiles=0)
    return dict(kernel="k_track2", threads=1024 if wl.depth else 512, lut_smem=int(bins <= 16), tiles=1, tma_mode=1)


# ---- A. histogram resolutions ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("modalities", ["region+depth", "region"])
@pytest.mark.parametrize("bins", [2, 4, 8, 64])
def test_histogram_resolution(capi, oracle, base, bins, modalities):
    wl = _variant(base, modalities, region=dict(n_histogram_bins=bins))
    _parity(capi, oracle, wl, f"bins{bins}_{modalities}", _default_launch(wl))


@pytest.mark.parametrize("upload", ["full", "pinned"])
@pytest.mark.parametrize("bins", [8, 64])
def test_histogram_resolution_legacy_staging(capi, oracle, base, monkeypatch, bins, upload):
    """M3TB_TMA=0 bins the colour tile inside k_track2. Its cells are 16 bits wide, so a 64-bin batch (18-bit indices)
    must go to k_track like under the TMA modes."""
    monkeypatch.setenv("M3TB_TMA", "0")
    wl = _variant(base, region=dict(n_histogram_bins=bins))
    launch = (dict(kernel="k_track2", threads=1024, lut_smem=1, tiles=1, tma_mode=0) if bins <= 32
              else dict(kernel="k_track", threads=256, lut_smem=0, tiles=0))
    _parity(capi, oracle, wl, f"bins{bins}_legacy_{upload}", launch, upload)


# ---- B. resolution change on a live context ----------------------------------------------------------------------------
def _step_outputs(ctx, wl, iteration):
    """start_modalities, histograms, a tracking step, poses / lines / points, calculate_results, histograms."""
    out = {}
    nb = wl.region.n_histogram_bins
    ctx.start_modalities(iteration)
    for b in range(wl.n_bodies):
        out[f"hist_start{b}"] = np.concatenate(ctx.get_histograms(b, nb))
    ctx.tracking_step(iteration, wl.n_corr_iterations, wl.n_update_iterations)
    launch = ctx.last_launch()
    out["poses"] = ctx.get_poses()
    for b in range(wl.n_bodies):
        out[f"lines{b}"] = ctx.get_region_lines(b, wl.lines_per_body)
        out[f"points{b}"] = ctx.get_depth_points(b, wl.points_per_body)
    ctx.calculate_results(iteration)
    for b in range(wl.n_bodies):
        out[f"hist_results{b}"] = np.concatenate(ctx.get_histograms(b, nb))
    return out, launch


@pytest.mark.parametrize("upload", ["full", "pinned", "prefetch"])
@pytest.mark.parametrize("first,second", [(16, 32), (32, 8), (64, 16), (16, 64)])
def test_resolution_change_on_live_context(capi, base, first, second, upload):
    """A context tracks a frame at one resolution, then m3tb_set_body switches every body to another and tracking goes
    on with the same frame. Everything must equal a fresh context that had the second resolution from the start: the
    bin-index images of the frame (rebuilt by k_bin for full copies; written by k_ingest for pinned frames, which cannot
    be rebuilt from their partial device copy) must not keep the first resolution's indices."""
    wl1 = _variant(base, region=dict(n_histogram_bins=first))
    wl2 = _variant(base, region=dict(n_histogram_bins=second))
    ctx, pin = _context(capi, wl1, upload)
    ctx.start_modalities(0)
    ctx.tracking_step(0, wl1.n_corr_iterations, wl1.n_update_iterations)
    poses = ctx.get_poses()
    op = capi.OptimizerParams(wl2.tikhonov_rotation, wl2.tikhonov_translation)
    for b in range(wl2.n_bodies):
        ctx.set_body(b, capi.region_params(wl2.region), capi.depth_params(wl2.depth), op, 0, 0, b, b)
    ctx.set_poses(poses)
    changed, launch = _step_outputs(ctx, wl2, 1)
    ctx.close()
    fresh_ctx, fresh_pin = _context(capi, wl2, upload)
    fresh_ctx.set_poses(poses)
    fresh, fresh_launch = _step_outputs(fresh_ctx, wl2, 1)
    fresh_ctx.close()
    del pin, fresh_pin
    record(f"resolution_{first}_to_{second}_{upload}", launch=launch, fresh_launch=fresh_launch)
    # one kernel on both sides (k_track and k_track2 sum in different orders); staging may differ, results may not
    assert launch["kernel"] == fresh_launch["kernel"] == _default_launch(wl2)["kernel"], (launch, fresh_launch)
    if launch["kernel"] == "k_track2":
        # full copies are re-binned and keep the TMA staging; a pinned frame's bins cannot be, so it bins in the kernel
        assert fresh_launch["tma_mode"] == 1 and launch["tma_mode"] == (1 if upload == "full" else 0), launch
    for k, v in fresh.items():
        assert np.array_equal(_bits(changed[k]), _bits(v)), (first, second, upload, k)
    n_valid = sum(int((fresh[f"lines{b}"]["valid"] != 0).sum()) for b in range(wl2.n_bodies))
    assert n_valid > 0.5 * wl2.lines_per_body * wl2.n_bodies, n_valid


# ---- C. update schedule ------------------------------------------------------------------------------------------------
SCHEDULES = [(u, g) for u in (1, 3, 5) for g in sorted({0, 1, 2, u})]


@pytest.mark.parametrize("kernel", ["k_track2", "k_track"])
@pytest.mark.parametrize("n_update,n_global", SCHEDULES)
def test_update_schedule(capi, oracle, base, monkeypatch, n_update, n_global, kernel):
    """n_global_iterations decides per update iteration between the global and the local gradient of the region
    modality; both kernels against the oracle for every split of the update loop."""
    if kernel == "k_track":
        monkeypatch.setenv("M3TB_KERNEL", "1")
    wl = _variant(base, region=dict(n_global_iterations=n_global), n_update_iterations=n_update)
    launch = (dict(kernel="k_track2", threads=1024, lut_smem=1, tiles=1) if kernel == "k_track2"
              else dict(kernel="k_track", threads=256, items_per_thread=1, lut_smem=1))
    _parity(capi, oracle, wl, f"schedule_u{n_update}_g{n_global}_{kernel}", launch)


def test_fused_step_equals_iteration_by_iteration_across_the_global_local_switch(capi, base):
    """3 updates with 2 global iterations switch to the local gradient inside every update loop: one fused
    m3tb_tracking_step == 7 x m3tb_corr_iteration, bit for bit."""
    wl = _variant(base, region=dict(n_global_iterations=2), n_update_iterations=3)
    ctx_a = capi.context_from_workload(wl)
    ctx_b = capi.context_from_workload(wl)
    for c in (ctx_a, ctx_b):
        c.start_modalities(0)
    ctx_a.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    assert ctx_a.last_launch()["kernel"] == "k_track2", ctx_a.last_launch()
    for corr in range(wl.n_corr_iterations):
        ctx_b.corr_iteration(0, corr, wl.n_update_iterations)
    assert ctx_b.last_launch()["kernel"] == "k_track2", ctx_b.last_launch()
    pa, pb = ctx_a.get_poses(), ctx_b.get_poses()
    assert np.array_equal(pa.view(np.uint32), pb.view(np.uint32))
    for b in range(wl.n_bodies):
        assert np.array_equal(_bits(ctx_a.get_region_lines(b, wl.lines_per_body)), _bits(ctx_b.get_region_lines(b, wl.lines_per_body)))
        assert np.array_equal(_bits(ctx_a.get_depth_points(b, wl.points_per_body)), _bits(ctx_b.get_depth_points(b, wl.points_per_body)))
    ctx_a.close()
    ctx_b.close()


# ---- D. schedules, lengths, learning rates -----------------------------------------------------------------------------
# name -> (region settings, depth settings, uploads, floors (valid lines, valid points) where the defaults do not hold)
SETTINGS = {
    # scales outside the specialised set {1, 2, 4, 6}, 8 entries, 2 standard deviations: k_track2's ROI reach grows
    # with the largest scale (the slow walk)
    "scales8": (dict(scales=(12, 9, 8, 5, 3, 3, 2, 1), standard_deviations=(15.0, 5.0)), {}, ("full", "pinned"), None),
    "step_function": (dict(function_slope=0.0, function_amplitude=0.49), {}, ("full",), None),
    "learning_rate_0.5": (dict(learning_rate=0.5), {}, ("full",), None),
    "learning_rate_2.0": (dict(learning_rate=2.0), {}, ("full",), None),
    # k_histogram's walk and k_ingest's reach depend on the line lengths
    "unconsidered_0": (dict(unconsidered_line_length=0.0), {}, ("full", "pinned"), None),
    "unconsidered_2": (dict(unconsidered_line_length=2.0), {}, ("full", "pinned"), None),
    "max_considered_5": (dict(max_considered_line_length=5.0), {}, ("full", "pinned"), None),
    "max_considered_60": (dict(max_considered_line_length=60.0), {}, ("full", "pinned"), None),
    "min_continuous_0": (dict(min_continuous_distance=0.0), {}, ("full",), None),
    "min_continuous_8": (dict(min_continuous_distance=8.0), {}, ("full",), None),
    "histogram_rates_1": (dict(learning_rate_f=1.0, learning_rate_b=1.0), {}, ("full",), None),
    "stride_0.002": ({}, dict(stride_length=0.002), ("full",), None),
    # a 2 cm stride leaves few search positions inside the considered distances: ~10 % of the points stay valid
    "stride_0.02": ({}, dict(stride_length=0.02), ("full",), (0.5, 0.05)),
    "distances8": ({}, dict(considered_distances=(0.08, 0.06, 0.05, 0.04, 0.03, 0.02, 0.015, 0.01),
                            standard_deviations=(0.06, 0.05, 0.04, 0.035, 0.03, 0.025, 0.02, 0.015)), ("full",), None),
    "distances1_deviations5": ({}, dict(considered_distances=(0.03,), standard_deviations=(0.05, 0.04, 0.03, 0.02, 0.01)),
                               ("full",), None),
}
_SETTING_CASES = [(name, up) for name, (_, _, ups, _) in SETTINGS.items() for up in ups]


@pytest.mark.parametrize("name,upload", _SETTING_CASES)
def test_region_and_depth_settings(capi, oracle, base, name, upload):
    region, depth, _, floors = SETTINGS[name]
    wl = _variant(base, region=region, depth=depth)
    kw = {} if floors is None else dict(min_valid_lines=floors[0], min_valid_points=floors[1])
    _parity(capi, oracle, wl, f"settings_{name}_{upload}", dict(kernel="k_track2", threads=1024, lut_smem=1, tiles=1),
            upload, **kw)


@pytest.mark.parametrize("field,value", [("function_length", 6), ("distribution_length", 10)])
def test_other_function_and_distribution_lengths_are_refused(capi, base, field, value):
    """function_length / distribution_length other than 8 / 12 are not implemented: refused, not run."""
    ctx = capi.context_from_workload(base)
    rp = capi.region_params(base.region)
    setattr(rp, field, value)
    with pytest.raises(capi.M3TBError, match="function_length / distribution_length"):
        ctx.set_body(0, rp, capi.depth_params(base.depth), None)
    ctx.close()
