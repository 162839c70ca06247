"""GPU parity at the shapes the bench and the untested k_track instantiations run (VERDICT r01, "what's weak" 1-4).

  * the BENCHMARKED shape: configs[3] bodies = 512 lines + 512 depth points, defaults, fused solve
    (m3tb_corr_iteration / m3tb_tracking_step -> the 512-items-per-modality instantiation with PH_SOLVE);
  * 1024 and 2048 lines / points per body (2 and 4 items per thread);
  * 32-bin histograms (k_histogram, the RBOT-shape config);
  * free-running trajectories against the GPU-mirror oracle (LINEAR / RODRIGUES: only the summation order differs),
    the fraction of bodies inside 1e-4 m / 1e-4 rad for the whole step is printed and appended to the JSON-lines file
    named by M3TB_PARITY_RECORD when that variable is set (>= 0.7 required, 0.75-0.92 measured);
  * the reference's own .bin sparse-viewpoint models (tests/golden/{region,depth}_model.bin: schauma, 162 views x 10
    points) read with model_io.read_model and fed through m3tb_set_region_model / m3tb_set_depth_model (SURVEY f2).
Bars as in test_gpu_parity.py: per-line / per-point state bit-exact, g / H <= 1e-5 of max|H|, pose after every
correspondence iteration <= 1e-4 m / 1e-4 rad against the reference-faithful oracle on identical inputs.
"""
import json
import os

import numpy as np
import pytest

from helpers import assert_lines_bit_equal, assert_points_bit_equal, pose_error, rel_to_max

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
TOL = 1e-4


def _record(name, **kv):
    print(f"[parity] {name}: " + ", ".join(f"{k}={v}" for k, v in kv.items()))
    path = os.environ.get("M3TB_PARITY_RECORD")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(dict(test=name, **kv)) + "\n")


def _per_iteration_parity(capi, oracle, wl, name, check_gh=True, min_valid_points=0.3, mirror_tol=1e-5):
    """Every correspondence iteration starts from the mirror oracle's pose on both sides. Checks, per iteration:
    closest views equal, per-line / per-point records of the FUSED launch bit-exact, g / H of the fine-grained calls,
    pose after the fused iteration vs the mirror oracle (tight) and vs the reference-faithful oracle (the 1e-4 gate)."""
    ctx = capi.context_from_workload(wl)
    mirror = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    faithful = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_POLAR, exp_mode=oracle.EXP_PADE)
    mirror.start_modalities(0)
    faithful.start_modalities(0)
    ctx.start_modalities(0)
    nl, npnt = wl.lines_per_body, wl.points_per_body
    worst = dict(mirror_m=0.0, mirror_rad=0.0, faithful_m=0.0, faithful_rad=0.0, H=0.0, g=0.0)
    n_valid_lines = n_valid_points = 0
    view_ties = 0   # (body, iteration) pairs where the two oracle modes themselves pick different template views
    mode_splits = 0  # ... or end the iteration more than the tolerance apart (a discrete event between the modes)
    for corr in range(wl.n_corr_iterations):
        start = mirror.get_poses()
        faithful.set_poses(start)
        if check_gh and corr in (0, wl.n_corr_iterations - 1):
            ctx.set_poses(start)
            if wl.region:
                ctx.region_correspondences(0, corr)
                g_r, H_r = ctx.region_gradient_hessian(0, corr, 0)
            if wl.depth:
                ctx.depth_correspondences(0, corr)
                g_d, H_d = ctx.depth_gradient_hessian(0, corr, 0)
            for b in range(wl.n_bodies):
                if wl.region:
                    mirror.region_correspondences(b, 0, corr)
                    og, oH = mirror.region_gradient_hessian(b, corr, 0)
                    worst["H"] = max(worst["H"], rel_to_max(H_r[b], oH))
                    worst["g"] = max(worst["g"], rel_to_max(g_r[b], og))
                if wl.depth:
                    mirror.depth_correspondences(b, 0, corr)
                    og, oH = mirror.depth_gradient_hessian(b, corr)
                    worst["H"] = max(worst["H"], rel_to_max(H_d[b], oH))
                    worst["g"] = max(worst["g"], rel_to_max(g_d[b], og))
        ctx.set_poses(start)
        ctx.corr_iteration(0, corr, wl.n_update_iterations)   # ONE fused launch: correspondences, g / H, solves
        gpu = ctx.get_poses()
        same_views = np.ones(wl.n_bodies, bool)
        for b in range(wl.n_bodies):
            if wl.region:
                n, view = mirror.region_correspondences(b, 0, corr)
                same_views[b] &= faithful.region_correspondences(b, 0, corr)[1] == view
                assert ctx.get_closest_views(b)[0] == view, (name, corr, b)
                lines = ctx.get_region_lines(b, nl)
                assert_lines_bit_equal(lines, mirror.lines[b][:n])
                n_valid_lines += int((lines["valid"] != 0).sum())
            if wl.depth:
                n, view = mirror.depth_correspondences(b, 0, corr)
                same_views[b] &= faithful.depth_correspondences(b, 0, corr)[1] == view
                assert ctx.get_closest_views(b)[1] == view, (name, corr, b)
                pts = ctx.get_depth_points(b, npnt)
                assert_points_bit_equal(pts, mirror.points[b][:n])
                n_valid_points += int((pts["valid"] != 0).sum())
        mirror.tracking_step(0, n_corr=corr + 1, corr_begin=corr)
        faithful.tracking_step(0, n_corr=corr + 1, corr_begin=corr)
        dt, dr = pose_error(gpu, mirror.get_poses())
        worst["mirror_m"], worst["mirror_rad"] = max(worst["mirror_m"], dt.max()), max(worst["mirror_rad"], dr.max())
        # The reference-faithful oracle takes the GetClosestView query from the polar factor of body2camera
        # (Transform::rotation()), the mirror oracle / the CUDA path from its linear block (~1e-7 apart). When the pose
        # sits on the boundary between two template views that 1e-7 decides which view is used - a discrete event of the
        # algorithm itself (two builds of the reference would disagree the same way). Such pairs are counted and
        # excluded from the 1e-4 gate; everything else must meet it.
        # The same holds for the other integer decisions of the path (int() of a line coordinate, the histogram bin pair of
        # the local-mode gradient): where the reference's two float realisations - the two oracle modes - themselves end
        # an iteration more than the tolerance apart, the comparison says nothing about the CUDA path.
        view_ties += int((~same_views).sum())
        st, sr = pose_error(mirror.get_poses(), faithful.get_poses())
        comparable = same_views & (st < TOL) & (sr < TOL)
        mode_splits += int((~comparable).sum())
        dt, dr = pose_error(gpu, faithful.get_poses())
        if comparable.any():
            worst["faithful_m"] = max(worst["faithful_m"], dt[comparable].max())
            worst["faithful_rad"] = max(worst["faithful_rad"], dr[comparable].max())
    ctx.close()
    _record(name, bodies=wl.n_bodies, lines=nl, points=npnt, valid_lines=n_valid_lines, valid_points=n_valid_points,
            view_ties=view_ties, oracle_mode_splits=mode_splits, **{k: float(f"{v:.3e}") for k, v in worst.items()})
    assert mode_splits <= max(1, 0.05 * wl.n_bodies * wl.n_corr_iterations), mode_splits
    if wl.region:
        assert n_valid_lines > 0.5 * nl * wl.n_bodies * wl.n_corr_iterations
    if wl.depth:
        assert n_valid_points > min_valid_points * npnt * wl.n_bodies * wl.n_corr_iterations
    assert worst["H"] < 1e-5 and worst["g"] < 1e-4, worst
    assert worst["mirror_m"] < mirror_tol and worst["mirror_rad"] < mirror_tol, worst   # only summation order + logf ulps differ
    assert worst["faithful_m"] < TOL and worst["faithful_rad"] < TOL, worst  # the contract gate


def test_benchmarked_shape_c4_per_iteration(capi, oracle, synth):
    """configs[3] bodies exactly as bench.py builds them (same preset, same seed, the first 8 of the 128-body shard)."""
    wl = synth.make_workload("c4", n_bodies=8, n_divides=4, seed=0)
    assert wl.lines_per_body == 512 and wl.points_per_body == 512
    _per_iteration_parity(capi, oracle, wl, "c4_512+512")


def test_benchmarked_shape_fused_step_equals_iterated(capi, synth):
    """m3tb_tracking_step (the launch bench.py times) == 7 x m3tb_corr_iteration bit for bit at 512 + 512."""
    wl = synth.make_workload("c4", n_bodies=8, n_divides=4, seed=0)
    a, b = capi.context_from_workload(wl), capi.context_from_workload(wl)
    for c in (a, b):
        c.start_modalities(0)
    a.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    for corr in range(wl.n_corr_iterations):
        b.corr_iteration(0, corr, wl.n_update_iterations)
    pa, pb = a.get_poses(), b.get_poses()
    assert np.array_equal(pa.view(np.uint32), pb.view(np.uint32))
    dt0, _ = pose_error(wl.start_body2world, wl.gt_body2world)
    dt1, _ = pose_error(pa, wl.gt_body2world)
    assert (dt1 < dt0).all()
    a.close()
    b.close()


@pytest.mark.parametrize("items", [1024, 2048])
def test_many_items_per_thread(capi, oracle, synth, items):
    """513..1024 and 1025..2048 lines / points per body: the 2- and 4-items-per-thread instantiations."""
    wl = synth.make_workload("c2", n_bodies=3, n_lines=items, n_points=items, n_divides=2, seed=31)
    # 4096 summands per sum: the warp-tree vs serial summation order shows at a few 1e-5 rad
    _per_iteration_parity(capi, oracle, wl, f"c2_{items}+{items}", mirror_tol=5e-5)


def test_region_only_32_bins_600_lines(capi, oracle, synth):
    """RBOT-shape parameters (32 bins: LUT in global memory, step-function lookup) with 600 lines (2 per thread)."""
    wl = synth.make_workload("c3", n_bodies=3, n_lines=600, n_divides=2, seed=33)
    _per_iteration_parity(capi, oracle, wl, "c3_600")


def test_histograms_32_bins_exact(capi, oracle, synth):
    """k_histogram with 32 bins (32768 bins per histogram): StartModality and CalculateResults bit-exact."""
    wl = synth.make_workload("c3", n_bodies=4, n_divides=3, seed=5)
    assert wl.region.n_histogram_bins == 32
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
            hf, hb = ctx.get_histograms(b, 32)
            assert np.array_equal(hf.view(np.uint32), orc.hist_f[b].view(np.uint32)), (stage, b)
            assert np.array_equal(hb.view(np.uint32), orc.hist_b[b].view(np.uint32)), (stage, b)
            assert np.count_nonzero(hf) > 10 and np.count_nonzero(hb) > 10
    ctx.close()


@pytest.mark.parametrize("which,n_bodies", [("c2", 24), ("c3", 24), ("c4", 12)])
def test_free_running_vs_mirror_oracle(capi, oracle, synth, which, n_bodies):
    """Both sides free-run the whole tracking step from the same start; the oracle in GPU-mirror mode differs from the
    CUDA path only in the summation order of g / H (~1e-7 relative). The fraction of bodies that stay inside 1e-4 m /
    1e-4 rad after EVERY correspondence iteration is recorded (measured on an H100: 0.75 - 0.92 depending on config,
    i.e. about one body in eight meets a discrete event - an int() of a line coordinate, a histogram bin pair of the local
    mode, a view switch - somewhere in its 7 x 2 iterations) and must be >= 0.7; the others may only deviate by the
    size of such an event."""
    wl = synth.make_workload(which, n_bodies=n_bodies, n_divides=4, seed=41)
    ctx = capi.context_from_workload(wl)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    orc.start_modalities(0)
    ctx.start_modalities(0)
    worst_t, worst_r = np.zeros(wl.n_bodies), np.zeros(wl.n_bodies)
    for corr in range(wl.n_corr_iterations):
        ctx.corr_iteration(0, corr, wl.n_update_iterations)
        orc.tracking_step(0, n_corr=corr + 1, corr_begin=corr)
        dt, dr = pose_error(ctx.get_poses(), orc.get_poses())
        worst_t, worst_r = np.maximum(worst_t, dt), np.maximum(worst_r, dr)
    within = (worst_t < TOL) & (worst_r < TOL)
    _record(f"free_running_{which}", bodies=wl.n_bodies, fraction_within_tol=float(within.mean()),
            worst_m=float(worst_t.max()), worst_rad=float(worst_r.max()),
            median_m=float(np.median(worst_t)), median_rad=float(np.median(worst_r)))
    assert within.mean() >= 0.7, (within.mean(), worst_t, worst_r)
    assert worst_t.max() < 3e-3 and worst_r.max() < 2e-2, (worst_t, worst_r)
    ctx.close()


def test_reference_bin_models_through_cuda_path(capi, oracle, pkg, synth):
    """SURVEY f2 on the device: the reference's checked-in .bin models (schauma, 162 views x 10 points; 8-bit-decoded,
    non-unit depth normals; FLT_MAX background distances) go through model_io.read_model ->
    m3tb_set_region_model / m3tb_set_depth_model and must give the oracle's closest views, per-line / per-point
    records (bit-exact) and poses."""
    rm = pkg.model_io.read_model(os.path.join(GOLDEN, "region_model.bin"))
    dm = pkg.model_io.read_model(os.path.join(GOLDEN, "depth_model.bin"))
    assert rm.model.n_views == 162 and rm.model.n_points == 10 and dm.model.n_points == 10
    wl = synth.make_workload("c2", n_bodies=6, n_lines=10, n_points=10, n_divides=2, seed=17,
                             models=(rm.model, dm.model))
    # (the synthetic frames show the triangle prism, not the schauma figure: few depth correspondences, irrelevant here)
    _per_iteration_parity(capi, oracle, wl, "reference_bin_models", min_valid_points=0.02)
