"""The device's rigid-body solve (SolveAndUpdateSerial, shared by k_track and k_track2) on the systems of
rigid_solve_cases, against the mirror oracle (orc_optimize_rigid, EXP_RODRIGUES) and the float64 restatement.

  * public C ABI: one context, one case per body, every case in one launch: m3tb_set_gradient_hessian for the region,
    depth and texture modalities, then m3tb_calculate_optimization (k_track). A refused update leaves the pose
    bit-identical; otherwise the pose equals the mirror oracle's bit for bit where ExpSkew takes its series
    (t2 < 0.01f) and within 4 ulps of the pose's largest entry where it calls sinf.
  * test aid (m3tb_debug_rigid_solve): the solve on both shared-memory layouts (k_track's and k_track2's) on every
    case, bit-identical to each other and theta bit-identical to the mirror oracle; on finite regular systems theta
    also meets the float64 gate of test_gpu_structure_limits.py (max(4 |theta_oracle32 - theta64|, 1e-6 |theta64|)).
  * end to end: correspondence iterations of k_track2 and of k_track (M3TB_KERNEL=1) with degenerate Tikhonov
    parameters, each started from the mirror oracle's pose: where the oracle refuses the update the device keeps the
    pose bit for bit, elsewhere the 1e-4 gate holds; and one refine_poses call with a NaN translation parameter.
"""
import numpy as np
import pytest

import rigid_solve_cases as rc
import structure_reference as sr
from helpers import pose_error, record
from test_rigid_solve_reference import CASES, oracle_solve, reference64

pytestmark = pytest.mark.gpu

F32 = np.float32
SINF_ULPS = 4
TRIANGLE = np.array([[[0.0, 0.0, 0.0], [0.05, 0.0, 0.0], [0.0, 0.05, 0.0]]], F32)


def same_bits(x, y):
    """bit-identical, NaN payloads aside"""
    x, y = np.asarray(x, F32), np.asarray(y, F32)
    nx, ny = np.isnan(x), np.isnan(y)
    return np.array_equal(nx, ny) and np.array_equal(x[~nx].view(np.uint32), y[~ny].view(np.uint32))


def t2_of(theta):
    w = np.asarray(theta[:3], F32)
    with np.errstate(over="ignore", invalid="ignore"):
        return (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]


def check_pose(name, theta, pose, pose_o):
    if t2_of(theta) < F32(0.01):
        assert same_bits(pose, pose_o), (name, pose, pose_o)
    else:  # sinf / cosf: a few ulps of the pose's largest finite entry; the same entries non-finite
        fin = np.isfinite(pose_o)
        assert np.array_equal(np.isfinite(pose), fin), (name, pose, pose_o)
        scale = max(float(np.abs(pose_o[fin]).max(initial=0.0)), 1.0)
        ulp = float(np.spacing(F32(scale)))
        dev = np.abs(pose[fin].astype(np.float64) - pose_o[fin].astype(np.float64))
        assert (dev <= SINF_ULPS * ulp).all(), (name, dev.max(), ulp)


def gate_theta(synth, case, theta, theta_o):
    if case.knife_edge or not case.finite_inputs() or case.group not in ("regular", "pivot", "exp", "sum"):
        return None
    upd, theta64, _ = reference64(synth, case)
    if not upd:
        return None
    gate = sr.theta_gates(theta_o, theta64, 6)[0]
    dev = sr.theta_deviations(theta, theta64, 6)[0]
    assert dev <= gate, (case.name, dev, gate)
    return dev


def test_both_solves_on_every_case(capi, oracle, synth):
    wl = synth.make_workload("c2", n_bodies=1, n_lines=16, n_points=16, n_divides=1, seed=5)
    ctx = capi.context_from_workload(wl)
    systems = [c.system() for c in CASES]
    a = np.stack([s[0] for s in systems])
    b = np.stack([s[1] for s in systems])
    poses = np.stack([c.pose for c in CASES])
    out = [ctx.debug_rigid_solve(solve, a, b, poses) for solve in (0, 1)]
    ctx.close()
    bad, worst = [], 0.0
    for i, c in enumerate(CASES):
        (tw, uw, pw), (ts, us, ps) = [(o[0][i], o[1][i], o[2][i]) for o in out]
        assert same_bits(tw, ts) and uw == us and same_bits(pw, ps), (c.name, tw, ts, uw, us)
        ok, theta_o, pose_o = oracle_solve(oracle, c, oracle.EXP_RODRIGUES)
        if uw != ok or not same_bits(tw, theta_o):
            bad.append((c.name, uw, ok, tw, theta_o))
            continue
        if not ok:
            assert same_bits(pw, c.pose), c.name
            continue
        check_pose(c.name, tw, pw, pose_o)
        dev = gate_theta(synth, c, tw, theta_o)
        worst = max(worst, dev or 0.0)
    record("rigid_solve_aid", cases=len(CASES), mismatches=[x[0] for x in bad], worst_theta_vs_float64=worst)
    assert not bad, [x[:3] for x in bad[:10]]


def test_public_abi_one_case_per_body(capi, oracle, synth):
    cases = [c for c in CASES if c.a_direct is None] * 2  # every case twice: more than a thousand bodies
    nb = len(cases)
    assert nb >= 1000
    wl = synth.make_workload("c2", n_bodies=nb, n_lines=16, n_points=16, n_divides=1, seed=7)
    ctx = capi.context_from_workload(wl)
    rp, dp = capi.region_params(wl.region), capi.depth_params(wl.depth)
    for k, c in enumerate(cases):
        ctx.set_body(k, rp, dp, capi.OptimizerParams(float(c.tikhonov[0]), float(c.tikhonov[1])), 0, 0, k, k)
        if c.texture:  # the texture modality needs a body geometry; one triangle will do, nothing is rendered
            ctx.set_body_geometry(k, TRIANGLE)
            ctx.set_texture_modality(k, capi.texture_params_default(), k)
    ctx.set_poses(np.stack([c.pose for c in cases]))
    for m in range(3):
        ctx.set_gradient_hessian(m, np.stack([c.g[m] for c in cases]), np.stack([c.H[m].reshape(36) for c in cases]))
    before = ctx.get_poses()
    ctx.calculate_optimization(0, 0, 0)
    assert ctx.last_launch()["kernel"] == "k_track"
    after = ctx.get_poses()
    # theta is not read back for a rigid body: it comes from the test aid on the same systems
    systems = [c.system() for c in cases]
    theta, upd, _ = ctx.debug_rigid_solve(0, np.stack([s[0] for s in systems]), np.stack([s[1] for s in systems]),
                                          before)
    ctx.close()
    bad = []
    for k, c in enumerate(cases):
        ok, theta_o, pose_o = oracle_solve(oracle, c, oracle.EXP_RODRIGUES)
        if ok != upd[k] or not same_bits(theta[k], theta_o):
            bad.append((c.name, ok, upd[k]))
            continue
        if not ok:
            if not same_bits(after[k], before[k]):
                bad.append((c.name, "moved"))
            continue
        check_pose(c.name, theta[k], after[k], pose_o)
        gate_theta(synth, c, theta[k], theta_o)
    record("rigid_solve_public_abi", bodies=nb, mismatches=[x[0] for x in bad])
    assert not bad, bad[:10]


# A NaN rotation parameter is left out: its NaN first pivot takes the zero-matrix exit, whose finite theta turns the pose
# non-finite in the oracle and on the device alike (test_both_solves_on_every_case covers that system), and tracking
# from a non-finite pose is not what this test is about.
TIKHONOV_E2E = [(1000.0, float("nan")), (0.0, 0.0), (1e30, 1e30), (10.0, 100.0), (1000.0, 30000.0)]


@pytest.mark.parametrize("kernel", ["k_track2", "k_track"])
def test_tracking_with_degenerate_tikhonov(capi, oracle, synth, monkeypatch, kernel):
    if kernel == "k_track":
        monkeypatch.setenv("M3TB_KERNEL", "1")
    nb = len(TIKHONOV_E2E)
    wl = synth.make_workload("c2", n_bodies=nb, n_lines=128, n_points=128, n_divides=2, seed=11)
    ctx = capi.context_from_workload(wl)
    mirror = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    rp, dp = capi.region_params(wl.region), capi.depth_params(wl.depth)
    for b, (tr, tt) in enumerate(TIKHONOV_E2E):
        ctx.set_body(b, rp, dp, capi.OptimizerParams(tr, tt), 0, 0, b, b)
        mirror.bodies[b].tikhonov_rotation, mirror.bodies[b].tikhonov_translation = tr, tt
    ctx.start_modalities(0)
    mirror.start_modalities(0)
    worst = {}
    for corr in range(wl.n_corr_iterations):
        s = mirror.get_poses()
        ctx.set_poses(s)
        ctx.corr_iteration(0, corr, wl.n_update_iterations)
        assert ctx.last_launch()["kernel"] == kernel
        mirror.tracking_step(0, n_corr=corr + 1, corr_begin=corr)
        got, want = ctx.get_poses(), mirror.get_poses()
        for b, (tr, tt) in enumerate(TIKHONOV_E2E):
            if same_bits(want[b], s[b]):  # the oracle refused every update: the pose is kept bit for bit
                assert same_bits(got[b], s[b]), (TIKHONOV_E2E[b], corr)
                continue
            dt, dr = pose_error(got[b:b + 1], want[b:b + 1])
            worst[b] = max(worst.get(b, 0.0), float(dt.max()), float(dr.max()))
    record(f"rigid_solve_e2e_{kernel}", worst={str(TIKHONOV_E2E[b]): v for b, v in worst.items()})
    ctx.close()
    for b, v in worst.items():
        assert v < 1e-4, (TIKHONOV_E2E[b], v)


def test_refine_poses_with_nan_translation_tikhonov(capi, synth):
    wl = synth.make_workload("c2", n_bodies=2, n_lines=128, n_points=128, n_divides=2, seed=13)
    ctx = capi.context_from_workload(wl)
    rp, dp = capi.region_params(wl.region), capi.depth_params(wl.depth)
    ctx.set_body(0, rp, dp, capi.OptimizerParams(1000.0, float("nan")), 0, 0, 0, 0)
    before = ctx.get_poses().copy()
    ctx.refine_poses(bodies=[0, 1], n_corr_iterations=2, n_update_iterations=2)
    after = ctx.get_poses()
    ctx.close()
    assert same_bits(after[0], before[0])
    assert not same_bits(after[1], before[1])
