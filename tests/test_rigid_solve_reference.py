"""The float32 oracle's rigid-body solve (orc_optimize_rigid, both exp modes) against the float64 restatement
(structure_reference: calculate_optimization of the implicit one-link structure), on every system of
rigid_solve_cases.

Outcome, on every case: whether the pose is updated, which theta entries are NaN and which are exactly 0, and whether
the new pose is finite. Knife-edge cases - where float32 rounding alone decides (a pivot at Eigen's tolerance, an exact
zero D of a singular float32 system, a signed-zero diagonal) - are judged against the float32 oracle only.

With a NaN or inf in g or H, the restatement's J^T H J (J = I, every product formed, as the reference's Eigen product
does) turns 0 * NaN into NaN across the whole system, so the reference refuses every such update. The oracle and the
device assemble a = 0 - H for the rigid body and keep the non-finite entries where they are; for those cases the
restatement's LDLT is run on that element-wise system, so that the solve itself is what is compared.
"""
import numpy as np
import pytest

import rigid_solve_cases as rc
import structure_reference as sr

F32 = np.float32
CASES = rc.all_cases()
EPS32 = float(np.finfo(F32).eps)


def oracle_solve(oracle, case, exp_mode):
    """(updated, theta [6], pose [3, 4]) of the float32 oracle: orc_optimize_rigid from the modality sums, or for a
    given system (Case.a_direct, which 0 - H cannot produce) the same three steps it takes: LDLT, NaN guard, update."""
    L = oracle.lib()
    theta = np.zeros(6, F32)
    pose = np.array(case.pose, F32).reshape(12)  # a copy: the oracle updates it in place
    if case.a_direct is None:
        g, H = case.sums()
        ok = L.orc_optimize_rigid(oracle.ptr(g), oracle.ptr(np.ascontiguousarray(H.reshape(36))), F32(case.tikhonov[0]),
                                  F32(case.tikhonov[1]), exp_mode, oracle.ptr(pose), oracle.ptr(theta))
        return bool(ok), theta, pose.reshape(3, 4)
    a, b = case.system()
    L.orc_ldlt_solve(6, oracle.ptr(np.ascontiguousarray(a)), oracle.ptr(b), oracle.ptr(theta))
    if np.isnan(theta).any():
        return False, theta, pose.reshape(3, 4)
    e = np.zeros(9, F32)
    L.orc_exp_skew(oracle.ptr(np.ascontiguousarray(theta[:3])), exp_mode, oracle.ptr(e))
    var = np.array([e[0], e[1], e[2], theta[3], e[3], e[4], e[5], theta[4], e[6], e[7], e[8], theta[5]], F32)
    out = np.zeros(12, F32)
    L.orc_pose_multiply(oracle.ptr(pose), oracle.ptr(var), oracle.ptr(out))
    return True, theta, out.reshape(3, 4)


def reference64(synth, case):
    """(updated, theta [6], pose [3, 4]) in float64"""
    spec = sr.implicit_structure(synth, 0, float(case.tikhonov[0]), float(case.tikhonov[1]))
    state = sr.State.from_arrays(case.pose.reshape(1, 12), np.eye(4)[None, :3], np.eye(4)[None, :3])
    if case.finite_inputs() and case.a_direct is None:
        n = 3 if case.texture else 2
        r = sr.calculate_optimization(spec, state, case.g[:n, None].astype(np.float64), case.H[:n, None].astype(np.float64))
        theta, updated, new = r.theta, r.updated, r.state
    else:  # the element-wise system of the oracle and the device (see the module docstring)
        a, b = case.system()
        if case.a_direct is None:
            with np.errstate(invalid="ignore", over="ignore"):
                n = 3 if case.texture else 2
                H = case.H[:n].astype(np.float64).sum(0)
                a = -H + np.diag([float(case.tikhonov[0])] * 3 + [float(case.tikhonov[1])] * 3)
                b = case.g[:n].astype(np.float64).sum(0)
        theta = sr.ldlt_solve(np.asarray(a, np.float64), np.asarray(b, np.float64))
        updated = not np.isnan(theta).any()
        new = sr.update_poses(spec, state, theta) if updated else state
    return updated, theta, new.link2world[0, :3]


def outcome(updated, theta, pose):
    return dict(updated=bool(updated), nan=tuple(np.isnan(theta)), zero=tuple(np.asarray(theta) == 0),
                finite_pose=bool(np.isfinite(pose).all()))


@pytest.mark.parametrize("exp_mode", ["rodrigues", "pade"])
def test_outcome_matches_float64(oracle, synth, exp_mode):
    mode = oracle.EXP_RODRIGUES if exp_mode == "rodrigues" else oracle.EXP_PADE
    bad = []
    for case in CASES:
        o = outcome(*oracle_solve(oracle, case, mode))
        if case.knife_edge:
            continue
        upd, theta64, pose64 = reference64(synth, case)
        r = outcome(upd, theta64, pose64)
        if np.abs(theta64[np.isfinite(theta64)]).max(initial=0.0) > 1e30:
            # a zero-matrix exit with a NaN first pivot solves with the unfactorised matrix: theta near 1e35, whose pose
            # product overflows float32 and not float64
            o.pop("finite_pose"), r.pop("finite_pose")
        if o != r:
            bad.append((case.name, o, r))
    assert not bad, bad[:5]


def test_knife_edge_cases_follow_float32_rounding(oracle):
    """Pivots at Eigen's float tolerance 1 / FLT_MAX: one ulp above divides, at or below gives exactly 0; an all-zero
    or NaN-headed diagonal is the zero-matrix exit (identity transpositions)."""
    by = {c.name: c for c in CASES}
    for name, zero in (("tolerance_above", False), ("tolerance_at", True), ("tolerance_below", True)):
        ok, theta, _ = oracle_solve(oracle, by[name], oracle.EXP_RODRIGUES)
        assert ok and (theta[5] == 0) == zero, (name, theta)
        if not zero:  # b5 = 0.75 D, both denormals
            assert abs(theta[5] - 0.75) < 1e-5, theta
    ok, theta, _ = oracle_solve(oracle, by["all_zero"], oracle.EXP_RODRIGUES)
    assert ok and (theta == 0).all()


def test_regular_numbers_within_gate(oracle, synth):
    """On regular systems the float32 oracle is within a backward-stable solve's forward error of float64:
    |theta32 - theta64| <= 16 eps32 cond(a) |theta64| (so theta_gates of structure_reference is a meaningful bar)."""
    worst = 0.0
    for case in CASES:
        if case.group not in ("regular", "pivot", "exp", "sum") or case.knife_edge or not case.finite_inputs():
            continue
        ok, theta, _ = oracle_solve(oracle, case, oracle.EXP_RODRIGUES)
        upd, theta64, _ = reference64(synth, case)
        assert ok and upd, case.name
        a, _ = case.system()
        a = np.tril(a.astype(np.float64)) + np.tril(a.astype(np.float64), -1).T
        bound = 16 * EPS32 * np.linalg.cond(a) * np.abs(theta64).max() + 1e-30
        dev = np.abs(theta.astype(np.float64) - theta64).max()
        if case.group != "sum":  # the float32 modality sum itself rounds: judged against the oracle only, on the GPU
            assert dev <= bound, (case.name, dev, bound)
            worst = max(worst, dev / bound)
    assert worst < 1.0


def test_catalogue_reaches_every_branch(oracle):
    tags = set().union(*(c.tags for c in CASES))
    for i in range(6):
        assert f"nan_g{i}" in tags and f"nan_diag{i}" in tags
    for t in ("zero_exit", "tolerance_zero", "tolerance_divides", "exp_series", "exp_closed", "sinf_large_argument",
              "order", "tie", "opposite_signs", "signed_zero", "rank", "negative_tikhonov", "nan_off", "nan_rowcol",
              "inf_diag", "inf_g", "nonfinite_tikhonov", "t2_branch_point", "theta_zero", "theta_zero_components",
              "drifted_pose", "modality_sum", "scaled"):
        assert t in tags, t
    assert len([c for c in CASES if "order" in c.tags]) == 720
    # the branches are reached by what the oracle actually computes, not only by construction
    t2s, series, closed, large = [], 0, 0, 0
    for c in CASES:
        ok, theta, _ = oracle_solve(oracle, c, oracle.EXP_RODRIGUES)
        if not ok:
            continue
        w = theta[:3]
        t2 = (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]
        series += t2 < F32(0.01)
        closed += t2 >= F32(0.01)
        large += np.isfinite(t2) and np.sqrt(np.float64(t2)) > rc.SINF_FAST_LIMIT
        if "t2_branch_point" in c.tags:
            t2s.append(t2)
    assert series and closed and large
    assert F32(0.01) in t2s and np.nextafter(F32(0.01), F32(0)) in t2s and np.nextafter(F32(0.01), F32(1)) in t2s
    # zero-matrix exit: a NaN or zero first pivot
    for c in CASES:
        if "zero_exit" in c.tags:
            a, _ = c.system()
            d = np.abs(np.diag(a))
            assert np.isnan(d[0]) or np.nanmax(d) == 0, c.name
