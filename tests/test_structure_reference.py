"""CPU anchors of the float64 restatement of Optimizer::CalculateOptimization (tests/structure_reference.py) that the
device's kinematic-structure solve is held to in test_gpu_structure_limits.py:

  * it agrees with the float32 oracle's structure functions to float32 rounding, on the shapes of
    test_gpu_structures.py and on the limit shapes (16 links, 96 DoF, 128 unknowns, 32 constraints, 3 extra bodies,
    body-less links below the root, n == 1);
  * its LDLT equals np.linalg.solve on nonsingular systems and gives Eigen's exact zeros on singular ones;
  * the GPU test's theta gate notices a single missing term of the system (one soft constraint, one hard row, one
    Tikhonov entry), so it is not vacuous.
"""
import numpy as np
import pytest

import structure_reference as sr
from test_gpu_structures import _random_structures


def _oracle_optimize(oracle, spec, state, g, H):
    """orc_optimize_structure (float32, the device's summation order) from the same state: (theta, ok, link2world)."""
    L = oracle.lib()
    so = oracle.OracleStructure(sr.with_joint_poses(spec, state.body2joint[:, :3], state.joint2parent[:, :3]))
    S = so.as_struct()
    gl, Hl = sr.link_gradients(spec, g, H)
    l2w = np.ascontiguousarray(state.link2world[:, :3].reshape(-1, 12), np.float32)
    theta = np.zeros(sr.n_unknowns(spec), np.float32)
    ok = L.orc_optimize_structure(S, oracle.ptr(gl.astype(np.float32)), oracle.ptr(Hl.reshape(-1, 36).astype(np.float32)),
                                  oracle.ROTATION_LINEAR, oracle.EXP_RODRIGUES, oracle.ptr(l2w), oracle.ptr(theta))
    return theta, ok, l2w, so, S


def _f32_state(state):
    """the state rounded to float32, as the device and the oracle hold it"""
    f = lambda a: a[:, :3].reshape(-1, 12).astype(np.float32)
    return sr.State.from_arrays(f(state.link2world), f(state.body2joint), f(state.joint2parent))


def _shapes(synth, seed):
    """(name, spec, n_bodies) of every shape the structure tests use"""
    rng = np.random.default_rng(seed)
    out = [(f"random_{k}", s, 8) for k, s in enumerate(_random_structures(synth, rng))]
    for name, (builder, nb) in sr.LIMIT_SHAPES.items():
        out.append((name, builder(synth, rng, list(range(nb))), nb))
    out.append(("seven_unknowns", sr.seven_unknowns(synth, rng, [0, 1]), 2))
    out.append(("constrained83", sr.constrained83(synth, rng, list(range(8))), 8))
    return out


def _setup(spec, nb, rng):
    world = np.stack([sr.rand_pose(rng, 2.0, 0.3) for _ in range(nb)])
    state = _f32_state(sr.start_state(spec, world))
    g, H = sr.random_gh(rng, nb)
    return state, g, H


def test_restatement_matches_float32_oracle(oracle, synth):
    L = oracle.lib()
    rng = np.random.default_rng(101)
    for name, spec, nb in _shapes(synth, 31):
        state, g, H = _setup(spec, nb, rng)
        theta_o, ok, l2w_o, so, S = _oracle_optimize(oracle, spec, state, g, H)
        dof = sr.dof_of(spec)
        # Link::CalculateJacobian
        J = sr.link_jacobians(spec, state)
        jo = np.zeros((len(spec.links), 6, dof), np.float32)
        so2 = oracle.OracleStructure(spec)
        S2 = so2.as_struct()
        L.orc_structure_jacobians(S2, oracle.ROTATION_LINEAR, oracle.ptr(jo))
        assert np.abs(jo - J).max() <= 1e-6 * max(1.0, np.abs(J).max()), (name, np.abs(jo - J).max())
        l2w32 = np.ascontiguousarray(state.link2world[:, :3].reshape(-1, 12), np.float32)
        # Constraint::CalculateResidualAndConstraintJacobian / SoftConstraint::AddGradientsAndHessiansToLinks
        hard = [c for c in spec.constraints if not c.soft]
        soft = [c for c in spec.constraints if c.soft]
        for k, c in enumerate(hard):
            res, cj = sr.constraint_residual_jacobian(c, state, J)
            ro = np.zeros(6, np.float32)
            co = np.zeros((6, max(dof, 1)), np.float32)
            nr = L.orc_constraint_residual_jacobian(S2, k, oracle.ptr(l2w32), oracle.ptr(jo), oracle.ROTATION_LINEAR,
                                                    oracle.ptr(ro), oracle.ptr(co))
            assert nr == len(res)
            assert np.abs(ro[:nr] - res).max() <= 2e-6 * max(1.0, np.abs(res).max()), (name, k)
            assert np.abs(co[:nr, :dof] - cj).max() <= 2e-6 * max(1.0, np.abs(cj).max()), (name, k)
        for k, c in enumerate(soft):
            ((g1, H1), (g2, H2)), _ = sr.soft_constraint_terms(c, state)
            go = np.zeros((len(spec.links), 6), np.float32)
            Ho = np.zeros((len(spec.links), 36), np.float32)
            L.orc_soft_constraint_add(S2, k, oracle.ptr(l2w32), oracle.ROTATION_LINEAR, oracle.ptr(go), oracle.ptr(Ho))
            gr = np.zeros((len(spec.links), 6))
            Hr = np.zeros((len(spec.links), 6, 6))
            gr[c.link1] += g1; Hr[c.link1] += H1
            gr[c.link2] += g2; Hr[c.link2] += H2
            assert np.abs(go - gr).max() <= 1e-5 * max(1.0, np.abs(gr).max()), (name, k)
            assert np.abs(Ho.reshape(-1, 6, 6) - Hr).max() <= 1e-5 * max(1.0, np.abs(Hr).max()), (name, k)
        # the whole CalculateOptimization
        r = sr.calculate_optimization(spec, state, g, H)
        assert ok == 1 and r.updated
        scale = np.abs(r.theta).max()
        # float32 solve of a (DoF + rows)^2 system: relative error ~ condition number x 6e-8
        cond = np.linalg.cond(r.system.a)
        err = np.abs(theta_o - r.theta).max()
        assert err <= max(1e-5, 2e-7 * cond) * scale, (name, err, scale, cond)
        lw = r.state.link2world[:, :3].reshape(-1, 12)
        assert np.abs(l2w_o - lw).max() <= 2e-5, (name, np.abs(l2w_o - lw).max())
        b2j_o, j2p_o = so.joint_poses()
        assert np.abs(b2j_o - r.state.body2joint[:, :3]).max() <= 2e-5
        assert np.abs(j2p_o - r.state.joint2parent[:, :3]).max() <= 2e-5


def test_restatement_covers_the_limit_shapes(synth):
    """What each limit shape claims: sizes at the C ABI's limits, active and inactive soft parts."""
    rng = np.random.default_rng(5)
    shapes = {name: builder(synth, rng, list(range(nb))) for name, (builder, nb) in sr.LIMIT_SHAPES.items()}
    s = shapes["dof96_rows32"]
    assert (len(s.links), sr.dof_of(s), sr.n_unknowns(s), len(s.constraints)) == (16, 96, 128, 32)
    assert sr.spec_smem_bytes(s) == 125120 > 48 * 1024
    state, g, H = _setup(s, 16, rng)
    parts = sr.calculate_optimization(s, state, g, H).system.soft_parts
    assert any(p[-1] for p in parts) and not all(p[-1] for p in parts)
    t = shapes["tree16"]
    assert len(t.links) == 16 and any(not l.fixed_body2joint_pose for l in t.links)
    assert len({sum(l.free_directions) for l in t.links}) >= 3 and len({l.parent for l in t.links if l.parent >= 0}) > 5
    assert max(len(l.extra_bodies) for l in shapes["extra3"].links) == 3
    assert any(l.body < 0 and l.parent >= 0 for l in shapes["bodyless_mid"].links)
    assert sr.n_unknowns(shapes["one_unknown"]) == 1


@pytest.mark.parametrize("n", [1, 2, 7, 83, 128])
def test_ldlt_matches_numpy_solve(n):
    rng = np.random.default_rng(n)
    for kind in ("definite", "indefinite", "kkt"):
        if kind == "kkt" and n < 7:
            continue
        A = rng.normal(size=(n, n))
        if kind == "definite":
            a = -(A @ A.T) - n * np.eye(n)
        elif kind == "indefinite":
            a = A + A.T + np.diag(rng.choice([-1.0, 1.0], n) * n)
        else:
            m = n // 3
            d = n - m
            B = rng.normal(size=(d, d))
            a = np.zeros((n, n))
            a[:d, :d] = -(B @ B.T) - d * np.eye(d)
            C = rng.normal(size=(m, d))
            a[d:, :d] = C
            a[:d, d:] = C.T
        b = rng.normal(size=n)
        x = sr.ldlt_solve(a, b)
        want = np.linalg.solve(a, b)
        assert np.abs(x - want).max() <= 1e-10 * np.abs(want).max(), (kind, np.abs(x - want).max())


def test_ldlt_singular_systems_pseudo_inverse():
    rng = np.random.default_rng(3)
    # all-zero matrix: the k == 0 exit, x = 0
    for n in (1, 2, 9):
        f = sr.ldlt_factor(np.zeros((n, n)))
        assert f.zero_matrix == (n > 1)
        assert np.array_equal(sr.ldlt_solve(np.zeros((n, n)), rng.normal(size=n)), np.zeros(n))
    # zero diagonal, non-zero constraint rows (g = H = 0, no Tikhonov, hard rows): also the k == 0 exit
    a = np.zeros((10, 10))
    a[7:, :7] = rng.normal(size=(3, 7))
    a[:7, 7:] = a[7:, :7].T
    f = sr.ldlt_factor(a)
    assert f.zero_matrix and np.array_equal(f.transpositions, np.arange(10))
    assert np.array_equal(sr.ldlt_solve(a, rng.normal(size=10)), np.zeros(10))
    # a zero row / column inside a definite system: exactly zero there, the definite part solved exactly
    for zero in ([0], [3, 5], [8]):
        n = 9
        keep = [i for i in range(n) if i not in zero]
        A = rng.normal(size=(len(keep), len(keep)))
        sub = -(A @ A.T) - np.eye(len(keep))
        a = np.zeros((n, n))
        a[np.ix_(keep, keep)] = sub
        b = rng.normal(size=n)
        x = sr.ldlt_solve(a, b)
        assert np.all(x[zero] == 0.0)
        want = np.linalg.solve(sub, b[keep])
        assert np.abs(x[keep] - want).max() <= 1e-10 * np.abs(want).max()
    # n == 1: a zero pivot gives 0, a tiny one is still inverted
    assert sr.ldlt_solve(np.array([[0.0]]), np.array([3.0]))[0] == 0.0
    assert sr.ldlt_solve(np.array([[1e-300]]), np.array([1e-300]))[0] == 1.0
    # a NaN first in the pivot tail stays (maxCoeff keeps its first entry), a later NaN never wins
    a = np.diag([1.0, np.nan, 5.0, np.nan])
    assert sr.ldlt_factor(a).transpositions[0] == 2
    a = np.diag([np.nan, 1.0, 5.0])
    assert sr.ldlt_factor(a).transpositions[0] == 0


def gpu_shape_cases(synth):
    """(name, spec, state, g, H) of the shapes that test_gpu_structure_limits.py holds to the restatement."""
    rng = np.random.default_rng(77)
    out = []
    for name, (builder, nb) in sr.LIMIT_SHAPES.items():
        spec = builder(synth, rng, list(range(nb)))
        out.append((name, spec) + _setup(spec, nb, rng))
    for name, builder, nb in (("constrained83", sr.constrained83, 8), ("seven_unknowns", sr.seven_unknowns, 2)):
        spec = builder(synth, rng, list(range(nb)))
        out.append((name, spec) + _setup(spec, nb, rng))
    spec = sr.implicit_structure(synth, 0, 1000.0, 30000.0)
    out.append(("implicit", spec) + _setup(spec, 1, rng))
    return out


def test_gates_notice_a_missing_term(oracle, synth):
    """The theta gate of the GPU test, max(4 |theta_oracle32 - theta64|, 1e-6 |theta64|) per block (joint variations,
    multipliers), is exceeded when one term is left out of the float64 system: an active soft constraint, a hard row,
    or the Tikhonov entry of one unknown."""
    n_checked = 0
    for name, spec, state, g, H in gpu_shape_cases(synth):
        r = sr.calculate_optimization(spec, state, g, H)
        theta_o = _oracle_optimize(oracle, spec, state, g, H)[0]
        dof, n = sr.dof_of(spec), sr.n_unknowns(spec)
        gates = sr.theta_gates(theta_o, r.theta, dof)
        # the Tikhonov entry of the root's first unknown and the one that weighs most against its diagonal entry (where
        # the modality Hessians or a hard constraint outweigh it a thousandfold, float32 cannot see it either)
        tik = np.array([spec.tikhonov_rotation if d < 3 else spec.tikhonov_translation
                        for l in spec.links for d in sr.free_dirs(l)])
        heavy = int(np.argmax(tik / np.abs(np.diag(r.system.a)[:dof])))
        mutations = [dict(drop_tikhonov=0), dict(drop_tikhonov=heavy)]
        active = sorted({p[0] for p in r.system.soft_parts if p[-1]})
        mutations += [dict(drop_soft=c) for c in active[:2]]
        if n > dof:
            mutations += [dict(drop_row=0), dict(drop_row=n - dof - 1)]
        for m in mutations:
            rm = sr.calculate_optimization(spec, state, g, H, **m)
            moved = sr.theta_deviations(rm.theta, r.theta, dof)
            assert moved[0] > gates[0] or moved[1] > gates[1], (name, m, moved, gates)
            n_checked += 1
    assert n_checked >= 20
