"""GPU parity for kinematic structures (SURVEY §8 a13-a16, BASELINE config 5): k_structure + the k_track phases around
it, through the C ABI, against the CPU oracle.

  * Optimizer::CalculateOptimization alone (random link trees, constraints, soft constraints, injected gradients):
    theta and every pose against the oracle in mirror mode (same expressions and summation order) - differences
    come only from atan2f / tanf / sinf.
  * config-5 chains (projected and constrained), pose after every correspondence iteration within 1e-4 m / 1e-4 rad
    of the reference-faithful oracle on identical inputs (body poses AND joint poses re-synchronised per iteration).
The reference has no known answers for this part: parity is against the oracle only (see oracle/m3t_oracle.h).
"""
import copy

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from helpers import pose_error

pytestmark = pytest.mark.gpu

TOL_POSE_M = 1e-4
TOL_POSE_RAD = 1e-4


def _rand_pose(rng, angle=1.0, trans=0.1):
    rv = rng.normal(size=3)
    rv *= rng.uniform(0, angle) / np.linalg.norm(rv)
    p = np.zeros((3, 4), np.float32)
    p[:, :3] = Rotation.from_rotvec(rv).as_matrix()
    p[:, 3] = rng.normal(size=3) * trans
    return p


@pytest.fixture(scope="module")
def wl_small(synth):
    return synth.make_chain_workload(n_chains=1, n_links=8, n_lines=32, n_points=32, n_divides=1, seed=1)


def _random_structures(synth, rng):
    """A few structure shapes over bodies 0..7: chains, a branching tree with a body-less fixed base, constraints."""
    I = synth.identity_pose
    out = []
    # (a) serial chain, mixed joint types, non-identity body2joint, one link that varies body2joint
    links = [synth.LinkSpec(body=0, parent=-1, body2joint=_rand_pose(rng, 0.3, 0.02), joint2parent=I())]
    for j in range(1, 8):
        free = [(1, 0, 0, 0, 0, 0), (0, 1, 0, 0, 0, 0), (0, 0, 1, 1, 0, 0), (1, 1, 1, 0, 0, 0)][j % 4]
        links.append(synth.LinkSpec(body=j, parent=j - 1, body2joint=_rand_pose(rng, 0.3, 0.02),
                                    joint2parent=_rand_pose(rng, 0.8, 0.05), free_directions=free,
                                    fixed_body2joint_pose=(j != 3)))
    out.append(synth.StructureSpec(links=links, tikhonov_rotation=100.0, tikhonov_translation=1000.0))
    # (b) fixed body-less base, two branches, hard constraint closing a loop + a soft constraint
    links = [synth.LinkSpec(body=-1, parent=-1, body2joint=I(), joint2parent=I(), free_directions=(0,) * 6,
                            link2world=_rand_pose(rng, 1.0, 0.3)),
             synth.LinkSpec(body=0, parent=0, body2joint=I(), joint2parent=_rand_pose(rng)),
             synth.LinkSpec(body=1, parent=1, body2joint=I(), joint2parent=_rand_pose(rng), free_directions=(1, 1, 0, 0, 0, 1)),
             synth.LinkSpec(body=2, parent=0, body2joint=_rand_pose(rng, 0.2, 0.01), joint2parent=_rand_pose(rng)),
             synth.LinkSpec(body=3, parent=3, body2joint=I(), joint2parent=_rand_pose(rng), free_directions=(0, 0, 1, 0, 0, 0))]
    cons = [synth.ConstraintSpec(link1=2, link2=4, body12joint1=_rand_pose(rng), body22joint2=_rand_pose(rng),
                                 directions=(1, 0, 1, 1, 1, 0)),
            synth.ConstraintSpec(link1=1, link2=3, body12joint1=_rand_pose(rng), body22joint2=_rand_pose(rng),
                                 directions=(1, 1, 1, 1, 1, 1), soft=True, max_distance_rotation=0.05,
                                 max_distance_translation=0.01, standard_deviation_rotation=0.1,
                                 standard_deviation_translation=0.02)]
    out.append(synth.StructureSpec(links=links, constraints=cons))
    # (c) optimization_time.cpp's constrained shape: 8 free links below the root, 7 x 5 constraint rows (83 x 83)
    links = [synth.LinkSpec(body=0, parent=-1, body2joint=I(), joint2parent=I())]
    cons = []
    for j in range(1, 8):
        links.append(synth.LinkSpec(body=j, parent=0, body2joint=I(), joint2parent=_rand_pose(rng, 0.5, 0.05)))
        cons.append(synth.ConstraintSpec(link1=j - 1, link2=j, body12joint1=synth.translation_pose(-0.01),
                                         body22joint2=I(), directions=(0, 1, 1, 1, 1, 1)))
    out.append(synth.StructureSpec(links=links, constraints=cons, tikhonov_rotation=100.0, tikhonov_translation=1000.0))
    return out


def test_calculate_optimization_matches_oracle(capi, oracle, synth, wl_small):
    L = oracle.lib()
    rng = np.random.default_rng(21)
    ctx = capi.context_from_workload(wl_small)
    nb = wl_small.n_bodies
    for spec in _random_structures(synth, rng):
        for rep in range(2):
            ctx.clear_structures()
            ctx.set_structure(0, spec)
            poses = np.stack([_rand_pose(rng, 2.0, 0.3) for _ in range(nb)])
            ctx.set_poses(poses)
            so = oracle.OracleStructure(copy.deepcopy(spec))
            S = so.as_struct()
            nl = len(spec.links)
            l2w = np.zeros((nl, 12), np.float32)
            for i, l in enumerate(spec.links):
                l2w[i] = (poses[l.body] if l.body >= 0 else l.link2world).reshape(12)
            # make the start consistent on both sides (Optimizer::SetUp / CalculateConsistentPoses)
            L.orc_structure_consistent_poses(S, oracle.EXP_RODRIGUES, oracle.ptr(l2w))
            ctx.calculate_consistent_poses()
            b2j, j2p, lw = ctx.get_link_poses(0, nl)
            assert np.allclose(lw.reshape(nl, 12), l2w, atol=2e-6)
            # gradients / Hessians of the two modalities (negative semi-definite Hessians like the real ones)
            g = np.zeros((2, nb, 6), np.float32)
            H = np.zeros((2, nb, 36), np.float32)
            for m in range(2):
                for b in range(nb):
                    A = rng.normal(size=(6, 6)) * np.array([30, 30, 30, 300, 300, 300])[:, None] * (0.2 + rep)
                    H[m, b] = -(A @ A.T).astype(np.float32).reshape(36)
                    g[m, b] = rng.normal(size=6) * np.array([3, 3, 3, 30, 30, 30]) * (0.2 + rep)
                ctx.set_gradient_hessian(m, g[m], H[m])
            gl = np.zeros((nl, 6), np.float32)
            Hl = np.zeros((nl, 36), np.float32)
            for i, l in enumerate(spec.links):
                if l.body >= 0:
                    gl[i] = np.float32(0) + g[0, l.body] + g[1, l.body]
                    Hl[i] = np.float32(0) + H[0, l.body] + H[1, l.body]
            n = spec.dof + spec.n_constraint_rows
            theta_o = np.zeros(n, np.float32)
            for it in range(3):  # three consecutive updates (joint poses evolve on the device)
                ok = L.orc_optimize_structure(S, oracle.ptr(gl), oracle.ptr(Hl), oracle.ROTATION_LINEAR,
                                              oracle.EXP_RODRIGUES, oracle.ptr(l2w), oracle.ptr(theta_o))
                assert ok == 1
                ctx.calculate_optimization(0, 0, it)
                theta_g, updated = ctx.get_structure_theta(0)
                assert updated and len(theta_g) == n
                scale = np.abs(theta_o).max()
                assert np.abs(theta_g - theta_o).max() <= 2e-4 * scale + 1e-7, (it, np.abs(theta_g - theta_o).max(), scale)
                b2j, j2p, lw = ctx.get_link_poses(0, nl)
                ob2j, oj2p = so.joint_poses()
                assert np.allclose(lw.reshape(nl, 12), l2w, atol=5e-6), np.abs(lw.reshape(nl, 12) - l2w).max()
                assert np.allclose(b2j, ob2j, atol=5e-6) and np.allclose(j2p, oj2p, atol=5e-6)
    ctx.close()


def test_constraint_convergence_on_device(capi, oracle, synth, wl_small):
    """examples/constraint_convergence.cpp on the GPU path: the violation of a fully constrained joint vanishes."""
    rng = np.random.default_rng(23)
    ctx = capi.context_from_workload(wl_small)
    nb = wl_small.n_bodies
    z6, z36 = np.zeros((nb, 6), np.float32), np.zeros((nb, 36), np.float32)
    for m in range(2):
        ctx.set_gradient_hessian(m, z6, z36)
    for run in range(5):
        b12j1, b22j2 = _rand_pose(rng, 1.0), _rand_pose(rng, 1.0)
        T = lambda p: np.vstack([np.asarray(p, np.float64), [0, 0, 0, 1]])
        j2p = (np.linalg.inv(T(b12j1)) @ T(_rand_pose(rng, 0.8, 0.2)))[:3].astype(np.float32)
        links = [synth.LinkSpec(body=0, parent=-1, body2joint=synth.identity_pose(), joint2parent=synth.identity_pose()),
                 synth.LinkSpec(body=1, parent=0, body2joint=b22j2, joint2parent=j2p)]
        spec = synth.StructureSpec(links=links, constraints=[synth.ConstraintSpec(
            link1=0, link2=1, body12joint1=b12j1, body22joint2=b22j2, directions=(1, 1, 1, 1, 1, 1))])
        ctx.clear_structures()
        ctx.set_structure(0, spec)
        ctx.set_poses(np.stack([_rand_pose(rng, 2.0, 0.3) for _ in range(nb)]))
        ctx.calculate_consistent_poses()
        errs = []
        for it in range(6):
            _, j2p_now, _ = ctx.get_link_poses(0, 2)
            err = T(b12j1) @ T(j2p_now[1])
            errs.append(max(np.linalg.norm(Rotation.from_matrix(err[:3, :3]).as_rotvec()), np.linalg.norm(err[:3, 3])))
            ctx.calculate_optimization(0, 0, it)
        assert errs[0] > 1e-2 and errs[-1] < 1e-5, errs
    ctx.close()


def _resync(ctx, orc, wl):
    """Identical inputs for the next iteration: body poses and joint poses of the oracle on the device."""
    for i, so in enumerate(orc.structure_objs):
        spec = copy.deepcopy(so.spec)
        b2j, j2p = so.joint_poses()
        for k, l in enumerate(spec.links):
            l.body2joint, l.joint2parent = b2j[k], j2p[k]
        ctx.set_structure(i, spec)
    ctx.set_poses(orc.get_poses())


@pytest.mark.parametrize("variant,soft", [("projected", False), ("constrained", False), ("constrained", True)])
def test_chain_pose_parity_per_iteration(capi, oracle, synth, variant, soft):
    """BASELINE config-5 shape: 8-link chains, RTB-shape parameters; the contract gate per correspondence iteration."""
    wl = synth.make_chain_workload(n_chains=3, n_links=8, n_lines=300, n_points=300, n_divides=4, variant=variant,
                                   soft=soft, seed=4)
    ctx = capi.context_from_workload(wl)
    assert ctx.n_structures() == 3
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_POLAR, exp_mode=oracle.EXP_PADE)
    orc.start_modalities(0)
    ctx.start_modalities(0)
    for corr in range(wl.n_corr_iterations):
        _resync(ctx, orc, wl)
        ctx.corr_iteration(0, corr, wl.n_update_iterations)
        orc.tracking_step(0, n_corr=corr + 1, corr_begin=corr)
        dt, dr = pose_error(ctx.get_poses(), orc.get_poses())
        assert dt.max() < TOL_POSE_M and dr.max() < TOL_POSE_RAD, (variant, corr, dt.max(), dr.max())
        for i, so in enumerate(orc.structure_objs):
            b2j, j2p, _ = ctx.get_link_poses(i, 8)
            ob2j, oj2p = so.joint_poses()
            assert np.abs(j2p - oj2p).max() < 1e-4 and np.abs(b2j - ob2j).max() < 1e-4
    ctx.close()


def test_chain_tracking_free_running(capi, oracle, synth):
    """Whole cycle free-running on both sides. With RTB's weak regularisation (lambda 100 / 1000) and 19 x 9 px lines
    the chain iteration is strongly expanding in its first steps (the oracle's own rotation error triples before it
    collapses, tests/diag/chain_free_running.py), so a 1e-7 difference in summation order grows to ~1e-5 m / 2e-3 rad within
    the first frame and further in the next one: the gate for parity is the per-iteration test above; here the
    first frame must stay within a loose band and both sides must converge towards the ground truth."""
    wl = synth.make_chain_workload(n_chains=4, n_links=8, n_lines=300, n_points=300, n_divides=4, seed=6)
    ctx = capi.context_from_workload(wl)
    orc = oracle.OracleTracker(wl)
    orc.start_modalities(0)
    ctx.start_modalities(0)
    e0t, e0r = pose_error(wl.start_body2world, wl.gt_body2world)
    for it in range(2):
        ctx.tracking_step(it, wl.n_corr_iterations, wl.n_update_iterations)
        ctx.calculate_results(it)
        orc.tracking_step(it)
        orc.calculate_results(it)
        if it == 0:
            dt, dr = pose_error(ctx.get_poses(), orc.get_poses())
            assert np.median(dt) < TOL_POSE_M and np.median(dr) < 5 * TOL_POSE_RAD, (dt, dr)
            assert dt.max() < 1e-3 and dr.max() < 2e-2, (dt, dr)
    for poses in (ctx.get_poses(), orc.get_poses()):
        e1t, e1r = pose_error(poses, wl.gt_body2world)
        assert np.median(e1t) < 0.4 * np.median(e0t) and np.median(e1r) < 0.4 * np.median(e0r), (e0t, e1t, e0r, e1r)
    ctx.close()


def test_rigid_bodies_through_structure_path(capi, synth):
    """A context with one declared structure runs every body through k_structure (implicit one-link structures for
    the rest); a free root link with body2joint = identity is the rigid-body optimiser of the fused kernel."""
    wl = synth.make_workload("c2", n_bodies=4, n_divides=3, seed=3)
    ctx_a = capi.context_from_workload(wl)
    ctx_b = capi.context_from_workload(wl)
    spec = synth.StructureSpec(links=[synth.LinkSpec(body=0, parent=-1, body2joint=synth.identity_pose(),
                                                     joint2parent=synth.identity_pose())],
                               tikhonov_rotation=wl.tikhonov_rotation, tikhonov_translation=wl.tikhonov_translation)
    ctx_b.set_structure(0, spec)
    for c in (ctx_a, ctx_b):
        c.start_modalities(0)
        c.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    pa, pb = ctx_a.get_poses(), ctx_b.get_poses()
    dt, dr = pose_error(pa, pb)
    # the two paths sum g / H in different orders (k_track2's two warp groups vs k_track + k_structure): equal to float
    # rounding, except where that rounding flips a discrete event of the free-running step (test_free_running_*)
    assert np.median(dt) < 2e-6 and np.median(dr) < 2e-6, (dt, dr)
    assert dt.max() < 3e-3 and dr.max() < 2e-2, (dt, dr)
    ctx_a.close()
    ctx_b.close()


def test_reset_joint_poses_keeps_other_structures_defaults(capi, synth):
    """Link::ResetJointPoses restores each link's OWN defaults (link.cpp:243-246): re-declaring structure 1 after
    tracking must not turn structure 0's tracked joint poses into its defaults (ADVICE r01)."""
    wl = synth.make_chain_workload(n_chains=2, n_links=4, n_lines=100, n_points=100, n_divides=2, seed=3)
    ctx = capi.context_from_workload(wl)
    ctx.start_modalities(0)
    _, j2p_default, _ = ctx.get_link_poses(0, 4)
    ctx.tracking_step(0, 2, 2)
    _, j2p_tracked, _ = ctx.get_link_poses(0, 4)
    assert np.abs(j2p_tracked - j2p_default).max() > 1e-6          # the joints moved
    ctx.set_structure(1, wl.structures[1])                          # touch the OTHER structure
    ctx.reset_joint_poses()
    _, j2p_reset, _ = ctx.get_link_poses(0, 4)
    assert np.array_equal(j2p_reset.view(np.uint32), j2p_default.view(np.uint32))
    ctx.close()
