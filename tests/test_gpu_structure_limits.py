"""The device's kinematic-structure solve (k_structure; the cluster-fused k_track) against the float64 restatement of
Optimizer::CalculateOptimization (tests/structure_reference.py) at the limits m3tb_set_structure accepts and in its
degenerate cases.

Every case feeds per-body gradients / Hessians through m3tb_set_gradient_hessian and runs three consecutive
calculate_optimization calls. Before each call the link and joint poses are read back from the device and handed to
the restatement and to the float32 oracle (mirror mode). Gates per structure and call:
  * theta, per block (joint variations, multipliers): |theta_gpu - theta64| <= max(4 |theta_oracle32 - theta64|,
    1e-6 |theta64|), i.e. no less accurate than the float32 reference arithmetic; and the mirror gate of
    test_gpu_structures.py, |theta_gpu - theta_oracle32| <= 2e-4 max|theta_oracle32|;
  * the updated link / joint poses equal the float64 Link::UpdatePoses of theta_gpu within 5e-6 (the update apart
    from the solve);
  * updated == (theta64 holds no NaN); a refused update leaves body and joint poses bit-identical.
"""
import numpy as np
import pytest

import structure_reference as sr
from helpers import pose_error, record

pytestmark = pytest.mark.gpu

TOL_POSE = 5e-6
SMEM_48K = 48 * 1024


@pytest.fixture(scope="module")
def wl64(synth):
    return synth.make_workload("c2", n_bodies=64, n_lines=16, n_points=16, n_divides=1, seed=5)


class Launch:
    """One context whose structures are `specs` (indices 0..) plus the device's implicit one-link structures for the
    unreferenced bodies, and the bookkeeping of the checks above."""

    def __init__(self, capi, oracle, synth, wl, specs, rng):
        self.oracle = oracle
        self.ctx = capi.context_from_workload(wl)
        self.nb = wl.n_bodies
        used = {b for s in specs for l in s.links for b in ((l.body,) + tuple(l.extra_bodies)) if b >= 0}
        self.implicit = [b for b in range(self.nb) if b not in used]
        self.specs = list(specs) + [sr.implicit_structure(synth, b, wl.tikhonov_rotation, wl.tikhonov_translation)
                                    for b in self.implicit]
        self.n_user = len(specs)
        for i, s in enumerate(specs):
            self.ctx.set_structure(i, s)
        self.ctx.set_poses(np.stack([sr.rand_pose(rng, 2.0, 0.3) for _ in range(self.nb)]))
        self.ctx.calculate_consistent_poses()
        self.worst = {}

    def smem_bytes(self):
        """k_structure's dynamic shared memory: sized for the largest structure of the launch"""
        return max(sr.spec_smem_bytes(s) for s in self.specs)

    def read(self, i):
        """(raw float32 body2joint, joint2parent, link2world) of structure i as the device holds them"""
        s = self.specs[i]
        if i < self.n_user:
            return self.ctx.get_link_poses(i, len(s.links))
        eye = np.eye(4, dtype=np.float32)[None, :3]
        return eye.copy(), eye.copy(), self.ctx.get_poses(s.links[0].body, 1)

    def step(self, g, H, check=None):
        """one calculate_optimization over the launch; returns [(float64 result, theta_gpu, updated)] per structure"""
        for m in range(2):
            self.ctx.set_gradient_hessian(m, g[m], H[m].reshape(self.nb, 36))
        before = [self.read(i) for i in range(len(self.specs))]
        poses_before = self.ctx.get_poses()
        states = [sr.State.from_arrays(lw, b2j, j2p) for b2j, j2p, lw in before]
        self.ctx.calculate_optimization(0, 0, 0)
        poses_after = self.ctx.get_poses()
        out = []
        for i, spec in enumerate(self.specs):
            if check is not None and i not in check:
                continue
            r = sr.calculate_optimization(spec, states[i], g, H)
            theta_g, upd = self.ctx.get_structure_theta(i)
            assert len(theta_g) == sr.n_unknowns(spec)
            assert upd == r.updated, (i, upd, np.isnan(r.theta).any())
            after = self.read(i)
            bodies = [b for l in spec.links for b in ((l.body,) + tuple(l.extra_bodies)) if b >= 0]
            if not r.updated:
                for x, y in zip(before[i][:2], after[:2]):
                    assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), i
                assert np.array_equal(poses_before[bodies].view(np.uint32), poses_after[bodies].view(np.uint32)), i
                out.append((r, theta_g, upd))
                continue
            dof = sr.dof_of(spec)
            theta_o, ok = sr.oracle_optimize(self.oracle, spec, states[i], g, H)
            assert ok == 1
            gates = sr.theta_gates(theta_o, r.theta, dof)
            dev = sr.theta_deviations(theta_g, r.theta, dof)
            dev_o = sr.theta_deviations(theta_o, r.theta, dof)
            assert dev[0] <= gates[0] and dev[1] <= gates[1], (i, dev, gates)
            scale = np.abs(theta_o).max()
            mirror = np.abs(theta_g - theta_o).max()
            assert mirror <= 2e-4 * scale + 1e-7, (i, mirror, scale)
            want = sr.update_poses(spec, states[i], theta_g)
            pose_dev = max(np.abs(after[k].reshape(-1, 12) - w[:, :3].reshape(-1, 12)).max()
                           for k, w in enumerate((want.body2joint, want.joint2parent, want.link2world)))
            assert pose_dev <= TOL_POSE, (i, pose_dev)
            for l, link in enumerate(spec.links):  # extra bodies take the link's pose, bit for bit
                for e in link.extra_bodies:
                    assert np.array_equal(poses_after[e].view(np.uint32), poses_after[link.body].view(np.uint32))
            key = "implicit" if i >= self.n_user else i
            w = self.worst.setdefault(key, dict(gpu_var=0.0, oracle_var=0.0, gpu_mult=0.0, oracle_mult=0.0, pose=0.0))
            w["gpu_var"], w["oracle_var"] = max(w["gpu_var"], dev[0]), max(w["oracle_var"], dev_o[0])
            w["gpu_mult"], w["oracle_mult"] = max(w["gpu_mult"], dev[1]), max(w["oracle_mult"], dev_o[1])
            w["pose"] = max(w["pose"], pose_dev)
            out.append((r, theta_g, upd))
        return out

    def report(self, name, **extra):
        worst = {str(k): {kk: float(f"{vv:.3e}") for kk, vv in v.items()} for k, v in self.worst.items()}
        record(name, smem_bytes=self.smem_bytes(), **extra, worst=worst)

    def close(self):
        self.ctx.close()


def _specs(synth, rng, names, first=0):
    """builders from structure_reference on consecutive bodies"""
    table = dict(sr.LIMIT_SHAPES, constrained83=(sr.constrained83, 8), seven_unknowns=(sr.seven_unknowns, 2))
    out = []
    for name in names:
        builder, nb = table[name]
        out.append(builder(synth, rng, list(range(first, first + nb))))
        first += nb
    return out


@pytest.mark.parametrize("shape", list(sr.LIMIT_SHAPES))
def test_limit_shape(capi, oracle, synth, wl64, shape):
    rng = np.random.default_rng(100 + list(sr.LIMIT_SHAPES).index(shape))
    spec = _specs(synth, rng, [shape])[0]
    run = Launch(capi, oracle, synth, wl64, [spec], rng)
    actives = []
    for it in range(3):
        g, H = sr.random_gh(rng, wl64.n_bodies, 0.2 + it)
        res = run.step(g, H)
        assert all(u for _, _, u in res)
        actives.append(sum(p[-1] for p in res[0][0].system.soft_parts))
    n = sr.n_unknowns(spec)
    if shape == "dof96_rows32":
        assert (len(spec.links), sr.dof_of(spec), n, len(spec.constraints)) == (16, 96, 128, 32)
        assert run.smem_bytes() > SMEM_48K
        parts = res[0][0].system.soft_parts
        assert any(p[-1] for p in parts) and not all(p[-1] for p in parts)
    if shape == "tree16":
        assert len(spec.links) == 16 and any(not l.fixed_body2joint_pose for l in spec.links)
    if shape == "extra3":
        assert max(len(l.extra_bodies) for l in spec.links) == 3
    if shape == "bodyless_mid":
        assert spec.links[1].body < 0 and spec.links[1].parent == 0
    if shape == "one_unknown":
        assert n == 1
    run.report(f"structure_limit_{shape}", unknowns=n, constraints=len(spec.constraints), active_soft_parts=actives)
    run.close()


@pytest.mark.parametrize("order", ["ascending", "descending"])
def test_mixed_launch(capi, oracle, synth, wl64, order):
    """1, 83, 128 and 7 unknowns in one k_structure launch, plus the implicit one-link structures of the other bodies:
    the shared memory is sized for the largest and carved per CTA."""
    rng = np.random.default_rng(61 if order == "ascending" else 62)
    names = ["one_unknown", "constrained83", "dof96_rows32", "seven_unknowns"]
    specs = _specs(synth, rng, names if order == "ascending" else names[::-1])
    run = Launch(capi, oracle, synth, wl64, specs, rng)
    assert sorted(sr.n_unknowns(s) for s in specs) == [1, 7, 83, 128] and len(run.implicit) == 64 - 27
    assert run.smem_bytes() > SMEM_48K
    for it in range(3):
        g, H = sr.random_gh(rng, wl64.n_bodies, 0.2 + it)
        res = run.step(g, H)
        assert len(res) == len(run.specs) and all(u for _, _, u in res)
    run.report(f"structure_mixed_launch_{order}", unknowns=[sr.n_unknowns(s) for s in specs],
               implicit=len(run.implicit))
    run.close()


def test_nan_and_inf_inputs(capi, oracle, synth, wl64):
    """NaN in one body's g refuses that structure's update (optimizer.cpp:165) and leaves its poses bit-identical; inf
    in H decides through the float64 restatement: at a one-unknown link it only makes the pivot -inf (theta = 0, the
    update goes through), at an implicit structure 0 * inf fills the system with NaNs (refused). The other structures of
    the launch are updated and pass the gates, and the next call with finite inputs updates everything again."""
    rng = np.random.default_rng(71)
    specs = _specs(synth, rng, ["one_unknown", "constrained83", "dof96_rows32", "seven_unknowns"])
    run = Launch(capi, oracle, synth, wl64, specs, rng)
    g, H = sr.random_gh(rng, wl64.n_bodies)
    run.step(g, H)
    # NaN in g of link 3 of the 83-unknown structure (body 1 + 3)
    g, H = sr.random_gh(rng, wl64.n_bodies)
    g[1, 4, 2] = np.nan
    res = run.step(g, H)
    status = [u for _, _, u in res]
    assert status[1] is False and np.isnan(res[1][0].theta).any()
    assert all(status[:1] + status[2:])
    # inf in H: the one-unknown structure (body 0) and the first implicit structure
    g, H = sr.random_gh(rng, wl64.n_bodies)
    bi = run.implicit[0]
    H[0, 0, 0, 0] = np.inf
    H[1, bi, 0, 0] = np.inf
    res = run.step(g, H)
    status = [u for _, _, u in res]
    k = run.n_user
    assert status[0] is True and res[0][1][0] == 0.0          # theta = b / -inf
    assert status[k] is False and np.isnan(res[k][0].theta).any()
    assert all(status[1:k] + status[k + 1:])
    # finite again: everything updates
    g, H = sr.random_gh(rng, wl64.n_bodies)
    res = run.step(g, H)
    assert all(u for _, _, u in res)
    run.report("structure_nan_inf", refused_nan_g=1, refused_inf_h=1, inf_pivot_updated=1)
    run.close()


def test_zero_system(capi, oracle, synth, wl64):
    """g = H = 0 and both Tikhonov parameters 0: the all-zero diagonal takes Eigen's zero-matrix exit (k == 0,
    pivot invalid), without constraints and with hard constraint rows. theta is exactly 0, the update goes through and
    the poses are UpdatePoses(0)."""
    rng = np.random.default_rng(81)
    tree, chain = _specs(synth, rng, ["tree16", "constrained83"])
    tree.constraints = []
    for s in (tree, chain):
        s.tikhonov_rotation = s.tikhonov_translation = 0.0
    run = Launch(capi, oracle, synth, wl64, [tree, chain], rng)
    z = np.zeros((2, wl64.n_bodies, 6), np.float32), np.zeros((2, wl64.n_bodies, 6, 6), np.float32)
    for it in range(3):
        res = run.step(*z)
        for i in range(2):
            r, theta_g, upd = res[i]
            assert r.factorization.zero_matrix and upd
            assert np.all(theta_g == 0.0) and np.all(r.theta == 0.0)
        assert np.all(np.diag(res[1][0].system.a) == 0.0) and np.abs(res[1][0].system.a[48:, :48]).max() > 0.1
    run.report("structure_zero_matrix", structures=["tree16 without constraints", "constrained83 (35 hard rows)"])
    run.close()


def test_singular_system_pseudo_inverse(capi, oracle, synth, wl64):
    """Translation Tikhonov 0 and a leaf link whose modality Hessians have a zero translation block: the leaf's three
    translation unknowns get all-zero rows, LDLT's D has exact zeros there and the pseudo-inverse sets them to 0; the
    other unknowns pass the gates."""
    rng = np.random.default_rng(91)
    links = [synth.LinkSpec(body=0, parent=-1, body2joint=sr.rand_pose(rng, 0.3, 0.02), joint2parent=synth.identity_pose()),
             synth.LinkSpec(body=1, parent=0, body2joint=sr.rand_pose(rng, 0.3, 0.02), joint2parent=sr.rand_pose(rng, 0.5, 0.04)),
             synth.LinkSpec(body=2, parent=1, body2joint=sr.rand_pose(rng, 0.3, 0.02), joint2parent=sr.rand_pose(rng, 0.5, 0.04),
                            fixed_body2joint_pose=False)]
    spec = synth.StructureSpec(links=links, tikhonov_rotation=100.0, tikhonov_translation=0.0)
    run = Launch(capi, oracle, synth, wl64, [spec], rng)
    leaf_t = [15, 16, 17]
    for it in range(3):
        g, H = sr.random_gh(rng, wl64.n_bodies, 0.2 + it)
        H[:, 2, 3:, :] = 0.0
        H[:, 2, :, 3:] = 0.0
        r, theta_g, upd = run.step(g, H, check={0})[0]
        assert upd
        d = np.abs(np.diag(r.factorization.mat))
        assert (d == 0.0).sum() == 3
        assert np.all(r.theta[leaf_t] == 0.0) and np.all(theta_g[leaf_t] == 0.0)
        assert np.all(np.delete(theta_g, leaf_t) != 0.0)
    run.report("structure_pseudo_inverse", zero_pivots=3, zeroed_unknowns=leaf_t)
    run.close()


def _cluster_limit_structure(synth, wl, chain):
    """The chain's constrained shape (8 six-DoF links, 7 constraints of 5 rows) with 9 of its constraints repeated:
    48 DoF + 80 hard rows = 128 unknowns, the largest system a cluster of 8 CTAs can be handed. The repeated rows are
    bit-identical copies, so the multipliers' split between copies is decided by rounding - but the same rounding on
    both paths, whose per-body sums agree bit for bit with at most 256 lines / points per body."""
    import copy
    spec = copy.deepcopy(wl.structures[chain])
    base = [c for c in spec.constraints if not c.soft]
    spec.constraints = base + [copy.deepcopy(base[k % len(base)]) for k in range(9)]
    return spec


def test_cluster_fused_solve_at_128_unknowns(capi, synth, monkeypatch):
    wl = synth.make_chain_workload(n_chains=2, n_links=8, n_lines=200, n_points=200, n_divides=2, variant="constrained",
                                   seed=8)
    wl.structures = [_cluster_limit_structure(synth, wl, c) for c in range(2)]
    spec = wl.structures[0]
    assert (sr.dof_of(spec), sr.n_unknowns(spec), len(spec.constraints)) == (48, 128, 16)
    smem = sr.spec_smem_bytes(spec)
    assert smem > SMEM_48K
    monkeypatch.setenv("M3TB_CLUSTER", "1")   # read at context creation
    ctx_a = capi.context_from_workload(wl)
    monkeypatch.delenv("M3TB_CLUSTER")
    ctx_b = capi.context_from_workload(wl)
    for c in (ctx_a, ctx_b):
        c.start_modalities(0)
    la, lb = ctx_a.launch_count, ctx_b.launch_count
    ctx_a.corr_iteration(0, 0, wl.n_update_iterations)
    ctx_b.corr_iteration(0, 0, wl.n_update_iterations)
    launch = ctx_a.last_launch()
    assert launch["kernel"] == "k_track_cluster" and ctx_a.launch_count - la == 1, launch
    assert ctx_b.launch_count - lb == 2 * wl.n_update_iterations
    dt, dr = pose_error(ctx_a.get_poses(), ctx_b.get_poses())
    assert dt.max() < 1e-5 and dr.max() < 1e-4, (dt.max(), dr.max())
    worst = 0.0
    for i in range(2):
        ta, ua = ctx_a.get_structure_theta(i)
        tb, ub = ctx_b.get_structure_theta(i)
        assert len(ta) == 128 and ua and ub
        dev = np.abs(ta - tb).max()
        assert dev <= 1e-3 * np.abs(tb).max(), (i, dev, np.abs(tb).max())
        worst = max(worst, dev / np.abs(tb).max())
    record("structure_cluster_128", kernel=launch["kernel"], struct_smem_bytes=smem,
           dyn_smem_bytes=32768 + (smem + 127) // 128 * 128, theta_rel_dev=float(f"{worst:.3e}"),
           pose_m=float(f"{dt.max():.3e}"), pose_rad=float(f"{dr.max():.3e}"))
    ctx_a.close()
    ctx_b.close()
