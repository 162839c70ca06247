"""m3tb_score_poses / m3tb_calculate_diameters / the reduced evaluation sets against the CPU restatement
(pose_score_oracle.cpp): bit-equal ADD, ADD-S, translation error, curves, AUCs and diameters; the rotation error within
acosf's ulp bound."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import pose_score_oracle as pso

pytestmark = pytest.mark.gpu

FIELDS = ["add_error", "adds_error", "add_auc", "adds_auc", "translation_error", "rotation_error", "tracking_success"]
ROTATION_ULPS = 4  # CUDA's acosf is within 2 ulp of the exact value, glibc's within 1; the argument is bit-equal


def mesh(n, seed, scale=0.1):
    return (np.random.default_rng(seed).standard_normal((n, 3)) * scale).astype(np.float32)


def poses(n, rng, rot=0.5, trans=0.3):
    out = np.zeros((n, 3, 4), np.float32)
    out[:, :, :3] = Rotation.from_rotvec(rng.normal(0, rot, (n, 3))).as_matrix()
    out[:, :, 3] = rng.normal(0, trans, (n, 3))
    return out


def perturb(p, rng, rot=0.05, trans=0.02):
    q = p.copy()
    d = Rotation.from_rotvec(rng.normal(0, rot, (len(p), 3))).as_matrix().astype(np.float32)
    q[:, :, :3] = np.einsum("nij,njk->nik", d, p[:, :, :3])
    q[:, :, 3] += rng.normal(0, trans, (len(p), 3))
    return q


def bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def check(ctx, bodies, models, model_of, gt, g2b=None, params=None, out=None):
    """Oracle results of `bodies` with the device's current poses, compared with the device's `out`."""
    p = params or {}
    kw = dict(threshold_max=p.get("threshold_max", 0.1), curve_scale=p.get("curve_scale", 1.0),
              auc_scale=p.get("auc_scale", 1.0))
    pose = ctx.get_poses(0, int(max(bodies)) + 1).reshape(-1, 3, 4)
    res, ca, cs = out
    for q, b in enumerate(bodies):
        m = model_of[b]
        r, ra, rs = pso.score_pose(models[m][0], models[m][1], pose[b], gt[q], None if g2b is None else g2b[b], **kw)
        for k, f in enumerate(FIELDS):
            if f == "rotation_error":
                x, y = np.float32(res[f][q]), r[k]
                assert (np.isnan(x) and np.isnan(y)) or abs(x - y) <= ROTATION_ULPS * np.spacing(max(abs(y), 1e-30)), (q, x, y)
            elif f == "tracking_success":
                near = abs(r[5] - pso.ROTATION_THRESHOLD) <= ROTATION_ULPS * np.spacing(pso.ROTATION_THRESHOLD)
                assert near or res[f][q] == r[k], (q, res[f][q], r[k])
            else:
                assert bits_equal(res[f][q], r[k]), (q, f, res[f][q], r[k])
        assert bits_equal(ca[q], ra) and bits_equal(cs[q], rs), q


def make_context(capi, n_bodies, n_models):
    return capi.Context(0, max_bodies=n_bodies, max_cameras=1, max_models=n_models)


@pytest.mark.parametrize("n,n_eval", [(1, 0), (5, 5), (2000, -1), (2000, 1000), (20000, 1000), (100000, 1000),
                                      (3, 10)])
def test_reduced_sets_equal_the_oracle(capi, n, n_eval):
    ctx = make_context(capi, 1, 1)
    v = mesh(n, n)
    ctx.set_evaluation_model(0, v, n_eval)
    assert bits_equal(ctx.get_evaluation_vertices(0), pso.reduce_vertices(v, n_eval))


@pytest.mark.parametrize("sizes,n_eval,n_bodies", [
    ((1, 7, 300), 0, 6),             # every vertex, tiny meshes
    ((2000, 513), 1000, 40),         # reduced sets, two models shared by many bodies
    ((20000,), 1000, 3),             # few bodies: the full set is searched in slices
    ((100000, 2000), 1000, 4),
    ((4000,), 4000, 300),            # n_vertices_evaluation == n
])
def test_scores_equal_the_oracle(capi, sizes, n_eval, n_bodies):
    rng = np.random.default_rng(sum(sizes) + n_bodies)
    ctx = make_context(capi, n_bodies, len(sizes))
    models = []
    for m, n in enumerate(sizes):
        v = mesh(n, 10 * m + n)
        ctx.set_evaluation_model(m, v, n_eval)
        models.append((pso.reduce_vertices(v, n_eval), v))
    model_of = rng.integers(0, len(sizes), n_bodies)
    for b in range(n_bodies):
        ctx.set_body_evaluation_model(b, int(model_of[b]))
    gt = poses(n_bodies, rng)
    est = perturb(gt, rng)
    est[::5] = perturb(gt[::5], rng, rot=0.002, trans=0.001)  # some near and below the thresholds
    ctx.set_poses(est)
    bodies = rng.permutation(n_bodies)
    out = ctx.score_poses(bodies, gt[bodies])
    check(ctx, bodies, models, model_of, gt[bodies], out=out)
    assert 0 < out[0]["tracking_success"].sum() < n_bodies or n_bodies < 10


def test_opt_geometry2body_and_diameter_scale(capi):
    rng = np.random.default_rng(11)
    n_bodies = 8
    ctx = make_context(capi, n_bodies, 1)
    v = mesh(3000, 12)
    ctx.set_evaluation_model(0, v, 1000)
    models = [(pso.reduce_vertices(v, 1000), v)]
    g2b = poses(n_bodies, rng, rot=1.0, trans=0.05)
    for b in range(n_bodies):
        ctx.set_body_evaluation_model(b, 0, g2b[b])
    d = ctx.calculate_diameters([0])[0]
    assert bits_equal(d, pso.diameter(v))
    gt = poses(n_bodies, rng)
    ctx.set_poses(perturb(gt, rng, rot=0.02, trans=0.01))
    params = dict(threshold_max=0.2, curve_scale=float(d), auc_scale=0.2)
    bodies = np.arange(n_bodies)
    out = ctx.score_poses(bodies, gt, capi.score_params(**params))
    check(ctx, bodies, models, [0] * n_bodies, gt, g2b=g2b, params=params, out=out)


@pytest.mark.parametrize("sizes", [(1, 2, 3), (511, 512, 513, 1025), (100000,)])
def test_diameters_equal_the_oracle(capi, sizes):
    ctx = make_context(capi, 1, len(sizes))
    vs = [mesh(n, n + 1) for n in sizes]
    for m, v in enumerate(vs):
        ctx.set_evaluation_model(m, v, 0)
    d = ctx.calculate_diameters(list(range(len(sizes)))[::-1])
    ref = [pso.diameter(v) for v in vs][::-1]
    assert bits_equal(d, ref), (d, ref)


def test_device_ground_truth_and_device_outputs(capi):
    import torch
    rng = np.random.default_rng(13)
    n_bodies = 20
    ctx = make_context(capi, n_bodies, 1)
    v = mesh(5000, 14)
    ctx.set_evaluation_model(0, v, 1000)
    for b in range(n_bodies):
        ctx.set_body_evaluation_model(b, 0)
    gt = poses(n_bodies, rng)
    ctx.set_poses(perturb(gt, rng))
    host = ctx.score_poses(np.arange(n_bodies), gt)
    dev = ctx.score_poses(np.arange(n_bodies), torch.from_numpy(gt).cuda())
    assert all(bits_equal(host[0][f], dev[0][f]) for f in FIELDS)
    launches = ctx.launch_count
    for bad in (torch.from_numpy(gt).double().cuda(), torch.from_numpy(gt[:-1]).cuda()):  # wrong dtype, too few poses
        with pytest.raises(capi.M3TBError):
            ctx.score_poses(np.arange(n_bodies), bad)
    assert ctx.launch_count == launches
    out = torch.zeros((n_bodies, 7), dtype=torch.float32, device="cuda")
    ca = torch.zeros((n_bodies, 100), dtype=torch.float32, device="cuda")
    cs = torch.zeros((n_bodies, 100), dtype=torch.float32, device="cuda")
    g = torch.from_numpy(gt).cuda()
    ctx.score_poses_to(np.arange(n_bodies), g.data_ptr(), 1, out.data_ptr(), ca.data_ptr(), cs.data_ptr())
    ctx.synchronize()
    rec = out.cpu().numpy().view(capi.POSE_SCORE_DTYPE).reshape(-1)
    assert all(bits_equal(host[0][f], rec[f]) for f in FIELDS)
    assert bits_equal(host[1], ca.cpu().numpy()) and bits_equal(host[2], cs.cpu().numpy())
    check(ctx, list(range(n_bodies)), [(pso.reduce_vertices(v, 1000), v)], [0] * n_bodies, gt, out=host)


def test_scoring_right_after_a_tracking_step(capi, synth):
    wl = synth.make_workload("c2", n_bodies=4, n_divides=2, seed=3)
    ctx = capi.context_from_workload(wl, device=0)
    rng = np.random.default_rng(15)
    v = mesh(2000, 16)
    ctx.set_evaluation_model(0, v, 500)
    for b in range(wl.n_bodies):
        ctx.set_body_evaluation_model(b, 0)
    gt = poses(wl.n_bodies, rng)
    ctx.start_modalities(0)
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    out = ctx.score_poses(np.arange(wl.n_bodies), gt)  # no synchronisation in between
    check(ctx, list(range(wl.n_bodies)), [(pso.reduce_vertices(v, 500), v)], [0] * wl.n_bodies, gt, out=out)


def test_nan_and_infinite_poses_and_acos_above_one(capi):
    """Bodies 0, 1: NaN poses; 3: ground truth 1e30 m away (every squared distance overflows); 4: an infinite
    ground-truth translation. As in nanoflann, their moved vertices are never added to the result set and keep FLT_MAX:
    ADD-S is sqrt(FLT_MAX), finite, with AUC 0 and a zero curve. Body 2: an acos argument above 1."""
    n = 5
    ctx = make_context(capi, n, 1)
    v = mesh(700, 17)
    ctx.set_evaluation_model(0, v, 0)
    for b in range(n):
        ctx.set_body_evaluation_model(b, 0)
    rng = np.random.default_rng(18)
    gt = poses(n, rng)
    est = perturb(gt, rng)
    est[0, 1, 3] = np.nan
    est[1, 0, 0] = np.nan
    for k in range(1, 400):  # body 2: scored against itself at an angle whose float trace exceeds 3
        R = Rotation.from_rotvec([0.0, 0.0, 1e-4 * k]).as_matrix()
        p = np.zeros((3, 4), np.float32)
        p[:, :3] = R
        if np.isnan(pso.score_pose(v[:3], v[:3], p, p)[0][5]):
            break
    est[2] = gt[2] = p
    gt[3, :, 3] = (1e30, -2e30, 0.5)
    gt[4, 0, 3] = np.inf
    ctx.set_poses(est)
    out = ctx.score_poses(np.arange(n), gt)
    check(ctx, list(range(n)), [(v, v)], [0] * n, gt, out=out)
    res = out[0]
    root_max = np.sqrt(np.float32(np.finfo(np.float32).max))
    for b in (0, 1, 3, 4):
        assert np.isfinite(res["adds_error"][b]) and res["adds_error"][b] == pytest.approx(root_max, rel=1e-3), b
        assert res["adds_auc"][b] == 0.0 and (out[2][b] == 0).all(), b
    assert np.isnan(res["add_auc"][:2]).all() and (out[1][:2] == 0).all()
    assert (res["tracking_success"][:3] == 1).all() and res["tracking_success"][3] == 0
    assert np.isnan(res["rotation_error"][2]) and res["add_error"][2] < 1e-6


def test_refusals_change_nothing(capi):
    ctx = make_context(capi, 2, 2)
    v = mesh(100, 19)
    ctx.set_evaluation_model(0, v, 10)
    ctx.set_body_evaluation_model(0, 0)
    gt = poses(2, np.random.default_rng(20))
    ctx.set_poses(gt[::-1].copy())
    before = ctx.score_poses([0], gt[:1])
    bad_v = v.copy()
    bad_v[3, 1] = np.inf
    for call in (lambda: ctx.set_evaluation_model(2, v, 0),           # not dense
                 lambda: ctx.set_evaluation_model(0, bad_v, 0),       # non-finite vertex
                 lambda: ctx.set_evaluation_model(-1, v, 0),
                 lambda: ctx.set_body_evaluation_model(0, 1),         # model 1 not set
                 lambda: ctx.set_body_evaluation_model(2, 0),         # body out of range
                 lambda: ctx.score_poses([1], gt[:1]),                # body 1 has no model
                 lambda: ctx.score_poses([2], gt[:1]),
                 lambda: ctx.score_poses([0], gt[:1], capi.score_params(threshold_max=0.0)),
                 lambda: ctx.score_poses([0], gt[:1], capi.score_params(curve_scale=float("nan"))),
                 lambda: ctx.calculate_diameters([1])):
        launches = ctx.launch_count
        with pytest.raises(capi.M3TBError):
            call()
        assert ctx.launch_count == launches
    assert bits_equal(ctx.get_evaluation_vertices(0), pso.reduce_vertices(v, 10))
    after = ctx.score_poses([0], gt[:1])
    assert all(bits_equal(before[0][f], after[0][f]) for f in FIELDS)


def test_failed_allocations_leave_the_context_as_it_was(capi):
    ctx = make_context(capi, 4, 2)
    v = mesh(3000, 21)
    ctx.set_evaluation_model(0, v, 1000)
    for b in range(4):
        ctx.set_body_evaluation_model(b, 0)
    gt = poses(4, np.random.default_rng(22))
    ctx.set_poses(gt)
    live = capi.debug_resources()
    for k in (1, 2):  # the two buffers of a new model
        capi.debug_resources(k)
        with pytest.raises(capi.M3TBError):
            ctx.set_evaluation_model(1, mesh(50, 23), 0)
        capi.debug_resources(0)
        assert capi.debug_resources() == live
    with pytest.raises(capi.M3TBError):
        ctx.set_body_evaluation_model(0, 1)  # model 1 was never stored
    capi.debug_resources(1)  # the first scratch buffer of a scoring call
    with pytest.raises(capi.M3TBError):
        ctx.score_poses(np.arange(4), gt)
    capi.debug_resources(0)
    assert capi.debug_resources() == live
    out = ctx.score_poses(np.arange(4), gt)
    check(ctx, list(range(4)), [(pso.reduce_vertices(v, 1000), v)], [0] * 4, gt, out=out)
