"""The group-cooperative closest-view search of k_track2 (ClosestViewPrunedGroup) against the oracle's full scan, in the
shapes tests/test_gpu_views.py does not reach: the 512-thread kernel (region-only and depth-only batches), cluster
tables read from global memory (more than 96 clusters), and exact ties between views split over different warps."""
import dataclasses

import numpy as np
import pytest

from test_gpu_views import _random_poses

pytestmark = pytest.mark.gpu


def _check_views(capi, oracle, wl, pose_sets):
    """One correspondence launch per pose set; every body's views equal the oracle's full scan. Returns the views."""
    ctx = capi.context_from_workload(wl)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    found = []
    for rep, poses in enumerate(pose_sets):
        ctx.set_poses(poses)
        orc.set_poses(poses)
        if wl.region:
            ctx.region_correspondences(0, 0)
        if wl.depth:
            ctx.depth_correspondences(0, 0)
        for b in range(wl.n_bodies):
            vr = orc.region_correspondences(b, 0, 0)[1] if wl.region else None
            vd = orc.depth_correspondences(b, 0, 0)[1] if wl.depth else None
            gr, gd = ctx.get_closest_views(b)
            got = (gr if wl.region else None, gd if wl.depth else None)
            assert got == (vr, vd), (rep, b, got, (vr, vd))
            found.append((vr, vd))
    ctx.close()
    return found


# The 512-thread k_track2 (region-only / depth-only batches) and cluster tables too large for shared memory (more
# than 96 clusters at n_divides = 5: the tables are read from global memory), for both kernel shapes.
@pytest.mark.parametrize("n_lines,n_points,n_divides", [(32, 0, 4), (0, 32, 4), (32, 32, 5), (32, 0, 5), (0, 32, 5)])
def test_closest_views_equal_full_scan_every_kernel_shape(capi, oracle, synth, n_lines, n_points, n_divides):
    wl = synth.make_workload("c2", n_bodies=96, n_lines=n_lines, n_points=n_points, n_divides=n_divides, seed=78)
    rng = np.random.default_rng(4)
    found = _check_views(capi, oracle, wl, [_random_poses(wl, rng) for _ in range(4)])
    assert len({v for f in found for v in f}) > 200  # the poses really covered the view sphere


def _rotation_onto(a, b):
    """Rotation (float64) that maps the unit vector a onto the unit vector b."""
    v, c = np.cross(a, b), float(a @ b)
    if c < -0.999999:  # opposite: half turn about any axis normal to a
        n = np.cross(a, [1.0, 0.0, 0.0] if abs(a[0]) < 0.9 else [0.0, 1.0, 0.0])
        n /= np.linalg.norm(n)
        return 2.0 * np.outer(n, n) - np.eye(3)
    K = np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])
    return np.eye(3) + K + K @ K / (1.0 + c)


def _tied(m):
    """The model with views k.. replaced by copies of views 0.. (k = a third of the views): orientations, points and
    scalars equal bit for bit, so two or three views give exactly the same dot product for any query. The triples are
    adjacent in the clustering's sort order but 32 is no multiple of 3, so many straddle two clusters (two warps)."""
    k = m.n_views // 3
    src = np.arange(m.n_views) % k
    return dataclasses.replace(m, orientations=m.orientations[src].copy(), points=m.points[src].copy(),
                               view_scalars=m.view_scalars[src].copy())


# Exact ties between views: the smallest view index wins, as in the reference's full scan (strict >, first maximum).
@pytest.mark.parametrize("n_lines,n_points", [(32, 32), (32, 0), (0, 32)])
def test_closest_view_ties_go_to_the_smallest_index(capi, oracle, synth, n_lines, n_points):
    base = synth.make_workload("c2", n_bodies=1, n_lines=max(n_lines, 1), n_points=max(n_points, 1), n_divides=4, seed=79)
    models = (_tied(base.region_model) if n_lines else None, _tied(base.depth_model) if n_points else None)
    wl = synth.make_workload("c2", n_bodies=96, n_lines=n_lines, n_points=n_points, n_divides=4, seed=79, models=models)
    rng = np.random.default_rng(6)
    k = (wl.region_model or wl.depth_model).n_views // 3
    for m, w2c, col in ((wl.region_model, wl.color_world2camera, 0), (wl.depth_model, wl.depth_world2camera, 1)):
        if m is None:
            continue
        aim = rng.choice(k, size=wl.n_bodies, replace=False)  # each a view with copies at aim + k (and aim + 2k)
        poses = wl.start_body2world.copy()
        Rw, tw = w2c[:, :3].astype(np.float64), w2c[:, 3].astype(np.float64)
        for b in range(wl.n_bodies):
            t = Rw @ poses[b, :, 3] + tw  # body origin in the camera; the query is R_b2c^T t / |t|
            o = m.orientations[aim[b]].astype(np.float64)
            R_b2c = _rotation_onto(o / np.linalg.norm(o), t / np.linalg.norm(t))
            poses[b, :, :3] = (Rw.T @ R_b2c).astype(np.float32)
        found = _check_views(capi, oracle, wl, [poses])
        assert [f[col] for f in found] == list(aim)
