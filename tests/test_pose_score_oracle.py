"""The CPU restatement of the evaluators' pose scoring (pose_score_oracle.cpp) against closed forms, numpy's MT19937 and
scipy; no GPU needed."""
import numpy as np
import pytest
from scipy.spatial.distance import pdist
from scipy.spatial.transform import Rotation

import pose_score_oracle as pso


def pose(R=None, t=(0.0, 0.0, 0.0)):
    p = np.zeros((3, 4), np.float32)
    p[:, :3] = np.eye(3) if R is None else R
    p[:, 3] = t
    return p


def mesh(n, seed, scale=0.1):
    return (np.random.default_rng(seed).standard_normal((n, 3)) * scale).astype(np.float32)


@pytest.mark.parametrize("n,n_eval", [(10, 3), (1000, 999), (5000, 1000), (100000, 1000), (7, 1)])
def test_reduced_set_is_mt19937_seed_7_modulo_n(n, n_eval):
    v = mesh(n, n)
    mt = np.random.MT19937()
    mt._legacy_seeding(7)  # std::mt19937{7}: init_genrand(7)
    idx = (mt.random_raw(n_eval) % n).astype(np.int64)
    np.testing.assert_array_equal(pso.reduce_vertices(v, n_eval), v[idx])


@pytest.mark.parametrize("n_eval", [0, -5, 50, 51])
def test_reduced_set_is_every_vertex_outside_0_n(n_eval):
    v = mesh(50, 3)
    np.testing.assert_array_equal(pso.reduce_vertices(v, n_eval), v)


def test_identity_scores_zero_errors_and_full_curves():
    v = mesh(300, 1)
    res, ca, cs = pso.score_pose(v, v, pose(), pose())
    assert list(res) == [0.0, 0.0, 1.0, 1.0, 0.0, 0.0, 1.0]
    assert (ca == 1.0).all() and (cs == 1.0).all()


def test_pure_translation_gives_add_equal_to_its_norm():
    v = (np.random.default_rng(2).integers(-8, 8, (64, 3)) / 8.0).astype(np.float32)
    t = np.array([0.03125, -0.0625, 0.0], np.float32)
    res, ca, _ = pso.score_pose(v, v, pose(), pose(t=t))
    assert res[0] == pytest.approx(np.linalg.norm(t.astype(np.float64)), rel=1e-6)
    # the curve is 0 below the first threshold 0.001 * (0.5 + i) the error falls below
    first = int(np.argmax(res[0] < np.float32(0.001) * (np.float32(0.5) + np.arange(100, dtype=np.float32))))
    assert (ca[:first] == 0.0).all() and (ca[first:] == 1.0).all()
    assert res[2] == np.float32(1.0) - np.float32(res[0] / np.float32(0.1))


def test_adds_never_exceeds_add():
    rng = np.random.default_rng(4)
    for k in range(20):
        v = mesh(500, 100 + k)
        R = Rotation.from_rotvec(rng.normal(0, 0.3, 3)).as_matrix()
        res, _, _ = pso.score_pose(v[::5], v, pose(), pose(R, rng.normal(0, 0.02, 3)))
        assert res[1] <= res[0]


def test_cube_under_a_symmetry_rotation_has_zero_adds():
    c = np.array([[x, y, z] for x in (-0.05, 0.05) for y in (-0.05, 0.05) for z in (-0.05, 0.05)], np.float32)
    Rz = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]], np.float32)
    res, _, cs = pso.score_pose(c, c, pose(), pose(Rz))
    assert res[1] == 0.0 and res[0] > 0.05
    assert (cs == 1.0).all()


def test_rbot_errors_against_float64():
    rng = np.random.default_rng(5)
    v = mesh(10, 6)
    for _ in range(50):
        R1 = Rotation.from_rotvec(rng.normal(0, 1.0, 3)).as_matrix()
        R2 = Rotation.from_rotvec(rng.normal(0, 1.0, 3)).as_matrix()
        p1, p2 = pose(R1, rng.normal(0, 0.1, 3)), pose(R2, rng.normal(0, 0.1, 3))
        res, _, _ = pso.score_pose(v, v, p1, p2)
        te = np.linalg.norm(p1[:, 3].astype(np.float64) - p2[:, 3])
        re = np.arccos(np.clip((np.trace(R1.T @ R2) - 1) / 2, -1, 1))
        assert res[4] == pytest.approx(te, rel=1e-6, abs=1e-8)
        assert res[5] == pytest.approx(re, abs=2e-3 if re < 0.05 else 1e-5)  # acos is ill-conditioned near 0
        assert res[6] == float(te <= 0.05 and re <= 5 * np.pi / 180)


def test_acos_above_one_is_nan_and_counts_as_success():
    res = nan_rotation_case()
    assert np.isnan(res[5]) and res[6] == 1.0


def nan_rotation_case():
    """A pose scored against itself whose float trace exceeds 3: acos of an argument above 1."""
    v = mesh(4, 7)
    for k in range(1, 400):
        R = Rotation.from_rotvec([0.0, 0.0, 1e-4 * k]).as_matrix()
        res, _, _ = pso.score_pose(v, v, pose(R), pose(R))
        if np.isnan(res[5]):
            return res
    raise AssertionError("no angle gives a trace above 3")


def test_nan_pose_gives_nan_add_and_a_flt_max_adds():
    """nanoflann starts the result set at FLT_MAX and takes a point only when dist < worst_dist: a NaN distance is
    never taken, so ADD-S is sqrt(FLT_MAX), AUC 0, while ADD and its AUC are NaN."""
    v = mesh(50, 8)
    p = pose()
    p[0, 3] = np.nan
    res, ca, cs = pso.score_pose(v, v, p, pose())
    assert np.isnan(res[0]) and np.isnan(res[2]) and np.isnan(res[4])
    assert res[1] == pytest.approx(np.sqrt(np.float32(np.finfo(np.float32).max)), rel=1e-5) and res[3] == 0.0
    assert (ca == 0).all() and (cs == 0).all()
    assert res[6] == 1.0  # NaN is not above the threshold


@pytest.mark.parametrize("t", [(1e30, 0.0, 0.0), (np.inf, 0.0, 0.0)])
def test_overflowing_or_infinite_translation_keeps_flt_max(t):
    v = mesh(50, 9)
    res, _, cs = pso.score_pose(v, v, pose(), pose(t=t))
    assert res[1] == pytest.approx(np.sqrt(np.float32(np.finfo(np.float32).max)), rel=1e-5)
    assert res[3] == 0.0 and (cs == 0).all() and res[6] == 0.0


def test_nearest_neighbour_is_the_minimum_below_flt_max():
    v = mesh(200, 10)
    q = v[:20] + np.float32(0.001)
    res, _, _ = pso.score_pose(q, v, pose(), pose())
    d = np.sqrt(((q[:, None, :].astype(np.float64) - v[None]) ** 2).sum(-1).min(1)).mean()
    assert res[1] == pytest.approx(d, rel=1e-5)


@pytest.mark.parametrize("n", [1, 2, 17, 3000])
def test_diameter_is_the_largest_pairwise_distance(n):
    v = mesh(n, 9 + n)
    d = pso.diameter(v)
    ref = pdist(v.astype(np.float64)).max() if n > 1 else 0.0
    assert d == pytest.approx(ref, rel=1e-6)
