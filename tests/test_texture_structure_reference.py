"""The two CPU restatements that the textured kinematic-structure tests compose, tied together without a GPU: a
one-link structure with identity joints and all six directions free, fed a texture gradient / Hessian from
texture_reference.gradient_hessian, is the rigid-body optimiser. structure_reference.calculate_optimization then gives
the same theta as texture_reference.optimize's solve to float64 rounding, and the same pose to the float32 rounding
that texture_reference.optimize ends with."""
from types import SimpleNamespace

import numpy as np
import pytest

import structure_reference as sr
import texture_reference as tr

INTR = dict(fu=614.0, fv=614.5, ppu=321.3, ppv=238.9, width=640, height=480)
TIKHONOV = (1000.0, 30000.0)


def _one_link():
    link = SimpleNamespace(body=0, parent=-1, free_directions=(1, 1, 1, 1, 1, 1), fixed_body2joint_pose=True,
                           extra_bodies=())
    return SimpleNamespace(links=[link], constraints=[], tikhonov_rotation=TIKHONOV[0],
                           tikhonov_translation=TIKHONOV[1])


def _texture_gh(rng, pose, true_pose, n=120, corr=0):
    """Data points on a 6 cm box seen at true_pose, the gradient / Hessian at pose."""
    cb = rng.uniform(-0.03, 0.03, (n, 3)).astype(np.float32)
    cc = tr.project(true_pose.reshape(12), INTR, cb) + rng.normal(0.0, 0.5, (n, 2)).astype(np.float32)
    return tr.gradient_hessian(pose, INTR, cb, cc, [15.0, 5.0][corr], 20.0)


def _rigid_pose(rot, t):
    p = np.zeros((3, 4), np.float32)
    p[:, :3] = sr.exp_so3(np.asarray(rot, np.float64))
    p[:, 3] = t
    return p


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_one_link_structure_is_the_rigid_texture_optimiser(seed):
    rng = np.random.default_rng(seed)
    spec = _one_link()
    pose = _rigid_pose(rng.normal(0.0, 0.2, 3), (0.01, -0.02, 0.5))
    true_pose = tr.pose_mul(_rigid_pose(rng.normal(0.0, 0.02, 3), rng.normal(0.0, 0.004, 3)), pose).reshape(3, 4)
    start = np.abs(pose - true_pose).max()
    for it in range(4):
        g, H = _texture_gh(rng, pose, true_pose, corr=min(it, 1))
        assert np.abs(g).max() > 0
        state = sr.State.from_arrays(pose.reshape(12), np.eye(4)[:3].reshape(12), np.eye(4)[:3].reshape(12))
        res = sr.calculate_optimization(spec, state, g[None, None], H[None, None])
        assert res.updated
        a = -H + np.diag([TIKHONOV[0]] * 3 + [TIKHONOV[1]] * 3)
        theta = np.linalg.solve(a, g)
        assert np.abs(res.theta - theta).max() <= 1e-12 * np.abs(theta).max()
        expected = tr.optimize(pose, g, H, *TIKHONOV)
        got = res.state.link2world[0, :3]
        # texture_reference.optimize rounds its float64 result to float32 once
        assert np.all(np.abs(got - expected) <= np.spacing(np.abs(expected).astype(np.float32))), it
        pose = expected
    # the iteration moved the pose towards the one the points were seen at
    assert np.abs(pose - true_pose).max() < start
