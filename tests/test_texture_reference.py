"""CPU checks of the texture modality's restatement (tests/texture_reference.py), which the GPU tests hold the device
to: TukeyNorm against its closed form, the reprojection Jacobian against finite differences, the kNN matcher against
cv2.BFMatcher fixtures (tests/golden/make_texture_knn.py), the focus region against hand-computed values, and the
keyframe rule evaluated with the pose of the last gradient pass."""
import os

import numpy as np
import pytest

import texture_reference as tr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "texture_knn.npz")
INTR = dict(fu=600.0, fv=600.0, ppu=320.0, ppv=240.0, width=640, height=480)


def _rot(axis, deg):
    c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
    i, j = [k for k in range(3) if k != axis]
    Q = np.eye(3)
    Q[i, i], Q[i, j], Q[j, i], Q[j, j] = c, -s, s, c
    return Q


def _pose(R=np.eye(3), t=(0.0, 0.0, 0.5)):
    return np.hstack([R, np.asarray(t, float)[:, None]]).astype(np.float32).reshape(12)


@pytest.mark.parametrize("c", [20.0, 3.5])
def test_tukey_norm_closed_form(c):
    for e in np.linspace(0.0, 2.5 * c, 41):
        exp = c * c / 6.0 * (1.0 - (1.0 - (e / c) ** 2) ** 3) if e <= c else c * c / 6.0
        assert abs(float(tr.tukey_norm(e, c)) - exp) <= 1e-5 * c * c
    assert tr.tukey_norm(-0.5 * c, c) == tr.tukey_norm(0.5 * c, c)


def test_reprojection_jacobian_against_finite_differences():
    """g = -w diff J for one point: J is d(projection) / d(theta) of body2world * [exp(skew(rot)) | trans]."""
    R = _rot(0, 12.0) @ _rot(1, -7.0)
    b2c = _pose(R, (0.02, -0.01, 0.45))
    X = np.array([[0.013, -0.021, 0.008]], np.float32)
    target = tr.project(b2c, INTR, X)[0] + np.array([1.5, -0.75], np.float32)
    sd, c = 5.0, 20.0
    g, H = tr.gradient_hessian(b2c, INTR, X, target[None], sd, c)

    def proj(theta):
        T = np.eye(4)
        T[:3, :] = np.asarray(b2c, float).reshape(3, 4)
        V = np.eye(4)
        from scipy.linalg import expm
        V[:3, :3] = expm(tr.skew(theta[:3]))
        V[:3, 3] = theta[3:]
        p = (T @ V)[:3] @ np.append(X[0].astype(float), 1.0)
        return np.array([p[0] * INTR["fu"] / p[2] + INTR["ppu"], p[1] * INTR["fv"] / p[2] + INTR["ppv"]])

    h = 1e-6
    J = np.stack([(proj(h * np.eye(6)[k]) - proj(-h * np.eye(6)[k])) / (2 * h) for k in range(6)], 1)
    diff = proj(np.zeros(6)) - target
    e2 = float(diff @ diff)
    w = float(tr.tukey_norm(np.sqrt(e2), c)) / e2 / sd ** 2
    np.testing.assert_allclose(g, -w * diff @ J, rtol=2e-4, atol=1e-6 * np.abs(g).max())
    np.testing.assert_allclose(H, -w * J.T @ J, rtol=2e-4, atol=1e-6 * np.abs(H).max())


@pytest.mark.parametrize("case", ["random", "ties", "equal_distance", "train_of_one", "empty_train"])
def test_knn_matches_cv2_bfmatcher(case):
    f = np.load(GOLDEN)
    got = tr.knn2(f[case + "_queries"], f[case + "_train"])
    for i, m in enumerate(got):
        idx = [j for j, _ in m] + [-1] * (2 - len(m))
        dist = [float(d) for _, d in m] + [-1.0] * (2 - len(m))
        assert idx == list(f[case + "_idx"][i]), (case, i)
        assert dist == [float(d) for d in f[case + "_dist"][i]], (case, i)


def test_ratio_test_keeps_zero_over_zero_and_drops_single_matches():
    f = np.load(GOLDEN)
    q, t = f["ties_queries"], f["ties_train"]
    assert list(f["ties_idx"][3]) == [70, 71] and list(f["ties_dist"][3]) == [0.0, 0.0]
    pts = np.arange(len(q) * 3, dtype=np.float32).reshape(-1, 3)
    xy = np.arange(len(t) * 2, dtype=np.float32).reshape(-1, 2)
    cb, cc = tr.match([(pts, q)], xy, t, 0.7)
    assert any(np.array_equal(p, pts[3]) for p in cb)  # d0 / d1 = 0 / 0 is NaN: kept
    cb1, _ = tr.match([(pts[:8], f["train_of_one_queries"])], xy[:1], f["train_of_one_train"], 0.7)
    cb0, _ = tr.match([(pts[:8], f["empty_train_queries"])], xy[:0], f["empty_train_train"], 0.7)
    assert len(cb1) == 0 and len(cb0) == 0


def test_focus_region_hand_computed():
    # x = y = 0: r_u = r_v = fu r / sqrt(z^2 - r^2) = 30 / sqrt(0.2475) = 60.3023
    roi, scale = tr.focus(INTR, _pose(t=(0.0, 0.0, 0.5)), 0.05, 200)
    assert roi == (250, 170, 140, 140)
    assert abs(float(scale) - 200.0 / (2 * 30 / np.sqrt(0.2475))) < 1e-4
    assert tr.focus(INTR, _pose(t=(0.0, 0.0, 0.07)), 0.05, 200) is None  # z < 1.5 r
    assert tr.focus(INTR, _pose(t=(1.0, 0.0, 0.5)), 0.05, 200) is None   # the region lies right of the image


def test_keyframe_rule_uses_the_pose_of_the_last_gradient_pass():
    max_rot = np.float32(10.0 * np.pi / 180.0)
    o_kf = tr.orientation(_pose())
    stale = _pose(_rot(1, 6.0))   # pose of the last gradient pass
    final = _pose(_rot(1, 12.0))  # pose after the final update
    assert tr.keyframe_fires(final, o_kf, 0, max_rot, 100)[0]
    fires, age = tr.keyframe_fires(stale, o_kf, 0, max_rot, 100)
    assert not fires and age == 1
    assert tr.keyframe_fires(stale, o_kf, 100, max_rot, 100) == (True, 101)  # age rule
    assert np.array_equal(tr.orientation(_pose(t=(0.0, 0.0, 0.0))), np.zeros(3, np.float32))
