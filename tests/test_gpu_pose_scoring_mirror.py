"""The C++ mirror's EvaluationModel and evaluators (examples/pose_scoring_selftest.cpp, plain g++ -std=c++17): its
closed-form checks hold and its results equal the CPU restatement for the same models and poses."""
import json
import subprocess

import numpy as np
import pytest

import pose_score_oracle as pso

pytestmark = pytest.mark.gpu


def pose(r00=1.0, r01=0.0, r10=0.0, r11=1.0, t=(0.0, 0.0, 0.0)):
    p = np.zeros((3, 4), np.float32)
    p[:, :3] = np.eye(3)
    p[0, 0], p[0, 1], p[1, 0], p[1, 1] = r00, r01, r10, r11
    p[:, 3] = t
    return p


def first_one(curve):
    return int(np.argmax(curve == 1.0)) if (curve == 1.0).any() else 100


def test_mirror_evaluators_equal_the_restatement(pkg):
    exe = pkg._build.build_pose_scoring_example()
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    out = json.loads(r.stdout.strip().splitlines()[-1])
    cube = np.array([[0.05 if (i >> k) & 1 else -0.05 for k in range(3)] for i in range(8)], np.float32)
    grid = np.array([[np.float32(0.02) * np.float32(k) for k in (i % 5, (i // 5) % 5, i // 25)] for i in range(125)],
                    np.float32)
    reduced = pso.reduce_vertices(grid, 50)
    assert out["n_reduced"] == len(reduced)
    assert np.float32(out["diameters"][0]) == pso.diameter(cube)
    assert np.float32(out["diameters"][1]) == pso.diameter(grid)
    models = [(cube, cube), (reduced, grid), (reduced, grid)]
    gt = [pose(0, -1, 1, 0), pose(t=(0.003, 0.004, 0.0)), pose(t=(0.0, 0.0, 0.002))]
    ident = pose()
    g2b = pose(0, -1, 1, 0, t=(0.01, 0.0, 0.0))  # body 2's geometry2body term
    errors = []
    for b in range(3):
        res, ca, cs = pso.score_pose(models[b][0], models[b][1], ident, gt[b], g2b if b == 2 else None)
        assert [np.float32(x) for x in out["ycb"][b]] == [res[2], res[3], first_one(ca), first_one(cs)]
        assert np.float32(out["rbot"][b][0]) == res[4] and np.float32(out["rbot"][b][2]) == res[6]
        assert abs(np.float32(out["rbot"][b][1]) - res[5]) <= 4 * np.spacing(np.float32(max(res[5], 1e-30)))
        errors.append(res[:2])
    d = pso.diameter(grid)
    res, ca, _ = pso.score_pose(reduced, grid, ident, gt[2], g2b, threshold_max=0.2, curve_scale=float(d), auc_scale=0.2)
    assert np.float32(out["opt"][0]) == res[2] and out["opt"][1] == first_one(ca)
    # RTBEvaluator: combined bodies {0} and {1, 2}, error threshold 0.1, averaged in float as the reference does
    f = np.float32
    for k, key in enumerate(("add", "adds")):
        c0 = errors[0][k] / f(1)
        c1 = (f(0) + errors[1][k] + errors[2][k]) / f(2)
        auc = (f(0) + (f(1) - min(c0 / f(0.1), f(1)))) + (f(1) - min(c1 / f(0.1), f(1)))
        assert np.float32(out["rtb"][k]) == f(auc / f(2)), key
