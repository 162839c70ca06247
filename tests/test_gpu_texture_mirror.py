"""The C++ mirror's TextureModality on the device (examples/texture_mirror_tracker.cpp): a textured rigid body and a
textured 3-link chain, with region + depth + texture on every body and seeded features generated in C++, tracked
through Tracker::ExecuteTrackingStep (k_track + k_structure per update) and ExecuteTrackingStepObjectWise (the
Modality / Optimizer methods one by one). The two paths agree within the gates of
test_gpu_host_mirror.py::test_cpp_tracker_kinematic_chains, and the step reduces the start perturbation."""
import json
import os
import subprocess

import numpy as np
import pytest

from helpers import pose_error

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cpp_texture_modality_rigid_and_chain(pkg, tmp_path):
    pkg._build.build_cuda()
    pkg._build.build_synth()
    csrc = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
    synth = os.path.join(ROOT, "3dobjecttracking_b200", "synth")
    exe = str(tmp_path / "texture_mirror_tracker")
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "3dobjecttracking_b200", "host"), "-I", synth,
           os.path.join(ROOT, "examples", "texture_mirror_tracker.cpp"), "-o", exe, "-L", csrc, "-L", synth,
           "-lm3t_b200", "-lm3t_synth", "-Wl,-rpath," + csrc, "-Wl,-rpath," + synth, "-fopenmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, "1", "300"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    out = json.loads(r.stdout.strip().split("\n")[-1])
    assert min(out["texture_points"]) > 20, out["texture_points"]
    fused, obj, start, gt = (np.array(out[k], np.float32).reshape(-1, 3, 4) for k in ("fused", "object_wise", "start", "gt"))
    dt, dr = pose_error(fused, obj)
    assert np.median(dt) < 2e-5 and np.median(dr) < 2e-4, (dt, dr)
    assert dt.max() < 1e-3 and dr.max() < 1e-2, (dt, dr)
    e0t, e0r = pose_error(start, gt)
    e1t, e1r = pose_error(fused, gt)
    assert np.median(e1t) < np.median(e0t) and np.median(e1r) < np.median(e0r), (e0t, e1t, e0r, e1r)
