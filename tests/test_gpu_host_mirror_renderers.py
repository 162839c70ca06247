"""The C++ mirror's renderer classes (RendererGeometry, FocusedSilhouetteRenderer, the ModelOcclusions /
UseRegionChecking / UseSilhouetteChecking overloads): an application that tracks with device renderers through
m3t_b200::Tracker reproduces the plain C-ABI calls bit for bit, and the object-wise fan-out (Tracker starting the
renderers before every correspondence iteration) follows it."""
import json
import subprocess

import numpy as np
import pytest

from helpers import pose_error

pytestmark = pytest.mark.gpu


def test_cpp_tracker_with_device_renderers(pkg):
    exe = pkg._build.build_host_example()
    r = subprocess.run([exe, "3", "200", "200", "2", "1", "1", "1"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads(r.stdout.strip().split("\n")[-1])
    assert out["renderers_visible"] is True
    fused = np.array(out["fused"], np.float32).reshape(-1, 3, 4)
    c_abi = np.array(out["c_abi"], np.float32).reshape(-1, 3, 4)
    obj = np.array(out["object_wise"], np.float32).reshape(-1, 3, 4)
    start = np.array(out["start"], np.float32).reshape(-1, 3, 4)
    assert np.array_equal(fused.view(np.uint32), c_abi.view(np.uint32))
    dt, dr = pose_error(fused, obj)
    # The object-wise fan-out runs the phases as separate launches (region / depth correspondences, per-modality
    # gradients, the optimiser) and sums region + depth in another order than k_track. Measured on an H100: bodies 1
    # and 2 agree to 4e-8 m / 2e-6 rad, body 0 deviates by 9.6e-5 m / 1.3e-3 rad after 7 x 2 iterations with the checks
    # on. This bound holds that measurement; bit equality is asserted only for the fused path above.
    assert dt.max() < 2e-4 and dr.max() < 3e-3, (dt, dr)
    assert np.median(dt) < 1e-6 and np.median(dr) < 1e-5, (dt, dr)
    moved_t, moved_r = pose_error(fused, start)
    assert moved_t.min() > 5e-4 and moved_r.min() > 5e-3
