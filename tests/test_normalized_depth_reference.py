"""The NumPy restatements of NormalizedDepthImage that the device is compared with: DepthCamera's (convertTo) equals
the cv2 outputs stored in tests/golden/normalized_depth.npz for every u16 value, and FullDepthRenderer's clamps,
truncates and treats the cleared depth value as the reference does (renderer.cpp:407-427)."""
import os

import numpy as np

import focused_normal_reference as fn
import viewer_reference as vr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "normalized_depth.npz")


def test_camera_restatement_equals_opencv_for_every_value():
    d = np.load(GOLDEN)
    values = np.arange(65536, dtype=np.uint16).reshape(256, 256)
    for (ds, lo, hi), exp in zip(d["ranges"], d["images"]):
        assert np.array_equal(vr.normalized_depth(values, ds, lo, hi), exp), (ds, lo, hi)
    tie = d["images"][2].reshape(-1)  # alpha = 0.5: half to even
    assert tie[1] == 0 and tie[3] == 2 and tie[5] == 2 and tie[7] == 4 and tie[509] == 254 and tie[511] == 255
    assert (d["images"][1].reshape(-1)[[0, 299, 300, 301, 700, 701, 65535]] == [0, 0, 0, 1, 255, 255, 255]).all()
    assert d["images"][5].reshape(-1)[0] == 204  # depth 0 with a negative min: 0.2 m of 0.25 m


def test_full_renderer_restatement():
    f32 = np.float32
    z_min, z_max = f32(0.1), f32(2.0)
    a = z_max * z_min * f32(65535) / (z_max - z_min)
    b = z_max * f32(65535) / (z_max - z_min)
    values = np.array([0, 1, 30000, 60000, 65534, 65535], np.uint16)
    depth = a / (b - values.astype(f32))
    got = fn.normalized_full_depth(values, a, b, 0.3, 1.5)
    scale = f32(255) / (f32(1.5) - f32(0.3))
    exp = [int(min(max(d - f32(0.3), f32(0)), f32(1.5) - f32(0.3)) * scale) for d in depth]
    assert list(got) == exp
    # the near plane clamps to 0, the cleared 65535 (about z_max) to delta, and delta * (255 / delta) is 254.99998 in
    # float32 here, which uchar() truncates
    assert got[0] == 0 and got[-1] == 254
    assert fn.normalized_full_depth(np.array([65535], np.uint16), a, b, 0.0, 5.0)[0] == int(depth[-1] * f32(51))
