"""m3tb_get_normalized_depth_image's one allocation, the device scratch image of a host destination: a refused call and
a call whose allocation fails leave the resource count unchanged, the next call gives the same bytes as in a context
that never failed, and destroying the context releases the scratch."""
import numpy as np
import pytest

import viewer_reference as vr
from test_gpu_viewers import I34, _intr

pytestmark = pytest.mark.gpu


def test_failed_and_refused_calls_leave_resources_as_they_were(capi):
    W, H = 333, 217
    frame = np.random.default_rng(2).integers(0, 1500, (H, W), dtype=np.uint16)
    exp = vr.normalized_depth(frame, 0.001, 0.1, 1.2)
    live0 = capi.debug_resources(-1)
    ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
    ctx.set_depth_camera(0, _intr(capi, W, H), I34, 0.001)
    ctx.upload_depth(0, frame)
    ctx.synchronize()
    live = capi.debug_resources(-1)
    buf = np.zeros((H, W), np.uint8)
    assert ctx.L.m3tb_get_normalized_depth_image(ctx.h, 0, 0, 1.2, 0.1, buf.ctypes.data, W) == -1  # refused
    assert capi.debug_resources(-1) == live
    capi.debug_resources(1)  # the scratch allocation fails
    try:
        with pytest.raises(capi.M3TBError):
            ctx.get_normalized_depth_image("camera", 0, 0.1, 1.2, W, H)
    finally:
        capi.debug_resources(0)
    assert capi.debug_resources(-1) == live
    assert np.array_equal(ctx.get_normalized_depth_image("camera", 0, 0.1, 1.2, W, H), exp)
    assert capi.debug_resources(-1) == live + 1  # the scratch, kept for later calls
    assert np.array_equal(ctx.get_normalized_depth_image("camera", 0, 0.1, 1.2, W, H), exp)
    assert capi.debug_resources(-1) == live + 1
    ctx.close()
    assert capi.debug_resources(-1) == live0
