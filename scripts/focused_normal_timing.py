"""m3tb_render_focused_normals and m3tb_get_normalized_depth_image timed with CUDA events. Focused normal renderers:
1, 16 and 128 of them, one per colour camera (640x480) on a ring around one schauma body (tests/golden/schauma_mesh.npz,
20,950 triangles) that each draws and references, at image sizes 200 and 480; every render is one call, four launches
for all renderers. Normalised depth: one call (one launch) into device memory for a 640x576 depth frame and for a full
renderer's 1280x720 depth image. Two numbers per case: ms_per_call, CUDA events around back-to-back calls, so it
includes each call's host work (table building and copies of a render; the destination's pointer query and the launch
of a normalised depth image); and kernel_ms, the device time of the call's kernels from torch.profiler over the same
number of calls, in a profiled pass of its own. Prints the card name and power limit, then one JSON line per case."""
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

capi = importlib.import_module("3dobjecttracking_b200.capi")
from full_render_timing import camera, schauma  # noqa: E402

K = int(sys.argv[1]) if len(sys.argv) > 1 else 200
K_DEPTH = 20 * K  # a normalised depth image is short: enough calls for a window of several milliseconds
I34 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def timed(ctx, call, n):
    """ms per call over n calls on a stream of our own, after a warm-up."""
    for _ in range(5):
        call()
    ctx.synchronize()
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(n):
        call()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_ms(call, n, prefix):
    """Summed device time per call of the kernels whose names start with `prefix`."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            call()
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.key_averages():
        if e.key.split("(")[0].split("::")[-1].startswith(prefix):
            total += getattr(e, "device_time_total", None) or e.cuda_time_total  # microseconds
    return total / 1000.0 / n


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)))
    tri, diam = schauma()
    W, H = 640, 480
    for S, n in ((200, 1), (200, 16), (200, 128), (480, 16)):
        ctx = capi.Context(0, max_bodies=1, max_cameras=n, max_models=1)
        for k in range(n):
            ctx.set_color_camera(k, capi.Intrinsics(0.96 * W, 0.96 * W, W / 2, H / 2, W, H), camera(k, n, 2.0 * diam))
        ctx.set_poses(I34[None])
        ctx.set_body_geometry(0, tri, None, diam, True, 1, 1)
        for k in range(n):
            ctx.set_focused_normal_renderer(k, "color", k, [0], [0], S)
        ms = timed(ctx, ctx.render_focused_normals, K)
        kms = kernel_ms(ctx.render_focused_normals, K, "k_view_")
        out = ctx.get_focused_normal_rendering(n - 1)
        print(json.dumps(dict(case="render_focused_normals", mesh="schauma", triangles=int(tri.shape[0]), image_size=S,
                              renderers=n, calls=K, ms_per_call=ms, kernel_ms=kms,
                              covered=float((out["depth"] != 65535).mean()))))
        ctx.close()
    # normalised depth: a depth camera frame and a full renderer's depth image, into device memory
    ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
    ctx.set_depth_camera(0, capi.Intrinsics(504.0, 504.0, 320.0, 288.0, 640, 576), I34, 0.001)
    ctx.upload_depth(0, np.random.default_rng(0).integers(0, 4000, (576, 640), dtype=np.uint16))
    dst = torch.zeros((576, 640), dtype=torch.uint8, device="cuda")
    call = lambda: ctx.get_normalized_depth_image_to("camera", 0, 0.2, 2.0, dst.data_ptr(), 640)  # noqa: E731
    ms, kms = timed(ctx, call, K_DEPTH), kernel_ms(call, K_DEPTH, "k_normalized_depth")
    print(json.dumps(dict(case="normalized_depth_camera", width=640, height=576, calls=K_DEPTH, ms_per_call=ms,
                          kernel_ms=kms)))
    ctx.close()
    W, H = 1280, 720
    ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
    ctx.set_color_camera(0, capi.Intrinsics(0.96 * W, 0.96 * W, W / 2, H / 2, W, H), camera(0, 1, 2.0 * diam))
    ctx.set_poses(I34[None])
    ctx.set_body_geometry(0, tri, None, diam, True, 1, 1)
    ctx.set_full_renderer(0, "color", 0, [0], 0.02, 10.0)
    ctx.render_full()
    dst = torch.zeros((H, W), dtype=torch.uint8, device="cuda")
    call = lambda: ctx.get_normalized_depth_image_to("full_renderer", 0, 0.2, 2.0, dst.data_ptr(), W)  # noqa: E731
    ms, kms = timed(ctx, call, K_DEPTH), kernel_ms(call, K_DEPTH, "k_normalized_depth")
    print(json.dumps(dict(case="normalized_depth_full_renderer", width=W, height=H, calls=K_DEPTH, ms_per_call=ms,
                          kernel_ms=kms)))
    ctx.close()


if __name__ == "__main__":
    main()
