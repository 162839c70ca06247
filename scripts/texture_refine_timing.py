"""Cost of a pose refinement with ORB texture bodies (m3tb_refine_poses_orb, Refiner::RefinePoses with TextureModality)
on a textured scene: the 11 bodies of tests/golden/texture_crops.npz (the prism at the fixture poses, region + depth +
texture, cv::ORB at M3T's settings, each body with a silhouette renderer of its own) in the cv2-golden 960x540 frame.
Times, with CUDA events around K calls (three windows per measurement, alternating), a refinement of 1 body and of all
11 bodies, 7 correspondence x 2 update iterations (the Refiner's defaults); for comparison one device detection of all
bodies (m3tb_texture_detect_orb: its host synchronisation is the one a refinement makes per correspondence iteration)
and the same 7 x 2 iterations as texture_detect_orb + start_modalities + corr_iteration. Counts the kernel launches of
one call each. Prints one JSON line with the card's name and power limit.

    python scripts/texture_refine_timing.py [K]"""
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pkg = importlib.import_module("3dobjecttracking_b200")
capi = importlib.import_module("3dobjecttracking_b200.capi")
synth = pkg.synth

K = int(sys.argv[1]) if len(sys.argv) > 1 else 50
REPEATS = 3  # timed windows per measurement, alternating between the measurements: their spread is reported
N_CORR, N_UPDATE = 7, 2
FIX = np.load(os.path.join(ROOT, "tests", "golden", "texture_crops.npz"))
W2C = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)


def gpu_info():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


def frame():
    path = os.path.join(ROOT, "tests", "golden", "color_camera_image_200.png")
    try:
        import cv2
        return cv2.imread(path, cv2.IMREAD_COLOR)
    except ImportError:
        from PIL import Image
        return np.ascontiguousarray(np.asarray(Image.open(path).convert("RGB"))[:, :, ::-1])


def scene(stream):
    poses = FIX["poses"]
    n = len(poses)
    fu, fv, ppu, ppv, w, h = (float(v) for v in FIX["intrinsics"])
    intr = synth.Intrinsics(fu, fv, ppu, ppv, int(w), int(h))
    ctx = capi.Context(0, max_bodies=n, max_cameras=1, max_models=1, stream=stream)
    ctx.set_color_camera(0, intr, W2C)
    ctx.set_depth_camera(0, intr, W2C, 0.001)
    ctx.upload_depth(0, np.zeros((intr.height, intr.width), np.uint16))
    ctx.upload_color(0, frame())
    tri, diam = synth.prism_triangles()
    for b in range(n):
        ctx.set_body_geometry(b, tri, W2C, diam, True, body_id=b + 1, region_id=b + 1)
    mp = capi.model_params(n_divides=1, n_points=40, image_size=200)
    ctx.generate_depth_model(0, 0, params=mp)
    ctx.generate_region_model(0, 0, params=mp)
    op = capi.OptimizerParams(1000.0, 30000.0)
    for b in range(n):
        ctx.set_body(b, capi.region_params(), capi.depth_params(), op, region_model=0, depth_model=0, color_camera=0,
                     depth_camera=0)
    ctx.set_poses(poses)
    params = capi.texture_params_default()
    params.focused_image_size = int(FIX["focused_image_size"])
    for b in range(n):
        ctx.set_focused_renderer(b, "color", 0, [b], [b], 200, id_type="body")
        ctx.set_texture_modality(b, params, 0)
        ctx.attach_renderer(b, "texture_silhouette", b)
    return ctx, poses


def time_ms(ctx, fn):
    """Mean milliseconds of fn() over K calls, CUDA events on the context's stream (after 3 warm-up calls)."""
    for _ in range(3):
        fn()
    ctx.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(STREAM)
    for _ in range(K):
        fn()
    end.record(STREAM)
    end.synchronize()
    return start.elapsed_time(end) / K


STREAM = torch.cuda.Stream()
ctx, poses = scene(STREAM.cuda_stream)
n = len(poses)
out = dict(bodies=n, n_corr_iterations=N_CORR, n_update_iterations=N_UPDATE, K=K, gpu=gpu_info())


def composition():
    for corr in range(N_CORR):
        ctx.texture_detect_orb(range(n))
        ctx.start_modalities(0)
        ctx.corr_iteration(0, corr, N_UPDATE)


cases = {"one_body": lambda: ctx.refine_poses_orb([1], (), N_CORR, N_UPDATE),
         "all_bodies": lambda: ctx.refine_poses_orb(range(n), (), N_CORR, N_UPDATE),
         "detection_all_bodies": lambda: ctx.texture_detect_orb(range(n)),
         "composition_all_bodies": composition}
for name, fn in cases.items():
    n0 = ctx.launch_count
    fn()
    out[name + "_launches"] = ctx.launch_count - n0
times = {name: [] for name in cases}
for _ in range(REPEATS):
    for name, fn in cases.items():
        ctx.set_poses(poses)
        times[name].append(round(time_ms(ctx, fn), 4))
for name, t in times.items():
    out[name + "_ms"] = sorted(t)[len(t) // 2]
    out[name + "_ms_windows"] = t
ctx.close()
print(json.dumps(out))
