"""Per-frame cost of the texture modality's front end at scripts/texture_timing.py's shape: 128 bodies (prism geometry,
one 640x480 colour / depth pair each), 300 ORB features per body. Detection itself is the caller's and is not timed.
Reports, with the card's name and power limit, host-clock milliseconds per frame (mean of K frames):
  - host path: m3tb_get_texture_focus, the full frame of every camera downloaded (m3tb_get_camera_image, what a
    caller whose frame lives only on the device needs before cropping), the grey crop on the CPU
    (tests/texture_crop_reference.py, the integers cv2 computes) and 128 m3tb_upload_texture_features calls, each
    ending in a stream synchronisation;
  - device path: one m3tb_texture_crop (one k_texture_crop launch) and one m3tb_upload_texture_features_device
    (one k_texture_features launch) from torch tensors, then a synchronisation.
Prints one JSON line.

    python scripts/texture_front_end_timing.py [K]"""
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import texture_crop_reference as cr  # noqa: E402

pkg = importlib.import_module("3dobjecttracking_b200")
capi = importlib.import_module("3dobjecttracking_b200.capi")
synth = pkg.synth

K = int(sys.argv[1]) if len(sys.argv) > 1 else 20
N_FEAT = 300
CAP = 512


def make():
    wl = synth.make_workload("c4", n_bodies=128, n_divides=2, seed=0)
    ctx = capi.context_from_workload(wl)
    tri, diam = synth.prism_triangles()
    params = capi.texture_params_default()
    for b in range(wl.n_bodies):
        ctx.set_body_geometry(b, tri, None, diam, True, b % 255 + 1, 7)
        ctx.set_focused_renderer(b, "color", b, [b], [b], id_type="body")
        ctx.set_texture_modality(b, params, b)
        ctx.attach_renderer(b, "texture_silhouette", b)
    return wl, ctx


def main():
    import torch
    wl, ctx = make()
    n = wl.n_bodies
    W, H = wl.color_intrinsics.width, wl.color_intrinsics.height
    rng = np.random.default_rng(0)
    xy = rng.uniform(0, 150, (n, N_FEAT, 2)).astype(np.float32)
    desc = rng.integers(0, 256, (n, N_FEAT, 32), dtype=np.uint8)
    d_xy, d_desc = torch.from_numpy(xy).cuda(), torch.from_numpy(desc).cuda()
    crops = torch.zeros((n, CAP, CAP), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    feats = [capi.DeviceFeatures(N_FEAT, 0, d_xy[b].data_ptr(), d_xy[b].data_ptr() + 4, 2, d_desc[b].data_ptr(), 32)
             for b in range(n)]
    bodies = list(range(n))
    frame = np.zeros((H, W, 3), np.uint8)

    def host_frame():
        roi, scale, valid = ctx.get_texture_focus()
        for b in range(n):
            ctx.get_camera_image_to(0, b, frame.ctypes.data, frame.strides[0])
            if valid[b]:
                cr.crop(frame, roi[b], scale[b])
                ctx.upload_texture_features(b, xy[b], desc[b], roi[b][0], roi[b][1], scale[b])

    def device_frame():
        ctx.texture_crop(bodies, crops.data_ptr(), CAP, CAP * CAP, CAP, CAP)
        ctx.upload_texture_features_device(bodies, feats)
        ctx.synchronize()

    out = {}
    for name, fn in (("host", host_frame), ("device", device_frame)):
        fn()
        ctx.synchronize()
        t0 = time.perf_counter()
        for _ in range(K):
            fn()
        ctx.synchronize()
        out["ms_per_frame_" + name] = (time.perf_counter() - t0) / K * 1e3
    roi, scale, size, valid = ctx.texture_crop(bodies, crops.data_ptr(), CAP, CAP * CAP, CAP, CAP)
    ctx.close()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps(dict(bodies=n, features_per_body=N_FEAT, K=K, mean_crop_pixels=float(np.mean(size[:, 0] * size[:, 1])),
                          valid_bodies=int(valid.sum()), **out, gpu=gpu)))


if __name__ == "__main__":
    main()
