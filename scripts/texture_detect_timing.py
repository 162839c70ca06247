"""Per-frame device time of m3tb_texture_detect_orb (crop + cv::ORB on the device) at 1, 8 and 128 bodies on the
golden frame, and, when cv2 is importable, the host arm it replaces: download each crop, cv2.ORB detect + compute,
upload the features (m3tb_upload_texture_features). Prints one JSON line; record the card and its power limit with it.

    python scripts/texture_detect_timing.py [--frames 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    args = ap.parse_args()
    import importlib
    import torch
    capi = importlib.import_module("3dobjecttracking_b200.capi")
    synth = importlib.import_module("3dobjecttracking_b200").synth
    from test_gpu_texture_device_front_end import FIX, FIX_FRAME, _scene
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        gpu = torch.cuda.get_device_name(0)
    out = {"gpu": gpu, "frames": args.frames, "device_ms": {}, "host_ms": {}}
    for n in (1, 8, 128):
        src = [b % len(FIX["poses"]) for b in range(n)]
        ctx = _scene(capi, synth, poses=FIX["poses"][src], own_geometry=True)
        bodies = list(range(n))
        ctx.texture_detect_orb(bodies)  # warm-up: scratch and tables
        ctx.synchronize()
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(args.frames):
            ctx.upload_color(0, FIX_FRAME)
            ctx.synchronize()
            start.record()
            ctx.texture_detect_orb(bodies)  # synchronises once (the poses), on the default stream
            stop.record()
            stop.synchronize()
            times.append(start.elapsed_time(stop))
        out["device_ms"][n] = round(float(np.median(times)), 4)
        try:
            import cv2
        except ImportError:
            ctx.close()
            continue
        cap = 512
        buf = torch.empty((n, cap, cap), dtype=torch.uint8, device="cuda")
        orb = cv2.ORB_create(300, 1.2, 3)
        host = []
        for _ in range(min(args.frames, 10)):
            ctx.upload_color(0, FIX_FRAME)
            ctx.synchronize()
            t0 = time.perf_counter()
            roi, scale, size, valid = ctx.texture_crop(bodies, buf.data_ptr(), cap, cap * cap, cap, cap)
            crops = buf.cpu().numpy()
            for b in bodies:
                w, h = size[b]
                img = np.ascontiguousarray(crops[b, :h, :w])
                kps = orb.detect(img, None)
                kps, desc = orb.compute(img, kps)
                xy = np.array([k.pt for k in kps], np.float32).reshape(-1, 2)
                desc = desc if desc is not None else np.zeros((0, 32), np.uint8)
                ctx.upload_texture_features(b, xy, desc, roi[b][0], roi[b][1], scale[b])
            host.append((time.perf_counter() - t0) * 1e3)
        out["host_ms"][n] = round(float(np.median(host)), 2)
        ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
