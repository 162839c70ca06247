"""Device time per undistorted upload (k_undistort, m3tb_set_camera_undistortion) next to cv2's host remap of the same
frames on the same machine, with the card's name and power limit. One command:

    python scripts/undistortion_timing.py [--reps 50] [--out results/undistortion_timing.json]

Per frame kind (1280x720 and 3840x2160 BGRA colour, 640x576 depth):
  - pageable / pinned / device: one m3tb_upload_* of one raw frame (CUDA events around the call: the host-to-device
    copy of a host frame included);
  - batch8_pageable / batch8_pinned: one m3tb_upload_*_batch of 8 raw frames (per batch);
  - zero_copy: k_undistort gathering straight from a pinned frame through its device alias (m3tb_upload_*_device on
    the pinned pointer), the alternative to the staging copy the library makes for pinned frames;
  - plain_pageable / plain_pinned_dma: a camera without an undistortion receiving an already rectified frame (a full
    pageable copy; a pinned frame followed by m3tb_detach_frames, i.e. one DMA of the whole frame);
  - cv2: cvtColor(RGBA2RGB) + remap (colour) or remap + add (depth) on the host, single call, median.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import importlib
    import torch
    capi = importlib.import_module("3dobjecttracking_b200.capi")
    synth = importlib.import_module("3dobjecttracking_b200.synth")
    name, power = card()
    results = dict(card=name, power_limit=power, reps=args.reps, frames={})
    k = np.array([0.52, -2.61, 6e-4, -3e-4, 1.45, 0.40, -2.43, 1.38], np.float32)
    for kind, W, H in (("color", 1280, 720), ("color", 3840, 2160), ("depth", 640, 576)):
        color = kind == "color"
        ch = 4 if color else 1
        f = 0.47 * W
        raw_i = synth.Intrinsics(f, f, W / 2 - 0.5, H / 2 - 0.5, W, H)
        rect_i = synth.Intrinsics(np.float32(f) * np.float32(1.05 if color else 1.0),
                                  np.float32(f) * np.float32(1.05 if color else 1.0), W / 2 - 0.5, H / 2 - 0.5, W, H)
        m = capi.undistortion_map(raw_i, k if color else k * 0.5, rect_i)
        rng = np.random.default_rng(0)
        if color:
            raws = rng.integers(0, 256, (8, H, W, 4), dtype=np.uint8)
        else:
            raws = rng.integers(0, 4000, (8, H, W), dtype=np.uint16)
        row = W * ch * raws.itemsize
        pinned = torch.from_numpy(raws).pin_memory()
        dev = torch.from_numpy(raws).cuda()
        ctx = capi.Context(max_cameras=9)
        eye = np.eye(4, dtype=np.float32)[:3]
        for cam in range(9):
            if color:
                ctx.set_color_camera(cam, rect_i, eye)
            else:
                ctx.set_depth_camera(cam, rect_i, eye, 0.001)
            if cam < 8:
                ctx.set_camera_undistortion(kind, cam, m, ch, -5 if not color else 0)
        L = ctx.L
        up = L.m3tb_upload_color if color else L.m3tb_upload_depth
        up_dev = L.m3tb_upload_color_device if color else L.m3tb_upload_depth_device
        up_batch = L.m3tb_upload_color_batch if color else L.m3tb_upload_depth_batch
        rect_frame = np.ascontiguousarray(raws[0][..., :3]) if color else raws[0]
        rect_pinned = torch.from_numpy(rect_frame).pin_memory()
        frame_bytes = H * row

        def pinned_dma():
            ctx._ck(up(ctx.h, 8, C.c_void_p(rect_pinned.data_ptr()), rect_frame.strides[0]))
            ctx.detach_frames()

        cases = {
            "pageable": lambda: ctx._ck(up(ctx.h, 0, raws[0].ctypes.data, row)),
            "pinned": lambda: ctx._ck(up(ctx.h, 1, C.c_void_p(pinned[1].data_ptr()), row)),
            "device": lambda: ctx._ck(up_dev(ctx.h, 2, C.c_void_p(dev[2].data_ptr()), row)),
            "zero_copy": lambda: ctx._ck(up_dev(ctx.h, 3, C.c_void_p(pinned[3].data_ptr()), row)),
            "batch8_pageable": lambda: ctx._ck(up_batch(ctx.h, 0, 8, raws.ctypes.data, frame_bytes, row)),
            "batch8_pinned": lambda: ctx._ck(up_batch(ctx.h, 0, 8, C.c_void_p(pinned.data_ptr()), frame_bytes, row)),
            "plain_pageable": lambda: ctx._ck(up(ctx.h, 8, rect_frame.ctypes.data, rect_frame.strides[0])),
            "plain_pinned_dma": pinned_dma,
        }
        res = {}
        for case, fn in cases.items():
            for _ in range(5):
                fn()
            ctx.synchronize()
            times = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            res[case] = dict(median_ms=round(statistics.median(times), 4), min_ms=round(min(times), 4))
        n_launch = ctx.launch_count
        ctx.close()
        try:
            import cv2
            host = []
            for i in range(args.reps):
                t0 = time.perf_counter()
                if color:
                    cv2.remap(cv2.cvtColor(raws[i % 8], cv2.COLOR_RGBA2RGB), m, None, cv2.INTER_NEAREST,
                              borderMode=cv2.BORDER_CONSTANT)
                else:
                    cv2.add(cv2.remap(raws[i % 8], m, None, cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT),
                            (-5.0, 0.0, 0.0, 0.0))
                host.append((time.perf_counter() - t0) * 1e3)
            res["cv2_host"] = dict(median_ms=round(statistics.median(host), 4), min_ms=round(min(host), 4),
                                   version=cv2.__version__, cpu_threads=cv2.getNumThreads())
        except ImportError:
            res["cv2_host"] = "cv2 not installed"
        res["launches"] = n_launch
        results["frames"][f"{kind}_{W}x{H}"] = res
        print(json.dumps({f"{kind}_{W}x{H}": res}), flush=True)
    print(json.dumps(dict(card=name, power_limit=power)), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
