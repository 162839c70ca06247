"""Depth-model (default) or, with --region, region-model generation at the reference's defaults: schauma (20950
triangles), 2562 views x 200 points at 2000 px (m3tb_model_params_default). Host clock around each synchronous
m3tb_generate_depth_model / m3tb_generate_region_model call (it ends with a device
synchronise), 3 runs after one warm-up. Peak scratch is measured: a second thread samples the device's free memory
(cudaMemGetInfo through torch) while each call runs, and the drop from before the call to the lowest sample is what the
call held at most (device-wide, so other work on the card would show up in it too). Prints one JSON line with the card's
name and power limit read in the same call; with --region also the device time of each kernel of one more call
(torch.profiler), to show which stage dominates."""
import importlib
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

capi = importlib.import_module("3dobjecttracking_b200.capi")
model_io = importlib.import_module("3dobjecttracking_b200.model_io")

golden = os.path.join(ROOT, "tests", "golden")
mf = model_io.read_model(os.path.join(golden, "depth_model.bin"))  # schauma's header values
mesh = np.load(os.path.join(golden, "schauma_mesh.npz"))
tri = mesh["vertices"][mesh["faces"]]
p = capi.model_params()
ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
ctx.set_body_geometry(0, tri, mf.body.geometry2body[:3], mf.body.maximum_body_diameter, True)
REGION = "--region" in sys.argv
args = [a for a in sys.argv[1:] if a != "--region"]


def generate():
    if REGION:
        ctx.generate_region_model(0, 0, (), p)
    else:
        ctx.generate_depth_model(0, 0, (), p)


generate()  # warm-up: module load
torch.cuda.init()


def generate_watched():
    """Seconds of one generation and the largest drop of free device memory while it ran."""
    free0 = torch.cuda.mem_get_info(0)[0]
    low = [free0]
    done = threading.Event()

    def watch():
        while not done.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info(0)[0])
            time.sleep(0.0005)
    w = threading.Thread(target=watch)
    w.start()
    t0 = time.perf_counter()
    generate()  # ctypes releases the GIL for the call
    dt = time.perf_counter() - t0
    done.set()
    w.join()
    return dt, free0 - low[0]


runs = [generate_watched() for _ in range(int(args[0]) if args else 3)]
times = [r[0] for r in runs]
stages = {}
if REGION:
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        generate()
    for e in prof.key_averages():
        if e.key.startswith(("void m3tb::k_", "m3tb::k_")) or "k_model" in e.key or "k_region" in e.key:
            stages[e.key.split("(")[0]] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1e6, 4)
m = ctx.get_region_model(0) if REGION else ctx.get_depth_model(0)
ctx.close()
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
print(json.dumps(dict(kind="region" if REGION else "depth", stage_seconds=stages, body="schauma", triangles=int(tri.shape[0]), views=m.n_views, points=m.n_points, image_size=p.image_size,
                      seconds_per_model=times, seconds_median=float(np.median(times)),
                      peak_scratch_bytes_measured=[int(r[1]) for r in runs], gpu=gpu)))
