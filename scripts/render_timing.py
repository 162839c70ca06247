"""k_render at the benchmark's shape: 128 bodies (prism), one renderer per body and camera (256 renderers, 200 x 200),
one m3tb_render per call. Host clock around K renders ending in a device synchronise; prints one JSON line."""
import importlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

pkg = importlib.import_module("3dobjecttracking_b200")
capi = importlib.import_module("3dobjecttracking_b200.capi")
synth = pkg.synth

K = int(sys.argv[1]) if len(sys.argv) > 1 else 200
wl = synth.make_workload("c4", n_bodies=128, n_divides=2, seed=0)
ctx = capi.context_from_workload(wl)
tri, diam = synth.prism_triangles()
for b in range(wl.n_bodies):
    ctx.set_body_geometry(b, tri, None, diam, True, b % 255 + 1, 7)
for b in range(wl.n_bodies):
    ctx.set_focused_renderer(2 * b, "color", b, [b], [b], id_type="region")
    ctx.set_focused_renderer(2 * b + 1, "depth", b, [b], [b], id_type="body")
for _ in range(20):
    ctx.render()
ctx.synchronize()
t0 = time.perf_counter()
for _ in range(K):
    ctx.render()
ctx.synchronize()
ms = (time.perf_counter() - t0) / K * 1e3
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
print(json.dumps(dict(renderers=256, image_size=200, ms_per_render=ms, write_out_bytes=256 * 200 * 200 * 3, gpu=gpu)))
