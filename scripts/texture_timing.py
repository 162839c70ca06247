"""Cost of the texture modality at the benchmark's shape: 128 bodies (prism geometry, one 640x480 colour / depth pair
each), 300 ORB-sized features per body and frame, one 200 x 200 silhouette renderer per body.
Reports, with the card's name and power limit, host-clock times around K calls ending in a device synchronise:
  - k_texture_match (m3tb_texture_correspondences at correspondence iteration 0, one launch);
  - one tracking step (n_corr x n_update of the workload) of the same bodies with and without the texture modality,
    and their difference, the per-step overhead of the texture term (renders before each correspondence iteration,
    the match, k_track instead of k_track2).
Prints one JSON line."""
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

pkg = importlib.import_module("3dobjecttracking_b200")
capi = importlib.import_module("3dobjecttracking_b200.capi")
synth = pkg.synth

K = int(sys.argv[1]) if len(sys.argv) > 1 else 100
N_FEAT = 300


def make(texture):
    wl = synth.make_workload("c4", n_bodies=128, n_divides=2, seed=0)
    ctx = capi.context_from_workload(wl)
    tri, diam = synth.prism_triangles()
    for b in range(wl.n_bodies):
        ctx.set_body_geometry(b, tri, None, diam, True, b % 255 + 1, 7)
    if texture:
        rng = np.random.default_rng(0)
        for b in range(wl.n_bodies):
            ctx.set_focused_renderer(b, "color", b, [b], [b], id_type="body")
            ctx.set_texture_modality(b, capi.texture_params_default(), b)
            ctx.attach_renderer(b, "texture_silhouette", b)
        roi, scale, valid = ctx.get_texture_focus()
        feats = []
        for b in range(wl.n_bodies):
            x, y, w, h = roi[b]
            xy = np.stack([rng.uniform(0, w, N_FEAT), rng.uniform(0, h, N_FEAT)], 1) * scale[b]
            desc = rng.integers(0, 256, (N_FEAT, 32), dtype=np.uint8)
            feats.append((xy.astype(np.float32), desc))
            ctx.upload_texture_features(b, xy, desc, x, y, scale[b] if valid[b] else 1.0)
        ctx.start_modalities(0)
        for b in range(wl.n_bodies):  # the next frame: the same features, a few descriptor bits flipped
            xy, desc = feats[b]
            desc = desc.copy()
            desc[:, ::4] ^= 1
            ctx.upload_texture_features(b, xy, desc, roi[b][0], roi[b][1], scale[b] if valid[b] else 1.0)
    return wl, ctx


def time_calls(ctx, fn):
    for _ in range(10):
        fn()
    ctx.synchronize()
    t0 = time.perf_counter()
    for _ in range(K):
        fn()
    ctx.synchronize()
    return (time.perf_counter() - t0) / K * 1e3


wl, plain = make(False)
step = lambda c: (lambda: c.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations))  # noqa: E731
ms_plain = time_calls(plain, step(plain))
plain_kernel = plain.last_launch()["kernel"]
wl, tex = make(True)
ms_match = time_calls(tex, lambda: tex.texture_correspondences(0, 0))
n_points = int(np.mean([len(tex.get_texture_points(b)) for b in range(wl.n_bodies)]))
ms_tex = time_calls(tex, step(tex))
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
print(json.dumps(dict(bodies=wl.n_bodies, features_per_body=N_FEAT, mean_data_points_per_body=n_points,
                      n_corr=wl.n_corr_iterations, n_update=wl.n_update_iterations, ms_texture_match=ms_match,
                      ms_step_without_texture=ms_plain, kernel_without_texture=plain_kernel, ms_step_with_texture=ms_tex,
                      kernel_with_texture=tex.last_launch()["kernel"], ms_texture_overhead_per_step=ms_tex - ms_plain,
                      gpu=gpu)))
