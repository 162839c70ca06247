"""Cost of the texture modality at the benchmark's shape: 128 bodies (prism geometry, one 640x480 colour / depth pair
each), 300 ORB-sized features per body and frame, one 200 x 200 silhouette renderer per body.
Reports, with the card's name and power limit, host-clock times around K calls ending in a device synchronise:
  - k_texture_match (m3tb_texture_correspondences at correspondence iteration 0, one launch);
  - one tracking step (n_corr x n_update of the workload) of the same bodies with and without the texture modality,
    and their difference, the per-step overhead of the texture term (renders before each correspondence iteration,
    the match, k_track instead of k_track2);
  - one tracking step (2 x 2 iterations) of 32 kinematic chains of 4 links (config-5 shape, 300 lines and points per
    link) with a texture modality on every link against the same chains without texture (k_track + k_structure per
    update either way).
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


def make(wl, texture):
    """A context of the workload; with texture, every body gets a texture modality on its own camera, a keyframe from
    the first frame's features and the next frame's features (the same ones, a few descriptor bits flipped)."""
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


wl = synth.make_workload("c4", n_bodies=128, n_divides=2, seed=0)
step = lambda c, n_corr, n_update: (lambda: c.tracking_step(0, n_corr, n_update))  # noqa: E731
wl, plain = make(wl, False)
ms_plain = time_calls(plain, step(plain, wl.n_corr_iterations, wl.n_update_iterations))
plain_kernel = plain.last_launch()["kernel"]
plain.close()
wl, tex = make(wl, True)
ms_match = time_calls(tex, lambda: tex.texture_correspondences(0, 0))
n_points = int(np.mean([len(tex.get_texture_points(b)) for b in range(wl.n_bodies)]))
ms_tex = time_calls(tex, step(tex, wl.n_corr_iterations, wl.n_update_iterations))
tex_kernel = tex.last_launch()["kernel"]
tex.close()
CHAINS, LINKS = 32, 4
cw = synth.make_chain_workload(n_chains=CHAINS, n_links=LINKS, n_divides=2, seed=0)
cw, chain_plain = make(cw, False)
ms_chain_plain = time_calls(chain_plain, step(chain_plain, 2, 2))
chain_plain.close()
cw, chain_tex = make(cw, True)
assert chain_tex.n_structures() == CHAINS
chain_tex.texture_correspondences(0, 0)
chain_points = int(np.mean([len(chain_tex.get_texture_points(b)) for b in range(cw.n_bodies)]))
ms_chain_tex = time_calls(chain_tex, step(chain_tex, 2, 2))
chain_tex_kernel = chain_tex.last_launch()["kernel"]
chain_tex.close()
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
print(json.dumps(dict(bodies=wl.n_bodies, features_per_body=N_FEAT, mean_data_points_per_body=n_points,
                      n_corr=wl.n_corr_iterations, n_update=wl.n_update_iterations, ms_texture_match=ms_match,
                      ms_step_without_texture=ms_plain, kernel_without_texture=plain_kernel, ms_step_with_texture=ms_tex,
                      kernel_with_texture=tex_kernel, ms_texture_overhead_per_step=ms_tex - ms_plain,
                      chains=CHAINS, links_per_chain=LINKS, chain_mean_data_points_per_link=chain_points,
                      chain_n_corr=2, chain_n_update=2, chain_ms_step_without_texture=ms_chain_plain,
                      chain_ms_step_with_texture=ms_chain_tex, chain_kernel_with_texture=chain_tex_kernel,
                      chain_ms_texture_overhead_per_step=ms_chain_tex - ms_chain_plain, gpu=gpu)))
