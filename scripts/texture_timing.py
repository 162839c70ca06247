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
Prints one JSON line.

With --descriptor sift|daisy it measures the L2 matcher instead (512 features per body of 128 / 104 floats, whole
numbers in 0 .. 255 for SIFT, unit-norm for DAISY, every query a keyframe point):
  - k_texture_knn_l2 per launch (torch.profiler CUDA activity over K calls of m3tb_texture_correspondences at
    correspondence iteration 0) for 1, 8 and 128 bodies and n_keyframes 1 and 4, with the FP32 rate from
    2 * queries * train * length against the 67 TFLOP/s data sheet;
  - one tracking step at the ORB shape above (128 bodies, 300 features) with ORB against the L2 descriptor.

With --features N (512 .. 4096) it measures a context whose bodies keep N features each (n_features_max N, every
feature near the body's centre, so all become keyframe points), for ORB and SIFT and for 1, 8 and 128 bodies:
  - the matcher's device time per launch (torch.profiler CUDA activity over K calls of m3tb_texture_correspondences at
    correspondence iteration 0): k_texture_knn_hamming for ORB above 512 (k_texture_match's in-CTA scan at 512) and
    k_texture_knn_l2 for SIFT;
  - one tracking step (n_corr x n_update of the workload).

With --descriptor brisk it measures the 64-byte Hamming matcher (random 64-byte descriptors, every feature near the
body's centre) at n_features_max 512, 2048 and 4096 for 1, 8 and 128 bodies: k_texture_knn_hamming per launch, and
one tracking step. In the same run it times k_texture_knn_hamming for ORB at 4096 features (8 and 128 bodies) on this
build and on the build given by --parent-lib PATH (another libm3t_b200.so, e.g. of the parent commit), alternating
between the two in fresh processes, three rounds each, so that a change of the 8-word path shows beside its spread.

    python scripts/texture_timing.py [K] [--descriptor sift|daisy|brisk] [--features N] [--parent-lib PATH]"""
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

ARGS = [a for a in sys.argv[1:] if not a.startswith("--")]
DESCRIPTOR = sys.argv[sys.argv.index("--descriptor") + 1] if "--descriptor" in sys.argv else None
FEATURES = int(sys.argv[sys.argv.index("--features") + 1]) if "--features" in sys.argv else None
PARENT_LIB = sys.argv[sys.argv.index("--parent-lib") + 1] if "--parent-lib" in sys.argv else None
ORB_KNN = "--orb-knn-4096" in sys.argv  # one round of the ORB comparison, run by brisk_main in a fresh process
ARGS = [a for a in ARGS if a not in (DESCRIPTOR, str(FEATURES), PARENT_LIB)]
K = int(ARGS[0]) if ARGS else 100
N_FEAT = 300
L2_LENGTH = {"sift": 128, "daisy": 104}
L2_TYPE = {"sift": capi.DESCRIPTOR_SIFT, "daisy": capi.DESCRIPTOR_DAISY}
TYPE = dict(L2_TYPE, brisk=capi.DESCRIPTOR_BRISK)


def descriptors(rng, kind, n):
    if kind is None:
        return rng.integers(0, 256, (n, 32), dtype=np.uint8)
    if kind == "brisk":
        return rng.integers(0, 256, (n, 64), dtype=np.uint8)
    if kind == "sift":
        return rng.integers(0, 256, (n, 128)).astype(np.float32)
    v = rng.random((n, L2_LENGTH[kind])).astype(np.float32)
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def perturbed(rng, kind, desc):
    if kind is None or kind == "brisk":
        desc = desc.copy()
        desc[:, ::4] ^= 1
        return desc
    noise = rng.integers(-3, 4, desc.shape) if kind == "sift" else rng.normal(0, 0.02, desc.shape)
    return np.clip(desc + noise, 0, None).astype(np.float32)


def make(wl, texture, kind=None, n_feat=N_FEAT, n_keyframes=1, central=False):
    """A context of the workload; with texture, every body gets a texture modality on its own camera, a keyframe from
    the first frame's features and the next frame's features (the same ones, a few descriptor bits flipped).
    kind: None (ORB), "brisk" or an L2 descriptor; n_keyframes > 1 refreshes the keyframe every frame until the deque is full;
    central puts every feature near the body's centre, so that all become keyframe points."""
    ctx = capi.context_from_workload(wl)
    tri, diam = synth.prism_triangles()
    for b in range(wl.n_bodies):
        ctx.set_body_geometry(b, tri, None, diam, True, b % 255 + 1, 7)
    if texture:
        rng = np.random.default_rng(0)
        params = capi.texture_params_default()
        if kind is not None:
            params.descriptor_type = TYPE[kind]
        params.n_keyframes = n_keyframes
        params.n_features_max = max(params.n_features_max, n_feat)
        params.max_keyframe_age = 0 if n_keyframes > 1 else params.max_keyframe_age
        for b in range(wl.n_bodies):
            ctx.set_focused_renderer(b, "color", b, [b], [b], id_type="body")
            ctx.set_texture_modality(b, params, b)
            ctx.attach_renderer(b, "texture_silhouette", b)
        roi, scale, valid = ctx.get_texture_focus()
        feats = []
        for b in range(wl.n_bodies):
            x, y, w, h = roi[b]
            if central:
                xy = np.stack([rng.uniform(0.47 * w, 0.53 * w, n_feat), rng.uniform(0.47 * h, 0.53 * h, n_feat)], 1)
            else:
                xy = np.stack([rng.uniform(0, w, n_feat), rng.uniform(0, h, n_feat)], 1)
            xy = xy * scale[b]
            desc = descriptors(rng, kind, n_feat)
            feats.append((xy.astype(np.float32), desc))
            ctx.upload_texture_features(b, xy, desc, x, y, scale[b] if valid[b] else 1.0)
        ctx.start_modalities(0)
        for frame in range(1, n_keyframes):
            ctx.calculate_results(frame)
        for b in range(wl.n_bodies):  # the next frame: the same features, descriptors perturbed
            xy, desc = feats[b]
            ctx.upload_texture_features(b, xy, perturbed(rng, kind, desc), roi[b][0], roi[b][1],
                                        scale[b] if valid[b] else 1.0)
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


def gpu_name():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()


step = lambda c, n_corr, n_update: (lambda: c.tracking_step(0, n_corr, n_update))  # noqa: E731


def knn_kernel_ms(ctx, kernel="k_texture_knn_l2"):
    """The kernel's mean device time per launch over K calls of the match (torch.profiler CUDA activity)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    for _ in range(10):
        ctx.texture_correspondences(0, 0)
    ctx.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(K):
            ctx.texture_correspondences(0, 0)
        ctx.synchronize()
        torch.cuda.synchronize()
    rows = [e for e in prof.key_averages() if kernel in e.key]
    assert len(rows) == 1 and 0 < rows[0].count <= K, [(e.key, e.count) for e in rows]
    # the profiler may drop a few events of a long run: the mean over the launches it recorded
    return max(rows[0].self_device_time_total, rows[0].device_time_total) / rows[0].count / 1e3


def l2_main(kind):
    import torch
    torch.cuda.init()
    length = L2_LENGTH[kind]
    shapes = []
    for n_bodies in (1, 8, 128):
        for n_keyframes in (1, 4):
            wl = synth.make_workload("c4", n_bodies=n_bodies, n_divides=2, seed=0)
            wl, ctx = make(wl, True, kind, n_feat=512, n_keyframes=n_keyframes, central=True)
            queries = sum(int(ctx.get_texture_keyframes(b)["sizes"].sum()) for b in range(n_bodies))
            ms = knn_kernel_ms(ctx)
            flop = 2.0 * queries * 512 * length
            ms_call = time_calls(ctx, lambda: ctx.texture_correspondences(0, 0))
            shapes.append(dict(bodies=n_bodies, n_keyframes=n_keyframes, queries=queries, train_per_body=512,
                               length=length, ms_knn_l2=ms, ms_match_call=ms_call, tflops=flop / ms / 1e9,
                               share_of_67_tflops=flop / ms / 1e9 / 67.0, datasheet_floor_ms=flop / 67e12 * 1e3))
            ctx.close()
    wl = synth.make_workload("c4", n_bodies=128, n_divides=2, seed=0)
    steps = {}
    for name, k in (("orb", None), (kind, kind)):
        wl, ctx = make(wl, True, k)
        steps[name] = time_calls(ctx, step(ctx, wl.n_corr_iterations, wl.n_update_iterations))
        ctx.close()
    print(json.dumps(dict(descriptor=kind, K=K, shapes=shapes, step_bodies=wl.n_bodies, step_features_per_body=N_FEAT,
                          n_corr=wl.n_corr_iterations, n_update=wl.n_update_iterations,
                          ms_step_orb=steps["orb"], **{"ms_step_" + kind: steps[kind]}, gpu=gpu_name())))


def features_main(n_feat):
    import torch
    torch.cuda.init()
    shapes = []
    for kind in ("orb", "sift"):
        kernel = "k_texture_knn_l2" if kind == "sift" else "k_texture_knn_hamming" if n_feat > 512 else "k_texture_match"
        for n_bodies in (1, 8, 128):
            wl = synth.make_workload("c4", n_bodies=n_bodies, n_divides=2, seed=0)
            wl, ctx = make(wl, True, None if kind == "orb" else kind, n_feat=n_feat, central=True)
            queries = sum(int(ctx.get_texture_keyframes(b)["sizes"].sum()) for b in range(n_bodies))
            ms = knn_kernel_ms(ctx, kernel)
            ms_step = time_calls(ctx, step(ctx, wl.n_corr_iterations, wl.n_update_iterations))
            points = int(np.mean([len(ctx.get_texture_points(b)) for b in range(n_bodies)]))
            shapes.append(dict(descriptor=kind, bodies=n_bodies, queries=queries, train_per_body=n_feat, kernel=kernel,
                               ms_kernel=ms, ms_step=ms_step, mean_data_points_per_body=points,
                               n_corr=wl.n_corr_iterations, n_update=wl.n_update_iterations))
            ctx.close()
    print(json.dumps(dict(features=n_feat, K=K, shapes=shapes, gpu=gpu_name())))


def orb_knn_round():
    """k_texture_knn_hamming for ORB at 4096 features per body, 8 and 128 bodies: {bodies: ms per launch}."""
    import torch
    torch.cuda.init()
    out = {}
    for n_bodies in (8, 128):
        wl = synth.make_workload("c4", n_bodies=n_bodies, n_divides=2, seed=0)
        wl, ctx = make(wl, True, None, n_feat=4096, central=True)
        out[n_bodies] = knn_kernel_ms(ctx, "k_texture_knn_hamming")
        ctx.close()
    return out


def brisk_main():
    import torch
    torch.cuda.init()
    shapes = []
    for n_feat in (512, 2048, 4096):
        for n_bodies in (1, 8, 128):
            wl = synth.make_workload("c4", n_bodies=n_bodies, n_divides=2, seed=0)
            wl, ctx = make(wl, True, "brisk", n_feat=n_feat, central=True)
            queries = sum(int(ctx.get_texture_keyframes(b)["sizes"].sum()) for b in range(n_bodies))
            ms = knn_kernel_ms(ctx, "k_texture_knn_hamming")
            ms_step = time_calls(ctx, step(ctx, wl.n_corr_iterations, wl.n_update_iterations))
            points = int(np.mean([len(ctx.get_texture_points(b)) for b in range(n_bodies)]))
            shapes.append(dict(descriptor="brisk", bodies=n_bodies, queries=queries, train_per_body=n_feat,
                               ms_knn_hamming=ms, ms_step=ms_step, mean_data_points_per_body=points,
                               n_corr=wl.n_corr_iterations, n_update=wl.n_update_iterations))
            ctx.close()
    orb = {"this": [], "parent": []}
    if PARENT_LIB:
        script = os.path.abspath(__file__)
        for _ in range(3):
            for name, lib_path in (("this", None), ("parent", PARENT_LIB)):
                env = dict(os.environ)
                env.pop("M3TB_LIB", None)
                if lib_path:
                    env["M3TB_LIB"] = os.path.abspath(lib_path)
                r = subprocess.run([sys.executable, script, str(K), "--orb-knn-4096"], env=env, capture_output=True,
                                   text=True, check=True)
                orb[name].append(json.loads(r.stdout.strip().split("\n")[-1]))
    print(json.dumps(dict(descriptor="brisk", K=K, shapes=shapes, orb_knn_hamming_4096_ms=orb, gpu=gpu_name())))


if ORB_KNN:
    print(json.dumps(orb_knn_round()))
    sys.exit(0)
if DESCRIPTOR == "brisk":
    brisk_main()
    sys.exit(0)
if FEATURES is not None:
    assert 512 <= FEATURES <= 4096, FEATURES
    features_main(FEATURES)
    sys.exit(0)
if DESCRIPTOR is not None:
    assert DESCRIPTOR in L2_LENGTH, DESCRIPTOR
    l2_main(DESCRIPTOR)
    sys.exit(0)
wl = synth.make_workload("c4", n_bodies=128, n_divides=2, seed=0)
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
gpu = gpu_name()
print(json.dumps(dict(bodies=wl.n_bodies, features_per_body=N_FEAT, mean_data_points_per_body=n_points,
                      n_corr=wl.n_corr_iterations, n_update=wl.n_update_iterations, ms_texture_match=ms_match,
                      ms_step_without_texture=ms_plain, kernel_without_texture=plain_kernel, ms_step_with_texture=ms_tex,
                      kernel_with_texture=tex_kernel, ms_texture_overhead_per_step=ms_tex - ms_plain,
                      chains=CHAINS, links_per_chain=LINKS, chain_mean_data_points_per_link=chain_points,
                      chain_n_corr=2, chain_n_update=2, chain_ms_step_without_texture=ms_chain_plain,
                      chain_ms_step_with_texture=ms_chain_tex, chain_kernel_with_texture=chain_tex_kernel,
                      chain_ms_texture_overhead_per_step=ms_chain_tex - ms_chain_plain, gpu=gpu)))
