"""m3tb_render_full timed with CUDA events: 1, 16 and 128 full renderers, one per colour camera at 640x480 (and 16 at
1280x720), each drawing one schauma body (tests/golden/schauma_mesh.npz, 20,950 triangles) that the camera sees from
its own side. Every render of a case is one m3tb_render_full call, three launches for all renderers. Prints the card
name and power limit, then one JSON line per case."""
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

capi = importlib.import_module("3dobjecttracking_b200.capi")

K = int(sys.argv[1]) if len(sys.argv) > 1 else 50


def schauma():
    z = np.load(os.path.join(ROOT, "tests", "golden", "schauma_mesh.npz"))
    t = np.ascontiguousarray(z["vertices"][z["faces"]], np.float32)
    return t, 2.0 * float(np.linalg.norm(t.reshape(-1, 3), axis=1).max())


def camera(k, n, dist):
    """world2camera of camera k of n on a ring around the origin, looking at it."""
    a = 2.0 * np.pi * k / n
    c, s = np.cos(a), np.sin(a)
    R = np.array([[c, 0, -s], [0, 1, 0], [s, 0, c]])  # camera z axis towards the origin
    t = np.array([0.0, 0.0, dist])
    return np.hstack([R, t[:, None]]).astype(np.float32)


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)))
    tri, diam = schauma()
    body2world = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)[None]
    for (W, H), n in (((640, 480), 1), ((640, 480), 16), ((640, 480), 128), ((1280, 720), 16)):
        ctx = capi.Context(0, max_bodies=1, max_cameras=n, max_models=1)
        for k in range(n):
            ctx.set_color_camera(k, capi.Intrinsics(0.96 * W, 0.96 * W, W / 2, H / 2, W, H), camera(k, n, 2.0 * diam))
        ctx.set_poses(body2world)
        ctx.set_body_geometry(0, tri, None, diam, True, 1, 1)
        for k in range(n):
            ctx.set_full_renderer(k, "color", k, [0], 0.02, 10.0)
        for _ in range(5):
            ctx.render_full()
        ctx.synchronize()
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        ctx.render_full()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(K):
            ctx.render_full()
        e1.record(stream)
        e1.synchronize()
        sil = ctx.get_full_rendering(n - 1, W, H)["silhouette"]
        print(json.dumps(dict(mesh="schauma", triangles=int(tri.shape[0]), width=W, height=H, renderers=n,
                              ms_per_render=e0.elapsed_time(e1) / K, covered=float((sil != 0).mean()))))
        ctx.close()


if __name__ == "__main__":
    main()
