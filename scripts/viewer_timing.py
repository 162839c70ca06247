"""m3tb_update_viewers timed with CUDA events: one NormalColorViewer over 1, 8 and 64 bodies at 640x480 and 1280x720,
with the 5120-triangle icosphere and the schauma mesh (tests/golden/schauma_mesh.npz). The bodies sit on a grid in front
of the camera, the single body close enough to fill a large part of the frame. Prints the card name and power limit,
then one JSON line per case."""
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

K = int(sys.argv[1]) if len(sys.argv) > 1 else 100


def meshes():
    tri, diam = synth.icosphere_triangles(0.04, 4)
    out = {"icosphere5120": (tri, diam)}
    z = np.load(os.path.join(ROOT, "tests", "golden", "schauma_mesh.npz"))
    t = np.ascontiguousarray(z["vertices"][z["faces"]], np.float32)
    out["schauma"] = (t, 2.0 * float(np.linalg.norm(t.reshape(-1, 3), axis=1).max()))
    return out


def poses(n, diam, W):
    """n bodies on a square grid, spaced by their diameter; one body alone sits at 2.5 diameters."""
    k = int(np.ceil(np.sqrt(n)))
    z = 2.5 * diam if n == 1 else 1.1 * diam * k
    out = np.zeros((n, 3, 4), np.float32)
    for b in range(n):
        a = 0.3 * b
        c, s = np.cos(a), np.sin(a)
        out[b, :, :3] = [[c, 0, s], [0, 1, 0], [-s, 0, c]]
        out[b, :, 3] = ((b % k - (k - 1) / 2) * diam, (b // k - (k - 1) / 2) * diam, z)
    return out


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps(dict(gpu=gpu)))
    w2c = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
    for name, (tri, diam) in meshes().items():
        for W, H in ((640, 480), (1280, 720)):
            for n in (1, 8, 64):
                ctx = capi.Context(0, max_bodies=n, max_cameras=1, max_models=1)
                ctx.set_color_camera(0, capi.Intrinsics(0.96 * W, 0.96 * W, W / 2, H / 2, W, H), w2c)
                ctx.set_poses(poses(n, diam, W))
                for b in range(n):
                    ctx.set_body_geometry(b, tri, None, diam, True)
                ctx.upload_color(0, np.random.default_rng(0).integers(0, 256, (H, W, 3), dtype=np.uint8))
                ctx.set_viewer(0, "color", 0, list(range(n)))
                for _ in range(10):
                    ctx.update_viewers()
                ctx.synchronize()
                stream = torch.cuda.Stream()
                ctx.set_stream(stream.cuda_stream)
                ctx.update_viewers()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(K):
                    ctx.update_viewers()
                e1.record(stream)
                e1.synchronize()
                _, normal = ctx.get_viewer_image(0, W, H)
                print(json.dumps(dict(mesh=name, triangles=int(tri.shape[0]), width=W, height=H, bodies=n,
                                      ms_per_update=e0.elapsed_time(e1) / K,
                                      covered=float((normal[..., 3] == 255).mean()))))
                ctx.close()


if __name__ == "__main__":
    main()
