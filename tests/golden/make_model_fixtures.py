"""Collects the fixtures of the depth-model generation known answers into tests/golden/.

Run in the build container (where /root/reference is mounted); the GPU box only sees the committed copies.
Sources (DLR-RM/3DObjectTracking @ f0210618, M3T/):
  data/_body/schauma.obj             the body of data/model_test/depth_model*.bin, written as vertices + faces after
                                     Body::LoadMeshData's unit scaling and winding handling (body.cpp:201-249)
  data/model_test/depth_model_occlusion.bin   the same body, 12 views, the triangle prism as occlusion body
  (depth_model.bin is already here, copied by make_golden.py)
These are data fixtures (numbers), not source code.
"""
import os
import shutil

import numpy as np

REF = "/root/reference/M3T"
HERE = os.path.dirname(os.path.abspath(__file__))


def read_obj(path, unit_in_meter=1.0, counterclockwise=True):
    """Vertices [n,3] float32 (scaled) and triangles [m,3] int32 (0-based, clockwise files reversed)."""
    verts, faces = [], []
    for line in open(path):
        parts = line.split()
        if not parts:
            continue
        if parts[0] == "v":
            verts.append([np.float32(float(x)) for x in parts[1:4]])
        elif parts[0] == "f":
            idx = [int(p.split("/")[0]) - 1 for p in parts[1:]]
            if len(idx) != 3:
                continue  # the reference skips non-triangles
            faces.append(idx if counterclockwise else idx[::-1])
    v = np.array(verts, np.float32)
    if unit_in_meter != 1.0:
        v = v * np.float32(unit_in_meter)
    return v, np.array(faces, np.int32)


def main():
    # schauma.yaml: geometry_unit_in_meter 1.0, geometry_counterclockwise 1
    v, f = read_obj(f"{REF}/data/_body/schauma.obj", 1.0, True)
    np.savez_compressed(os.path.join(HERE, "schauma_mesh.npz"), vertices=v, faces=f)
    shutil.copy(f"{REF}/data/model_test/depth_model_occlusion.bin", os.path.join(HERE, "depth_model_occlusion.bin"))
    print("schauma:", v.shape, f.shape)


if __name__ == "__main__":
    main()
