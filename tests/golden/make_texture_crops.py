"""Writes texture_crops.npz: the texture modality's focused grey images of color_camera_image_200.png, made by cv2
itself (cvtColor BGR2GRAY, the focus region, resize by scale with INTER_LINEAR), at body poses whose focus region
and scale tests/texture_reference.py computes, and the cv2.ORB and cv2.SIFT features detected on each crop. The poses
cover downscaled and upscaled crops, a distant body, scale exactly 0.5 (on an even and on an odd region) and exactly 1, and focus regions clipped at each
image border. The GPU tests compare k_texture_crop with these crops and feed these features to the device upload,
so they need no cv2.

    python tests/golden/make_texture_crops.py
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import texture_reference as tr  # noqa: E402

MAX_FEATURES = 512
FOCUSED_IMAGE_SIZE = 200
DIAMETER = np.float32(0.07764273136854172)  # synth.prism_triangles()' maximum body diameter
# world = camera; intrinsics of the 960 x 540 frame
INTR = dict(fu=614.0, fv=614.5, ppu=480.3, ppv=270.1, width=960, height=540)


def pose(t, rot_deg=0.0):
    c, s = np.cos(np.radians(rot_deg)), np.sin(np.radians(rot_deg))
    R = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
    return np.hstack([R, np.array(t, float)[:, None]]).astype(np.float32)


def radius():
    return np.float32(0.5) * DIAMETER


def exact_scale(target, odd=False):
    """A pose straight ahead whose focus scale is exactly `target`: bisect z (the scale grows with z), then walk the
    float32 values around the crossing; another small x offset when none hits. odd: the focus region must also have
    an odd width and height (at 0.5, cv::resize's 2x INTER_AREA path then averages a cut last column and row)."""
    for xi in range(200):
        x = np.float32((1.7e-3 if odd else 1e-4) * xi)
        y = np.float32(1.1e-3 * xi if odd else 0.0)
        lo, hi = np.float32(0.06), np.float32(3.0)
        for _ in range(60):
            mid = np.float32((lo + hi) / 2)
            f = tr.focus(INTR, pose((x, y, mid)).reshape(12), radius(), FOCUSED_IMAGE_SIZE)
            if f is None or f[1] < target:
                lo = mid
            else:
                hi = mid
        for direction in (np.float32(0), np.float32(np.inf)):
            z = hi
            for _ in range(40):
                f = tr.focus(INTR, pose((x, y, z)).reshape(12), radius(), FOCUSED_IMAGE_SIZE)
                if f is not None and f[1] == np.float32(target) and (not odd or (f[0][2] % 2 and f[0][3] % 2)):
                    return pose((x, y, z))
                z = np.nextafter(z, direction)
    raise RuntimeError("no pose with scale %r" % target)


def poses():
    z = 0.3
    edge = lambda u, v: (float((u - INTR["ppu"]) * z / INTR["fu"]), float((v - INTR["ppv"]) * z / INTR["fv"]), z)
    return np.stack([
        pose((0.0, 0.0, 0.2)),                 # downscaled
        pose((0.01, -0.005, 0.5), 20.0),       # upscaled
        pose((-0.02, 0.01, 2.0)),              # distant: a large scale
        exact_scale(0.5),
        exact_scale(1.0),
        pose(edge(15.0, 270.0)),               # clipped at the left border
        pose(edge(945.0, 270.0)),              # right
        pose(edge(480.0, 12.0)),               # top
        pose(edge(480.0, 528.0)),              # bottom
        pose((0.03, 0.02, 0.35), -15.0),
        exact_scale(0.5, odd=True),
    ])


def main(out_dir=HERE):
    cv2.setNumThreads(1)
    image = cv2.imread(os.path.join(HERE, "color_camera_image_200.png"), cv2.IMREAD_COLOR)
    grey = cv2.cvtColor(image, cv2.COLOR_BGR2GRAY)
    P = poses()
    n = len(P)
    rois = np.zeros((n, 4), np.int32)
    scales = np.zeros(n, np.float32)
    crops = []
    orb_n = np.zeros(n, np.int32)
    orb_xy = np.zeros((n, MAX_FEATURES, 2), np.float32)
    orb_desc = np.zeros((n, MAX_FEATURES, 32), np.uint8)
    sift_n = np.zeros(n, np.int32)
    sift_xy = np.zeros((n, MAX_FEATURES, 2), np.float32)
    sift_desc = np.zeros((n, MAX_FEATURES, 128), np.float32)
    orb = cv2.ORB_create(MAX_FEATURES)
    sift = cv2.SIFT_create(0, 5, 0.04, 10, 0.7)  # M3T's SIFT settings (texture_modality.h)
    for b in range(n):
        roi, scale = tr.focus(INTR, P[b].reshape(12), radius(), FOCUSED_IMAGE_SIZE)
        x, y, w, h = roi
        s = float(scale)
        crop = cv2.resize(grey[y:y + h, x:x + w], None, fx=s, fy=s, interpolation=cv2.INTER_LINEAR)
        rois[b], scales[b] = roi, scale
        crops.append(crop)
        for det, nn, xy, desc in ((orb, orb_n, orb_xy, orb_desc), (sift, sift_n, sift_xy, sift_desc)):
            kps, d = det.detectAndCompute(crop, None)
            k = min(len(kps), MAX_FEATURES)
            nn[b] = k
            if k:
                xy[b, :k] = np.array([kp.pt for kp in kps[:k]], np.float32)
                desc[b, :k] = d[:k]
    cap_h = max(c.shape[0] for c in crops)
    cap_w = max(c.shape[1] for c in crops)
    crop_arr = np.zeros((n, cap_h, cap_w), np.uint8)
    sizes = np.zeros((n, 2), np.int32)
    for b, c in enumerate(crops):
        crop_arr[b, :c.shape[0], :c.shape[1]] = c
        sizes[b] = (c.shape[1], c.shape[0])
    np.savez_compressed(os.path.join(out_dir, "texture_crops.npz"), poses=P, rois=rois, scales=scales, crops=crop_arr,
                        sizes=sizes, intrinsics=np.array([INTR[k] for k in ("fu", "fv", "ppu", "ppv", "width",
                                                                             "height")], np.float32),
                        diameter=DIAMETER, focused_image_size=np.int32(FOCUSED_IMAGE_SIZE), orb_n=orb_n, orb_xy=orb_xy,
                        orb_desc=orb_desc, sift_n=sift_n, sift_xy=sift_xy, sift_desc=sift_desc)


if __name__ == "__main__":
    main()
