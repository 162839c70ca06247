"""Writes texture_knn_l2.npz: cv2.BFMatcher(NORM_L2).knnMatch(k=2) on float descriptor sets that pin the matcher's
semantics the SIFT and DAISY texture modality depends on: real SIFT descriptors of color_camera_image_200.png against
those of an affinely warped copy (M3T's SIFT settings, at most 512 per set), exact ties (the earlier train descriptor
wins), distance 0 to both neighbours (the ratio test's 0 / 0), equal distances in reverse index order, a train set of
one (a single match), an empty train set (no match), and unit-norm DAISY-like sets of lengths 104 and 200.

    python tests/golden/make_texture_knn_l2.py
"""
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
MAX_FEATURES = 512


def sift(gray):
    # M3T's SIFT settings (texture_modality.h): nfeatures 0, n_octave_layers 5, contrast 0.04, edge 10, sigma 0.7
    _, d = cv2.SIFT_create(0, 5, 0.04, 10, 0.7).detectAndCompute(gray, None)
    return np.ascontiguousarray(d[:MAX_FEATURES], np.float32)


def daisy_like(rng, n, length):
    v = rng.random((n, length)).astype(np.float32)
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def cases():
    gray = cv2.cvtColor(cv2.imread(os.path.join(HERE, "color_camera_image_200.png")), cv2.COLOR_BGR2GRAY)
    warp = cv2.getRotationMatrix2D((gray.shape[1] / 2, gray.shape[0] / 2), 12.0, 1.1)
    q, t = sift(gray), sift(cv2.warpAffine(gray, warp, (gray.shape[1], gray.shape[0])))
    yield "sift", q, t
    tie = t.copy()
    tie[10] = tie[40]  # two equal train rows: every query sees a tie between 10 and 40
    tie[70] = q[3]
    tie[71] = q[3]     # query 3: distance 0 to 70 and 71
    yield "ties", q[:64], tie[:96]
    a, b = q[0].copy(), q[0].copy()  # train rows at equal distance 1 from query 0, in reverse index order
    a[5] += 1
    b[9] -= 1
    yield "equal_distance", q[:4], np.stack([b, a, q[1], q[2]])
    yield "train_of_one", q[:8], t[:1]
    yield "empty_train", q[:8], t[:0]
    rng = np.random.default_rng(2025)
    for length in (104, 200):
        dq = daisy_like(rng, 100, length)
        noisy = dq[:75] + rng.normal(0, 0.02, (75, length)).astype(np.float32)
        noisy = (noisy / np.linalg.norm(noisy, axis=1, keepdims=True)).astype(np.float32)
        dt = np.vstack([noisy, daisy_like(rng, 75, length)])[rng.permutation(150)]
        yield "daisy%d" % length, dq, np.ascontiguousarray(dt, np.float32)


def main(out_dir=HERE):
    cv2.setNumThreads(1)
    m = cv2.BFMatcher(cv2.NORM_L2)
    out = {}
    for name, q, t in cases():
        res = m.knnMatch(q, t, k=2) if len(t) else [[] for _ in range(len(q))]
        idx = np.full((len(q), 2), -1, np.int32)
        dist = np.full((len(q), 2), -1.0, np.float32)
        for i, r in enumerate(res):
            for k, d in enumerate(r):
                idx[i, k], dist[i, k] = d.trainIdx, d.distance
        out[name + "_queries"], out[name + "_train"] = q, t
        out[name + "_idx"], out[name + "_dist"] = idx, dist
    np.savez_compressed(os.path.join(out_dir, "texture_knn_l2.npz"), **out)


if __name__ == "__main__":
    main()
