"""Writes texture_knn_binary64.npz: cv2.BFMatcher(NORM_HAMMING).knnMatch(k=2) on 64-byte descriptor sets that pin the
matcher's semantics the BRISK and FREAK texture modality depends on:

- brisk: real BRISK(25, 3, 0.6) descriptors (M3T's BRISK settings) of a focused crop of texture_crops.npz against
  those of an affinely warped copy, at most 512 per set (one chunk of the kNN kernel);
- brisk_large: BRISK of color_camera_image_200.png against a warped copy, 1024 queries and 4096 train rows (eight
  512-row chunks);
- orb_brisk: BRISK descriptors computed at ORB(300, 1.2, 3) keypoints, FREAK's pipeline shape (cv::ORB detects, a
  64-byte binary descriptor describes) with the descriptor cv2 has;
- ties (the earlier train descriptor wins), zero_zero (distance 0 to both neighbours, the ratio test's 0 / 0),
  equal_distance (equal distances in reverse index order), train_of_one (a single match), empty_train (no match);
- float_patterns: rows whose 32-bit words read as float NaN, inf and denormals (all 0xFF bytes among them), which a
  binary descriptor may hold and which must be matched bit for bit.

The ratio-test outcome follows from idx / dist (threshold 0.7: keep = idx[:, 1] >= 0 and not dist0 / dist1 >= 0.7).

    python tests/golden/make_texture_knn_binary64.py
"""
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
MAX_FEATURES = 512
CROP = 5  # a focused crop of texture_crops.npz with a few hundred BRISK keypoints


def brisk():
    return cv2.BRISK_create(25, 3, 0.6)  # texture_modality.h:413-415


def warped(gray, angle=12.0, scale=1.1):
    warp = cv2.getRotationMatrix2D((gray.shape[1] / 2, gray.shape[0] / 2), angle, scale)
    return cv2.warpAffine(gray, warp, (gray.shape[1], gray.shape[0]))


def describe(gray, limit):
    _, d = brisk().detectAndCompute(gray, None)
    d = np.zeros((0, 64), np.uint8) if d is None else d
    return np.ascontiguousarray(d[:limit], np.uint8)


def orb_brisk(gray):
    keypoints = cv2.ORB_create(300, 1.2, 3).detect(gray, None)  # texture_modality.h:410-412
    _, d = brisk().compute(gray, keypoints)
    return np.ascontiguousarray(d, np.uint8)


def float_patterns(rng):
    words = np.array([0xFFFFFFFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0x00000001, 0x80000001, 0x007FFFFF, 0],
                     np.uint32)
    q = words[rng.integers(0, len(words), (48, 16))]
    q[0] = 0xFFFFFFFF  # all 0xFF bytes
    q[1] = 0x7F800000  # every word +inf
    t = words[rng.integers(0, len(words), (80, 16))]
    t[:40] = q[:40]
    flips = rng.integers(0, 32, (40, 3))
    for k in range(3):  # a few flipped bits per copy, so that each query has a clear nearest row
        t[np.arange(40), rng.integers(0, 16, 40)] ^= np.uint32(1) << flips[:, k].astype(np.uint32)
    t = t[rng.permutation(80)]
    return q.view(np.uint8).reshape(48, 64), np.ascontiguousarray(t.view(np.uint8).reshape(80, 64))


def cases():
    crop = np.load(os.path.join(HERE, "texture_crops.npz"))["crops"][CROP]
    q, t = describe(crop, MAX_FEATURES), describe(warped(crop), MAX_FEATURES)
    yield "brisk", q, t
    image = cv2.cvtColor(cv2.imread(os.path.join(HERE, "color_camera_image_200.png")), cv2.COLOR_BGR2GRAY)
    yield "brisk_large", describe(image, 1024), describe(warped(image), 4096)
    yield "orb_brisk", orb_brisk(image), orb_brisk(warped(image))
    tie = t.copy()
    tie[10] = tie[40]  # two equal train rows: every query sees a tie between 10 and 40
    yield "ties", q[:64], tie[:96]
    zero = t[:96].copy()
    zero[70] = q[3]
    zero[71] = q[3]    # query 3: distance 0 to 70 and 71
    yield "zero_zero", q[:64], zero
    a, b = q[0].copy(), q[0].copy()  # train rows at equal distance 1 from query 0, in reverse index order
    a[5] ^= 1
    b[9] ^= 4
    yield "equal_distance", q[:4], np.stack([b, a, q[1], q[2]])
    yield "train_of_one", q[:8], t[:1]
    yield "empty_train", q[:8], t[:0]
    yield ("float_patterns",) + float_patterns(np.random.default_rng(64))


def main(out_dir=HERE):
    cv2.setNumThreads(1)
    m = cv2.BFMatcher(cv2.NORM_HAMMING)
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
    np.savez_compressed(os.path.join(out_dir, "texture_knn_binary64.npz"), **out)


if __name__ == "__main__":
    main()
