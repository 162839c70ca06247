"""Writes texture_knn.npz: cv2.BFMatcher(NORM_HAMMING).knnMatch(k=2) on 32-byte descriptor sets that pin the matcher's
semantics the texture modality depends on: exact ties (the earlier train descriptor wins), distance 0 to both
neighbours (the ratio test's 0 / 0), a train set of one (a single match) and an empty train set (no match).

    python tests/golden/make_texture_knn.py
"""
import os

import cv2
import numpy as np


def cases():
    rng = np.random.default_rng(2024)
    q = rng.integers(0, 256, (64, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (96, 32), dtype=np.uint8)
    yield "random", q, t
    tie = t.copy()
    tie[10] = tie[40]  # two equal train rows: every query sees a tie between 10 and 40
    tie[70] = q[3]
    tie[71] = q[3]    # query 3: distance 0 to 70 and 71
    yield "ties", q, tie
    flip = q.copy()   # train rows at equal distance 1 from query 0, in reverse order
    a, b = flip[0].copy(), flip[0].copy()
    a[5] ^= 1
    b[9] ^= 4
    yield "equal_distance", q[:4], np.stack([b, a, q[1], q[2]])
    yield "train_of_one", q[:8], t[:1]
    yield "empty_train", q[:8], t[:0]


def main():
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
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "texture_knn.npz"), **out)


if __name__ == "__main__":
    main()
