"""Writes texture_knn_large.npz: cv2.BFMatcher kNN (k = 2) on train sets above 512 descriptors, for the texture
modality's large-capacity matchers (n_features_max up to 4096, k_texture_knn_l2 / k_texture_knn_hamming):

- sift_*: M3T's default SIFT (cv2.SIFT_create(0, 5, 0.04, 10, 0.7), every keypoint kept) of the committed focused crops
  (texture_crops.npz), untruncated: sift_n holds the keypoint count of every crop (16 to 2339), sift_desc the
  descriptors of the crops in SIFT_CROPS (sift_crops, sift_offset), as uint8 (SIFT writes whole numbers up to 255,
  asserted here); sift_pairs lists (query crop, train crop) and sift_idx / sift_dist the NORM_L2 kNN of each pair,
  concatenated in pair order.
- orb_*: cv2.ORB_create(4096, 1.2, 3) on color_camera_image_200.png against an affinely warped copy, NORM_HAMMING.
- syn_{ham,l2}_{511,512,513,1024,4096}_{idx,dist}: the kNN of the synthetic sets of tests/texture_knn_sets.py (made
  from a fixed hash, so only the results are stored).

    python tests/golden/make_texture_knn_large.py
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import texture_knn_sets  # noqa: E402

SIFT_CROPS = (3, 5, 9)  # 2339, 560 and 398 keypoints
SIFT_PAIRS = [(3, 5), (5, 3), (5, 9)]


def knn(matcher, q, t):
    res = matcher.knnMatch(q, t, k=2) if len(t) else [[] for _ in range(len(q))]
    idx = np.full((len(q), 2), -1, np.int32)
    dist = np.full((len(q), 2), -1.0, np.float32)
    for i, r in enumerate(res):
        for k, d in enumerate(r):
            idx[i, k], dist[i, k] = d.trainIdx, d.distance
    return idx, dist


def sift_crops():
    z = np.load(os.path.join(HERE, "texture_crops.npz"))
    sift = cv2.SIFT_create(0, 5, 0.04, 10, 0.7)
    out = []
    for crop, (w, h) in zip(z["crops"], z["sizes"]):
        _, d = sift.detectAndCompute(np.ascontiguousarray(crop[:h, :w]), None)
        d = np.zeros((0, 128), np.float32) if d is None else d
        assert np.all(d == np.round(d)) and d.min() >= 0 and d.max() <= 255, "SIFT descriptors are whole numbers"
        out.append(d.astype(np.uint8))
    return out


def orb_sets():
    gray = cv2.cvtColor(cv2.imread(os.path.join(HERE, "color_camera_image_200.png")), cv2.COLOR_BGR2GRAY)
    warp = cv2.getRotationMatrix2D((gray.shape[1] / 2, gray.shape[0] / 2), 12.0, 1.1)
    orb = cv2.ORB_create(4096, 1.2, 3)
    _, q = orb.detectAndCompute(gray, None)
    _, t = orb.detectAndCompute(cv2.warpAffine(gray, warp, (gray.shape[1], gray.shape[0])), None)
    return q, t


def main(out_dir=HERE):
    cv2.setNumThreads(1)
    l2, ham = cv2.BFMatcher(cv2.NORM_L2), cv2.BFMatcher(cv2.NORM_HAMMING)
    out = {}
    crops = sift_crops()
    out["sift_n"] = np.array([len(d) for d in crops], np.int32)
    out["sift_crops"] = np.array(SIFT_CROPS, np.int32)
    out["sift_offset"] = np.concatenate([[0], np.cumsum([len(crops[c]) for c in SIFT_CROPS])[:-1]]).astype(np.int32)
    out["sift_desc"] = np.concatenate([crops[c] for c in SIFT_CROPS])
    out["sift_pairs"] = np.array(SIFT_PAIRS, np.int32)
    idx, dist = zip(*(knn(l2, crops[a].astype(np.float32), crops[b].astype(np.float32)) for a, b in SIFT_PAIRS))
    out["sift_idx"], out["sift_dist"] = np.concatenate(idx), np.concatenate(dist)
    q, t = orb_sets()
    out["orb_queries"], out["orb_train"] = q, t
    out["orb_idx"], out["orb_dist"] = knn(ham, q, t)
    for name, hamming in (("ham", True), ("l2", False)):
        for n in texture_knn_sets.SIZES:
            q, t = texture_knn_sets.synthetic(n, hamming)
            m = ham if hamming else l2
            cast = (lambda a: a) if hamming else (lambda a: a.astype(np.float32))
            out["syn_%s_%d_idx" % (name, n)], out["syn_%s_%d_dist" % (name, n)] = knn(m, cast(q), cast(t))
    np.savez_compressed(os.path.join(out_dir, "texture_knn_large.npz"), **out)


if __name__ == "__main__":
    main()
