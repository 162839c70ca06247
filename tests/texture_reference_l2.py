"""CPU restatement of the texture modality's L2 matcher for float descriptors (SIFT / DAISY): brute-force
cv::BFMatcher(NORM_L2) kNN (k = 2) and the ratio test of CalculateCorrespondences, as k_texture_knn_l2 and
k_texture_match compute them. Everything else of the modality (keyframes, projection, gradients) is the ORB
restatement's, tests/texture_reference.py."""
import numpy as np

f32 = np.float32


def knn2_l2(queries, train):
    """cv::BFMatcher(NORM_L2).knnMatch(k = 2): per query [(train_idx, distance), ...] (at most 2, best first). The sum
    of squared differences is exact (int64) for whole-number descriptors and float64 otherwise, then rounded to float32
    and passed through sqrt; a distance enters only if strictly below the second (FLT_MAX at first), so NaN and inf
    never do, and ties keep the earlier train index."""
    q = np.asarray(queries, f32)
    t = np.asarray(train, f32)
    q = q.reshape(len(q), -1)
    t = t.reshape(len(t), q.shape[1])
    whole = bool(np.all(q == np.round(q)) and np.all(t == np.round(t)))
    dtype = np.int64 if whole else np.float64
    qd, td = q.astype(dtype), t.astype(dtype)
    out = []
    for i in range(len(q)):
        with np.errstate(over="ignore", invalid="ignore"):
            s = ((qd[i][None, :] - td) ** 2).sum(1)
            d = np.sqrt(s.astype(f32))
        best = []
        for j, dj in enumerate(d):
            if not dj < (best[1][1] if len(best) == 2 else f32(3.4028235e38)):
                continue
            k = len(best) if len(best) < 2 else 1
            while k > 0 and best[k - 1][1] > dj:
                k -= 1
            best.insert(k, (j, f32(dj)))
            best = best[:2]
        out.append(best)
    return out


def match_l2(keyframes, frame_xy, frame_desc, threshold):
    """match for float descriptors (SIFT / DAISY, knn2_l2): keyframes = [(points [n, 3], descriptors [n, length])]."""
    cb, cc = [], []
    for pts, desc in keyframes:
        if len(desc) == 0 or len(frame_desc) == 0:
            continue
        for q, m in enumerate(knn2_l2(desc, frame_desc)):
            if len(m) < 2:
                continue
            with np.errstate(invalid="ignore", divide="ignore"):
                if f32(m[0][1]) / f32(m[1][1]) >= f32(threshold):
                    continue
            cb.append(pts[q])
            cc.append(frame_xy[m[0][0]])
    return np.array(cb, f32).reshape(-1, 3), np.array(cc, f32).reshape(-1, 2)
