"""Vectorised restatement of the texture modality's Hamming matcher at any descriptor width (ORB's 32 bytes, BRISK /
FREAK's 64): cv::BFMatcher(NORM_HAMMING).knnMatch(k = 2) and the ratio test of CalculateCorrespondences, as
k_texture_knn_hamming and k_texture_match compute them. It gives what tests/texture_reference.py's knn2 / match give,
at sizes (4096 x 4096) that restatement's Python loops cannot reach."""
import numpy as np

f32 = np.float32
_POPCOUNT = np.unpackbits(np.arange(256, dtype=np.uint8)[:, None], axis=1).sum(1).astype(np.int32)


def distances(queries, train):
    """[nq, nt] int32 bit counts of queries XOR train."""
    q = np.asarray(queries, np.uint8)
    t = np.asarray(train, np.uint8).reshape(-1, q.shape[1])
    d = np.zeros((len(q), len(t)), np.int32)
    for c in range(q.shape[1]):
        d += _POPCOUNT[q[:, c, None] ^ t[None, :, c]]
    return d


def knn2(queries, train):
    """(idx [nq, 2] int32, dist [nq, 2] float32), -1 where there is no neighbour: the two first train rows of each
    query under (distance, index) order, which is what the insertion gives (a strictly smaller distance enters, ties
    keep the earlier index)."""
    q = np.asarray(queries, np.uint8)
    idx = np.full((len(q), 2), -1, np.int32)
    dist = np.full((len(q), 2), -1.0, f32)
    n = len(np.asarray(train).reshape(-1, q.shape[1])) if len(q) else 0
    if n == 0:
        return idx, dist
    d = distances(q, train)
    rows = np.arange(len(q))
    idx[:, 0] = np.argmin(d, 1)  # the first index of the minimum
    dist[:, 0] = d[rows, idx[:, 0]]
    if n > 1:
        d[rows, idx[:, 0]] = np.iinfo(np.int32).max
        idx[:, 1] = np.argmin(d, 1)
        dist[:, 1] = d[rows, idx[:, 1]]
    return idx, dist


def knn2_insertion(queries, train):
    """knn2 as cv::batchDistance's K = 2 insertion computes it, train row by train row in index order (a strictly
    smaller distance enters, ties keep the earlier index): per query [(train_idx, distance), ...], at most 2."""
    out = []
    for row in distances(queries, train):
        best = []
        for j, d in enumerate(row.tolist()):
            if len(best) < 2 or d < best[1][1]:
                k = len(best) if len(best) < 2 else 1
                while k > 0 and best[k - 1][1] > d:
                    k -= 1
                best.insert(k, (j, d))
                best = best[:2]
        out.append(best)
    return out


def kept(idx, dist, threshold):
    """The ratio test: a second neighbour and not dist0 / dist1 >= threshold (0 / 0 is NaN and keeps the match)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        return (idx[:, 1] >= 0) & ~(dist[:, 0] / dist[:, 1] >= f32(threshold))


def match(keyframes, frame_xy, frame_desc, threshold):
    """CalculateCorrespondences at corr_iteration 0: keyframes = [(points [n, 3], descriptors [n, width])] front to
    back. Returns (center_f_body [m, 3], correspondence_center [m, 2])."""
    cb, cc = [np.zeros((0, 3), f32)], [np.zeros((0, 2), f32)]
    for pts, desc in keyframes:
        if len(desc) == 0 or len(frame_desc) == 0:
            continue
        idx, dist = knn2(desc, frame_desc)
        keep = kept(idx, dist, threshold)
        cb.append(np.asarray(pts, f32)[keep])
        cc.append(np.asarray(frame_xy, f32)[idx[keep, 0]])
    return np.concatenate(cb).astype(f32), np.concatenate(cc).astype(f32)
