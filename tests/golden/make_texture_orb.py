"""Writes tests/golden/texture_orb.npz: cv2's ORB (detect, then compute, as M3T runs it) on the 11 focused crops of
texture_crops.npz at every setting of texture_orb_reference.SETTINGS, and on golden body 3's crop of
texture_orb_reference.dot_frame() (ties at both cuts, more keypoints than n_features) at TIE_SETTING, in the canonical
order (level ascending, then row-major by the keypoint's pixel in its level), so the GPU tests need no cv2.

Each set is cv2's output; the NumPy restatement (tests/texture_orb_reference.py) supplies the order and must equal it
as a multiset, or the script stops. Run from the repository root: python tests/golden/make_texture_orb.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import texture_orb_reference as R  # noqa: E402


def main():
    import cv2
    crops = np.load(os.path.join(HERE, "texture_crops.npz"))
    out = {"settings": np.array([(n, s, l) for n, s, l in R.SETTINGS], np.float64), "cv2_version": np.array(cv2.__version__)}
    for si, (n, s, l) in enumerate(R.SETTINGS):
        counts, rows = [], {k: [] for k in ("xy", "angle", "response", "octave", "descriptors")}
        for i, (w, h) in enumerate(crops["sizes"]):
            img = np.ascontiguousarray(crops["crops"][i, :h, :w])
            mine, ref = R.orb(img, n, s, l), R.cv2_orb(img, n, s, l)
            if R.as_multiset(mine) != R.as_multiset(ref):
                raise SystemExit(f"the restatement differs from cv2 on crop {i} at {(n, s, l)}")
            counts.append(len(mine["angle"]))
            for k in rows:
                rows[k].append(mine[k])
        out[f"s{si}_n"] = np.array(counts, np.int32)
        for k, v in rows.items():
            out[f"s{si}_{k}"] = np.concatenate(v)
    # the tie frame: DetectAndComputeCorrKeypoints' crop of it (cvtColor, roi, resize by scale) as cv2 makes it
    roi, scale = crops["rois"][R.TIE_BODY], float(crops["scales"][R.TIE_BODY])
    grey = cv2.cvtColor(R.dot_frame(), cv2.COLOR_BGR2GRAY)
    x, y, w, h = (int(v) for v in roi)
    tie = cv2.resize(grey[y:y + h, x:x + w], None, fx=scale, fy=scale)
    mine, ref = R.orb(tie, *R.TIE_SETTING), R.cv2_orb(tie, *R.TIE_SETTING)
    if R.as_multiset(mine) != R.as_multiset(ref):
        raise SystemExit("the restatement differs from cv2 on the tie crop")
    if len(ref["angle"]) <= R.TIE_SETTING[0]:
        raise SystemExit("the tie crop keeps no more than n_features keypoints")
    out["tie_crop"] = tie
    for k in ("xy", "angle", "response", "octave", "descriptors"):
        out[f"tie_{k}"] = mine[k]
    np.savez_compressed(os.path.join(HERE, "texture_orb.npz"), **out)
    print("wrote texture_orb.npz:", {f"s{si}": [int(v) for v in out[f"s{si}_n"]] for si in range(len(R.SETTINGS))},
          "tie:", len(out["tie_angle"]))


if __name__ == "__main__":
    main()
