"""The NumPy restatement of cv::ORB (tests/texture_orb_reference.py) against cv2: bit-equal detect + compute as a
multiset of (x, y, angle, response, octave, descriptor) on the golden crops, random textured images of several sizes
and tie-heavy dot grids and a checkerboard, at every setting; stage checks against cv2's resize, sepFilter2D and
FastFeatureDetector; the committed rBRIEF pattern against cv2's binary; the golden file against the restatement."""
import os

import numpy as np
import pytest

import texture_orb_reference as R

cv2 = pytest.importorskip("cv2")
HERE = os.path.dirname(os.path.abspath(__file__))
CROPS = np.load(os.path.join(HERE, "golden", "texture_crops.npz"))


def _inputs():
    out = [(f"crop{i}", np.ascontiguousarray(CROPS["crops"][i, :h, :w])) for i, (w, h) in enumerate(CROPS["sizes"])]
    out += [(f"random{s}", R.textured(s, s, s)) for s in R.RANDOM_SIZES]
    out += [("random640x480", R.textured(480, 640, 5)), ("dots", R.dot_grid()), ("dense_dots", R.dot_grid(spacing=6)),
            ("checkerboard", R.checkerboard())]
    return out


INPUTS = _inputs()


@pytest.mark.parametrize("setting", R.SETTINGS, ids=lambda s: "%d-%g-%d" % s)
def test_restatement_equals_cv2(setting):
    compared = 0
    for name, img in INPUTS:
        mine = R.orb(img, *setting)
        try:
            ref = R.cv2_orb(img, *setting)
        except cv2.error:  # cv::resize refuses an empty level (a 1-pixel image at 8 levels); nothing is detected
            assert len(mine["angle"]) == 0, name
            continue
        assert R.as_multiset(mine) == R.as_multiset(ref), (name, len(mine["angle"]), len(ref["angle"]))
        compared += len(ref["angle"])
        # canonical order: level ascending, then row-major in the level
        key = mine["octave"].astype(np.int64) << 40 | mine["lxy"][:, 1].astype(np.int64) << 20 | mine["lxy"][:, 0]
        assert (np.diff(key) > 0).all(), name
    assert compared > 1000


def test_ties_are_kept_at_both_cuts():
    # cv::ORB keeps more than n_features when scores tie at a cut
    assert len(R.cv2_orb(R.dot_grid(), 300)["angle"]) == len(R.orb(R.dot_grid(), 300)["angle"]) == 444
    assert len(R.orb(R.dot_grid(), 20)["angle"]) == 366
    assert len(R.orb(R.dot_grid(spacing=6), 300)["angle"]) == 1453


def test_stages_equal_cv2():
    rng = np.random.default_rng(3)
    for h, w in [(216, 216), (240, 242), (100, 120), (369, 369), (7, 9), (1, 1), (64, 65)]:
        img = rng.integers(0, 256, (h, w)).astype(np.uint8)
        for lw, lh in R.level_sizes(w, h, 1.2, 8)[1:] + R.level_sizes(w, h, 2.0, 3)[1:]:
            if lw >= 1 and lh >= 1:
                assert np.array_equal(R.resize_linear_exact(img, lw, lh),
                                      cv2.resize(img, (lw, lh), interpolation=cv2.INTER_LINEAR_EXACT)), ((h, w), (lw, lh))
    k = cv2.getGaussianKernel(7, 2, ktype=cv2.CV_32F)
    assert np.array_equal(R.GAUSS, k.ravel())
    for i, (w, h) in enumerate(CROPS["sizes"]):
        img = np.ascontiguousarray(CROPS["crops"][i, :h, :w])
        assert np.array_equal(R.gaussian_blur(img), cv2.sepFilter2D(img, -1, k, k, borderType=cv2.BORDER_REFLECT_101))
        fd = cv2.FastFeatureDetector_create(R.FAST_THRESHOLD, True)
        kps = fd.detect(img)
        ref = sorted((int(p.pt[1]), int(p.pt[0]), int(p.response)) for p in kps)
        xs, ys, sc = R.fast_corners(img)
        assert ref == sorted(zip(ys.tolist(), xs.tolist(), sc.tolist()))
    for y, x in [(0, 0), (3, -4), (-7, 2), (5, 5), (-9, -9), (1000, -1), (0, -3)]:
        assert R.fast_atan2(np.float32(y), np.float32(x)) == np.float32(cv2.fastAtan2(float(y), float(x)))


def test_bit_pattern_is_cv2s():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_orb_pattern", os.path.join(R.ROOT, "scripts", "make_orb_pattern.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert np.array_equal(mod.pattern_from_header(), mod.pattern_from_cv2())


def test_golden_file_matches_the_restatement():
    g = np.load(os.path.join(HERE, "golden", "texture_orb.npz"))
    for si, setting in enumerate(R.SETTINGS):
        at = 0
        for i, (w, h) in enumerate(CROPS["sizes"]):
            mine = R.orb(np.ascontiguousarray(CROPS["crops"][i, :h, :w]), *setting)
            n = int(g[f"s{si}_n"][i])
            assert n == len(mine["angle"])
            for k in ("xy", "angle", "response", "octave", "descriptors"):
                assert np.array_equal(g[f"s{si}_{k}"][at:at + n].view(np.uint8), mine[k].view(np.uint8)), (si, i, k)
            at += n


def test_golden_tie_crop():
    """The tie crop in the golden file is the device crop's restatement of dot_frame at golden body 3's focus, and cv::ORB
    keeps more keypoints there than n_features."""
    import texture_crop_reference as C
    g = np.load(os.path.join(HERE, "golden", "texture_orb.npz"))
    crop = C.crop(R.dot_frame(), CROPS["rois"][R.TIE_BODY], CROPS["scales"][R.TIE_BODY])
    assert np.array_equal(g["tie_crop"], crop)
    mine = R.orb(crop, *R.TIE_SETTING)
    assert len(mine["angle"]) == len(g["tie_angle"]) == 566 > R.TIE_SETTING[0]
    for k in ("xy", "angle", "response", "octave", "descriptors"):
        assert np.array_equal(g[f"tie_{k}"].view(np.uint8), mine[k].view(np.uint8)), k
    assert R.as_multiset(mine) == R.as_multiset(R.cv2_orb(crop, *R.TIE_SETTING))
