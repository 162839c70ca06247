"""The NumPy restatement of cv::ORB (tests/texture_orb_reference.py) against cv2: bit-equal detect + compute as a
multiset of (x, y, angle, response, octave, descriptor) on the golden crops, random textured images of several sizes
and tie-heavy dot grids and a checkerboard, at every setting; the same at every setting of R.SWEEP on noise, 0 / 255
noise, constant, ramp and textured images with a side of 63 px; no keypoints wherever cv2 raises on an empty pyramid
level, although the earlier levels have some; stage checks against cv2's resize, sepFilter2D and FastFeatureDetector;
the committed rBRIEF pattern against cv2's binary; the golden file against the restatement."""
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


def _compare(name, img, setting):
    """R against cv2 on one image: equal multisets where cv2 detects, nothing where cv2 raises. Returns the keypoint
    count compared, or None where cv2 raised."""
    mine = R.orb(img, *setting)
    try:
        ref = R.cv2_orb(img, *setting)
    except cv2.error:  # cv::resize refuses an empty pyramid level: nothing is detected
        assert R.empty_pyramid(img.shape[1], img.shape[0], setting[1], setting[2]), name
        assert len(mine["angle"]) == 0, name
        return None
    assert R.as_multiset(mine) == R.as_multiset(ref), (name, len(mine["angle"]), len(ref["angle"]))
    # canonical order: level ascending, then row-major in the level
    key = mine["octave"].astype(np.int64) << 40 | mine["lxy"][:, 1].astype(np.int64) << 20 | mine["lxy"][:, 0]
    assert (np.diff(key) > 0).all(), name
    return len(ref["angle"])


@pytest.mark.parametrize("setting", R.SETTINGS, ids=lambda s: "%d-%g-%d" % s)
def test_restatement_equals_cv2(setting):
    compared = sum(_compare(name, img, setting) or 0 for name, img in INPUTS)
    assert compared > 1000


def _sweep_inputs():
    crop = lambda i: np.ascontiguousarray(CROPS["crops"][i, :CROPS["sizes"][i][1], :CROPS["sizes"][i][0]])
    return [("noise200", R.noise(200, 200, 1)), ("binary150x170", R.binary_noise(150, 170, 2)),
            ("constant", np.full((100, 100), 128, np.uint8)), ("ramp120x90", R.ramp(120, 90)),
            ("textured63x200", R.textured(63, 200, 11)), ("textured200x63", R.textured(200, 63, 12)),
            ("textured300", R.textured(300, 300, 13)), ("textured320_block8", R.textured(320, 320, 14, block=8)),
            ("dots", R.dot_grid()), ("checkerboard", R.checkerboard()), ("crop3", crop(3)), ("crop9", crop(9))]


SWEEP_INPUTS = _sweep_inputs()


@pytest.mark.parametrize("setting", R.SWEEP, ids=lambda s: "%d-%.9g-%d" % s)
def test_restatement_equals_cv2_across_the_sweep(setting):
    counts = [_compare(name, img, setting) for name, img in SWEEP_INPUTS]
    if setting[2] < 5:  # no sweep input is small enough for an empty level there
        assert None not in counts
    if setting[0] >= 20 and setting[1] < 3.0:
        assert sum(c or 0 for c in counts) > 20 * setting[2]


def test_an_empty_pyramid_level_gives_no_keypoints():
    """cv::ORB builds every level before it detects: where one level has a side of 0 pixels cv2 raises and detects
    nothing, although the earlier levels have keypoints. 10 of the 11 golden crops at (300, 2.5, 8), and a textured
    63 x 200 image at (300, 3.0, 8)."""
    cases = [(f"crop{i}", np.ascontiguousarray(CROPS["crops"][i, :h, :w]), (300, 2.5, 8))
             for i, (w, h) in enumerate(CROPS["sizes"])]
    cases.append(("textured63x200", R.textured(63, 200, 11), (300, 3.0, 8)))
    empty = 0
    for name, img, (n, sf, nl) in cases:
        h, w = img.shape
        if not R.empty_pyramid(w, h, sf, nl):
            assert name == "crop2"  # 369 px: level 7 is 1 px, and the crop has no keypoints at any setting
            assert _compare(name, img, (n, sf, nl)) == 0
            continue
        empty += 1
        with pytest.raises(cv2.error):
            R.cv2_orb(img, n, sf, nl)
        stages = {}
        assert len(R.orb(img, n, sf, nl, stages=stages)["angle"]) == 0
        assert stages["empty_pyramid"] and "levels" not in stages
        # the levels before the first empty one do have keypoints, which cv::ORB does not return
        full = next(k for k in range(1, nl + 1) if R.empty_pyramid(w, h, sf, k + 1))
        assert len(R.orb(img, n, sf, full)["angle"]) > 0, name
    assert empty == 11


def test_stage_counts():
    """orb(stages=...) records the FAST corners of each level, those inside the border the first cut ranks, and the
    counts after both cuts; the GPU sweep reads them for its branch coverage."""
    stages = {}
    res = R.orb(R.dot_grid(), 20, stages=stages)
    assert stages["per_level"] == R.features_per_level(20, 1.2, 3) == [8, 7, 5] and not stages["empty_pyramid"]
    assert stages["n_corners"] == [0, 625, 615] and stages["n_fast"] == [0, 361, 289]
    xs, ys, _ = R.fast_corners(stages["levels"][2])
    h, w = stages["levels"][2].shape
    assert ((xs >= 31) & (xs < w - 31) & (ys >= 31) & (ys < h - 31)).sum() == 289
    # level 1 ties at both cuts and keeps every candidate; level 2 ties at the Harris cut only
    assert stages["n_first_cut"] == [0, 361, 16] and stages["n_second_cut"] == [0, 361, 5]
    assert sum(stages["n_second_cut"]) == len(res["angle"]) == 366


def test_nonpositive_harris_responses_are_kept_like_cv2():
    """At n_features 2^24 the cuts keep everything, so keypoints with a Harris response <= 0 survive."""
    img = R.textured(300, 300, 13)
    mine = R.orb(img, 1 << 24, 1.2, 3)
    assert (mine["response"] <= 0).sum() > 0
    assert R.as_multiset(mine) == R.as_multiset(R.cv2_orb(img, 1 << 24, 1.2, 3))


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
