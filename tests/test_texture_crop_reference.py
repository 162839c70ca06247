"""tests/texture_crop_reference.py (the integers k_texture_crop computes) against cv2 itself: the grey conversion on
every BGR triple, and the crop over a sweep of focus regions and scales (up and down, 0.5 and 1 exactly, 1-px-wide
regions, regions clipped at each image border)."""
import os

import numpy as np
import pytest

import texture_crop_reference as cr

cv2 = pytest.importorskip("cv2")

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def test_grey_equals_cvtcolor_on_every_triple():
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.empty((4096, 4096, 3), np.uint8)
    flat = img.reshape(-1, 3)
    flat[:, 0] = v & 255
    flat[:, 1] = (v >> 8) & 255
    flat[:, 2] = v >> 16
    del v
    assert np.array_equal(cr.grey(img), cv2.cvtColor(img, cv2.COLOR_BGR2GRAY))


def _frame():
    img = cv2.imread(os.path.join(GOLDEN, "color_camera_image_200.png"), cv2.IMREAD_COLOR)
    assert img is not None
    return img


def _check(img, roi, scale):
    x, y, w, h = roi
    s = float(np.float32(scale))
    expected = cv2.resize(cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)[y:y + h, x:x + w], None, fx=s, fy=s,
                          interpolation=cv2.INTER_LINEAR)
    got = cr.crop(img, roi, scale)
    assert got.shape == expected.shape, (roi, scale)
    assert np.array_equal(got, expected), (roi, scale, int(np.count_nonzero(got != expected)))


SCALES = [0.5, 1.0, 0.2731, 0.4999, 0.5001, 0.61, 0.913, 0.999, 1.0004, 1.1, 1.37, 2.0, 2.5, 3.3, 5.17]


@pytest.mark.parametrize("scale", SCALES)
def test_resize_sweep(scale):
    img = _frame()
    H, W = img.shape[:2]
    rng = np.random.default_rng(int(scale * 1e4))
    rois = [(10, 12, 219, 219), (3, 5, 178, 150), (0, 0, 64, 64), (1, 1, 63, 65), (7, 9, 33, 17)]
    for _ in range(12):
        w, h = int(rng.integers(2, min(W, 230))), int(rng.integers(2, min(H, 230)))
        rois.append((int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1)), w, h))
    # regions clipped at each border: they start at 0 or end at the last pixel
    rois += [(0, 40, 57, 81), (W - 57, 40, 57, 81), (30, 0, 81, 57), (30, H - 57, 81, 57), (0, 0, W, H)]
    for roi in rois:
        x, y, w, h = roi
        if min(cr.output_size(w, h, scale)) < 1:
            continue  # cv::resize refuses an empty output; the focus region is then not used
        _check(img, roi, scale)


@pytest.mark.parametrize("scale", [1.0, 1.5, 2.0, 3.7, 7.0, 12.25])
def test_one_pixel_wide_and_high_regions(scale):
    img = _frame()
    for roi in [(5, 7, 1, 40), (0, 0, 1, 9), (20, 3, 40, 1), (img.shape[1] - 1, 10, 1, 31), (13, 17, 1, 1)]:
        _check(img, roi, scale)


def test_exactly_half_on_odd_and_even_sizes():
    img = _frame()
    for w in range(2, 14):
        for h in range(2, 14):
            _check(img, (11, 13, w, h), 0.5)


def test_output_size_rounds_half_to_even():
    assert cr.output_size(201, 3, 0.5) == (100, 2)
    assert cr.output_size(203, 5, 0.5) == (102, 2)
    for w, s in [(201, 0.5), (33, 1.5), (75, 1.1), (199, 0.913), (5, 0.1)]:
        img = np.zeros((4, w), np.uint8)
        try:
            out = cv2.resize(img, None, fx=float(np.float32(s)), fy=float(np.float32(s)), interpolation=cv2.INTER_LINEAR)
        except cv2.error:
            assert min(cr.output_size(w, 4, s)) < 1
            continue
        assert cr.output_size(w, 4, s) == (out.shape[1], out.shape[0])


def test_fixture_crops_are_the_restatement():
    """tests/golden/texture_crops.npz (cv2's crops, which the GPU tests compare k_texture_crop with) equals the
    restatement at the fixture's focus regions and scales."""
    z = np.load(os.path.join(GOLDEN, "texture_crops.npz"))
    img = _frame()
    assert {0.5, 1.0} <= set(float(s) for s in z["scales"])
    for b in range(len(z["poses"])):
        w, h = z["sizes"][b]
        got = cr.crop(img, z["rois"][b], z["scales"][b])
        assert got.shape == (h, w) and np.array_equal(got, z["crops"][b, :h, :w])


def test_front_end_kernels_have_no_local_memory(pkg):
    import re
    pkg._build.build_cuda()
    log = open(os.path.join(os.path.dirname(GOLDEN), "..", "3dobjecttracking_b200", "csrc", "build.log")).read()
    for name in ("_ZN4m3tb14k_texture_cropENS_11TexCropArgsE", "_ZN4m3tb18k_texture_featuresENS_11TexFeatArgsE"):
        m = re.search(r"Function properties for " + name + r"\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads", log)
        if m is None:
            pytest.skip("the library was built before this run (no ptxas report in build.log)")
        assert m.groups() == ("0", "0", "0"), m.group(0)
