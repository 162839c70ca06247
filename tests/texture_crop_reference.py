"""Integer restatement of the texture modality's focused grey image, DetectAndComputeCorrKeypoints
(texture_modality.cpp:862-868): resize(cvtColor(image, BGR2GRAY)(roi), Size(), scale, scale, INTER_LINEAR), as
OpenCV computes it for 8-bit images. k_texture_crop computes the same integers; tests/test_texture_crop_reference.py
holds this restatement to cv2 itself.

- grey: (3735 B + 19235 G + 9798 R + 2^14) >> 15, equal to cv2.cvtColor on all 2^24 BGR triples.
- output size: saturate_cast<int>(roi.w * double(scale)) x saturate_cast<int>(roi.h * double(scale)), rounded half to
  even; equal to the input size: a plain copy.
- scale == 0.5 (cv::resize switches to the fast INTER_AREA path at exactly 2x): full 2 x 2 blocks
  (a + b + c + d + 2) >> 2; a block cut by an odd last row or column: cvRound(float(sum) / count) over its pixels, and
  the whole last output row takes that path when the source has an odd number of rows.
- otherwise linear, fixed point with 2048 = 1 << 11:
  - coefficient of output position d: f = float((d + 0.5) * (1.0 / scale) - 0.5), s = floor(f), f -= s, weights
    cvRound((1 - f) * 2048) and cvRound(f * 2048) (half to even);
  - columns: s < 0 -> (s, f) = (0, 0); s >= w - 1 -> (s, f) = (w - 1, 0);
  - rows keep their weights; only the two source rows are clamped to [0, h - 1] (this is the border-row rule);
  - horizontal: H = g[s] * w0 + g[s + 1] * w1;
  - vertical, as OpenCV's vectorised pass: (((b0 * (H0 >> 4)) >> 16) + ((b1 * (H1 >> 4)) >> 16) + 2) >> 2.
"""
import numpy as np

GREY_B, GREY_G, GREY_R, GREY_SHIFT = 3735, 19235, 9798, 15


def grey(bgr):
    """cv2.cvtColor(bgr, COLOR_BGR2GRAY) for uint8 [..., 3]."""
    b = bgr[..., 0].astype(np.int64)
    g = bgr[..., 1].astype(np.int64)
    r = bgr[..., 2].astype(np.int64)
    return ((GREY_B * b + GREY_G * g + GREY_R * r + (1 << (GREY_SHIFT - 1))) >> GREY_SHIFT).astype(np.uint8)


def output_size(w, h, scale):
    """cv::resize's dsize for Size() and factors (scale, scale): saturate_cast<int> rounds half to even."""
    s = float(np.float32(scale))
    return int(np.rint(w * s)), int(np.rint(h * s))


def _coefficients(n_out, n_in, scale, clamp):
    inv = 1.0 / float(np.float32(scale))
    d = np.arange(n_out, dtype=np.float64)
    f = ((d + 0.5) * inv - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp:
        lo, hi = s < 0, s >= n_in - 1
        f = np.where(lo | hi, np.float32(0), f).astype(np.float32)
        s = np.where(lo, 0, np.where(hi, n_in - 1, s))
    w0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    w1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return np.clip(s, 0, n_in - 1), np.clip(s + 1, 0, n_in - 1), w0, w1


def resize(g, scale):
    """cv2.resize(g, None, fx=scale, fy=scale, interpolation=INTER_LINEAR) for a uint8 [h, w] image."""
    h, w = g.shape
    dw, dh = output_size(w, h, scale)
    if (dw, dh) == (w, h):
        return g.copy()
    if float(np.float32(scale)) == 0.5:
        return _area2(g, dw, dh)
    x0, x1, a0, a1 = _coefficients(dw, w, scale, True)
    y0, y1, b0, b1 = _coefficients(dh, h, scale, False)
    gi = g.astype(np.int64)
    H = gi[:, x0] * a0 + gi[:, x1] * a1  # [h, dw]
    v = (((b0[:, None] * (H[y0] >> 4)) >> 16) + ((b1[:, None] * (H[y1] >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def _area2(g, dw, dh):
    h, w = g.shape
    out = np.zeros((dh, dw), np.uint8)
    gi = g.astype(np.int64)
    fw, fh = w // 2, h // 2
    full = gi[:2 * fh:2, :2 * fw:2] + gi[1:2 * fh:2, :2 * fw:2] + gi[:2 * fh:2, 1:2 * fw:2] + gi[1:2 * fh:2, 1:2 * fw:2]
    out[:fh, :fw] = ((full + 2) >> 2)[:dh, :dw]
    for dy in range(dh):
        for dx in range(dw):
            if dy < fh and dx < fw:
                continue
            block = gi[2 * dy:2 * dy + 2, 2 * dx:2 * dx + 2]
            out[dy, dx] = int(np.rint(np.float32(block.sum()) / np.float32(block.size))) if block.size else 0
    return out


def crop(image_bgr, roi, scale):
    """The focused grey image of a focus region roi = (x, y, w, h) at `scale`."""
    x, y, w, h = (int(v) for v in roi)
    return resize(grey(image_bgr[y:y + h, x:x + w]), scale)
