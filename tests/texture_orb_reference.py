"""NumPy restatement of cv::ORB (OpenCV 4) at M3T's settings: detect, then compute, on an 8-bit grey image.

Only n_features, scale_factor and n_levels vary; everything else is cv::ORB's default (edgeThreshold 31, firstLevel
0, WTA_K 2, HARRIS_SCORE, patchSize 31, fastThreshold 20). Every stage is integer or float32 arithmetic in the order
OpenCV evaluates it, so the result is bit-equal to cv2's as a multiset of keypoints and descriptors
(tests/test_texture_orb_reference.py). The order is this project's canonical one, which k_texture_orb shares: level
ascending, then row-major by the keypoint's pixel in its level. cv2's order within a level comes from nth_element /
partition and is not reproduced.
"""
import math
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EDGE_THRESHOLD = 31
PATCH_SIZE = 31
HALF_PATCH = PATCH_SIZE // 2
FAST_THRESHOLD = 20
HARRIS_BLOCK = 7
HARRIS_K = np.float32(0.04)

# FAST's 16-pixel circle of radius 3, (dx, dy), fast.cpp's offsets16
FAST_CIRCLE = ((0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3),
               (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0), (-3, 1), (-2, 2), (-1, 3))


def bit_pattern():
    """The 256 point pairs as [512][2] (x, y), from the committed header the kernels compile."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_orb_pattern",
                                                  os.path.join(ROOT, "scripts", "make_orb_pattern.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.pattern_from_header().reshape(512, 2)


def cv_round(v):
    """cvRound: round half to even, as lrint does."""
    return np.rint(v).astype(np.int64)


def level_scales(scale_factor, n_levels):
    """layerScale: (float)pow(scaleFactor, level), scaleFactor the double of cv::ORB::create's float argument."""
    sf = float(np.float32(scale_factor))
    return [np.float32(math.pow(sf, level)) for level in range(n_levels)]


def level_sizes(width, height, scale_factor, n_levels):
    """Size(cvRound(cols * (1.f / scale)), cvRound(rows * (1.f / scale))) per level, as (width, height)."""
    out = []
    for s in level_scales(scale_factor, n_levels):
        inv = np.float32(1.0) / s
        out.append((int(cv_round(np.float32(width) * inv)), int(cv_round(np.float32(height) * inv))))
    return out


def features_per_level(n_features, scale_factor, n_levels):
    """nfeaturesPerLevel: a geometric series in 1 / scaleFactor rounded with cvRound; the last level the remainder."""
    sf = float(np.float32(scale_factor))
    factor = np.float32(1.0 / sf)
    one = np.float32(1.0)
    desired = np.float32(np.float32(n_features) * (one - factor)) / (one - np.float32(math.pow(float(factor), n_levels)))
    desired = np.float32(desired)
    out, total = [], 0
    for _ in range(n_levels - 1):
        k = int(cv_round(desired))
        out.append(k)
        total += k
        desired = np.float32(desired * factor)
    out.append(max(n_features - total, 0))
    return out


def _linear_exact_taps(src_n, dst_n):
    """resize_bitExact's interpolationLinear: per output position the source offset and the two weights in 1/256,
    and the output ranges pinned to the first / last source pixel ([0, lo) and [hi, dst_n))."""
    scale = 1.0 / (float(dst_n) / float(src_n))
    offs = np.zeros(dst_n, np.int64)
    c1 = np.zeros(dst_n, np.int64)
    lo, hi = 0, dst_n
    for d in range(dst_n):
        f = scale * (d + 0.5) - 0.5
        i = math.floor(f)
        if i >= 0 and src_n > 1:
            if i < src_n - 1:
                offs[d] = i
                c1[d] = int(np.rint((f - i) * 256.0))
            else:
                offs[d] = src_n - 1
                hi = min(hi, d)
        else:
            lo = max(lo, d + 1)
    return offs, 256 - c1, c1, lo, hi


def resize_linear_exact(src, width, height):
    """cv::resize(src, Size(width, height), 0, 0, INTER_LINEAR_EXACT) on uint8: 8-bit fixed-point weights, rows
    exact in 1/256, the vertical sum rounded half up from 1/65536; outside the interior the edge row / column."""
    src = src.astype(np.int64)
    sh, sw = src.shape
    xo, xc0, xc1, xlo, xhi = _linear_exact_taps(sw, width)
    yo, yc0, yc1, ylo, yhi = _linear_exact_taps(sh, height)
    rows = np.empty((sh, width), np.int64)  # every source row resized horizontally, in 1/256
    rows[:, :xlo] = src[:, :1] * 256
    mid = np.arange(xlo, xhi)
    if len(mid):
        rows[:, mid] = src[:, xo[mid]] * xc0[mid] + src[:, np.minimum(xo[mid] + 1, sw - 1)] * xc1[mid]
    rows[:, xhi:] = src[:, [xo[width - 1]]] * 256
    out = np.empty((height, width), np.int64)
    out[:ylo] = (rows[0] + 128) >> 8
    mid = np.arange(ylo, yhi)
    if len(mid):
        acc = rows[yo[mid]] * yc0[mid, None] + rows[np.minimum(yo[mid] + 1, sh - 1)] * yc1[mid, None]
        out[mid] = (acc + (1 << 15)) >> 16
    out[yhi:] = (rows[sh - 1] + 128) >> 8
    return np.clip(out, 0, 255).astype(np.uint8)


def empty_pyramid(width, height, scale_factor, n_levels):
    """Whether a level of the pyramid has a side of 0 pixels. cv::ORB builds every level before it detects, and
    cv::resize refuses an empty size, so cv2 raises and detects nothing at all, on the earlier levels neither."""
    return any(lw < 1 or lh < 1 for lw, lh in level_sizes(width, height, scale_factor, n_levels))


def pyramid(image, scale_factor, n_levels):
    """imagePyramid's levels: level 0 the image, level l resize(level l - 1, INTER_LINEAR_EXACT). Every level has at
    least one pixel (see empty_pyramid)."""
    h, w = image.shape
    assert not empty_pyramid(w, h, scale_factor, n_levels)
    levels = [np.ascontiguousarray(image, dtype=np.uint8)]
    for (lw, lh) in level_sizes(w, h, scale_factor, n_levels)[1:]:
        levels.append(resize_linear_exact(levels[-1], lw, lh))
    return levels


def fast_scores(img, threshold=FAST_THRESHOLD):
    """FAST-9/16's corner score per pixel (cornerScore<16>), 0 where the pixel is no corner or outside the rows and
    columns fast.cpp tests ([3, rows - 3) x [3, cols - 3))."""
    h, w = img.shape
    score = np.zeros((h, w), np.int64)
    if h < 7 or w < 7:
        return score
    v = img[3:h - 3, 3:w - 3].astype(np.int64)
    d = np.stack([v - img[3 + dy:h - 3 + dy, 3 + dx:w - 3 + dx].astype(np.int64) for dx, dy in FAST_CIRCLE])
    d = np.concatenate([d, d[:9]])
    best = np.full(v.shape, -1 << 20, np.int64)
    for sign in (1, -1):
        for k in range(16):
            best = np.maximum(best, (sign * d[k:k + 9]).min(axis=0))
    score[3:h - 3, 3:w - 3] = np.where(best > threshold, best - 1, 0)
    return score


def fast_corners(img, threshold=FAST_THRESHOLD):
    """FastFeatureDetector(threshold, nonmaxSuppression=true): corners whose score beats all 8 neighbours', as
    (x, y, score) in row-major order."""
    s = fast_scores(img, threshold)
    h, w = s.shape
    p = np.pad(s, 1)
    keep = s > 0
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dx or dy:
                keep &= s > p[1 + dy:1 + dy + h, 1 + dx:1 + dx + w]
    ys, xs = np.nonzero(keep)
    return xs, ys, s[ys, xs]


def retain_best(values, n):
    """KeyPointsFilter::retainBest as a mask: every point whose response is at least the n-th largest (ties at the
    cut all stay); n = 0 keeps nothing."""
    if len(values) <= n:
        return np.ones(len(values), bool)
    if n == 0:
        return np.zeros(len(values), bool)
    kth = np.sort(values)[::-1][n - 1]
    return values >= kth


def harris(img, xs, ys):
    """HarrisResponses, block 7, k 0.04: integer Sobel sums, then the float formula evaluated as OpenCV does."""
    img = img.astype(np.int64)
    r = HARRIS_BLOCK // 2
    a = np.zeros(len(xs), np.int64)
    b = np.zeros(len(xs), np.int64)
    c = np.zeros(len(xs), np.int64)
    for by in range(-r, r + 1):
        for bx in range(-r, r + 1):
            y, x = ys + by, xs + bx
            ix = (img[y, x + 1] - img[y, x - 1]) * 2 + (img[y - 1, x + 1] - img[y - 1, x - 1]) + \
                 (img[y + 1, x + 1] - img[y + 1, x - 1])
            iy = (img[y + 1, x] - img[y - 1, x]) * 2 + (img[y + 1, x - 1] - img[y - 1, x - 1]) + \
                 (img[y + 1, x + 1] - img[y - 1, x + 1])
            a += ix * ix
            b += iy * iy
            c += ix * iy
    f32 = np.float32
    scale = f32(1.0) / f32(f32(4 * HARRIS_BLOCK) * f32(255.0))
    sss = f32(f32(f32(scale * scale) * scale) * scale)
    fa, fb, fc = a.astype(f32), b.astype(f32), c.astype(f32)
    s = (fa + fb).astype(f32)
    with np.errstate(over="ignore"):
        t = ((fa * fb).astype(f32) - (fc * fc).astype(f32)).astype(f32)
        t = (t - ((HARRIS_K * s).astype(f32) * s).astype(f32)).astype(f32)
    return (t * sss).astype(f32)


def _umax():
    """ICAngles' row ends of the radius-15 circular patch (orb.cpp's u_max, made symmetric)."""
    half = HALF_PATCH
    umax = [0] * (half + 2)
    vmax = math.floor(float(np.float32(np.float32(half) * np.float32(math.sqrt(2.0)) / np.float32(2)) + np.float32(1)))
    vmin = math.ceil(float(np.float32(np.float32(half) * np.float32(math.sqrt(2.0)) / np.float32(2))))
    for v in range(vmax + 1):
        umax[v] = int(cv_round(math.sqrt(float(half * half - v * v))))
    v0 = 0
    for v in range(half, vmin - 1, -1):
        while umax[v0] == umax[v0 + 1]:
            v0 += 1
        umax[v] = v0
        v0 += 1
    return umax


UMAX = _umax()


def fast_atan2(y, x):
    """cv::fastAtan2 on float32 arrays, in degrees [0, 360)."""
    f32 = np.float32
    deg = f32(180.0 / math.pi)
    p1, p3 = f32(f32(0.9997878412794807) * deg), f32(f32(-0.3258083974640975) * deg)
    p5, p7 = f32(f32(0.1555786518463281) * deg), f32(f32(-0.04432655554792128) * deg)
    eps = f32(2.220446049250313e-16)
    y, x = np.asarray(y, f32), np.asarray(x, f32)
    ax, ay = np.abs(x), np.abs(y)
    big = ax >= ay
    num, den = np.where(big, ay, ax), np.where(big, ax, ay)
    c = (num / (den + eps).astype(f32)).astype(f32)
    c2 = (c * c).astype(f32)
    a = (p7 * c2).astype(f32)
    a = ((a + p5).astype(f32) * c2).astype(f32)
    a = ((a + p3).astype(f32) * c2).astype(f32)
    a = ((a + p1).astype(f32) * c).astype(f32)
    a = np.where(big, a, (f32(90.0) - a).astype(f32))
    a = np.where(x < 0, (f32(180.0) - a).astype(f32), a)
    a = np.where(y < 0, (f32(360.0) - a).astype(f32), a)
    return a.astype(f32)


def angles(img, xs, ys):
    """ICAngles: the intensity-centroid angle over the radius-15 circle."""
    img = img.astype(np.int64)
    m01 = np.zeros(len(xs), np.int64)
    m10 = np.zeros(len(xs), np.int64)
    for u in range(-HALF_PATCH, HALF_PATCH + 1):
        m10 += u * img[ys, xs + u]
    for v in range(1, HALF_PATCH + 1):
        d = UMAX[v]
        vsum = np.zeros(len(xs), np.int64)
        for u in range(-d, d + 1):
            plus, minus = img[ys + v, xs + u], img[ys - v, xs + u]
            vsum += plus - minus
            m10 += u * (plus + minus)
        m01 += v * vsum
    return fast_atan2(m01.astype(np.float32), m10.astype(np.float32))


def _fma(a, b, c):
    """fmaf on float32 arrays: the product and sum are exact in x87 extended precision, rounded once to float32."""
    ld = np.longdouble
    return (np.asarray(a, np.float32).astype(ld) * ld(b) + np.asarray(c, np.float32).astype(ld)).astype(np.float32)


def gaussian_kernel():
    """getGaussianKernel(7, 2, CV_32F): the double taps, normalised to sum 1, cast to float."""
    x = np.arange(7, dtype=np.float64) - 3.0
    k = np.exp(-(x * x) / (2.0 * 2.0 * 2.0))
    return (k / k.sum()).astype(np.float32)


GAUSS = gaussian_kernel()


def gaussian_blur(img):
    """GaussianBlur(7 x 7, sigma 2, BORDER_REFLECT_101) of a pyramid level as ORB runs it: in place on a view of the
    padded pyramid, which OpenCV filters with its separable float path (sepFilter2D), not the fixed-point one it uses
    for whole images. Rows: s = k0 p0, then s = fma(p_t, k_t, s) for t = 1 .. 6; columns, symmetric about the centre:
    s = k3 S0, then s = fma(S_t + S_-t, k_(3+t), s) for t = 1 .. 3; the result rounded half to even and saturated.
    This is what OpenCV's AVX2 / AVX-512 builds compute (v_muladd is a fused multiply-add there)."""
    h, w = img.shape
    p = np.pad(img.astype(np.float32), 3, mode="reflect")
    rows = (p[:, 0:w] * GAUSS[0]).astype(np.float32)
    for t in range(1, 7):
        rows = _fma(p[:, t:t + w], GAUSS[t], rows)
    out = (rows[3:3 + h] * GAUSS[3]).astype(np.float32)
    for t in range(1, 4):
        out = _fma((rows[3 + t:3 + t + h] + rows[3 - t:3 - t + h]).astype(np.float32), GAUSS[3 + t], out)
    return np.clip(np.rint(out), 0, 255).astype(np.uint8)


def descriptors(blurred, xs, ys, angle, pattern):
    """computeOrbDescriptors (WTA_K 2): the pattern rotated by cos / sin of the angle (in double, cast to float),
    points at cvRound, bit k of byte i = (value of point 16 i + 2 k < value of point 16 i + 2 k + 1)."""
    f32 = np.float32
    rad = (angle.astype(f32) * f32(math.pi / 180.0)).astype(f32)
    a = np.cos(rad.astype(np.float64)).astype(f32)
    b = np.sin(rad.astype(np.float64)).astype(f32)
    px = pattern[:, 0].astype(f32)[None, :]
    py = pattern[:, 1].astype(f32)[None, :]
    a, b = a[:, None], b[:, None]
    x = ((px * a).astype(f32) - (py * b).astype(f32)).astype(f32)
    y = ((px * b).astype(f32) + (py * a).astype(f32)).astype(f32)
    vals = blurred[ys[:, None] + cv_round(y), xs[:, None] + cv_round(x)].astype(np.int64)
    bits = (vals[:, 0::2] < vals[:, 1::2]).astype(np.uint8).reshape(len(xs), 32, 8)
    return (bits << np.arange(8, dtype=np.uint8)).sum(axis=2).astype(np.uint8)


def orb(image, n_features=300, scale_factor=1.2, n_levels=3, pattern=None, stages=None):
    """cv::ORB::create(n_features, scale_factor, n_levels): detect, then compute, in canonical order.

    Returns a dict of arrays: xy [n][2] float32 (level-0 coordinates, KeyPoint::pt), angle, response (float32),
    octave (int32), descriptors [n][32] uint8, and lxy [n][2] the pixel in its level; nothing when a level of the
    pyramid is empty (empty_pyramid). `stages`, when a dict, receives "empty_pyramid", the per-level counts
    ("per_level") and, per level, the pyramid, blurred levels, the FAST corners found ("n_corners") and those inside
    the border that the first cut ranks ("n_fast"), and the counts after each cut."""
    image = np.ascontiguousarray(image, dtype=np.uint8)
    if pattern is None:
        pattern = bit_pattern()
    per_level = features_per_level(n_features, scale_factor, n_levels)
    empty = empty_pyramid(image.shape[1], image.shape[0], scale_factor, n_levels)
    if stages is not None:
        stages["empty_pyramid"] = empty
        stages["per_level"] = per_level
    levels = [] if empty else pyramid(image, scale_factor, n_levels)
    scales = level_scales(scale_factor, n_levels)
    out = {k: [np.zeros((0,) + s, t)] for k, s, t in (("xy", (2,), np.float32), ("lxy", (2,), np.int32),
                                                        ("angle", (), np.float32), ("response", (), np.float32),
                                                        ("octave", (), np.int32), ("descriptors", (32,), np.uint8))}
    for level, img in enumerate(levels):
        h, w = img.shape
        xs, ys, sc = fast_corners(img)
        n_corners = len(xs)
        if h <= 2 * EDGE_THRESHOLD or w <= 2 * EDGE_THRESHOLD:
            inside = np.zeros(len(xs), bool)
        else:
            inside = (xs >= EDGE_THRESHOLD) & (xs < w - EDGE_THRESHOLD) & (ys >= EDGE_THRESHOLD) & (ys < h - EDGE_THRESHOLD)
        xs, ys, sc = xs[inside], ys[inside], sc[inside]
        n_fast = len(xs)
        keep = retain_best(sc.astype(np.float32), 2 * per_level[level])
        xs, ys = xs[keep], ys[keep]
        n_first = len(xs)
        resp = harris(img, xs, ys)
        keep = retain_best(resp, per_level[level])
        xs, ys, resp = xs[keep], ys[keep], resp[keep]
        ang = angles(img, xs, ys)
        blurred = gaussian_blur(img) if len(xs) else img
        desc = descriptors(blurred, xs, ys, ang, pattern)
        s = scales[level]
        out["xy"].append(np.stack([(xs.astype(np.float32) * s).astype(np.float32),
                                   (ys.astype(np.float32) * s).astype(np.float32)], axis=1).reshape(-1, 2))
        out["lxy"].append(np.stack([xs, ys], axis=1).reshape(-1, 2).astype(np.int32))
        out["angle"].append(ang)
        out["response"].append(resp)
        out["octave"].append(np.full(len(xs), level, np.int32))
        out["descriptors"].append(desc.reshape(-1, 32))
        if stages is not None:
            stages.setdefault("levels", []).append(img)
            stages.setdefault("blurred", []).append(blurred)
            stages.setdefault("n_corners", []).append(n_corners)
            stages.setdefault("n_fast", []).append(n_fast)
            stages.setdefault("n_first_cut", []).append(n_first)
            stages.setdefault("n_second_cut", []).append(len(xs))
    res = {k: np.concatenate(v) for k, v in out.items()}
    res["xy"] = res["xy"].astype(np.float32).reshape(-1, 2)
    res["angle"] = res["angle"].astype(np.float32)
    res["response"] = res["response"].astype(np.float32)
    return res


def cv2_orb(image, n_features=300, scale_factor=1.2, n_levels=3):
    """What M3T runs (texture_modality.cpp:858-888): cv::ORB detect, then compute, as the same dict (cv2's order)."""
    import cv2
    o = cv2.ORB_create(n_features, scale_factor, n_levels)
    kps = o.detect(image, None)
    kps, desc = o.compute(image, kps)
    n = len(kps)
    return {
        "xy": np.array([k.pt for k in kps], np.float32).reshape(n, 2),
        "angle": np.array([k.angle for k in kps], np.float32),
        "response": np.array([k.response for k in kps], np.float32),
        "octave": np.array([k.octave for k in kps], np.int32),
        "descriptors": (desc if desc is not None else np.zeros((0, 32), np.uint8)).reshape(n, 32),
    }


def as_multiset(res):
    """The keypoints as a sorted list of byte strings (x, y, angle, response, octave, descriptor)."""
    rows = []
    for i in range(len(res["angle"])):
        rows.append(res["xy"][i].tobytes() + res["angle"][i:i + 1].tobytes() + res["response"][i:i + 1].tobytes() +
                    res["octave"][i:i + 1].tobytes() + res["descriptors"][i].tobytes())
    return sorted(rows)


# ---- inputs shared by the CPU test and the golden generator ------------------------------------------------------

def textured(h, w, seed, block=4):
    """A random textured image: random blocks of `block` pixels plus noise, so FAST finds corners at every level."""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, size=(max(h // block, 1) + 2, max(w // block, 1) + 2)).astype(np.float64)
    up = np.kron(base, np.ones((block, block)))[:h, :w]
    noise = rng.integers(-40, 41, size=(h, w))
    img = np.clip(up + noise, 0, 255).astype(np.uint8)
    return img


def noise(h, w, seed):
    """Uniform noise: FAST corners on most pixels, long candidate lists and many equal FAST scores."""
    return np.random.default_rng(seed).integers(0, 256, size=(h, w)).astype(np.uint8)


def binary_noise(h, w, seed):
    """0 / 255 noise: FAST scores saturate, so the first cut ties on nearly every candidate."""
    return (np.random.default_rng(seed).integers(0, 2, size=(h, w)) * 255).astype(np.uint8)


def ramp(h, w):
    """A smooth diagonal ramp: no FAST corner anywhere."""
    yy, xx = np.mgrid[0:h, 0:w]
    return ((xx + 2 * yy) * 255 // max(w + 2 * h - 3, 1)).astype(np.uint8)


def as_frame(grey):
    """A BGR frame whose grey image (BGR2GRAY) is `grey` itself."""
    return np.ascontiguousarray(np.repeat(grey[:, :, None], 3, axis=2))


def dot_grid(h=300, w=300, spacing=12):
    """Identical dots on a flat ground: many equal FAST and Harris scores, so both cuts keep ties (444 keypoints at
    n_features 300 and 366 at 20; at spacing 6, 1453 keypoints at n_features 300)."""
    img = np.full((h, w), 40, np.uint8)
    for y in range(6, h - 4, spacing):
        for x in range(6, w - 4, spacing):
            img[y - 1:y + 2, x - 1:x + 2] = 220
    return img


def dot_frame(h=540, w=960, spacing=6, dot=3):
    """A BGR camera frame of identical grey dots. Golden body 3's focus (scale 0.5) crops it into a grid whose corners
    tie at both cuts: cv::ORB keeps 566 keypoints at n_features 300."""
    img = np.full((h, w), 40, np.uint8)
    for y in range(0, h, spacing):
        for x in range(0, w, spacing):
            img[y:y + dot, x:x + dot] = 220
    return np.ascontiguousarray(np.repeat(img[:, :, None], 3, axis=2))


TIE_BODY = 3
TIE_SETTING = (300, 1.2, 3)


def checkerboard(h=200, w=200, cell=5):
    yy, xx = np.mgrid[0:h, 0:w]
    return np.where(((yy // cell) + (xx // cell)) % 2 == 0, 30, 225).astype(np.uint8)


SETTINGS = [(300, 1.2, 3), (20, 1.2, 3), (500, 1.2, 8), (300, 2.0, 3), (300, 1.2, 1), (4096, 1.2, 3)]
RANDOM_SIZES = [1, 7, 62, 63, 64, 65, 70, 100, 200, 369]

# The float just above 1, the smallest scale_factor cv::ORB accepts: every level has the size of level 0.
NEXT_ABOVE_1 = float(np.nextafter(np.float32(1.0), np.float32(2.0)))
# (n_features, scale_factor, n_levels) beyond SETTINGS: every n_features of {1, 2, 5, 20, 300, 1000, 4096, 2^24}, every
# scale_factor of {NEXT_ABOVE_1, 1.05, 1.2, 1.3, 1.5, 2.0, 2.5, 3.0} and n_levels 1 .. 8. It has per-level counts of 0
# (n_features up to 5, and 300 at 8 levels of 2.5 or 3.0), pyramids with an empty level (3.0 at 8 levels below 1094 px,
# 2.5 at 8 levels below 305 px and at 5 levels below 20 px) and n_features 2^24, where the cuts keep everything and
# keypoints with a Harris response <= 0 survive.
SWEEP = [(1, 1.2, 3), (1, 3.0, 1), (2, NEXT_ABOVE_1, 8), (2, 2.5, 2), (5, 1.05, 4), (5, 1.5, 6), (20, 1.3, 7),
         (20, 2.0, 5), (300, 1.2, 3), (300, 2.5, 8), (300, 3.0, 8), (300, NEXT_ABOVE_1, 2), (1000, 1.3, 4),
         (1000, 1.5, 8), (1000, 2.0, 6), (4096, 1.2, 8), (4096, 1.05, 8), (4096, 3.0, 3), (1 << 24, 1.2, 3),
         (1 << 24, 1.5, 1), (1 << 24, 2.5, 5), (1 << 24, NEXT_ABOVE_1, 4)]
