"""Writes tests/golden/normalized_depth.npz: DepthCamera::NormalizedDepthImage (camera.cpp:108-115) as cv2 computes it,
convertTo(CV_8UC1, alpha, beta) with alpha = 255 / ((max - min) / depth_scale) and beta = -(min / depth_scale) * alpha in
float32, for every u16 depth value (the 256 x 256 image of 0 .. 65535, row-major) and each range below.
tests/viewer_reference.normalized_depth and the device (m3tb_get_normalized_depth_image) are compared with it.

    python tests/golden/make_normalized_depth.py
"""
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# (depth_scale, min_depth, max_depth)
RANGES = [
    (0.001, 0.0, 1.0),     # the NormalDepthViewer default: 0 .. 1000 mm onto 0 .. 255
    (0.001, 0.3, 0.7),     # saturation at both ends
    (1.0, 0.0, 510.0),     # alpha = 0.5: every odd value is a rounding tie
    (0.25, 10.0, 20.0),    # alpha = 6.375, beta = -255
    (0.0001, 0.5, 6.5),    # a fine depth scale
    (0.001, -0.2, 0.05),   # a negative min: depth 0 maps above 0
]


def depth_values():
    return np.arange(65536, dtype=np.uint16).reshape(256, 256)


def convert(src, alpha, beta):
    """cv::Mat::convertTo(CV_8U, alpha, beta) through cv2.normalize(NORM_MINMAX), which calls it with
    scale = (dmax - dmin) / (smax - smin) and shift = dmin - smin * scale; with smin = 0 they equal alpha and beta."""
    assert src.min() == 0
    dmin = float(beta)
    dmax = dmin + float(alpha) * float(src.max())
    assert (dmax - dmin) / float(src.max()) == float(alpha)
    return cv2.normalize(src, None, alpha=dmin, beta=dmax, norm_type=cv2.NORM_MINMAX, dtype=cv2.CV_8U)


def main():
    f32 = np.float32
    images = []
    for ds, lo, hi in RANGES:
        alpha = f32(255) / ((f32(hi) - f32(lo)) / f32(ds))
        beta = -(f32(lo) / f32(ds)) * alpha
        images.append(convert(depth_values(), alpha, beta))
    np.savez_compressed(os.path.join(HERE, "normalized_depth.npz"), ranges=np.array(RANGES, np.float64),
                        images=np.stack(images), opencv_version=np.array(cv2.__version__))


if __name__ == "__main__":
    main()
