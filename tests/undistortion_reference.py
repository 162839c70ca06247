"""NumPy restatement of the frame undistortion of AzureKinectColorCamera / AzureKinectDepthCamera::UpdateImage
(azure_kinect_camera.cpp:175-195, 321-345): cv::cvtColor(RGBA2RGB) on BGRA frames, cv::remap(INTER_NEAREST,
BORDER_CONSTANT) through a CV_16SC2 map and, for depth, `image_ += short(offset)` with saturation. Held to cv2 by
tests/test_undistortion_map.py; the oracle of tests/test_gpu_undistortion.py."""
import os

import numpy as np

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "undistortion")


def remap_nearest(raw, map_xy):
    """cv2.remap(raw, map_xy, None, INTER_NEAREST, BORDER_CONSTANT) for an (H, W, 2) int16 map: output pixel (i, j) is
    raw[y][x] with (x, y) = map_xy[i, j] when 0 <= x < W and 0 <= y < H, and 0 otherwise."""
    x = map_xy[..., 0].astype(np.int64)
    y = map_xy[..., 1].astype(np.int64)
    h, w = raw.shape[:2]
    inside = (x >= 0) & (x < w) & (y >= 0) & (y < h)
    out = np.zeros(map_xy.shape[:2] + raw.shape[2:], raw.dtype)
    out[inside] = raw[y[inside], x[inside]]
    return out


def undistort_color(raw, map_xy):
    """A BGRA (4 channels: COLOR_RGBA2RGB keeps bytes 0..2 in order) or BGR raw frame -> the rectified BGR frame."""
    return remap_nearest(np.ascontiguousarray(raw[..., :3]), map_xy)


def add_depth_offset(depth, offset):
    """image_ += short(offset) on a CV_16UC1 image: saturated to 0 .. 65535, invalid (0) pixels included."""
    return np.clip(depth.astype(np.int64) + int(offset), 0, 65535).astype(np.uint16)


def undistort_depth(raw, map_xy, offset=0):
    out = remap_nearest(raw, map_xy)
    return add_depth_offset(out, offset) if offset else out


def load_golden_map(name):
    """A cv2-made map stored by tests/golden/undistortion/make_undistortion_maps.py: (map_xy (H, W, 2) int16, dict of
    the calibration: fx fy cx cy (raw), fu fv (rectified), coefficients, width, height)."""
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    # stored as the first column and the differences along each row (small integers, which compress well)
    first = z["first_column"].astype(np.int64)
    diff = z["row_differences"].astype(np.int64)
    m = np.concatenate([first[:, None, :], diff], axis=1).cumsum(axis=1).astype(np.int16)
    calib = {k: z[k].item() if z[k].ndim == 0 else z[k] for k in z.files if k not in ("first_column", "row_differences")}
    return m, calib


def golden_names():
    return sorted(f[:-4] for f in os.listdir(GOLDEN_DIR) if f.endswith(".npz"))
