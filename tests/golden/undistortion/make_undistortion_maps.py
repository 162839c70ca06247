"""Writes the cv2-made undistortion maps the GPU tests compare against (tests/undistortion_reference.py loads them):
cv2.initUndistortRectifyMap(CV_32FC1) + cv2.convertMaps(CV_16SC2, nninterpolation=True) with float32 camera matrices,
R = I and fu / fv scaled by image_scale, as AzureKinect*Camera::GetIntrinsicsAndDistortionMap builds them
(azure_kinect_camera.cpp:234-265, 387-419). Each map is stored as its first column and the differences along each row.

    python tests/golden/undistortion/make_undistortion_maps.py
"""
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# name: (width, height, fx, fy, cx, cy, k1, k2, p1, p2, k3, k4, k5, k6, image_scale)
CALIBRATIONS = {
    # an Azure Kinect-like 720p colour calibration (the reference's default colour mode)
    "color_1280x720": (1280, 720, 605.9, 605.7, 637.8, 366.2, 0.52, -2.61, 6e-4, -3e-4, 1.45, 0.40, -2.43, 1.38, 1.0),
    # an NFOV unbinned depth calibration
    "depth_640x576": (640, 576, 504.2, 504.3, 319.5, 335.9, 3.12, 1.88, 4e-5, -1e-5, 0.09, 3.45, 2.85, 0.48, 1.0),
    "color_640x480": (640, 480, 520.0, 521.0, 318.0, 242.0, 0.0, 0.0, 4e-3, -3e-3, 0.0, 0.0, 0.0, 0.0, 1.1),
    "odd_333x217": (333, 217, 250.0, 248.0, 166.0, 108.0, -0.21, 0.05, 1e-3, 2e-3, -0.01, 0.1, -0.02, 0.01, 0.8),
}


def cv2_map(width, height, fx, fy, cx, cy, coefficients, image_scale):
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    fu, fv = np.float32(fx) * np.float32(image_scale), np.float32(fy) * np.float32(image_scale)
    Kn = np.array([[fu, 0, cx], [0, fv, cy], [0, 0, 1]], np.float32)
    D = np.asarray(coefficients, np.float32).reshape(1, 8)
    m1, m2 = cv2.initUndistortRectifyMap(K, D, None, Kn, (width, height), cv2.CV_32FC1)
    m, _ = cv2.convertMaps(m1, m2, cv2.CV_16SC2, nninterpolation=True)
    return m, fu, fv


def main():
    for name, c in CALIBRATIONS.items():
        w, h, fx, fy, cx, cy = c[:6]
        k1, k2, p1, p2, k3, k4, k5, k6 = c[6:14]
        coefficients = np.array([k1, k2, p1, p2, k3, k4, k5, k6], np.float32)  # OpenCV order
        m, fu, fv = cv2_map(w, h, fx, fy, cx, cy, coefficients, c[14])
        m64 = m.astype(np.int64)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), first_column=m[:, 0, :],
                            row_differences=np.diff(m64, axis=1).astype(np.int32), width=w, height=h,
                            fx=np.float32(fx), fy=np.float32(fy), cx=np.float32(cx), cy=np.float32(cy), fu=fu, fv=fv,
                            coefficients=coefficients, opencv_version=cv2.__version__)


if __name__ == "__main__":
    main()
