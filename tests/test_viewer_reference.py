"""The CPU restatement of the device viewers (tests/viewer_reference.py) against independent computations: OpenCV 4.13's
convertTo and GRAY2BGR, the alpha blend compiled by the host C++ compiler, closed forms of the prism seen along its axis
at a non-square size with an off-centre principal point, and the model-generation renderer at W = H = S."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import model_generation_reference as mg
import render_reference as rr
import viewer_reference as vr

I34 = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
Intr = type("Intr", (), {})


def _intr(fu, fv, ppu, ppv, width, height):
    i = Intr()
    i.fu, i.fv, i.ppu, i.ppv, i.width, i.height = fu, fv, ppu, ppv, width, height
    return i


def _opencv_convert(src, alpha, beta):
    """cv::Mat::convertTo(CV_8U, alpha, beta) through cv2.normalize(NORM_MINMAX), which calls it with
    scale = (dmax - dmin) / (smax - smin) and shift = dmin - smin * scale; with smin = 0 both round to alpha and beta."""
    cv2 = pytest.importorskip("cv2")
    assert src.min() == 0
    dmin = float(beta)
    dmax = dmin + float(alpha) * float(src.max())
    assert dmax > dmin
    return cv2.normalize(src, None, alpha=dmin, beta=dmax, norm_type=cv2.NORM_MINMAX, dtype=cv2.CV_8U)


@pytest.mark.parametrize("min_depth,max_depth", [(0.0, 1.0), (0.3, 0.9), (0.01, 7.3), (0.5, 0.6), (0.123, 0.3456),
                                                 (0.45, 0.47)])
@pytest.mark.parametrize("width", [640, 333, 17, 1])
def test_normalized_depth_equals_opencv(min_depth, max_depth, width):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(width)
    src = rng.integers(0, 65536, (97, width), dtype=np.uint16)
    src[:, : (width + 1) // 2] = rng.integers(0, 3000, (97, (width + 1) // 2))
    src[0, 0], src[1, 0] = 0, 65535
    ds = np.float32(0.001)
    alpha = np.float32(255) / ((np.float32(max_depth) - np.float32(min_depth)) / ds)
    beta = -(np.float32(min_depth) / ds) * alpha
    exp = _opencv_convert(src, alpha, beta)
    got = vr.normalized_depth(src, ds, min_depth, max_depth)
    assert np.array_equal(got, exp)
    assert (got == 0).any() and (got == 255).any()  # saturates at both ends
    gray = cv2.cvtColor(exp, cv2.COLOR_GRAY2BGR)
    assert np.array_equal(np.repeat(got[..., None], 3, axis=2), gray)


_BLEND_SRC = r"""
#include <cstddef>
extern "C" void blend(const unsigned char* cam, const unsigned char* rend, unsigned char* out, size_t n, float opacity) {
  const float alpha_scale = opacity / 255.0f;
  for (size_t k = 0; k < n; ++k) {
    const float alpha = float(rend[4 * k + 3]) * alpha_scale;
    const float alpha_inv = 1.0f - alpha;
    for (int c = 0; c < 3; ++c) out[3 * k + c] = char(cam[3 * k + c] * alpha_inv + rend[4 * k + c] * alpha);
  }
}
"""


@pytest.fixture(scope="module")
def host_blend():
    """The blend as the host compiler builds it (g++, x86-64, no -ffast-math): the char() rule comes from the compiler."""
    if shutil.which("g++") is None:
        pytest.skip("no host C++ compiler")
    d = tempfile.mkdtemp()
    src, lib = os.path.join(d, "blend.cpp"), os.path.join(d, "blend.so")
    with open(src, "w") as f:
        f.write(_BLEND_SRC)
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-fPIC", "-shared", src, "-o", lib], check=True)
    L = ctypes.CDLL(lib)
    L.blend.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_float]
    yield L
    shutil.rmtree(d, ignore_errors=True)


@pytest.mark.parametrize("opacity", [0.0, 0.3, 0.5, 1.0, 1.7, -0.4, 3e7])
def test_alpha_blend_equals_host_compiler(host_blend, opacity):
    rng = np.random.default_rng(7)
    cam = rng.integers(0, 256, (61, 83, 3), dtype=np.uint8)
    rend = rng.integers(0, 256, (61, 83, 4), dtype=np.uint8)
    rend[..., 3] = np.where(rng.random((61, 83)) < 0.5, 0, 255)
    rend[:5, :, 3] = rng.integers(0, 256, (5, 83))  # any alpha, not only the renderer's 0 / 255
    exp = np.zeros_like(cam)
    host_blend.blend(cam.ctypes.data, rend.ctypes.data, exp.ctypes.data, cam.shape[0] * cam.shape[1], opacity)
    got = vr.alpha_blend(cam, rend, opacity)
    assert np.array_equal(got, exp)
    bg = rend[..., 3] == 0
    assert np.array_equal(got[bg], cam[bg])  # background pixels keep the camera pixel


def _convex_hull_inside(pu, pv, u, v):
    pts = np.stack([pu, pv], 1)
    c = pts.mean(0)
    hull = pts[np.argsort(np.arctan2(pts[:, 1] - c[1], pts[:, 0] - c[0]))]

    def turn(p, q, s):
        return (q[0] - p[0]) * (s[1] - q[1]) - (q[1] - p[1]) * (s[0] - q[0])
    hull = hull[[k for k in range(len(hull)) if turn(hull[k - 1], hull[k], hull[(k + 1) % len(hull)]) > 1e-12]]
    dist = np.full(u.shape, np.inf)
    inside = np.ones(u.shape, bool)
    for k in range(len(hull)):
        a, b = hull[k], hull[(k + 1) % len(hull)]
        e = ((b[0] - a[0]) * (v - a[1]) - (b[1] - a[1]) * (u - a[0])) / np.hypot(*(b - a))
        inside &= e > 0
        dist = np.minimum(dist, np.abs(e))
    return inside, dist


@pytest.mark.parametrize("kind", ["color", "depth"])
def test_prism_along_its_axis_closed_forms(synth, kind):
    intr = _intr(410.0, 395.5, 201.7, 93.2, 333, 217)  # non-square, principal point off centre
    tri, diam = synth.prism_triangles()
    geo = {0: rr.Geometry(tri, I34.copy(), diam, True)}
    pose = I34.copy()
    pose[:, 3] = (0.012, -0.008, 0.25)  # axis along the optical axis, off the principal ray
    normal, _ = vr.render_normal(intr, I34, {0: pose}, geo, [0])
    H, W = 217, 333
    jj, ii = np.mgrid[0:H, 0:W].astype(np.float64)
    u, v = ii, jj  # pixel centre (i + 0.5) maps to u = i (FullRenderer's ppu + 0.5)
    verts = synth.PRISM_VERTICES + pose[:, 3].astype(np.float64)
    pu = intr.fu * verts[:, 0] / verts[:, 2] + intr.ppu
    pv = intr.fv * verts[:, 1] / verts[:, 2] + intr.ppv
    inside, dist = _convex_hull_inside(pu, pv, u, v)
    sure = dist > 1e-3
    covered = normal[..., 3] == 255
    assert np.array_equal(covered[sure], inside[sure])  # the exact projected silhouette
    assert inside.sum() > 500
    near = verts[:, 2] < pose[2, 3]  # the cap facing the camera, outward normal (0, 0, -1)
    cap, cdist = _convex_hull_inside(pu[near], pv[near], u, v)
    cap &= cdist > 1e-3
    assert cap.sum() > 300
    # 0.5 - 0.5 * (0, 0, -1) = (0.5, 0.5, 1) -> unorm8 (128, 128, 255) (127.5 rounds to even)
    assert np.all(normal[cap] == np.array([128, 128, 255, 255], np.uint8))
    assert np.all(normal[~covered] == 0)
    rng = np.random.default_rng(3)
    if kind == "color":
        frame = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        cam = frame
    else:
        frame = rng.integers(0, 1400, (H, W), dtype=np.uint16)
        g = vr.normalized_depth(frame, 0.001, 0.0, 1.0)
        cam = np.repeat(g[..., None], 3, axis=2)
    img = vr.viewer_image(kind, frame, normal, 0.5, 0.001, 0.0, 1.0)
    assert np.array_equal(img[~covered], cam[~covered])  # every background pixel is the camera pixel
    a = np.float32(255) * (np.float32(0.5) / np.float32(255))
    exp = (cam[cap].astype(np.float32) * (np.float32(1) - a) + np.array([128, 128, 255], np.float32) * a).astype(np.uint8)
    assert np.array_equal(img[cap], exp)


@pytest.mark.parametrize("mesh,view", [("prism", 0), ("prism", 7), ("icosphere", 3)])
def test_square_viewer_equals_model_generation_renderer(synth, mesh, view):
    if mesh == "prism":
        tri, diam = synth.prism_triangles()
    else:
        tri, diam = synth.icosphere_triangles(radius=0.04, n_divides=1)
    body = rr.Geometry(tri, I34.copy(), diam, True)
    S = 120
    st = mg.Setup(body, [], 0.8, S)
    c2b = mg.geodesic_poses(1, 0.8)[view]
    exp = mg.render_view(st, c2b)["normal"]
    intr = _intr(st.fu, st.fu, st.pp, st.pp, S, S)
    got, _ = vr.render_normal(intr, mg.pose_inverse(c2b), {0: I34}, {0: body}, [0], st.z_min, st.z_max)
    assert np.array_equal(got, exp)
    assert (got[..., 3] == 255).sum() > 100
