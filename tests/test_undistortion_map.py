"""m3tb_undistortion_map (host only) against OpenCV's initUndistortRectifyMap(CV_32FC1) + convertMaps(CV_16SC2,
nninterpolation=True), the refusals, the NumPy restatement of the remap / depth offset against cv2, the stored cv2 maps
of tests/golden/undistortion/, and the mirror's AzureKinect cameras (examples/undistortion_selftest.cpp, host checks).

The bar: every map entry that lies inside the raw frame in either map is identical, and so is the remapped image.
Entries far outside the frame (|value| beyond the int16 range) may saturate differently and select the border value
either way."""
import json
import os
import subprocess

import numpy as np
import pytest

import undistortion_reference as ur

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Azure Kinect colour modes (720p .. 3072p), depth modes (NFOV binned / unbinned, WFOV unbinned / binned), an odd size
RESOLUTIONS = [(1280, 720), (1920, 1080), (2560, 1440), (2048, 1536), (3840, 2160), (4096, 3072),
               (320, 288), (640, 576), (512, 512), (1024, 1024), (333, 217)]


def _intr(synth, w, h, fu, fv, cx, cy):
    return synth.Intrinsics(float(fu), float(fv), float(cx), float(cy), int(w), int(h))


def _calibration(rng, w, h, kind):
    f = np.float32(rng.uniform(0.45, 0.8) * w)
    fx, fy = f, np.float32(f * rng.uniform(0.995, 1.005))
    cx = np.float32(w / 2 + rng.uniform(-0.03, 0.03) * w)
    cy = np.float32(h / 2 + rng.uniform(-0.03, 0.03) * h)
    if kind == "rational":
        k = [rng.uniform(-0.6, 0.6), rng.uniform(-2.5, 2.5), rng.uniform(-2e-3, 2e-3), rng.uniform(-2e-3, 2e-3),
             rng.uniform(-1.5, 1.5), rng.uniform(-0.6, 0.6), rng.uniform(-2.5, 2.5), rng.uniform(-1.5, 1.5)]
    elif kind == "tangential":
        k = [0.0, 0.0, rng.uniform(-5e-3, 5e-3), rng.uniform(-5e-3, 5e-3), 0.0, 0.0, 0.0, 0.0]
    else:
        k = [0.0] * 8
    scale = np.float32(1.0 if kind == "zero" else rng.uniform(0.5, 1.2))
    return fx, fy, cx, cy, np.asarray(k, np.float32), scale


def _cv2_map(cv2, w, h, fx, fy, cx, cy, k, scale):
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    fu, fv = np.float32(fx) * scale, np.float32(fy) * scale
    Kn = np.array([[fu, 0, cx], [0, fv, cy], [0, 0, 1]], np.float32)
    m1, m2 = cv2.initUndistortRectifyMap(K, k.reshape(1, 8), None, Kn, (w, h), cv2.CV_32FC1)
    m, _ = cv2.convertMaps(m1, m2, cv2.CV_16SC2, nninterpolation=True)
    return m, fu, fv


def _inside(m, w, h):
    return (m[..., 0] >= 0) & (m[..., 0] < w) & (m[..., 1] >= 0) & (m[..., 1] < h)


CASES = [(w, h, "rational", i) for i, (w, h) in enumerate(RESOLUTIONS)] + \
        [(w, h, "tangential", 50 + i) for i, (w, h) in enumerate(RESOLUTIONS[::3])] + \
        [(w, h, "zero", 80 + i) for i, (w, h) in enumerate(RESOLUTIONS[::2])]


@pytest.mark.parametrize("w,h,kind,seed", CASES)
def test_map_equals_opencv(capi, synth, w, h, kind, seed):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy, k, scale = _calibration(rng, w, h, kind)
    ref, fu, fv = _cv2_map(cv2, w, h, fx, fy, cx, cy, k, scale)
    got = capi.undistortion_map(_intr(synth, w, h, fx, fy, cx, cy), k, _intr(synth, w, h, fu, fv, cx, cy))
    assert got.shape == (h, w, 2) and got.dtype == np.int16
    either = _inside(ref, w, h) | _inside(got, w, h)
    bad = either & np.any(got != ref, axis=2)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:5])
    differing = int(np.any(got != ref, axis=2).sum())
    assert differing <= max(8, w * h // 100000), differing  # only far out-of-frame saturations may differ
    if kind == "zero":  # the exact identity
        jj, ii = np.meshgrid(np.arange(w), np.arange(h))
        assert np.array_equal(got[..., 0], jj) and np.array_equal(got[..., 1], ii)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    a = cv2.remap(img, ref, None, cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT)
    b = cv2.remap(img, got, None, cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT)
    assert np.array_equal(a, b)


@pytest.mark.parametrize("name", ur.golden_names())
def test_map_equals_the_stored_opencv_maps(capi, synth, name):
    m, c = ur.load_golden_map(name)
    w, h = int(c["width"]), int(c["height"])
    got = capi.undistortion_map(_intr(synth, w, h, c["fx"], c["fy"], c["cx"], c["cy"]), c["coefficients"],
                                _intr(synth, w, h, c["fu"], c["fv"], c["cx"], c["cy"]))
    either = _inside(m, w, h) | _inside(got, w, h)
    assert not (either & np.any(got != m, axis=2)).any()


def test_map_pitch(capi, synth):
    intr = _intr(synth, 64, 48, 50.0, 50.0, 32.0, 24.0)
    k = np.array([0.1, -0.05, 1e-3, 0, 0, 0, 0, 0], np.float32)
    dense = capi.undistortion_map(intr, k, intr)
    padded = np.full((48, 64 * 4 + 12), 0x7f, np.uint8)
    rc = capi.lib().m3tb_undistortion_map(capi.C.byref(intr), capi._p(k), capi.C.byref(intr), padded.ctypes.data,
                                          padded.strides[0])
    assert rc == 0
    assert np.array_equal(padded[:, :256].copy().view(np.int16).reshape(48, 64, 2), dense)
    assert (padded[:, 256:] == 0x7f).all()  # the row padding is not written


def test_refusals(capi, synth):
    C = capi.C
    L = capi.lib()
    good = _intr(synth, 64, 48, 50.0, 50.0, 32.0, 24.0)
    k = np.zeros(8, np.float32)
    out = np.zeros((48, 64, 2), np.int16)

    def call(raw=good, coeff=k, rect=good, ptr=out.ctypes.data, pitch=256):
        return L.m3tb_undistortion_map(C.byref(raw) if raw is not None else None,
                                       capi._p(coeff) if coeff is not None else None,
                                       C.byref(rect) if rect is not None else None, ptr, pitch)

    assert call() == 0
    assert call(pitch=255) != 0
    assert call(ptr=None) != 0
    assert call(raw=None) != 0 and call(rect=None) != 0 and call(coeff=None) != 0
    assert call(rect=_intr(synth, 65, 48, 50.0, 50.0, 32.0, 24.0)) != 0
    assert call(rect=_intr(synth, 64, 47, 50.0, 50.0, 32.0, 24.0)) != 0
    assert call(raw=_intr(synth, 0, 48, 50.0, 50.0, 32.0, 24.0), rect=_intr(synth, 0, 48, 50.0, 50.0, 32.0, 24.0)) != 0
    for bad in ((0.0, 50.0, 32.0, 24.0), (50.0, -1.0, 32.0, 24.0), (np.nan, 50.0, 32.0, 24.0),
                (50.0, 50.0, np.inf, 24.0), (50.0, 50.0, 32.0, -np.inf), (50.0, 50.0, -3.0, 24.0)):
        b = _intr(synth, 64, 48, *bad)
        assert call(raw=b) != 0 and call(rect=b) != 0, bad
    for i in range(8):
        for v in (np.nan, np.inf, -np.inf):
            kk = np.zeros(8, np.float32)
            kk[i] = v
            assert call(coeff=kk) != 0, (i, v)
    with pytest.raises(capi.M3TBError):
        capi.undistortion_map(good, k, _intr(synth, 64, 49, 50.0, 50.0, 32.0, 24.0))


@pytest.mark.parametrize("channels", [3, 4])
def test_remap_restatement_equals_cv2(capi, synth, channels):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(channels)
    m, _ = ur.load_golden_map("color_1280x720")
    raw = rng.integers(0, 256, (720, 1280, channels), dtype=np.uint8)
    bgr = cv2.cvtColor(raw, cv2.COLOR_RGBA2RGB) if channels == 4 else raw
    ref = cv2.remap(bgr, m, None, cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT)
    assert np.array_equal(ur.undistort_color(raw, m), ref)


@pytest.mark.parametrize("offset", [-37, 0, 37, -32768, 32767])
def test_depth_restatement_equals_cv2(offset):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(abs(offset))
    m, _ = ur.load_golden_map("depth_640x576")
    m[:3] = -1          # entries outside the raw frame (this calibration has none of its own)
    m[:, -2:, 0] = 641
    raw = rng.integers(0, 65536, (576, 640), dtype=np.uint16)
    raw[::7, ::5] = 0
    raw[3::11, 2::3] = 65535
    img = cv2.remap(raw, m, None, cv2.INTER_NEAREST, borderMode=cv2.BORDER_CONSTANT)
    if offset:
        img = cv2.add(img, (float(offset), 0.0, 0.0, 0.0))  # image_ += short(offset): saturating
    assert np.array_equal(ur.undistort_depth(raw, m, offset), img)
    border = ~_inside(m, 640, 576)
    assert border.any()
    assert (ur.undistort_depth(raw, m, offset)[border] == max(offset, 0)).all()  # border pixels get the offset too


def test_mirror_selftest_host_checks(pkg, tmp_path):
    pkg._build.build_cuda()
    csrc = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
    exe = str(tmp_path / "undistortion_selftest")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "3dobjecttracking_b200", "host"), os.path.join(ROOT, "examples", "undistortion_selftest.cpp"),
           "-o", exe, "-L", csrc, "-lm3t_b200", "-Wl,-rpath," + csrc]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True)
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["host_checks_failed"] == 0, r.stderr
    assert out["depth"]["depth_value_offset"] == -37  # short(-0.0375f / 0.001f)
    c = out["color"]
    assert np.float32(c["fu"]) == np.float32(c["fx"]) * np.float32(1.05)
    assert r.returncode == 0, r.stderr
