"""cv::ORB on the device (m3tb_texture_detect_orb, k_texture_orb): detections bit-equal to cv2's golden sets in the
canonical order at every setting; tracking from them equal to a context fed the same features through the host
upload, on rigid bodies, a kinematic chain and more than one launch's worth of bodies; bodies without a focus;
the n_features_max capacity with ties; refusals and a failed scratch allocation that leave the context as it was; the
C++ mirror's DetectFeatures (examples/texture_orb_device_mirror_tracker.cpp) against the C ABI read-back path."""
import json
import os
import subprocess

import numpy as np
import pytest

import texture_orb_reference as R
from test_gpu_texture_device_front_end import CHAIN_POSES, FIX, FIX_FRAME, _crop, _same, _scene

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "texture_orb.npz"))
FIELDS = ("xy", "angle", "response", "octave", "descriptors")


def _golden(si, i):
    n = GOLD[f"s{si}_n"]
    at = int(n[:i].sum())
    return {k: GOLD[f"s{si}_{k}"][at:at + int(n[i])] for k in FIELDS}


def _texture_params(capi, n_features_max):
    p = capi.texture_params_default()
    p.descriptor_type = capi.DESCRIPTOR_ORB
    p.focused_image_size = int(FIX["focused_image_size"])
    p.n_features_max = n_features_max
    return p


@pytest.mark.parametrize("si", range(len(R.SETTINGS)), ids=["%d-%g-%d" % s for s in R.SETTINGS])
def test_detections_equal_cv2(capi, synth, si):
    ctx = _scene(capi, synth)
    n = len(FIX["poses"])
    for b in range(n):
        ctx.set_texture_modality(b, _texture_params(capi, 4096), 0)
    before = ctx.launch_count
    ctx.texture_detect_orb(list(range(n)), R.SETTINGS[si])
    assert ctx.launch_count == before + 2
    found = ctx.get_texture_detections()
    for i in range(n):
        gold = _golden(si, i)
        assert found[i] == len(gold["angle"])
        got = ctx.get_texture_orb_keypoints(i)
        for k in FIELDS:
            assert _same(got[k], gold[k]), (i, k)
    ctx.close()


def _feed_host(ctx_d, ctx_h, bodies):
    """The device detections of ctx_d uploaded to ctx_h through the host path (same roi and scale)."""
    roi, scale, _ = ctx_d.get_texture_focus()
    for b in bodies:
        got = ctx_d.get_texture_orb_keypoints(b)
        ctx_h.upload_texture_features(b, got["xy"], got["descriptors"], roi[b][0], roi[b][1], scale[b])


def _track_equal(capi, synth, scene, bodies, n_min):
    ctx_d = _scene(capi, synth, **scene)
    ctx_h = _scene(capi, synth, **scene)
    ctx_d.texture_detect_orb(bodies)
    _feed_host(ctx_d, ctx_h, bodies)
    for ctx in (ctx_d, ctx_h):
        ctx.start_modalities(0)
    total = 0
    for b in bodies:
        kd, kh = ctx_d.get_texture_keyframes(b), ctx_h.get_texture_keyframes(b)
        assert _same(kd["sizes"], kh["sizes"]) and _same(kd["points"], kh["points"])
        assert _same(kd["descriptors"], kh["descriptors"])
        total += int(kd["sizes"].sum())
    assert total >= n_min
    for it in (1, 2):
        for ctx in (ctx_d, ctx_h):
            ctx.upload_color(0, FIX_FRAME)
        ctx_d.texture_detect_orb(bodies)
        _feed_host(ctx_d, ctx_h, bodies)
        for ctx in (ctx_d, ctx_h):
            ctx.tracking_step(it, 2, 2)
            ctx.calculate_results(it)
        assert _same(ctx_d.get_poses(), ctx_h.get_poses())
        for b in bodies:
            assert _same(ctx_d.get_texture_points(b), ctx_h.get_texture_points(b))
            kd, kh = ctx_d.get_texture_keyframes(b), ctx_h.get_texture_keyframes(b)
            assert _same(kd["points"], kh["points"]) and _same(kd["descriptors"], kh["descriptors"])
    ctx_d.close()
    ctx_h.close()


def test_tracking_equals_the_host_upload_rigid(capi, synth):
    _track_equal(capi, synth, dict(bodies=[0, 3, 9]), [0, 1, 2], 50)


def test_tracking_equals_the_host_upload_chain(capi, synth):
    _track_equal(capi, synth, dict(poses=CHAIN_POSES, chain=True), [0, 1, 2], 20)


def test_more_bodies_than_one_launch_takes(capi, synth):
    n = 131
    src = [b % len(FIX["poses"]) for b in range(n)]
    ctx = _scene(capi, synth, poses=FIX["poses"][src], own_geometry=True)
    order = [int(b) for b in np.random.default_rng(7).permutation(n)]
    before = ctx.launch_count
    ctx.texture_detect_orb(order)
    assert ctx.launch_count == before + 4  # a crop and a detection launch per 128 bodies
    found = ctx.get_texture_detections()
    for b in range(n):
        gold = _golden(0, src[b])
        assert found[b] == len(gold["angle"])
        got = ctx.get_texture_orb_keypoints(b)
        assert all(_same(got[k], gold[k]) for k in FIELDS), b
    ctx.close()
    _track_equal(capi, synth, dict(poses=FIX["poses"][src], own_geometry=True), list(range(n)), 1000)


def test_the_detection_crop_is_m3tb_texture_crop(capi, synth):
    ctx = _scene(capi, synth)
    n = len(FIX["poses"])
    out, roi, scale, size, valid = _crop(ctx, list(range(n)))
    host = out.cpu().numpy()
    ctx.texture_detect_orb(list(range(n)))
    for i in range(n):
        w, h = size[i]
        mine = R.orb(host[i, :h, :w])
        got = ctx.get_texture_orb_keypoints(i)
        assert all(_same(got[k], mine[k]) for k in FIELDS), i
    ctx.close()


def test_bodies_without_a_focus_get_no_features(capi, synth):
    poses = FIX["poses"][[0, 3]].copy()
    poses[1, 2, 3] = 0.01  # in front of the camera by less than 1.5 radii: no focus
    ctx = _scene(capi, synth, poses=poses)
    ctx.texture_detect_orb([0, 1])
    assert list(ctx.get_texture_detections()) == [int(GOLD["s0_n"][0]), 0]
    assert len(ctx.get_texture_orb_keypoints(1)["angle"]) == 0
    ctx.start_modalities(0)
    assert int(ctx.get_texture_keyframes(0)["sizes"].sum()) > 0
    assert int(ctx.get_texture_keyframes(1)["sizes"].sum()) == 0
    ctx.close()


def test_capacity(capi, synth):
    """Crop 3 keeps 958 keypoints at n_features 4096: dropped at n_features_max 512, kept at 2048."""
    si = R.SETTINGS.index((4096, 1.2, 3))
    gold = _golden(si, 3)
    assert len(gold["angle"]) == 958
    ctx = _scene(capi, synth, bodies=[3])
    ctx.texture_detect_orb([0], (4096, 1.2, 3))
    assert list(ctx.get_texture_detections()) == [958]
    assert len(ctx.get_texture_orb_keypoints(0)["angle"]) == 0
    ctx.start_modalities(0)
    assert int(ctx.get_texture_keyframes(0)["sizes"].sum()) == 0
    ctx.set_texture_modality(0, _texture_params(capi, 2048), 0)
    ctx.texture_detect_orb([0], (4096, 1.2, 3))
    assert list(ctx.get_texture_detections()) == [958]
    got = ctx.get_texture_orb_keypoints(0)
    assert all(_same(got[k], gold[k]) for k in FIELDS)
    ctx.close()


def test_ties_keep_more_than_n_features(capi, synth):
    """A frame of identical dots: cv::ORB keeps 566 keypoints at n_features 300 (ties at both cuts). The body is
    dropped at n_features_max 512 with the count reported, and kept at 2048, equal to cv2."""
    tie = {k: GOLD[f"tie_{k}"] for k in FIELDS}
    n = len(tie["angle"])
    assert n == 566 > R.TIE_SETTING[0]
    ctx = _scene(capi, synth, bodies=[R.TIE_BODY], upload=False)
    ctx.upload_color(0, R.dot_frame())
    out, _, _, size, valid = _crop(ctx, [0])
    w, h = size[0]
    assert valid[0] and np.array_equal(out.cpu().numpy()[0, :h, :w], GOLD["tie_crop"])
    ctx.texture_detect_orb([0], R.TIE_SETTING)
    assert list(ctx.get_texture_detections()) == [n]
    assert len(ctx.get_texture_orb_keypoints(0)["angle"]) == 0
    ctx.start_modalities(0)
    assert int(ctx.get_texture_keyframes(0)["sizes"].sum()) == 0
    ctx.set_texture_modality(0, _texture_params(capi, 2048), 0)
    assert list(ctx.get_texture_detections()) == [0]  # setting the modality forgets the detection
    ctx.texture_detect_orb([0], R.TIE_SETTING)
    assert list(ctx.get_texture_detections()) == [n]
    got = ctx.get_texture_orb_keypoints(0)
    assert all(_same(got[k], tie[k]) for k in FIELDS)
    ctx.start_modalities(0)
    assert int(ctx.get_texture_keyframes(0)["sizes"].sum()) > 0
    ctx.close()


def test_read_back_is_the_detections_own(capi, synth):
    """A later host upload replaces the feature slot, not the read-back; setting or removing the modality forgets it;
    a detection that grows the parity tables forgets the other bodies'."""
    ctx = _scene(capi, synth, bodies=[0, 3])
    ctx.texture_detect_orb([0, 1])
    gold0 = _golden(0, 0)
    roi, scale, _ = ctx.get_texture_focus()
    ctx.upload_texture_features(0, np.zeros((3, 2), np.float32), np.full((3, 32), 7, np.uint8), roi[0][0], roi[0][1],
                                scale[0])
    got = ctx.get_texture_orb_keypoints(0)
    assert all(_same(got[k], gold0[k]) for k in FIELDS)
    ctx.set_texture_modality(1, None, 0)
    assert list(ctx.get_texture_detections()) == [len(gold0["angle"]), 0]
    assert len(ctx.get_texture_orb_keypoints(1)["angle"]) == 0
    ctx.set_texture_modality(1, _texture_params(capi, 512), 0)
    ctx.texture_detect_orb([1])
    ctx.set_texture_modality(1, _texture_params(capi, 1024), 0)  # the context's feature capacity grows
    ctx.texture_detect_orb([1])                                   # new parity tables: body 0's detection is gone
    assert list(ctx.get_texture_detections()) == [0, int(GOLD["s0_n"][3])]
    assert len(ctx.get_texture_orb_keypoints(0)["angle"]) == 0
    got = ctx.get_texture_orb_keypoints(1)
    assert all(_same(got[k], _golden(0, 3)[k]) for k in FIELDS)
    ctx.close()


def _state(ctx, n):
    return (ctx.get_texture_detections().tolist(), [ctx.get_texture_orb_keypoints(b)["descriptors"].tobytes() for b in range(n)],
            ctx.get_poses().tobytes())


def test_refusals_leave_the_context_as_it_was(capi, synth):
    ctx = _scene(capi, synth, bodies=[0, 3, 4, 5])
    sift = capi.texture_params_default()
    sift.descriptor_type = capi.DESCRIPTOR_SIFT
    ctx.set_texture_modality(2, sift, 0)
    ctx.set_texture_modality(3, None, 0)  # a body without a texture modality
    ctx.texture_detect_orb([0, 1])
    state = _state(ctx, 2)

    def refused(code, bodies, params=None):
        before = ctx.launch_count
        with pytest.raises(capi.M3TBError, match="status %d" % code):
            ctx.texture_detect_orb(bodies, params)
        assert ctx.launch_count == before
        assert _state(ctx, 2) == state

    refused(-1, [0, 2])                      # SIFT body
    refused(-1, [0, 3])                      # no texture modality
    refused(-1, [0, 0])                      # listed twice
    refused(-1, [0, 7])                      # no such body
    refused(-3, [0], ((1 << 24) + 1, 1.2, 3))  # n_features above 2^24
    refused(-1, [0], (0, 1.2, 3))            # n_features < 1
    refused(-1, [0], (300, 1.0, 3))          # scale_factor <= 1
    refused(-1, [0], (300, float("nan"), 3))
    refused(-1, [0], (300, float("inf"), 3))
    refused(-1, [0], (300, 1.2, 0))          # n_levels < 1
    refused(-3, [1], (300, 1.2, 9))          # n_levels above the device limit
    refused(-3, [0, 1], [(300, 1.2, 3), (300, 1.2, 9)])
    ctx.close()


def test_a_failed_scratch_allocation_leaves_the_context_as_it_was(capi, synth):
    import ctypes as C
    ctx = _scene(capi, synth, bodies=[0, 3])
    ctx.texture_detect_orb([0])
    state = _state(ctx, 2)
    live = C.c_longlong(0)
    for fail_after in range(1, 8):
        ctx.L.m3tb_debug_resources(fail_after, C.byref(live))
        try:
            ctx.texture_detect_orb([0, 1], (300, 1.2, 3))
            ok = True
        except capi.M3TBError:
            ok = False
        finally:
            ctx.L.m3tb_debug_resources(0, C.byref(live))
        if ok:
            break
        assert _state(ctx, 2) == state
    else:
        pytest.fail("no allocation budget let the detection through")
    found = ctx.get_texture_detections()
    assert list(found) == [int(GOLD["s0_n"][0]), int(GOLD["s0_n"][3])]
    ctx.close()


def test_cpp_mirror_detects_on_the_device(pkg, tmp_path):
    """examples/texture_orb_device_mirror_tracker.cpp: a rigid body and a 3-link chain tracked by
    Tracker::ExecuteTrackingStep with features from TextureModality::DetectFeatures (one body alone, then lists), against
    the same scene fed the C ABI read-back through the host SetFeatures: equal texture points and poses, bit for bit."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg._build.build_cuda()
    pkg._build.build_synth()
    csrc = os.path.join(root, "3dobjecttracking_b200", "csrc")
    synth_dir = os.path.join(root, "3dobjecttracking_b200", "synth")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "texture_orb_device_mirror_tracker")
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(root, "include"), "-I",
           os.path.join(root, "3dobjecttracking_b200", "host"), "-I", synth_dir, "-I", os.path.join(cuda, "include"),
           os.path.join(root, "examples", "texture_orb_device_mirror_tracker.cpp"), "-o", exe, "-L", csrc, "-L", synth_dir,
           "-L", os.path.join(cuda, "lib64"), "-lm3t_b200", "-lm3t_synth", "-lcudart", "-Wl,-rpath," + csrc,
           "-Wl,-rpath," + synth_dir, "-Wl,-rpath," + os.path.join(cuda, "lib64"), "-fopenmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, "1", "300"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    out = json.loads(r.stdout.strip().split("\n")[-1])
    assert out["orb_n_features"] == 300
    assert min(out["found_start"]) > 50 and min(out["found"]) > 50
    assert min(out["texture_points_device"]) > 10 and out["texture_points_device"] == out["texture_points_host"]
    host, dev = (np.array(out[k], np.float32).reshape(-1, 12) for k in ("host", "device"))
    assert _same(host, dev)
    start = np.array(out["start"], np.float32).reshape(-1, 12)
    assert not _same(dev, start)  # the step moved the bodies
