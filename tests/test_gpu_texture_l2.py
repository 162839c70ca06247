"""SIFT and DAISY texture modalities on the device (m3tb_upload_texture_float_features, k_texture_knn_l2): the
cv2.BFMatcher(NORM_L2) fixtures through the C ABI, the fine-grained and fused paths against the CPU restatement
(tests/texture_reference_l2.py knn2_l2 / match_l2) on seeded SIFT-like (whole numbers) and DAISY-like (unit-norm) features,
a textured kinematic structure with SIFT links against the restatement and the structure oracle, a mixed context whose
ORB and texture-free bodies are unchanged by L2 bodies beside them, the refusals, the all-or-nothing float tables, and
the C++ mirror's SIFT tracker."""
import json
import os
import subprocess

import numpy as np
import pytest

import test_gpu_texture as rigid
import test_gpu_texture_structures as ts
import texture_reference as tr
import texture_reference_l2 as tr2
from helpers import pose_error

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "texture_knn_l2.npz")
SIFT, DAISY = 3, 1
KIND = {"sift": (SIFT, 128), "daisy": (DAISY, 104)}
INTR = rigid.INTR


def _descriptors(rng, kind, n):
    if kind == "sift":
        return rng.integers(0, 256, (n, 128)).astype(np.float32)
    v = rng.random((n, KIND[kind][1])).astype(np.float32)
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def _perturbed(rng, kind, d):
    if kind == "sift":
        return np.clip(d + rng.integers(-3, 4, d.shape), 0, 255).astype(np.float32)
    v = (d + rng.normal(0, 0.02, d.shape)).astype(np.float32)
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def _clear(queries, train, threshold=0.7, rel=1e-5):
    """Per query: the ratio of its two best (float64) distances lies more than `rel` from the threshold, so no
    summation order can change whether it is kept; a kept query's best is then ahead of the second by 30 %."""
    if len(train) < 2:
        return np.ones(len(queries), bool)
    d = np.sqrt(((queries[:, None, :].astype(np.float64) - train[None, :, :]) ** 2).sum(-1))
    s = np.sort(d, 1)
    with np.errstate(invalid="ignore", divide="ignore"):
        return ~(np.abs(s[:, 0] / s[:, 1] - threshold) <= rel)


def _start(capi, synth, rng, kind, n_feat=200, **texture):
    ctx, params, _ = rigid._scene(capi, synth, descriptor_type=KIND[kind][0], **texture)
    roi, scale, valid = ctx.get_texture_focus()
    assert valid[0]
    crop, _ = rigid._features(rng, roi[0], scale[0], n_feat)
    desc = _descriptors(rng, kind, n_feat)
    xy = rigid._upload(ctx, 0, crop, desc, roi[0], scale[0])
    ctx.start_modalities(0)
    idx, pts = tr.reconstruct(xy, ctx.get_rendering(0), INTR, tr.pose_inverse(rigid._b2c(ctx.get_poses()[0])), 1)
    kf = ctx.get_texture_keyframes(0)
    assert list(kf["sizes"]) == [len(idx)] and len(idx) > 20
    assert np.array_equal(kf["points"].view(np.uint32), pts.view(np.uint32))
    assert kf["descriptors"].dtype == np.float32 and np.array_equal(kf["descriptors"].view(np.uint32),
                                                                     desc[idx].view(np.uint32))
    return ctx, params, pts, desc[idx]


def _next_frame(ctx, rng, kind, true_pose, kf_pts, kf_desc, n_noise=40):
    roi, scale, _ = ctx.get_texture_focus()
    proj = tr.project(rigid._b2c(true_pose), INTR, kf_pts)
    crop = ((proj - roi[0][:2].astype(np.float32)) * scale[0]).astype(np.float32)
    nc, _ = rigid._features(rng, roi[0], scale[0], n_noise)
    crop = np.vstack([crop, nc]).astype(np.float32)
    desc = np.vstack([_perturbed(rng, kind, kf_desc), _descriptors(rng, kind, n_noise)]).astype(np.float32)
    return rigid._upload(ctx, 0, crop, desc, roi[0], scale[0]), desc


# ---- the OpenCV fixtures through the C ABI ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["sift", "ties", "equal_distance", "train_of_one", "empty_train", "daisy104",
                                  "daisy200"])
def test_opencv_fixtures_through_the_c_abi(capi, synth, name):
    """Queries become keyframe points (all inside the silhouette, at distinct places), the train set the next frame's
    features at distinct coordinates, so each data point names its query and the train index it matched."""
    z = np.load(GOLDEN)
    q, t, ref_idx, ref_dist = (z[name + k] for k in ("_queries", "_train", "_idx", "_dist"))
    daisy = name.startswith("daisy")
    ctx, params, _ = rigid._scene(capi, synth, descriptor_type=DAISY if daisy else SIFT)
    roi, scale, _ = ctx.get_texture_focus()
    center = tr.project(rigid._b2c(ctx.get_poses()[0]), INTR, np.zeros((1, 3), np.float32))[0]
    rng = np.random.default_rng(31)
    qxy = (center + rng.uniform(-8.0, 8.0, (len(q), 2))).astype(np.float32)
    qcrop = ((qxy - roi[0][:2].astype(np.float32)) * scale[0]).astype(np.float32)
    rigid._upload(ctx, 0, qcrop, q, roi[0], scale[0])
    ctx.start_modalities(0)
    kf = ctx.get_texture_keyframes(0)
    assert list(kf["sizes"]) == [len(q)]
    kf_rows = {p.tobytes(): i for i, p in enumerate(kf["points"])}
    assert len(kf_rows) == len(q)
    tcrop = np.stack([np.arange(len(t), dtype=np.float32), np.full(len(t), 3.0, np.float32)], 1)
    txy = rigid._upload(ctx, 0, tcrop, t, roi[0], scale[0])
    t_rows = {p.tobytes(): j for j, p in enumerate(txy)}
    assert len(t_rows) == len(t)
    ctx.texture_correspondences(1, 0)
    got = ctx.get_texture_points(0)
    device = np.full(len(q), -1)
    for p in got:
        device[kf_rows[p["center_f_body"].tobytes()]] = t_rows[p["correspondence_center"].tobytes()]
    with np.errstate(invalid="ignore", divide="ignore"):
        keep = (ref_idx[:, 1] >= 0) & ~(ref_dist[:, 0] / ref_dist[:, 1] >= np.float32(params.descriptor_distance_threshold))
    expected = np.where(keep, ref_idx[:, 0], -1)
    if not daisy:
        assert np.array_equal(device, expected)
        # data points keep query order
        assert [kf_rows[p["center_f_body"].tobytes()] for p in got] == sorted(kf_rows[p["center_f_body"].tobytes()]
                                                                               for p in got)
    else:
        clear = _clear(q, t, np.float32(params.descriptor_distance_threshold))
        assert clear.sum() > 0.9 * len(q)
        assert np.array_equal(device[clear], expected[clear])
    if name == "sift":
        assert 20 < (device >= 0).sum() < len(q)


# ---- tracking against the restatement ---------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["sift", "daisy"])
def test_fine_grained_iterations_match_the_restatement(capi, synth, kind):
    rng = np.random.default_rng(5)
    ctx, params, kf_pts, kf_desc = _start(capi, synth, rng, kind)
    true_pose = rigid._pose((2.0, -1.5, 1.0), (0.004, -0.003, 0.505))
    xy, desc = _next_frame(ctx, rng, kind, true_pose, kf_pts, kf_desc)
    if kind == "daisy":  # SIFT sums whole numbers, exact in any order; DAISY needs a clear ratio
        assert _clear(kf_desc, desc).all()
    cb, cc = tr2.match_l2([(kf_pts, kf_desc)], xy, desc, params.descriptor_distance_threshold)
    assert len(cb) > 20
    pose = ctx.get_poses()[0]
    for corr in range(2):
        ctx.texture_correspondences(1, corr)
        got = ctx.get_texture_points(0)
        assert np.array_equal(got["center_f_body"].view(np.uint32), cb.view(np.uint32))
        assert np.array_equal(got["correspondence_center"].view(np.uint32), cc.view(np.uint32))
        assert np.array_equal(got["center"].view(np.uint32),
                              tr.project(rigid._b2c(ctx.get_poses()[0]), INTR, cb).view(np.uint32))
        for upd in range(2):
            g, H = ctx.texture_gradient_hessian(1, corr, upd)
            eg, eH = tr.gradient_hessian(rigid._b2c(pose), INTR, cb, cc, params.standard_deviations[min(corr, 1)], 20.0)
            scale = np.abs(eH).max()
            assert np.abs(g[0] - eg).max() <= 1e-5 * scale and np.abs(H[0] - eH).max() <= 1e-5 * scale
            ctx.calculate_optimization(1, corr, upd)
            pose = tr.optimize(pose, g[0].astype(np.float64), H[0].astype(np.float64))
            assert np.abs(ctx.get_poses()[0].reshape(12) - pose.reshape(12)).max() < 1e-4


@pytest.mark.parametrize("kind,n_keyframes", [("sift", 1), ("sift", 4), ("daisy", 1), ("daisy", 4)])
def test_fused_step_and_keyframe_refresh(capi, synth, kind, n_keyframes):
    """tracking_step against the restatement iteration by iteration, the keyframe deque refreshed every frame (age
    rule) and matched keyframe by keyframe."""
    rng = np.random.default_rng(11 + n_keyframes)
    ctx, params, kf_pts, kf_desc = _start(capi, synth, rng, kind, n_keyframes=n_keyframes, max_keyframe_age=0)
    keyframes = [(kf_pts, kf_desc)]
    pose = ctx.get_poses()[0]
    for frame in range(1, 6):
        true_pose = rigid._pose((1.0 * frame, 0.5, -0.5 * frame), (0.002 * frame, 0.001, 0.5 + 0.002 * frame))
        xy, desc = _next_frame(ctx, rng, kind, true_pose, *keyframes[-1])
        for _, d in keyframes:
            assert kind == "sift" or _clear(d, desc).all()
        cb, cc = tr2.match_l2(keyframes, xy, desc, params.descriptor_distance_threshold)
        ctx.tracking_step(frame, 2, 2)
        assert ctx.last_launch()["kernel"] == "k_track"
        stale = pose
        for corr in range(2):
            for upd in range(2):
                g, H = tr.gradient_hessian(rigid._b2c(pose), INTR, cb, cc, params.standard_deviations[min(corr, 1)], 20.0)
                stale = pose
                pose = tr.optimize(pose, g, H)
        assert np.abs(ctx.get_poses()[0].reshape(12) - pose.reshape(12)).max() < 1e-4, frame
        got = ctx.get_texture_points(0)
        assert np.array_equal(got["center_f_body"].view(np.uint32), cb.view(np.uint32))
        assert np.array_equal(got["correspondence_center"].view(np.uint32), cc.view(np.uint32))
        ctx.calculate_results(frame)
        kf = ctx.get_texture_keyframes(0)
        idx, pts = tr.reconstruct(xy, ctx.get_rendering(0), INTR, tr.pose_inverse(rigid._b2c(stale)), 1)
        new = kf["points"][-kf["sizes"][-1]:]
        assert len(new) == len(idx) and np.abs(new - pts).max() < 1e-3
        assert np.array_equal(kf["descriptors"][-kf["sizes"][-1]:], desc[idx])
        keyframes.append((new.copy(), desc[idx]))
        keyframes = keyframes[-n_keyframes:]
        assert len(kf["sizes"]) == min(frame + 1, n_keyframes)
        pose = ctx.get_poses()[0].reshape(3, 4)


def test_textured_chain_with_sift_links(capi, oracle, synth, monkeypatch):
    """The root and two revolute children with SIFT texture modalities: the structure test's fine-grained iteration
    (restatement + structure oracle at every update) with the L2 matcher, and the fused step held to it."""
    monkeypatch.setattr(ts.tr, "match", tr2.match_l2)  # the structure helpers' matcher is the L2 one here
    spec = ts._chain(synth)
    ctxs = []
    for _ in range(2):
        ctx, params = ts._context(capi, synth, ts.CHAIN_POSES, texture=(0, 1, 2), descriptor_type=SIFT)
        ctx.set_structure(0, spec)
        roi, scale, valid = ctx.get_texture_focus()
        for b in range(3):
            rng = np.random.default_rng(100 + b)
            x, y, w, h = roi[b]
            pts = np.stack([rng.uniform(x, x + w, 200), rng.uniform(y, y + h, 200)], 1).astype(np.float32)
            crop = ((pts - np.array([x, y], np.float32)) * np.float32(scale[b])).astype(np.float32)
            ctx.upload_texture_features(b, crop, _descriptors(rng, "sift", 200), x, y, scale[b])
        ctx.start_modalities(0)
        kfs = {b: ctx.get_texture_keyframes(b) for b in range(3)}
        roi, scale, _ = ctx.get_texture_focus()
        poses = ctx.get_poses()
        frame = {}
        for b, kf in kfs.items():
            rng = np.random.default_rng(200 + b)
            proj = tr.project(ts._b2c(tr.pose_mul(ts.MOTION, poses[b])), INTR, kf["points"])
            crop = ((proj - roi[b][:2].astype(np.float32)) * scale[b]).astype(np.float32)
            desc = _perturbed(rng, "sift", kf["descriptors"])
            ctx.upload_texture_features(b, crop, desc, roi[b][0], roi[b][1], scale[b])
            frame[b] = (tr.crop_to_image(crop, roi[b][0], roi[b][1], scale[b]), desc)
        ctxs.append((ctx, kfs, frame))
    (fine, kfs, frame), (fused, _, _) = ctxs
    matches = {}
    for corr in range(2):
        ts._fine_iteration(fine, oracle, spec, params, corr, kfs, frame, matches)
        before = fused.launch_count
        fused.corr_iteration(1, corr, ts.N_UPDATE)
        assert fused.last_launch()["kernel"] == "k_track"
        # one k_render, k_texture_knn_l2 + k_texture_match at iteration 0 only, then k_track + k_structure per update
        assert fused.launch_count - before == 1 + 2 * (corr == 0) + 2 * ts.N_UPDATE, corr
        assert np.abs(fused.get_poses() - fine.get_poses()).max() < 1e-4, corr


def test_mixed_context_orb_and_texture_free_bodies_are_unchanged(capi, synth):
    """Bodies ORB (0), SIFT (1), DAISY (2) and texture-free (3): the ORB body's data points and the poses of bodies 0
    and 3 are bit-identical to those of a context whose bodies 1 and 2 have no texture modality."""
    runs = []
    for tex in ([0, 1, 2], [0]):
        rng = np.random.default_rng(14)
        ctx, params, _ = rigid._scene(capi, synth, n_bodies=4, depth_frame=rigid._plane(), texture_bodies=[])
        ctx.set_poses(np.stack([rigid._pose(t=(0.12 * b - 0.18, 0.0, 0.5)) for b in range(4)]))
        for b, kind in zip(tex, ("orb", "sift", "daisy")):
            p = capi.texture_params_default()
            p.descriptor_type = {"orb": 4, "sift": SIFT, "daisy": DAISY}[kind]
            ctx.set_texture_modality(b, p, 0)
            ctx.attach_renderer(b, "texture_silhouette", b)
        roi, scale, valid = ctx.get_texture_focus()
        feats = {}
        for b, kind in zip(tex, ("orb", "sift", "daisy")):
            assert valid[b]
            crop, orb = rigid._features(rng, roi[b], scale[b], 200)
            desc = orb if kind == "orb" else _descriptors(rng, kind, 200)
            ctx.upload_texture_features(b, crop, desc, roi[b][0], roi[b][1], scale[b])
            feats[b] = (crop, desc, kind)
        ctx.start_modalities(0)
        for b, (crop, desc, kind) in feats.items():  # the next frame: the same keypoints shifted, descriptors perturbed
            if kind == "orb":
                desc = desc.copy()
                desc[:, ::4] ^= 1
            else:
                desc = _perturbed(rng, kind, desc)
            ctx.upload_texture_features(b, crop + 1.5, desc, roi[b][0], roi[b][1], scale[b])
        poses, points = [], []
        for frame in range(1, 4):
            ctx.tracking_step(frame, 2, 2)
            poses.append(ctx.get_poses()[[0, 3]].copy())
            points.append(ctx.get_texture_points(0).copy())
        if len(tex) == 3:
            assert all(len(ctx.get_texture_points(b)) > 20 for b in (1, 2))
        runs.append((poses, points))
    (poses_l2, points_l2), (poses_orb, points_orb) = runs
    assert len(points_orb[0]) > 20
    for a, b in zip(poses_l2, poses_orb):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    for a, b in zip(points_l2, points_orb):
        assert a.tobytes() == b.tobytes()


# ---- refusals and resources -------------------------------------------------------------------------------------------
def test_refusals(capi, synth):
    ctx, params, _ = rigid._scene(capi, synth, n_bodies=2, texture_bodies=[0])
    p = capi.texture_params_default()
    p.descriptor_type = SIFT
    ctx.set_texture_modality(1, p, 0)
    ctx.attach_renderer(1, "texture_silhouette", 1)
    xy = np.zeros((4, 2), np.float32)
    with pytest.raises(capi.M3TBError, match="status -1"):  # the wrong upload call for the body's type
        ctx.upload_texture_features(0, xy, np.zeros((4, 128), np.float32), 0, 0, 1.0)
    with pytest.raises(capi.M3TBError, match="status -1"):
        ctx.upload_texture_features(1, xy, np.zeros((4, 32), np.uint8), 0, 0, 1.0)
    with pytest.raises(capi.M3TBError, match="status -1"):  # SIFT is 128 floats
        ctx.upload_texture_features(1, xy, np.zeros((4, 64), np.float32), 0, 0, 1.0)
    bad = np.zeros((4, 128), np.float32)
    for v in (np.nan, np.inf, -np.inf):
        bad[2, 17] = v
        with pytest.raises(capi.M3TBError, match="status -1"):
            ctx.upload_texture_features(1, xy, bad, 0, 0, 1.0)
    with pytest.raises(capi.M3TBError, match="status -3"):
        ctx.upload_texture_features(1, np.zeros((513, 2), np.float32), np.zeros((513, 128), np.float32), 0, 0, 1.0)
    p.descriptor_type = DAISY
    ctx.set_texture_modality(1, p, 0)
    for length in (0, 257):
        with pytest.raises(capi.M3TBError, match="status -1"):
            ctx.upload_texture_features(1, xy, np.zeros((4, length), np.float32), 0, 0, 1.0)
    ctx.upload_texture_features(1, xy, np.ones((4, 104), np.float32), 0, 0, 1.0)
    with pytest.raises(capi.M3TBError, match="status -1"):  # the first upload fixed the length
        ctx.upload_texture_features(1, xy, np.ones((4, 200), np.float32), 0, 0, 1.0)
    ctx.upload_texture_features(1, xy[:0], np.ones((0, 104), np.float32), 0, 0, 1.0)
    ctx.set_texture_modality(1, p, 0)  # setting the modality again clears the length
    ctx.upload_texture_features(1, xy, np.ones((4, 200), np.float32), 0, 0, 1.0)
    for t in (0, 2, 5):  # BRISK, FREAK, ORB_CUDA
        p.descriptor_type = t
        with pytest.raises(capi.M3TBError, match="status -3"):
            ctx.set_texture_modality(1, p, 0)


@pytest.mark.parametrize("fail_at", [1, 2, 3, 4])
def test_failed_float_table_allocation_leaves_the_context_as_it_was(capi, synth, fail_at):
    """Fault injection on the first SIFT modality: of a context without texture tables (fail_at 1 .. 3 the float
    tables, 4 the first base table) and of one whose ORB body made the base tables."""
    for orb_first in (False, True):
        ctx, params, _ = rigid._scene(capi, synth, n_bodies=2, texture_bodies=[0] if orb_first else [])
        live0 = capi.debug_resources()
        p = capi.texture_params_default()
        p.descriptor_type = SIFT
        capi.debug_resources(fail_after=fail_at)
        try:
            if orb_first and fail_at == 4:  # the base tables exist: three allocations only
                ctx.set_texture_modality(1, p, 0)
                capi.debug_resources(fail_after=0)
                assert capi.debug_resources() == live0 + 3
                continue
            with pytest.raises(capi.M3TBError, match="status -2"):
                ctx.set_texture_modality(1, p, 0)
        finally:
            capi.debug_resources(fail_after=0)
        assert capi.debug_resources() == live0
        with pytest.raises(capi.M3TBError, match="status -1"):
            ctx.get_texture_points(1)  # no texture modality
        if orb_first:
            ctx.tracking_step(0, 1, 1)
        ctx.set_texture_modality(1, p, 0)
        assert len(ctx.get_texture_points(1)) == 0


def test_cpp_mirror_sift_tracker(pkg, tmp_path):
    """examples/texture_mirror_tracker.cpp in its SIFT mode: Tracker::ExecuteTrackingStep against the object-wise path."""
    pkg._build.build_cuda()
    pkg._build.build_synth()
    csrc = os.path.join(ROOT, "3dobjecttracking_b200", "csrc")
    synth_dir = os.path.join(ROOT, "3dobjecttracking_b200", "synth")
    exe = str(tmp_path / "texture_mirror_tracker")
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-I",
           os.path.join(ROOT, "3dobjecttracking_b200", "host"), "-I", synth_dir,
           os.path.join(ROOT, "examples", "texture_mirror_tracker.cpp"), "-o", exe, "-L", csrc, "-L", synth_dir,
           "-lm3t_b200", "-lm3t_synth", "-Wl,-rpath," + csrc, "-Wl,-rpath," + synth_dir, "-fopenmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, "1", "300", "sift"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    out = json.loads(r.stdout.strip().split("\n")[-1])
    assert out["descriptor"] == "sift" and min(out["texture_points"]) > 20, out["texture_points"]
    fused, obj, start, gt = (np.array(out[k], np.float32).reshape(-1, 3, 4) for k in ("fused", "object_wise", "start", "gt"))
    dt, dr = pose_error(fused, obj)  # the gates of test_gpu_texture_mirror.py
    assert np.median(dt) < 2e-5 and np.median(dr) < 2e-4, (dt, dr)
    assert dt.max() < 1e-3 and dr.max() < 1e-2, (dt, dr)
    e0t, e0r = pose_error(start, gt)
    e1t, e1r = pose_error(fused, gt)
    assert np.median(e1t) < np.median(e0t) and np.median(e1r) < np.median(e0r), (e0t, e1t, e0r, e1r)
