"""The texture modality above 512 features per body (m3tb_texture_params::n_features_max up to 4096): the OpenCV kNN
fixtures of tests/golden/texture_knn_large.npz (untruncated M3T-default SIFT of the committed crops, 4096-feature ORB,
synthetic sets around the 512-row chunk) through the C ABI at capacities 1024 and 4096; a full deque of 8 x 4096
keyframe points matched and summed; fused against fine-grained tracking with the Hamming and L2 kNN kernels; a
kinematic chain with large-capacity links; a mixed context whose default ORB body is bit-identical to one without the
large body; the device front end at the capacity; the refusals; allocation failures while the capacity grows; the
launches of default and large contexts; and the C++ mirror's tracker with 2000 features per body."""
import json
import os
import subprocess

import numpy as np
import pytest

import test_gpu_texture as rigid
import test_gpu_texture_device_front_end as dfe
import test_gpu_texture_structures as ts
import test_texture_knn_large as kl
import texture_knn_sets
import texture_reference as tr
from helpers import pose_error

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Z = np.load(kl.GOLDEN)
ORB, SIFT = 4, 3
INTR = rigid.INTR
f32 = np.float32


def _match(keyframes, xy, desc, threshold, hamming):
    """CalculateCorrespondences at corr_iteration 0 with the vectorised kNN (tests/test_texture_knn_large.py)."""
    cb, cc = [np.zeros((0, 3), f32)], [np.zeros((0, 2), f32)]
    for pts, d in keyframes:
        if len(d) == 0 or len(desc) == 0:
            continue
        idx, dist = kl.knn2(d, desc, hamming)
        keep = kl.ratio_keep(idx, dist, f32(threshold))
        cb.append(np.asarray(pts, f32)[keep])
        cc.append(np.asarray(xy, f32)[idx[keep, 0]])
    return np.concatenate(cb), np.concatenate(cc)


def _grid(ctx, n):
    """n distinct image positions 0.25 px apart around the body's centre, all inside its silhouette."""
    center = tr.project(rigid._b2c(ctx.get_poses()[0]), INTR, np.zeros((1, 3), f32))[0]
    g = np.arange(64, dtype=f32) * f32(0.25) - f32(8.0)
    return (center + np.stack(np.meshgrid(g, g), -1).reshape(-1, 2)[:n]).astype(f32)


def _to_crop(xy, roi, scale):
    return ((xy - roi[:2].astype(f32)) * f32(scale)).astype(f32)


def _case(name):
    """(queries, train, idx, dist, descriptor type) of a fixture case."""
    if name == "orb":
        return Z["orb_queries"], Z["orb_train"], Z["orb_idx"], Z["orb_dist"], ORB
    if name.startswith("sift"):
        q, t, idx, dist = kl.sift_pair(Z, int(name[4:]))
        return q, t, idx, dist, SIFT
    _, kind, n = name.split("_")
    q, t = texture_knn_sets.synthetic(int(n), kind == "ham")
    idx, dist = Z[name + "_idx"], Z[name + "_dist"]
    if kind == "l2":
        return q.astype(f32), t.astype(f32), idx, dist, SIFT
    return q, t, idx, dist, ORB


CASES = [("orb", 4096), ("sift0", 4096), ("sift1", 4096), ("sift2", 1024), ("sift2", 4096), ("syn_ham_511", 1024),
         ("syn_ham_1024", 1024), ("syn_ham_4096", 4096), ("syn_l2_513", 1024), ("syn_l2_1024", 1024),
         ("syn_l2_4096", 4096), ("syn_l2_512", 4096)]


@pytest.mark.parametrize("name,cap", CASES)
def test_opencv_fixtures_through_the_c_abi(capi, synth, name, cap):
    """Queries become keyframe points at distinct places, the train set the next frame's features at distinct
    coordinates, so each data point names its query and the train index it matched: equal to cv2.BFMatcher's kNN and
    the ratio test, in query order."""
    q, t, ref_idx, ref_dist, dtype = _case(name)
    assert max(len(q), len(t)) <= cap and max(len(q), len(t)) > 500
    ctx, params, _ = rigid._scene(capi, synth, descriptor_type=dtype, n_features_max=cap)
    roi, scale, _ = ctx.get_texture_focus()
    rigid._upload(ctx, 0, _to_crop(_grid(ctx, len(q)), roi[0], scale[0]), q, roi[0], scale[0])
    ctx.start_modalities(0)
    kf = ctx.get_texture_keyframes(0)
    assert list(kf["sizes"]) == [len(q)]
    kf_rows = {p.tobytes(): i for i, p in enumerate(kf["points"])}
    assert len(kf_rows) == len(q)
    tcrop = np.stack([np.arange(len(t), dtype=f32), np.full(len(t), 3.0, f32)], 1)
    txy = rigid._upload(ctx, 0, tcrop, t, roi[0], scale[0])
    t_rows = {p.tobytes(): j for j, p in enumerate(txy)}
    assert len(t_rows) == len(t)
    before = ctx.launch_count
    ctx.texture_correspondences(1, 0)
    assert ctx.launch_count - before == 2  # one kNN kernel, then k_texture_match
    got = ctx.get_texture_points(0)
    device = np.full(len(q), -1)
    for p in got:
        device[kf_rows[p["center_f_body"].tobytes()]] = t_rows[p["correspondence_center"].tobytes()]
    keep = kl.ratio_keep(ref_idx, ref_dist, f32(params.descriptor_distance_threshold))
    assert np.array_equal(device, np.where(keep, ref_idx[:, 0], -1))
    order = [kf_rows[p["center_f_body"].tobytes()] for p in got]
    assert order == sorted(order) and len(got) == keep.sum()
    assert keep.sum() > 0 or (name.startswith("syn") and len(t) <= 512)  # random queries past no ratio test


@pytest.mark.parametrize("cap", [1024, 4096])
def test_full_deque_of_large_keyframes(capi, synth, cap):
    """8 keyframes of `cap` ORB points each (n_keyframes 8, the age rule fires every frame) are matched in full:
    8 x cap data points in keyframe and query order, and their gradient / Hessian hold to the restatement."""
    rng = np.random.default_rng(cap)
    ctx, params, _ = rigid._scene(capi, synth, n_features_max=cap, n_keyframes=8, max_keyframe_age=0)
    roi, scale, _ = ctx.get_texture_focus()
    xy = _grid(ctx, cap)
    desc = rng.integers(0, 256, (cap, 32), dtype=np.uint8)
    image_xy = rigid._upload(ctx, 0, _to_crop(xy, roi[0], scale[0]), desc, roi[0], scale[0])
    ctx.start_modalities(0)
    for frame in range(1, 8):
        ctx.calculate_results(frame)
    kf = ctx.get_texture_keyframes(0)
    assert list(kf["sizes"]) == [cap] * 8
    assert np.array_equal(kf["descriptors"], np.tile(desc, (8, 1)))
    ctx.set_poses(rigid._pose((0.5, -0.3, 0.2), (0.001, -0.001, 0.501))[None])
    ctx.texture_correspondences(1, 0)
    got = ctx.get_texture_points(0)
    assert len(got) == 8 * cap
    assert np.array_equal(got["center_f_body"].view(np.uint32), kf["points"].view(np.uint32))
    assert np.array_equal(got["correspondence_center"].view(np.uint32), np.tile(image_xy, (8, 1)).view(np.uint32))
    pose = ctx.get_poses()[0]
    g, H = ctx.texture_gradient_hessian(1, 0, 0)
    eg, eH = tr.gradient_hessian(rigid._b2c(pose), INTR, kf["points"], np.tile(image_xy, (8, 1)),
                                 params.standard_deviations[0], 20.0)
    s = np.abs(eH).max()
    assert np.abs(g[0] - eg).max() <= 1e-5 * s and np.abs(H[0] - eH).max() <= 1e-5 * s


def _large_start(capi, synth, kind, n, cap, rng):
    ctx, params, _ = rigid._scene(capi, synth, descriptor_type=ORB if kind == "orb" else SIFT, n_features_max=cap)
    roi, scale, _ = ctx.get_texture_focus()
    crop, orb = rigid._features(rng, roi[0], scale[0], n)
    desc = orb if kind == "orb" else rng.integers(0, 256, (n, 128)).astype(f32)
    xy = rigid._upload(ctx, 0, crop, desc, roi[0], scale[0])
    ctx.start_modalities(0)
    idx, pts = tr.reconstruct(xy, ctx.get_rendering(0), INTR, tr.pose_inverse(rigid._b2c(ctx.get_poses()[0])), 1)
    kf = ctx.get_texture_keyframes(0)
    assert list(kf["sizes"]) == [len(idx)] and len(idx) > 400
    assert np.array_equal(kf["points"].view(np.uint32), pts.view(np.uint32))
    return ctx, params, pts, desc[idx]


def _large_frame(ctx, rng, kind, true_pose, kf_pts, kf_desc, n_noise=300):
    roi, scale, _ = ctx.get_texture_focus()
    crop = _to_crop(tr.project(rigid._b2c(true_pose), INTR, kf_pts), roi[0], scale[0])
    nc, nd = rigid._features(rng, roi[0], scale[0], n_noise)
    if kind == "orb":
        desc = kf_desc.copy()
        desc[:, ::3] ^= rng.integers(0, 256, desc[:, ::3].shape, dtype=np.uint8) & np.uint8(0x11)
    else:
        desc = np.clip(kf_desc + rng.integers(-3, 4, kf_desc.shape), 0, 255).astype(f32)
        nd = rng.integers(0, 256, (n_noise, 128)).astype(f32)
    crop, desc = np.vstack([crop, nc]).astype(f32), np.vstack([desc, nd])
    return rigid._upload(ctx, 0, crop, desc, roi[0], scale[0]), desc


@pytest.mark.parametrize("kind,n,cap", [("orb", 2000, 2048), ("orb", 4000, 4096), ("sift", 2000, 4096)])
def test_fused_and_fine_grained_tracking_agree(capi, synth, kind, n, cap):
    """Two identical contexts: one tracks with m3tb_tracking_step, the other through the fine-grained calls, whose
    data points equal the restatement bit for bit at correspondence iteration 0; the poses agree."""
    runs = []
    for _ in range(2):
        rng = np.random.default_rng(77)
        ctx, params, kf_pts, kf_desc = _large_start(capi, synth, kind, n, cap, rng)
        true_pose = rigid._pose((1.5, -1.0, 0.8), (0.003, -0.002, 0.504))
        xy, desc = _large_frame(ctx, rng, kind, true_pose, kf_pts, kf_desc)
        runs.append((ctx, params, xy, desc, kf_pts, kf_desc))
    (fused, params, xy, desc, kf_pts, kf_desc), (fine, *_) = runs
    cb, cc = _match([(kf_pts, kf_desc)], xy, desc, params.descriptor_distance_threshold, kind == "orb")
    assert len(cb) > 300 and len(desc) > 512
    before = fused.launch_count
    fused.tracking_step(1, 2, 2)
    assert fused.last_launch()["kernel"] == "k_track"
    pose = fine.get_poses()[0]
    for corr in range(2):
        fine.texture_correspondences(1, corr)
        if corr == 0:
            got = fine.get_texture_points(0)
            assert np.array_equal(got["center_f_body"].view(np.uint32), cb.view(np.uint32))
            assert np.array_equal(got["correspondence_center"].view(np.uint32), cc.view(np.uint32))
        for upd in range(2):
            g, H = fine.texture_gradient_hessian(1, corr, upd)
            fine.calculate_optimization(1, corr, upd)
            pose = tr.optimize(pose, g[0].astype(np.float64), H[0].astype(np.float64))
            assert np.abs(fine.get_poses()[0].reshape(12) - pose.reshape(12)).max() < 1e-4
    assert np.abs(fused.get_poses()[0] - fine.get_poses()[0]).max() < 1e-4
    start = np.abs(np.array([0.0, 0.0, 0.5], f32) - true_pose[:, 3]).max()
    assert np.abs(fused.get_poses()[0].reshape(3, 4)[:, 3] - true_pose[:, 3]).max() < start
    assert fused.launch_count > before


def test_textured_chain_with_large_capacity_links(capi, oracle, synth, monkeypatch):
    """The root and two revolute children with ORB texture modalities at n_features_max 2048 (Hamming kNN), 2000
    features per link: the structure test's fine-grained iteration held to the restatement and the structure oracle,
    and the fused step held to it."""
    monkeypatch.setattr(ts.tr, "match", lambda k, xy, d, thr: _match(k, xy, d, thr, True))
    spec = ts._chain(synth)
    ctxs = []
    for _ in range(2):
        ctx, params = ts._context(capi, synth, ts.CHAIN_POSES, texture=(0, 1, 2), n_features_max=2048)
        ctx.set_structure(0, spec)
        roi, scale, valid = ctx.get_texture_focus()
        for b in range(3):
            rng = np.random.default_rng(300 + b)
            crop, desc = rigid._features(rng, roi[b], scale[b], 2000)
            ctx.upload_texture_features(b, crop, desc, roi[b][0], roi[b][1], scale[b])
        ctx.start_modalities(0)
        kfs = {b: ctx.get_texture_keyframes(b) for b in range(3)}
        roi, scale, _ = ctx.get_texture_focus()
        poses = ctx.get_poses()
        frame = {}
        for b, kf in kfs.items():
            rng = np.random.default_rng(400 + b)
            proj = tr.project(ts._b2c(tr.pose_mul(ts.MOTION, poses[b])), INTR, kf["points"])
            crop = _to_crop(proj, roi[b], scale[b])
            desc = kf["descriptors"].copy()
            desc[:, ::5] ^= np.uint8(0x01)
            nc, nd = rigid._features(rng, roi[b], scale[b], 600)  # distractors: more than 512 train rows
            crop, desc = np.vstack([crop, nc]).astype(f32), np.vstack([desc, nd])
            ctx.upload_texture_features(b, crop, desc, roi[b][0], roi[b][1], scale[b])
            frame[b] = (tr.crop_to_image(crop, roi[b][0], roi[b][1], scale[b]), desc)
        assert all(len(kf["points"]) > 100 and len(frame[b][1]) > 512 for b, kf in kfs.items())
        ctxs.append((ctx, kfs, frame))
    (fine, kfs, frame), (fused, _, _) = ctxs
    matches = {}
    for corr in range(2):
        ts._fine_iteration(fine, oracle, spec, params, corr, kfs, frame, matches)
        before = fused.launch_count
        fused.corr_iteration(1, corr, ts.N_UPDATE)
        assert fused.last_launch()["kernel"] == "k_track"
        # one k_render, k_texture_knn_hamming + k_texture_match at iteration 0 only, then k_track + k_structure per update
        assert fused.launch_count - before == 1 + 2 * (corr == 0) + 2 * ts.N_UPDATE, corr
        assert np.abs(fused.get_poses() - fine.get_poses()).max() < 1e-4, corr


def test_mixed_context_default_body_is_unchanged(capi, synth):
    """Bodies ORB at the default capacity (0), SIFT at 4096 with 3000 features (1) and texture-free (2): body 0's
    keyframes, data points, gradient / Hessian and the poses of bodies 0 and 2 are bit-identical to those of a context
    whose body 1 has no texture modality."""
    runs = []
    for large in (True, False):
        rng = np.random.default_rng(19)
        ctx, params, _ = rigid._scene(capi, synth, n_bodies=3, depth_frame=rigid._plane(), texture_bodies=[])
        ctx.set_poses(np.stack([rigid._pose(t=(0.12 * b - 0.12, 0.0, 0.5)) for b in range(3)]))
        bodies = [(0, "orb", 512)] + ([(1, "sift", 4096)] if large else [])
        for b, kind, cap in bodies:
            p = capi.texture_params_default()
            p.descriptor_type = ORB if kind == "orb" else SIFT
            p.n_features_max = cap
            ctx.set_texture_modality(b, p, 0)
            ctx.attach_renderer(b, "texture_silhouette", b)
        roi, scale, valid = ctx.get_texture_focus()
        crop0, desc0 = rigid._features(rng, roi[0], scale[0], 400)
        ctx.upload_texture_features(0, crop0, desc0, roi[0][0], roi[0][1], scale[0])
        if large:
            crop1, _ = rigid._features(np.random.default_rng(5), roi[1], scale[1], 3000)
            desc1 = np.random.default_rng(6).integers(0, 256, (3000, 128)).astype(f32)
            ctx.upload_texture_features(1, crop1, desc1, roi[1][0], roi[1][1], scale[1])
        ctx.start_modalities(0)
        kf0 = ctx.get_texture_keyframes(0)
        d0 = desc0.copy()
        d0[:, ::4] ^= 1
        ctx.upload_texture_features(0, crop0 + 1.5, d0, roi[0][0], roi[0][1], scale[0])
        if large:
            d1 = np.clip(desc1 + 1, 0, 255).astype(f32)
            ctx.upload_texture_features(1, crop1 + 1.5, d1, roi[1][0], roi[1][1], scale[1])
        ctx.texture_correspondences(1, 0)
        g, H = ctx.texture_gradient_hessian(1, 0, 0)
        gh = (g[0].copy(), H[0].copy())
        poses, points = [], []
        for frame in range(1, 4):
            ctx.tracking_step(frame, 2, 2)
            poses.append(ctx.get_poses()[[0, 2]].copy())
            points.append(ctx.get_texture_points(0).copy())
        if large:
            assert len(ctx.get_texture_points(1)) > 512
        runs.append((kf0, gh, poses, points))
    (kf_a, gh_a, poses_a, points_a), (kf_b, gh_b, poses_b, points_b) = runs
    assert len(points_b[0]) > 20
    assert np.array_equal(kf_a["points"].view(np.uint32), kf_b["points"].view(np.uint32))
    assert np.array_equal(kf_a["descriptors"], kf_b["descriptors"])
    for a, b in zip(gh_a, gh_b):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    for a, b in zip(poses_a, poses_b):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    for a, b in zip(points_a, points_b):
        assert a.tobytes() == b.tobytes()


def test_device_front_end_at_the_capacity(capi, synth):
    """m3tb_upload_texture_features_device takes n = n_features_max (the same keyframe as the host upload) and refuses
    n_features_max + 1 with nothing launched."""
    import torch
    xy, _ = dfe._features("sift", 0)
    rows = Z["sift_desc"][:1024].astype(f32)  # the first 1024 of crop 3's 2339 SIFT descriptors
    xy = np.resize(xy, (1024, 2)).astype(f32) + np.repeat(np.arange(2, dtype=f32), 512)[:, None] * f32(0.5)
    kfs = []
    for device in (True, False):
        ctx = dfe._scene(capi, synth, [0], capi.DESCRIPTOR_SIFT)
        p = capi.texture_params_default()
        p.descriptor_type = SIFT
        p.focused_image_size = int(dfe.FIX["focused_image_size"])
        p.n_features_max = 1024
        ctx.set_texture_modality(0, p, 0)
        out, roi, scale, size, valid = dfe._crop(ctx, [0])
        assert valid[0]
        if device:
            f, keep = dfe._device(capi, xy, rows, "interleaved")
            big, keep2 = dfe._device(capi, np.resize(xy, (1025, 2)), np.resize(rows, (1025, 128)), "interleaved")
            torch.cuda.synchronize()
            before = ctx.launch_count
            with pytest.raises(capi.M3TBError, match="status -3"):
                ctx.upload_texture_features_device([0], [big])
            assert ctx.launch_count == before
            ctx.upload_texture_features_device([0], [f])
            assert ctx.launch_count == before + 1
        else:
            with pytest.raises(capi.M3TBError, match="status -3"):
                ctx.upload_texture_features(0, np.resize(xy, (1025, 2)), np.resize(rows, (1025, 128)), roi[0][0],
                                            roi[0][1], scale[0])
            ctx.upload_texture_features(0, xy, rows, roi[0][0], roi[0][1], scale[0])
        ctx.start_modalities(0)
        kfs.append(ctx.get_texture_keyframes(0))
        ctx.close()
    assert kfs[0]["sizes"][0] > 100 and list(kfs[0]["sizes"]) == list(kfs[1]["sizes"])
    assert np.array_equal(kfs[0]["points"].view(np.uint32), kfs[1]["points"].view(np.uint32))
    assert np.array_equal(kfs[0]["descriptors"], kfs[1]["descriptors"])


def test_refusals(capi, synth):
    ctx, params, _ = rigid._scene(capi, synth)
    for cap, status in ((511, -1), (0, -1), (4097, -3), (8192, -3)):
        p = capi.texture_params_default()
        p.n_features_max = cap
        with pytest.raises(capi.M3TBError, match="status %d" % status):
            ctx.set_texture_modality(0, p, 0)
    assert capi.texture_params_default().n_features_max == 512
    p = capi.texture_params_default()
    p.n_features_max = 600
    ctx.set_texture_modality(0, p, 0)
    ctx.upload_texture_features(0, np.zeros((600, 2), f32), np.zeros((600, 32), np.uint8), 0, 0, 1.0)
    with pytest.raises(capi.M3TBError, match="status -3"):
        ctx.upload_texture_features(0, np.zeros((601, 2), f32), np.zeros((601, 32), np.uint8), 0, 0, 1.0)
    for t in (0, 2, 5):  # BRISK, FREAK and ORB_CUDA stay refused at any capacity
        p.descriptor_type = t
        with pytest.raises(capi.M3TBError, match="status -3"):
            ctx.set_texture_modality(0, p, 0)


def _orb_body_with_keyframe(capi, synth, rng):
    ctx, params, _ = rigid._scene(capi, synth, n_bodies=2, texture_bodies=[0])
    roi, scale, _ = ctx.get_texture_focus()
    crop, desc = rigid._features(rng, roi[0], scale[0], 300)
    ctx.upload_texture_features(0, crop, desc, roi[0][0], roi[0][1], scale[0])
    ctx.start_modalities(0)
    return ctx


@pytest.mark.parametrize("kind", ["orb", "sift"])
def test_failed_growth_leaves_the_context_as_it_was(capi, synth, kind):
    """Fault injection at every allocation of the step that raises the capacity to 4096 (a second body's modality):
    the resources, the first body's keyframes and data points are as they were and the second body has no modality;
    then the same call succeeds and the first body's keyframe survives the growth."""
    p = capi.texture_params_default()
    p.descriptor_type = ORB if kind == "orb" else SIFT
    p.n_features_max = 4096
    ctx = _orb_body_with_keyframe(capi, synth, np.random.default_rng(8))
    kf0 = ctx.get_texture_keyframes(0)
    live0 = capi.debug_resources()
    n_alloc = 5 + (1 if kind == "orb" else 3)  # xy, desc, kf_desc, kf_points, points and the match / float tables
    for fail_at in range(1, n_alloc + 1):
        capi.debug_resources(fail_after=fail_at)
        try:
            with pytest.raises(capi.M3TBError, match="status -2"):
                ctx.set_texture_modality(1, p, 0)
        finally:
            capi.debug_resources(fail_after=0)
        assert capi.debug_resources() == live0, fail_at
        with pytest.raises(capi.M3TBError, match="status -1"):
            ctx.get_texture_points(1)
        kf = ctx.get_texture_keyframes(0)
        assert np.array_equal(kf["points"].view(np.uint32), kf0["points"].view(np.uint32))
    ctx.set_texture_modality(1, p, 0)
    ctx.attach_renderer(1, "texture_silhouette", 1)
    assert capi.debug_resources() == live0 + 1 + (0 if kind == "orb" else 2)  # the new tables replace the old ones
    kf = ctx.get_texture_keyframes(0)
    assert np.array_equal(kf["points"].view(np.uint32), kf0["points"].view(np.uint32))
    assert np.array_equal(kf["descriptors"], kf0["descriptors"])
    ctx.tracking_step(1, 1, 1)
    # the same context grown from the start holds the same data points as one that never grew
    ref = _orb_body_with_keyframe(capi, synth, np.random.default_rng(8))
    ref.tracking_step(1, 1, 1)
    assert ctx.get_texture_points(0).tobytes() == ref.get_texture_points(0).tobytes()


def test_launch_counts(capi, synth):
    """A default context launches what it launched before (k_texture_match alone at iteration 0); an ORB body above
    512 adds one k_texture_knn_hamming launch per frame, at correspondence iteration 0 only."""
    deltas = {}
    for cap in (512, 1024):
        rng = np.random.default_rng(2)
        ctx, params, _ = rigid._scene(capi, synth, n_features_max=cap)
        roi, scale, _ = ctx.get_texture_focus()
        crop, desc = rigid._features(rng, roi[0], scale[0], 300)
        ctx.upload_texture_features(0, crop, desc, roi[0][0], roi[0][1], scale[0])
        ctx.start_modalities(0)
        before = ctx.launch_count
        ctx.tracking_step(1, 2, 2)
        step = ctx.launch_count - before
        before = ctx.launch_count
        ctx.texture_correspondences(1, 0)
        corr0 = ctx.launch_count - before
        before = ctx.launch_count
        ctx.texture_correspondences(1, 1)
        corr1 = ctx.launch_count - before
        deltas[cap] = (step, corr0, corr1, ctx.get_texture_points(0).tobytes())
    assert deltas[512][1:3] == (1, 1)
    assert deltas[1024][0] == deltas[512][0] + 1 and deltas[1024][1:3] == (2, 1)
    assert deltas[512][3] == deltas[1024][3]  # the Hamming kNN matches as the in-CTA scan does


def test_cpp_mirror_tracker_with_2000_features(pkg, tmp_path):
    """examples/texture_mirror_tracker.cpp with 2000 ORB features per body (n_features_max 2000): Tracker::
    ExecuteTrackingStep against the object-wise path."""
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
    r = subprocess.run([exe, "1", "2000", "orb"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    out = json.loads(r.stdout.strip().split("\n")[-1])
    assert out["n_features_max"] == 2000 and min(out["texture_points"]) > 200, out["texture_points"]
    fused, obj, start, gt = (np.array(out[k], np.float32).reshape(-1, 3, 4) for k in ("fused", "object_wise", "start", "gt"))
    dt, dr = pose_error(fused, obj)  # the gates of test_gpu_texture_mirror.py
    assert np.median(dt) < 2e-5 and np.median(dr) < 2e-4, (dt, dr)
    assert dt.max() < 1e-3 and dr.max() < 1e-2, (dt, dr)
    e0t, e0r = pose_error(start, gt)
    e1t, e1r = pose_error(fused, gt)
    assert np.median(e1t) < np.median(e0t) and np.median(e1r) < np.median(e0r), (e0t, e1t, e0r, e1r)
