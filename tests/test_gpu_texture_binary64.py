"""BRISK and FREAK texture modalities on the device (64-byte NORM_HAMMING rows in the wide tables, matched by
k_texture_knn_hamming): the cv2.BFMatcher(NORM_HAMMING) fixtures through the C ABI, fine-grained and fused tracking
against the vectorised restatement (tests/texture_reference_binary64.py) at n_features_max 512, 2048 and 4096 with host
and device uploads, a textured chain with BRISK links against the restatement and the structure oracle, a mixed context
whose ORB, SIFT, DAISY and texture-free bodies are bit-identical to a context without the BRISK / FREAK bodies, the
refusals, the all-or-nothing wide tables, and the C++ mirror's BRISK tracker."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import test_gpu_texture as rigid
import test_gpu_texture_device_front_end as front
import test_gpu_texture_l2 as l2
import test_gpu_texture_structures as ts
import texture_reference as tr
import texture_reference_binary64 as tb
from helpers import pose_error

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "texture_knn_binary64.npz")
BRISK, FREAK, ORB, SIFT, DAISY = 0, 2, 4, 3, 1
KIND = {"brisk": BRISK, "freak": FREAK}
INTR = rigid.INTR
# words that read as float NaN, inf and denormals: binary rows holding them are copied, never checked
FLOAT_WORDS = np.array([0xFFFFFFFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0x00000001, 0x007FFFFF], np.uint32)


def _descriptors(rng, n, patterns=False):
    d = rng.integers(0, 256, (n, 64), dtype=np.uint8)
    if patterns:  # every third row made of NaN / inf / denormal words
        d[::3] = FLOAT_WORDS[rng.integers(0, len(FLOAT_WORDS), (len(d[::3]), 16))].view(np.uint8).reshape(-1, 64)
    return d


def _perturbed(rng, d, bits=10):
    d = d.copy()
    rows = np.repeat(np.arange(len(d)), bits)
    cols = rng.integers(0, d.shape[1], len(rows))
    np.bitwise_xor.at(d, (rows, cols), (1 << rng.integers(0, 8, len(rows))).astype(np.uint8))
    return d


class Uploader:
    """Host uploads, or device uploads (m3tb_texture_crop of a fresh colour frame, then descriptors from device memory
    in rows 72 bytes apart), of one body's crop-coordinate features."""

    def __init__(self, capi, ctx, device):
        self.capi, self.ctx, self.device, self.keep = capi, ctx, device, []
        if device:
            import torch
            self.torch = torch
            self.out = torch.zeros(512 * 512, dtype=torch.uint8, device="cuda")
            self.frame = np.full((INTR["height"], INTR["width"], 3), 90, np.uint8)

    def __call__(self, b, crop, desc, roi, scale):
        if not self.device:
            self.ctx.upload_texture_features(b, crop, desc, roi[0], roi[1], scale)
        else:
            self.ctx.upload_color(0, self.frame)
            croi, cscale, _, valid = self.ctx.texture_crop([b], self.out.data_ptr(), 512, 512 * 512, 512, 512)
            assert valid[0] and tuple(croi[0]) == tuple(roi) and cscale[0] == np.float32(scale)
            f, bufs = front._device(self.capi, crop, desc, "interleaved")
            assert f.descriptor_pitch == 72 and f.length == 0
            self.ctx.upload_texture_features_device([b], [f])
            self.keep.append(bufs)
            self.ctx.synchronize()
            assert not self.ctx.get_texture_feature_flags().any()
        return tr.crop_to_image(crop, roi[0], roi[1], scale)


def _start(capi, synth, rng, kind, n_feat, device, **texture):
    ctx, params, _ = rigid._scene(capi, synth, descriptor_type=KIND[kind], **texture)
    upload = Uploader(capi, ctx, device)
    roi, scale, valid = ctx.get_texture_focus()
    assert valid[0]
    crop, _ = rigid._features(rng, roi[0], scale[0], n_feat)
    desc = _descriptors(rng, n_feat, patterns=True)
    xy = upload(0, crop, desc, roi[0], scale[0])
    ctx.start_modalities(0)
    idx, pts = tr.reconstruct(xy, ctx.get_rendering(0), INTR, tr.pose_inverse(rigid._b2c(ctx.get_poses()[0])), 1)
    kf = ctx.get_texture_keyframes(0)
    assert list(kf["sizes"]) == [len(idx)] and len(idx) > 20
    assert np.array_equal(kf["points"].view(np.uint32), pts.view(np.uint32))
    assert kf["descriptors"].dtype == np.uint8 and np.array_equal(kf["descriptors"], desc[idx])
    return ctx, params, upload, pts, desc[idx]


def _next_frame(ctx, upload, rng, true_pose, kf_pts, kf_desc, n_noise):
    roi, scale, _ = ctx.get_texture_focus()
    proj = tr.project(rigid._b2c(true_pose), INTR, kf_pts)
    crop = ((proj - roi[0][:2].astype(np.float32)) * scale[0]).astype(np.float32)
    nc, _ = rigid._features(rng, roi[0], scale[0], n_noise)
    crop = np.vstack([crop, nc]).astype(np.float32)
    desc = np.vstack([_perturbed(rng, kf_desc), _descriptors(rng, n_noise, patterns=True)])
    return upload(0, crop, desc, roi[0], scale[0]), desc


# ---- the OpenCV fixtures through the C ABI ----------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["brisk", "brisk_large", "orb_brisk", "ties", "zero_zero", "equal_distance",
                                  "train_of_one", "empty_train", "float_patterns"])
@pytest.mark.parametrize("kind", ["brisk", "freak"])
def test_opencv_fixtures_through_the_c_abi(capi, synth, name, kind):
    """Queries become keyframe points (all inside the silhouette, at distinct places), the train set the next frame's
    features at distinct coordinates, so each data point names its query and the train index it matched."""
    z = np.load(GOLDEN)
    q, t, ref_idx, ref_dist = (z[name + k] for k in ("_queries", "_train", "_idx", "_dist"))
    cap = 512 if max(len(q), len(t)) <= 512 else 4096
    ctx, params, _ = rigid._scene(capi, synth, descriptor_type=KIND[kind], n_features_max=cap)
    roi, scale, _ = ctx.get_texture_focus()
    center = tr.project(rigid._b2c(ctx.get_poses()[0]), INTR, np.zeros((1, 3), np.float32))[0]
    rng = np.random.default_rng(31)
    qxy = (center + rng.uniform(-8.0, 8.0, (len(q), 2))).astype(np.float32)
    qcrop = ((qxy - roi[0][:2].astype(np.float32)) * scale[0]).astype(np.float32)
    rigid._upload(ctx, 0, qcrop, q, roi[0], scale[0])
    ctx.start_modalities(0)
    kf = ctx.get_texture_keyframes(0)
    assert list(kf["sizes"]) == [len(q)] and np.array_equal(kf["descriptors"], q)
    kf_rows = {p.tobytes(): i for i, p in enumerate(kf["points"])}
    assert len(kf_rows) == len(q)
    tcrop = np.stack([np.arange(len(t), dtype=np.float32) * 0.25, np.full(len(t), 3.0, np.float32)], 1)
    txy = rigid._upload(ctx, 0, tcrop, t, roi[0], scale[0])
    t_rows = {p.tobytes(): j for j, p in enumerate(txy)}
    assert len(t_rows) == len(t)
    before = ctx.launch_count
    ctx.texture_correspondences(1, 0)
    assert ctx.launch_count - before == 2  # k_texture_knn_hamming + k_texture_match
    got = ctx.get_texture_points(0)
    device = np.full(len(q), -1)
    for p in got:
        device[kf_rows[p["center_f_body"].tobytes()]] = t_rows[p["correspondence_center"].tobytes()]
    keep = tb.kept(ref_idx, ref_dist, params.descriptor_distance_threshold)
    assert np.array_equal(device, np.where(keep, ref_idx[:, 0], -1))
    order = [kf_rows[p["center_f_body"].tobytes()] for p in got]
    assert order == sorted(order)  # data points keep query order


# ---- tracking against the restatement ---------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,cap,device", [("brisk", 4096, False), ("freak", 512, True), ("brisk", 2048, True)])
def test_fine_grained_iterations_match_the_restatement(capi, synth, kind, cap, device):
    rng = np.random.default_rng(5)
    n_feat = cap * 3 // 4
    ctx, params, upload, kf_pts, kf_desc = _start(capi, synth, rng, kind, n_feat, device, n_features_max=cap)
    true_pose = rigid._pose((2.0, -1.5, 1.0), (0.004, -0.003, 0.505))
    xy, desc = _next_frame(ctx, upload, rng, true_pose, kf_pts, kf_desc, n_feat // 4)
    cb, cc = tb.match([(kf_pts, kf_desc)], xy, desc, params.descriptor_distance_threshold)
    assert len(cb) > 20
    pose = ctx.get_poses()[0]
    for corr in range(2):
        ctx.texture_correspondences(1, corr)
        got = ctx.get_texture_points(0)
        assert np.array_equal(got["center_f_body"].view(np.uint32), cb.view(np.uint32))
        assert np.array_equal(got["correspondence_center"].view(np.uint32), cc.view(np.uint32))
        for upd in range(2):
            g, H = ctx.texture_gradient_hessian(1, corr, upd)
            eg, eH = tr.gradient_hessian(rigid._b2c(pose), INTR, cb, cc, params.standard_deviations[min(corr, 1)], 20.0)
            scale = np.abs(eH).max()
            assert np.abs(g[0] - eg).max() <= 1e-5 * scale and np.abs(H[0] - eH).max() <= 1e-5 * scale
            ctx.calculate_optimization(1, corr, upd)
            pose = tr.optimize(pose, g[0].astype(np.float64), H[0].astype(np.float64))
            assert np.abs(ctx.get_poses()[0].reshape(12) - pose.reshape(12)).max() < 1e-4


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("cap", [512, 2048, 4096])
@pytest.mark.parametrize("kind", ["brisk", "freak"])
def test_fused_step_and_keyframe_refresh(capi, synth, kind, cap, device):
    """tracking_step against the restatement, the keyframe deque (4 entries) refreshed every frame and matched
    keyframe by keyframe."""
    rng = np.random.default_rng(11 + cap)
    n_feat = cap * 3 // 4
    ctx, params, upload, kf_pts, kf_desc = _start(capi, synth, rng, kind, n_feat, device, n_features_max=cap,
                                                  n_keyframes=4, max_keyframe_age=0)
    keyframes = [(kf_pts, kf_desc)]
    pose = ctx.get_poses()[0]
    for frame in range(1, 4):
        true_pose = rigid._pose((1.0 * frame, 0.5, -0.5 * frame), (0.002 * frame, 0.001, 0.5 + 0.002 * frame))
        kp, kd = keyframes[-1]
        xy, desc = _next_frame(ctx, upload, rng, true_pose, kp, kd, min(cap - len(kp), n_feat // 4))
        cb, cc = tb.match(keyframes, xy, desc, params.descriptor_distance_threshold)
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
        keyframes = keyframes[-4:]
        assert len(kf["sizes"]) == min(frame + 1, 4)
        pose = ctx.get_poses()[0].reshape(3, 4)
    if device:
        assert not ctx.get_texture_feature_flags().any()


def test_textured_chain_with_brisk_links(capi, oracle, synth, monkeypatch):
    """The root and two revolute children with BRISK texture modalities: the structure test's fine-grained iteration
    (restatement + structure oracle at every update) with the 64-byte matcher, and the fused step held to it."""
    monkeypatch.setattr(ts.tr, "match", tb.match)  # the structure helpers' matcher is the 64-byte one here
    spec = ts._chain(synth)
    ctxs = []
    for _ in range(2):
        ctx, params = ts._context(capi, synth, ts.CHAIN_POSES, texture=(0, 1, 2), descriptor_type=BRISK)
        ctx.set_structure(0, spec)
        roi, scale, valid = ctx.get_texture_focus()
        for b in range(3):
            rng = np.random.default_rng(100 + b)
            x, y, w, h = roi[b]
            pts = np.stack([rng.uniform(x, x + w, 200), rng.uniform(y, y + h, 200)], 1).astype(np.float32)
            crop = ((pts - np.array([x, y], np.float32)) * np.float32(scale[b])).astype(np.float32)
            ctx.upload_texture_features(b, crop, _descriptors(rng, 200), x, y, scale[b])
        ctx.start_modalities(0)
        kfs = {b: ctx.get_texture_keyframes(b) for b in range(3)}
        roi, scale, _ = ctx.get_texture_focus()
        poses = ctx.get_poses()
        frame = {}
        for b, kf in kfs.items():
            rng = np.random.default_rng(200 + b)
            proj = tr.project(ts._b2c(tr.pose_mul(ts.MOTION, poses[b])), INTR, kf["points"])
            crop = ((proj - roi[b][:2].astype(np.float32)) * scale[b]).astype(np.float32)
            desc = _perturbed(rng, kf["descriptors"])
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
        # one k_render, k_texture_knn_hamming + k_texture_match at iteration 0 only, then k_track + k_structure
        assert fused.launch_count - before == 1 + 2 * (corr == 0) + 2 * ts.N_UPDATE, corr
        assert np.abs(fused.get_poses() - fine.get_poses()).max() < 1e-4, corr


# ---- a mixed context --------------------------------------------------------------------------------------------------
MIXED = [("orb", 512), ("orb", 4096), ("sift", 512), ("daisy", 512), ("brisk", 2048), ("freak", 512), (None, 0)]


def _mixed_run(capi, synth, with_binary64):
    rng = np.random.default_rng(14)
    n = len(MIXED)
    ctx, params, _ = rigid._scene(capi, synth, n_bodies=n, depth_frame=rigid._plane(), texture_bodies=[])
    ctx.set_poses(np.stack([rigid._pose(t=(0.06 * b - 0.18, 0.0, 0.5)) for b in range(n)]))
    bodies = [b for b, (kind, _) in enumerate(MIXED) if kind and (with_binary64 or kind not in KIND)]
    for b in bodies:
        kind, cap = MIXED[b]
        p = capi.texture_params_default()
        p.descriptor_type = {"orb": ORB, "sift": SIFT, "daisy": DAISY, **KIND}[kind]
        p.n_features_max = cap
        ctx.set_texture_modality(b, p, 0)
        ctx.attach_renderer(b, "texture_silhouette", b)
    roi, scale, valid = ctx.get_texture_focus()
    feats = {}
    for b in bodies:
        kind, cap = MIXED[b]
        assert valid[b]
        crop, orb = rigid._features(rng, roi[b], scale[b], min(cap, 600))
        desc = orb if kind == "orb" else _descriptors(rng, len(crop)) if kind in KIND else l2._descriptors(rng, kind,
                                                                                                          len(crop))
        ctx.upload_texture_features(b, crop, desc, roi[b][0], roi[b][1], scale[b])
        feats[b] = (crop, desc, kind)
    ctx.start_modalities(0)
    for b, (crop, desc, kind) in feats.items():
        desc = _perturbed(rng, desc, 4) if desc.dtype == np.uint8 else l2._perturbed(rng, kind, desc)
        ctx.upload_texture_features(b, crop + 1.5, desc, roi[b][0], roi[b][1], scale[b])
    before = ctx.launch_count
    ctx.texture_correspondences(0, 0)
    launches = ctx.launch_count - before
    run = dict(launches=launches, poses=[], points=[], keyframes=[])
    for frame in range(1, 4):
        ctx.tracking_step(frame, 2, 2)
        run["poses"].append(ctx.get_poses().copy())
        run["points"].append({b: ctx.get_texture_points(b).tobytes() for b in bodies})
    ctx.calculate_results(4)
    run["keyframes"] = {b: ctx.get_texture_keyframes(b) for b in bodies}
    return run


def test_mixed_context_other_bodies_are_unchanged(capi, synth):
    """ORB (512 and 4096), SIFT, DAISY, BRISK, FREAK and texture-free bodies: every body but BRISK and FREAK has the
    data points, poses and keyframes it has in a context whose BRISK and FREAK bodies have no texture modality, and
    one k_texture_knn_hamming launch matches the ORB-4096, BRISK and FREAK bodies together."""
    with_b, without = _mixed_run(capi, synth, True), _mixed_run(capi, synth, False)
    # k_texture_knn_l2, k_texture_knn_hamming (one launch for every binary kNN body) and k_texture_match
    assert with_b["launches"] == without["launches"] == 3
    others = [b for b, (kind, _) in enumerate(MIXED) if kind not in KIND]
    for a, b in zip(with_b["poses"], without["poses"]):
        assert np.array_equal(a[others].view(np.uint32), b[others].view(np.uint32))
    for a, b in zip(with_b["points"], without["points"]):
        assert all(a[k] == b[k] for k in b)
    assert all(len(with_b["points"][-1][b]) > 20 for b in with_b["points"][-1])
    for k, kf in without["keyframes"].items():
        got = with_b["keyframes"][k]
        assert list(got["sizes"]) == list(kf["sizes"]) and got["points"].tobytes() == kf["points"].tobytes()
        assert got["descriptors"].tobytes() == kf["descriptors"].tobytes()
    assert with_b["keyframes"][4]["descriptors"].shape[1] == 64


# ---- refusals and resources -------------------------------------------------------------------------------------------
def _state(ctx):
    kf = ctx.get_texture_keyframes(0)
    return (kf["points"].tobytes(), kf["descriptors"].tobytes(), ctx.get_texture_points(0).tobytes(),
            ctx.get_poses().tobytes())


def test_refusals_leave_the_context_unchanged(capi, synth):
    """Each refusal leaves the BRISK body's keyframes, data points and pose as they were."""
    rng = np.random.default_rng(8)
    ctx, params, upload, kf_pts, kf_desc = _start(capi, synth, rng, "brisk", 300, False)
    roi, scale, _ = ctx.get_texture_focus()
    ctx.upload_texture_features(0, *rigid._features(rng, roi[0], scale[0], 100)[:1], _descriptors(rng, 100),
                                roi[0][0], roi[0][1], scale[0])
    ctx.texture_correspondences(1, 0)
    state = _state(ctx)
    xy = np.zeros((4, 2), np.float32)
    fp = C.POINTER(C.c_float)
    with pytest.raises(capi.M3TBError, match="status -1"):  # a float upload to a BRISK body
        ctx.upload_texture_features(0, xy, np.zeros((4, 128), np.float32), 0, 0, 1.0)
    assert ctx.L.m3tb_upload_texture_float_features(ctx.h, 0, xy.ctypes.data_as(fp),
                                                    np.zeros((4, 16), np.float32).ctypes.data_as(fp), 4, 16, 0, 0,
                                                    C.c_float(1.0)) == -1
    with pytest.raises(ValueError):  # the binding checks the width
        ctx.upload_texture_features(0, xy, np.zeros((4, 32), np.uint8), 0, 0, 1.0)
    with pytest.raises(capi.M3TBError, match="status -3"):  # more features than n_features_max
        ctx.upload_texture_features(0, np.zeros((513, 2), np.float32), np.zeros((513, 64), np.uint8), 0, 0, 1.0)
    import torch
    out = torch.zeros(512 * 512, dtype=torch.uint8, device="cuda")
    ctx.upload_color(0, np.full((INTR["height"], INTR["width"], 3), 90, np.uint8))
    ctx.texture_crop([0], out.data_ptr(), 512, 512 * 512, 512, 512)
    f, bufs = front._device(capi, xy, np.zeros((4, 64), np.uint8), "interleaved")
    for length, pitch in ((16, 72), (64, 72), (0, 63)):  # a nonzero device length, a pitch below 64 bytes
        g = capi.DeviceFeatures(4, length, f.x, f.y, f.xy_stride, f.descriptors, pitch)
        with pytest.raises(capi.M3TBError, match="status -1"):
            ctx.upload_texture_features_device([0], [g])
    with pytest.raises(capi.M3TBError, match="status -1"):  # detection is cv::ORB
        ctx.texture_detect_orb([0])
    with pytest.raises(capi.M3TBError, match="status -3"):  # no device detector between iterations
        ctx.refine_poses_orb([0], n_corr_iterations=1, n_update_iterations=1)
    p = capi.texture_params_default()
    # ORB_CUDA; and ORB, SIFT, DAISY in place of the BRISK modality: the binary upload and the keyframe read-back take
    # no width, so the body changes across the 64-byte width only through the removal of its modality
    for t in (5, ORB, SIFT, DAISY):
        p.descriptor_type = t
        with pytest.raises(capi.M3TBError, match="status -3"):
            ctx.set_texture_modality(0, p, 0)
    assert ctx.get_texture_keyframes(0)["descriptors"].shape[1] == 64
    ctx.upload_texture_features(0, *rigid._features(rng, roi[0], scale[0], 100)[:1], _descriptors(rng, 100),
                                roi[0][0], roi[0][1], scale[0])  # the frame changed: features again
    assert _state(ctx)[:2] == state[:2] and _state(ctx)[3] == state[3]
    del bufs
    p.descriptor_type = FREAK  # the same width: in place
    ctx.set_texture_modality(0, p, 0)
    assert len(ctx.get_texture_keyframes(0)["sizes"]) == 0
    p.descriptor_type = ORB
    ctx.set_texture_modality(0, None, 0)  # removed first: any type
    ctx.set_texture_modality(0, p, 0)
    ctx.attach_renderer(0, "texture_silhouette", 0)
    ctx.upload_texture_features(0, np.zeros((4, 2), np.float32), np.zeros((4, 32), np.uint8), 0, 0, 1.0)
    p.descriptor_type = BRISK
    with pytest.raises(capi.M3TBError, match="status -3"):  # and back: the ORB modality stays
        ctx.set_texture_modality(0, p, 0)
    ctx.upload_texture_features(0, np.zeros((4, 2), np.float32), np.zeros((4, 32), np.uint8), 0, 0, 1.0)


@pytest.mark.parametrize("fail_at", [1, 2, 3, 4])
def test_failed_wide_table_allocation_leaves_the_context_as_it_was(capi, synth, fail_at):
    """Fault injection on the first BRISK modality: of a context without texture tables (fail_at 1 .. 3 the wide and
    match tables, 4 the first base table) and of one whose ORB body made the base tables."""
    for orb_first in (False, True):
        ctx, params, _ = rigid._scene(capi, synth, n_bodies=2, texture_bodies=[0] if orb_first else [])
        live0 = capi.debug_resources()
        p = capi.texture_params_default()
        p.descriptor_type = BRISK
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


def test_cpp_mirror_brisk_tracker(pkg, tmp_path):
    """examples/texture_mirror_tracker.cpp in its BRISK mode: Tracker::ExecuteTrackingStep against the object-wise
    path."""
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
    r = subprocess.run([exe, "1", "300", "brisk"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    out = json.loads(r.stdout.strip().split("\n")[-1])
    assert out["descriptor"] == "brisk" and min(out["texture_points"]) > 20, out["texture_points"]
    fused, obj, start, gt = (np.array(out[k], np.float32).reshape(-1, 3, 4) for k in ("fused", "object_wise", "start", "gt"))
    dt, dr = pose_error(fused, obj)  # the gates of test_gpu_texture_mirror.py
    assert np.median(dt) < 2e-5 and np.median(dr) < 2e-4, (dt, dr)
    assert dt.max() < 1e-3 and dr.max() < 1e-2, (dt, dr)
    e0t, e0r = pose_error(start, gt)
    e1t, e1r = pose_error(fused, gt)
    assert np.median(e1t) < np.median(e0t) and np.median(e1r) < np.median(e0r), (e0t, e1t, e0r, e1r)
