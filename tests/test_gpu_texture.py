"""Texture modality on the device (m3tb_set_texture_modality ... k_texture_keyframe / k_texture_match / the texture term
of k_track) against the CPU restatement in tests/texture_reference.py, on seeded synthetic ORB-like features: keyframe
points and data points bit for bit, gradients / Hessians within 1e-5 of max|H|, poses of the fine-grained and the fused
path within 1e-4 at every iteration, the stale-pose keyframe refresh of CalculateResults, and the refusals."""
import numpy as np
import pytest

import texture_reference as tr

pytestmark = pytest.mark.gpu

W2C = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
INTR = dict(fu=614.0, fv=614.5, ppu=321.3, ppv=238.9, width=640, height=480)


def _pose(rot_deg=(0.0, 0.0, 0.0), t=(0.0, 0.0, 0.5)):
    R = np.eye(3)
    for axis, deg in enumerate(rot_deg):
        c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
        i, j = [k for k in range(3) if k != axis]
        Q = np.eye(3)
        Q[i, i], Q[i, j], Q[j, i], Q[j, j] = c, -s, s, c
        R = R @ Q
    return np.hstack([R, np.array(t)[:, None]]).astype(np.float32)


def _scene(capi, synth, n_bodies=1, region=False, depth_frame=None, color_frame=None, texture_bodies=None, **texture):
    """Depth (+ region) + texture bodies on the synthetic prism, one silhouette renderer per body. The default depth
    frame is empty (the depth modality finds no correspondence, so the texture term alone moves the pose).
    texture_bodies: the bodies that get a texture modality (default all)."""
    intr = synth.default_color_intrinsics()
    ctx = capi.Context(0, max_bodies=n_bodies + 1, max_cameras=1, max_models=1)
    ctx.set_color_camera(0, intr, W2C)
    ctx.set_depth_camera(0, intr, W2C, 0.001)
    ctx.upload_depth(0, np.zeros((intr.height, intr.width), np.uint16) if depth_frame is None else depth_frame)
    if region:
        ctx.upload_color(0, np.full((intr.height, intr.width, 3), 40, np.uint8) if color_frame is None else color_frame)
    tri, diam = synth.prism_triangles()
    op = capi.OptimizerParams(1000.0, 30000.0)
    for b in range(n_bodies):
        ctx.set_body_geometry(b, tri, W2C, diam, True, body_id=b + 1, region_id=b + 1)
    mp = capi.model_params(n_divides=1, n_points=40, image_size=200)
    ctx.generate_depth_model(0, 0, params=mp)
    if region:
        ctx.generate_region_model(0, 0, params=mp)
    params = capi.texture_params_default()
    for k, v in texture.items():
        setattr(params, k, v)
    for b in range(n_bodies):
        ctx.set_body(b, capi.region_params() if region else None, capi.depth_params(), op, region_model=0,
                     depth_model=0, color_camera=0, depth_camera=0)
    ctx.set_poses(np.stack([_pose(t=(0.03 * b, 0.0, 0.5)) for b in range(n_bodies)]))
    for b in range(n_bodies):
        ctx.set_focused_renderer(b, "color", 0, list(range(n_bodies)), [b], 200, id_type="body")
        if texture_bodies is None or b in texture_bodies:
            ctx.set_texture_modality(b, params, 0)
            ctx.attach_renderer(b, "texture_silhouette", b)
    return ctx, params, diam


def _features(rng, roi, scale, n):
    """n keypoints inside the focus region (crop coordinates) with random descriptors."""
    x, y, w, h = roi
    xy = np.stack([rng.uniform(x, x + w, n), rng.uniform(y, y + h, n)], 1).astype(np.float32)
    crop = ((xy - np.array([x, y], np.float32)) * np.float32(scale)).astype(np.float32)
    return crop, rng.integers(0, 256, (n, 32), dtype=np.uint8)


def _upload(ctx, b, crop, desc, roi, scale):
    ctx.upload_texture_features(b, crop, desc, roi[0], roi[1], scale)
    return tr.crop_to_image(crop, roi[0], roi[1], scale)


def _b2c(pose):
    return tr.pose_mul(W2C, pose)


def _start(capi, synth, rng, n_feat=200, **texture):
    ctx, params, diam = _scene(capi, synth, **texture)
    roi, scale, valid = ctx.get_texture_focus()
    assert valid[0]
    exp = tr.focus(INTR, _b2c(ctx.get_poses()[0]), np.float32(0.5) * np.float32(diam), params.focused_image_size)
    assert tuple(roi[0]) == exp[0] and np.float32(scale[0]) == exp[1]
    crop, desc = _features(rng, roi[0], scale[0], n_feat)
    xy = _upload(ctx, 0, crop, desc, roi[0], scale[0])
    ctx.start_modalities(0)
    rend = ctx.get_rendering(0)
    idx, pts = tr.reconstruct(xy, rend, INTR, tr.pose_inverse(_b2c(ctx.get_poses()[0])), 1)
    kf = ctx.get_texture_keyframes(0)
    assert list(kf["sizes"]) == [len(idx)] and len(idx) > 20
    assert np.array_equal(kf["points"].view(np.uint32), pts.view(np.uint32))
    assert np.array_equal(kf["descriptors"], desc[idx])
    return ctx, params, pts, desc[idx]


def _next_frame(ctx, rng, true_pose, kf_pts, kf_desc, n_noise=40, flips=12):
    """Features of the next frame: the keyframe points seen at `true_pose` with a few descriptor bits flipped, plus
    random distractors."""
    roi, scale, _ = ctx.get_texture_focus()
    proj = tr.project(_b2c(true_pose), INTR, kf_pts)
    crop = ((proj - roi[0][:2].astype(np.float32)) * scale[0]).astype(np.float32)
    desc = kf_desc.copy()
    for r in range(len(desc)):
        for bit in rng.choice(256, flips, replace=False):
            desc[r, bit // 8] ^= np.uint8(1 << (bit % 8))
    nc, nd = _features(rng, roi[0], scale[0], n_noise)
    crop, desc = np.vstack([crop, nc]), np.vstack([desc, nd])
    return _upload(ctx, 0, crop, desc, roi[0], scale[0]), desc


def test_fine_grained_iterations_match_the_restatement(capi, synth):
    rng = np.random.default_rng(5)
    ctx, params, kf_pts, kf_desc = _start(capi, synth, rng)
    true_pose = _pose((2.0, -1.5, 1.0), (0.004, -0.003, 0.505))
    xy, desc = _next_frame(ctx, rng, true_pose, kf_pts, kf_desc)
    cb, cc = tr.match([(kf_pts, kf_desc)], xy, desc, params.descriptor_distance_threshold)
    assert len(cb) > 20
    pose = ctx.get_poses()[0]
    for corr in range(2):
        ctx.texture_correspondences(1, corr)
        got = ctx.get_texture_points(0)
        assert np.array_equal(got["center_f_body"].view(np.uint32), cb.view(np.uint32))
        assert np.array_equal(got["correspondence_center"].view(np.uint32), cc.view(np.uint32))
        assert np.array_equal(got["center"].view(np.uint32), tr.project(_b2c(ctx.get_poses()[0]), INTR, cb).view(np.uint32))
        for upd in range(2):
            g, H = ctx.texture_gradient_hessian(1, corr, upd)
            eg, eH = tr.gradient_hessian(_b2c(pose), INTR, cb, cc, params.standard_deviations[min(corr, 1)], 20.0)
            scale = np.abs(eH).max()
            assert np.abs(g[0] - eg).max() <= 1e-5 * scale and np.abs(H[0] - eH).max() <= 1e-5 * scale
            ctx.calculate_optimization(1, corr, upd)
            pose = tr.optimize(pose, g[0].astype(np.float64), H[0].astype(np.float64))
            assert np.abs(ctx.get_poses()[0].reshape(12) - pose.reshape(12)).max() < 1e-4
    # the pose moved towards the one the features were seen at
    start = np.abs(np.array([0.0, 0.0, 0.5], np.float32) - true_pose[:, 3]).max()
    assert np.abs(ctx.get_poses()[0].reshape(3, 4)[:, 3] - true_pose[:, 3]).max() < start


@pytest.mark.parametrize("n_keyframes", [1, 3])
def test_fused_step_and_keyframe_refresh(capi, synth, n_keyframes):
    """tracking_step against the restatement iteration by iteration; CalculateResults refreshes the keyframe (age rule)
    with the pose of the last gradient pass while the silhouette renderer draws the final pose."""
    rng = np.random.default_rng(11 + n_keyframes)
    ctx, params, kf_pts, kf_desc = _start(capi, synth, rng, n_keyframes=n_keyframes, max_keyframe_age=0)
    keyframes = [(kf_pts, kf_desc)]
    pose = ctx.get_poses()[0]
    for frame in range(1, 4):
        true_pose = _pose((1.0 * frame, 0.5, -0.5 * frame), (0.002 * frame, 0.001, 0.5 + 0.002 * frame))
        xy, desc = _next_frame(ctx, rng, true_pose, *keyframes[-1])
        cb, cc = tr.match(keyframes, xy, desc, params.descriptor_distance_threshold)
        ctx.tracking_step(frame, 2, 2)
        assert ctx.last_launch()["kernel"] == "k_track"
        stale = pose
        for corr in range(2):
            for upd in range(2):
                g, H = tr.gradient_hessian(_b2c(pose), INTR, cb, cc, params.standard_deviations[min(corr, 1)], 20.0)
                stale = pose
                pose = tr.optimize(pose, g, H)
        assert np.abs(ctx.get_poses()[0].reshape(12) - pose.reshape(12)).max() < 1e-4, frame
        got = ctx.get_texture_points(0)
        assert np.array_equal(got["center_f_body"].view(np.uint32), cb.view(np.uint32))
        ctx.calculate_results(frame)
        rend = ctx.get_rendering(0)  # drawn at the final pose
        kf = ctx.get_texture_keyframes(0)
        assert kf["age"] == 0
        # reconstructed with camera2body of the pose before the final update (within the pose gate: the device's stale
        # pose is its own iterate, not the restatement's)
        idx, pts = tr.reconstruct(xy, rend, INTR, tr.pose_inverse(_b2c(stale)), 1)
        new = kf["points"][-kf["sizes"][-1]:]
        assert len(new) == len(idx)
        assert np.abs(new - pts).max() < 1e-3
        keyframes.append((new.copy(), desc[idx]))
        keyframes = keyframes[-n_keyframes:]
        assert len(kf["sizes"]) == min(frame + 1, n_keyframes)
        pose = ctx.get_poses()[0].reshape(3, 4)


def test_stale_pose_rotation_rule_and_zero_features(capi, synth):
    """No refresh under the default rules after a small motion; a frame without features leaves no data points and
    does not move the pose."""
    rng = np.random.default_rng(3)
    ctx, params, kf_pts, kf_desc = _start(capi, synth, rng)
    ctx.upload_texture_features(0, np.zeros((0, 2), np.float32), np.zeros((0, 32), np.uint8), 0, 0, 1.0)
    before = ctx.get_poses()[0].reshape(12).copy()
    ctx.tracking_step(1, 2, 2)
    assert len(ctx.get_texture_points(0)) == 0
    assert np.abs(ctx.get_poses()[0].reshape(12) - before).max() < 1e-6
    ctx.calculate_results(1)
    kf = ctx.get_texture_keyframes(0)
    assert kf["age"] == 1 and list(kf["sizes"]) == [len(kf_pts)]
    fires, age = tr.keyframe_fires(_b2c(before), kf["orientation"], 0, params.max_keyframe_rotation_difference,
                                   params.max_keyframe_age)
    assert not fires and age == 1


def test_invisible_body_keeps_no_keyframe(capi, synth):
    rng = np.random.default_rng(4)
    ctx, params, _ = _scene(capi, synth)
    roi, scale, _ = ctx.get_texture_focus()
    crop, desc = _features(rng, roi[0], scale[0], 50)
    ctx.upload_texture_features(0, crop, desc, roi[0][0], roi[0][1], scale[0])
    ctx.set_poses(_pose(t=(0.0, 0.0, -0.5))[None])  # behind the camera
    roi2, _, valid = ctx.get_texture_focus()
    assert not valid[0] and not roi2.any()
    ctx.start_modalities(0)
    assert len(ctx.get_texture_keyframes(0)["sizes"]) == 0


def test_refusals(capi, synth):
    ctx, params, _ = _scene(capi, synth)
    p = capi.texture_params_default()
    p.descriptor_type = 0  # BRISK
    with pytest.raises(capi.M3TBError, match="status -3"):
        ctx.set_texture_modality(0, p, 0)
    p = capi.texture_params_default()
    p.n_keyframes = 9
    with pytest.raises(capi.M3TBError, match="status -3"):
        ctx.set_texture_modality(0, p, 0)
    with pytest.raises(capi.M3TBError, match="status -1"):
        ctx.set_texture_modality(0, capi.texture_params_default(), 5)
    with pytest.raises(capi.M3TBError, match="status -3"):
        ctx.upload_texture_features(0, np.zeros((513, 2), np.float32), np.zeros((513, 32), np.uint8), 0, 0, 1.0)
    with pytest.raises(capi.M3TBError, match="status -1"):
        ctx.upload_texture_features(0, np.zeros((1, 2), np.float32), np.zeros((1, 32), np.uint8), 0, 0, 0.0)
    ctx.set_focused_renderer(1, "color", 0, [0], [0], 200, id_type="region")
    with pytest.raises(capi.M3TBError, match="status -1"):
        ctx.attach_renderer(0, "texture_silhouette", 1)
    ctx.attach_renderer(0, "texture_silhouette", -1)
    with pytest.raises(capi.M3TBError, match="status -4"):
        ctx.tracking_step(0, 1, 1)
    ctx.set_texture_modality(0, None, 0)
    ctx.tracking_step(0, 1, 1)  # without the texture modality the body tracks as before


def test_failed_table_allocation_leaves_the_context_as_it_was(capi, synth):
    """Fault injection: the texture tables are made all or nothing by the first m3tb_set_texture_modality."""
    intr = synth.default_color_intrinsics()
    ctx = capi.Context(0, max_bodies=1, max_cameras=1, max_models=1)
    ctx.set_color_camera(0, intr, W2C)
    ctx.set_depth_camera(0, intr, W2C, 0.001)
    tri, diam = synth.prism_triangles()
    ctx.set_body_geometry(0, tri, W2C, diam, True, body_id=1, region_id=1)
    ctx.generate_depth_model(0, 0, params=capi.model_params(n_divides=1, n_points=40, image_size=200))
    ctx.set_body(0, None, capi.depth_params(), capi.OptimizerParams(1000.0, 30000.0), depth_model=0)
    live0 = capi.debug_resources()
    capi.debug_resources(fail_after=3)
    try:
        with pytest.raises(capi.M3TBError, match="status -2"):
            ctx.set_texture_modality(0, capi.texture_params_default(), 0)
    finally:
        capi.debug_resources(fail_after=0)
    assert capi.debug_resources() == live0
    with pytest.raises(capi.M3TBError, match="status -1"):
        ctx.get_texture_points(0)  # no texture modality
    ctx.set_texture_modality(0, capi.texture_params_default(), 0)
    assert len(ctx.get_texture_points(0)) == 0


def _plane(z_mm=530):
    return np.full((480, 640), z_mm, np.uint16)


def test_set_body_again_keeps_the_texture_modality(capi, synth):
    """m3tb_set_body on a body with a texture modality keeps it (keyframes, renderers, parameters); removing it brings
    back what a context without texture launches."""
    rng = np.random.default_rng(21)
    ctx, params, kf_pts, kf_desc = _start(capi, synth, rng)
    ctx.set_body(0, None, capi.depth_params(), capi.OptimizerParams(1000.0, 30000.0), depth_model=0)
    _next_frame(ctx, rng, _pose(t=(0.002, 0.0, 0.5)), kf_pts, kf_desc)
    ctx.tracking_step(1, 1, 1)
    assert ctx.last_launch()["kernel"] == "k_track"
    assert len(ctx.get_texture_points(0)) > 20
    assert list(ctx.get_texture_keyframes(0)["sizes"]) == [len(kf_pts)]
    ctx.set_texture_modality(0, params, 0)  # set again: still one modality, an empty deque
    assert len(ctx.get_texture_keyframes(0)["sizes"]) == 0
    ctx.set_texture_modality(0, None, 0)
    with pytest.raises(capi.M3TBError, match="status -1"):
        ctx.get_texture_points(0)
    ctx.tracking_step(2, 1, 1)
    plain, _, _ = _scene(capi, synth, texture_bodies=[])
    plain.tracking_step(2, 1, 1)
    assert ctx.last_launch() == plain.last_launch()


def test_rotation_rule_refreshes_with_the_pose_of_the_last_gradient_pass(capi, synth):
    """CalculateResults with a rotation above max_keyframe_rotation_difference: pop-front happens first (n_keyframes
    2 keeps the old keyframe), the new keyframe is reconstructed bit for bit with camera2body of the pose of the last
    gradient pass from the silhouette rendered at the final pose."""
    rng = np.random.default_rng(8)
    ctx, params, kf_pts, kf_desc = _start(capi, synth, rng, n_keyframes=2)
    o0 = ctx.get_texture_keyframes(0)["orientation"].copy()
    rotated = _pose((0.0, 14.0, 0.0))
    xy, desc = _next_frame(ctx, rng, _pose((0.0, 14.5, 0.0), (0.003, -0.002, 0.505)), kf_pts, kf_desc)
    ctx.set_poses(rotated[None])
    ctx.texture_correspondences(1, 0)
    ctx.texture_gradient_hessian(1, 0, 0)
    stale = ctx.get_poses()[0].reshape(12).copy()
    ctx.calculate_optimization(1, 0, 0)
    assert np.abs(ctx.get_poses()[0].reshape(12) - stale).max() > 0  # the final pose differs
    fires, _ = tr.keyframe_fires(_b2c(stale), o0, 0, params.max_keyframe_rotation_difference, params.max_keyframe_age)
    assert fires
    ctx.calculate_results(1)
    rend = ctx.get_rendering(0)
    idx, pts = tr.reconstruct(xy, rend, INTR, tr.pose_inverse(_b2c(stale)), 1)
    kf = ctx.get_texture_keyframes(0)
    assert list(kf["sizes"]) == [len(kf_pts), len(idx)] and len(idx) > 10 and kf["age"] == 0
    assert np.array_equal(kf["points"][len(kf_pts):].view(np.uint32), pts.view(np.uint32))
    assert np.array_equal(kf["descriptors"][len(kf_pts):], desc[idx])
    assert np.array_equal(kf["orientation"].view(np.uint32), tr.orientation(_b2c(stale)).view(np.uint32))


def test_measured_occlusions(capi, synth):
    """A depth frame with a near surface over the left half: keyframe points whose depth window sees it are dropped."""
    rng = np.random.default_rng(9)
    frame = np.zeros((480, 640), np.uint16)
    frame[:, :321] = 300
    ctx, params, _ = _scene(capi, synth, depth_frame=frame, measure_occlusions=1)
    roi, scale, _ = ctx.get_texture_focus()
    crop, desc = _features(rng, roi[0], scale[0], 300)
    xy = _upload(ctx, 0, crop, desc, roi[0], scale[0])
    ctx.start_modalities(0)
    b2c = _b2c(ctx.get_poses()[0])
    m = dict(image=frame, intr=INTR, depth_scale=0.001, b2d=b2c, radius=params.measured_occlusion_radius,
             threshold=params.measured_occlusion_threshold)
    rend = ctx.get_rendering(0)
    idx, pts = tr.reconstruct(xy, rend, INTR, tr.pose_inverse(b2c), 1, measured=m)
    all_idx, _ = tr.reconstruct(xy, rend, INTR, tr.pose_inverse(b2c), 1)
    assert 10 < len(idx) < len(all_idx)
    kf = ctx.get_texture_keyframes(0)
    assert np.array_equal(kf["points"].view(np.uint32), pts.view(np.uint32))
    assert np.array_equal(kf["descriptors"], desc[idx])


def test_modeled_occlusions(capi, synth):
    """A second body in front of part of the first, drawn only by the depth renderer attached for model_occlusions."""
    rng = np.random.default_rng(10)
    ctx, params, _ = _scene(capi, synth, model_occlusions=1)
    tri, diam = synth.prism_triangles()
    ctx.set_body_geometry(1, tri, W2C, diam, True, body_id=2, region_id=2)
    ctx.set_poses(np.stack([_pose(), _pose(t=(0.045, 0.0, 0.42))]))
    with pytest.raises(capi.M3TBError, match="status -4"):  # model_occlusions needs its depth renderer
        ctx.start_modalities(0)
    ctx.set_focused_renderer(1, "color", 0, [0, 1], [0], 200, id_type="body")
    ctx.attach_renderer(0, "texture_depth", 1)
    roi, scale, _ = ctx.get_texture_focus()
    crop, desc = _features(rng, roi[0], scale[0], 300)
    xy = _upload(ctx, 0, crop, desc, roi[0], scale[0])
    ctx.start_modalities(0)
    b2c = _b2c(ctx.get_poses()[0])
    m = dict(rendering=ctx.get_rendering(1), intr=INTR, b2c=b2c, radius=params.modeled_occlusion_radius,
             threshold=params.modeled_occlusion_threshold)
    rend = ctx.get_rendering(0)
    idx, pts = tr.reconstruct(xy, rend, INTR, tr.pose_inverse(b2c), 1, modeled=m)
    all_idx, _ = tr.reconstruct(xy, rend, INTR, tr.pose_inverse(b2c), 1)
    assert 10 < len(idx) < len(all_idx)
    kf = ctx.get_texture_keyframes(0)
    assert np.array_equal(kf["points"].view(np.uint32), pts.view(np.uint32))


def test_ties_zero_distances_and_a_single_train_descriptor(capi, synth):
    """Every keyframe descriptor twice in the frame: d0 = d1 = 0, 0 / 0 is NaN and keeps the match, and the earlier
    train descriptor wins the tie. A frame of one descriptor gives no data point (fewer than two matches)."""
    rng = np.random.default_rng(12)
    ctx, params, kf_pts, kf_desc = _start(capi, synth, rng)
    roi, scale, _ = ctx.get_texture_focus()
    proj = tr.project(_b2c(_pose(t=(0.001, 0.0, 0.5))), INTR, kf_pts)
    crop = ((proj - roi[0][:2].astype(np.float32)) * scale[0]).astype(np.float32)
    crop2, desc2 = np.vstack([crop, crop + 1.0]).astype(np.float32), np.vstack([kf_desc, kf_desc])
    xy = _upload(ctx, 0, crop2, desc2, roi[0], scale[0])
    cb, cc = tr.match([(kf_pts, kf_desc)], xy, desc2, params.descriptor_distance_threshold)
    assert len(cb) == len(kf_pts) and np.array_equal(cc, xy[:len(kf_pts)])
    ctx.texture_correspondences(1, 0)
    got = ctx.get_texture_points(0)
    assert np.array_equal(got["center_f_body"].view(np.uint32), cb.view(np.uint32))
    assert np.array_equal(got["correspondence_center"].view(np.uint32), cc.view(np.uint32))
    _upload(ctx, 0, crop[:1], kf_desc[:1], roi[0], scale[0])
    ctx.texture_correspondences(1, 0)
    assert len(ctx.get_texture_points(0)) == 0


@pytest.mark.parametrize("region", [False, True])
def test_link_sums_region_depth_texture_and_fused_step(capi, synth, region):
    """Link::CalculateGradientAndHessian adds region, depth and texture: the fine-grained calls' pose equals the
    restatement's Optimizer step from the three sums, and the fused step gives the same poses."""
    color = np.full((480, 640, 3), 40, np.uint8)
    color[180:300, 250:400] = (200, 120, 60)
    ctxs, kf = [], None
    for _ in range(2):
        rng = np.random.default_rng(13)
        ctx, params, _ = _scene(capi, synth, region=region, depth_frame=_plane(), color_frame=color)
        roi, scale, _ = ctx.get_texture_focus()
        crop, desc = _features(rng, roi[0], scale[0], 200)
        _upload(ctx, 0, crop, desc, roi[0], scale[0])
        ctx.start_modalities(0)
        kf = ctx.get_texture_keyframes(0)
        _next_frame(ctx, rng, _pose((1.0, -1.0, 0.5), (0.003, -0.002, 0.503)), kf["points"], kf["descriptors"])
        ctxs.append(ctx)
    fine, fused = ctxs
    pose = fine.get_poses()[0].reshape(3, 4)
    fused_poses = []
    for corr in range(2):
        if region:
            fine.region_correspondences(1, corr)
        fine.depth_correspondences(1, corr)
        fine.texture_correspondences(1, corr)
        for upd in range(2):
            g = np.zeros(6)
            H = np.zeros((6, 6))
            if region:
                gr, Hr = fine.region_gradient_hessian(1, corr, upd)
                g, H = g + gr[0], H + Hr[0]
            gd, Hd = fine.depth_gradient_hessian(1, corr, upd)
            gt, Ht = fine.texture_gradient_hessian(1, corr, upd)
            assert np.abs(gt[0]).max() > 0
            g, H = g + gd[0] + gt[0], H + Hd[0] + Ht[0]
            fine.calculate_optimization(1, corr, upd)
            pose = tr.optimize(pose, g, H)
            assert np.abs(fine.get_poses()[0].reshape(12) - pose.reshape(12)).max() < 1e-4
        fused.corr_iteration(1, corr, 2)
        assert fused.last_launch()["kernel"] == "k_track"
        fused_poses.append(fused.get_poses()[0].reshape(12))
        assert np.abs(fused_poses[-1] - fine.get_poses()[0].reshape(12)).max() < 1e-4


def test_mixed_batch_non_texture_bodies_track_as_without_texture(capi, synth):
    """Body 0 with a texture modality, body 1 without: body 1's poses equal those of a context without any texture
    modality, whose launches are those of a context that never had one."""
    runs = []
    for tex in ([0], []):
        rng = np.random.default_rng(14)
        ctx, params, _ = _scene(capi, synth, n_bodies=2, depth_frame=_plane(), texture_bodies=tex)
        if tex:
            roi, scale, _ = ctx.get_texture_focus(0, 1)
            crop, desc = _features(rng, roi[0], scale[0], 200)
            _upload(ctx, 0, crop, desc, roi[0], scale[0])
        ctx.start_modalities(0)
        if tex:
            kf = ctx.get_texture_keyframes(0)
            _next_frame(ctx, rng, _pose((1.0, 0.0, 0.0), (0.002, 0.0, 0.502)), kf["points"], kf["descriptors"])
        poses = []
        for frame in range(1, 4):
            ctx.tracking_step(frame, 2, 2)
            poses.append(ctx.get_poses()[1].reshape(12).copy())
        runs.append((poses, ctx.last_launch()))
    (with_tex, launch_tex), (without, launch_plain) = runs
    assert launch_tex["kernel"] == "k_track"
    for a, b in zip(with_tex, without):
        assert np.abs(a - b).max() < 1e-4
    assert np.abs(without[-1] - _pose(t=(0.03, 0.0, 0.5)).reshape(12)).max() > 1e-4  # the depth term moved body 1
