"""Texture modalities on the links of kinematic structures, on the device, against the two CPU restatements: the texture
modality's (tests/texture_reference.py: data points bit for bit, gradients / Hessians within 1e-5 of max|H|) and the
structure solve's (orc_optimize_structure fed the device's region + depth + texture sums: theta within 2e-4 of
max|theta|, link and joint poses within 5e-6), on the synthetic prism with seeded ORB-like features. The fused step
(k_track + k_structure per update, the texture match once per frame) is held to the fine-grained calls; a link seen by
two cameras sums both sets' texture terms; keyframes on links keep only their own body's pixels; mixed contexts and the
removal of a link's texture modality change nothing for the bodies without one."""
import numpy as np
import pytest

import structure_reference as sr
import texture_reference as tr

pytestmark = pytest.mark.gpu

W2C = np.hstack([np.eye(3), np.zeros((3, 1))]).astype(np.float32)
INTR = dict(fu=614.0, fv=614.5, ppu=321.3, ppv=238.9, width=640, height=480)
N_UPDATE = 2


def _pose(rot_deg=(0.0, 0.0, 0.0), t=(0.0, 0.0, 0.5)):
    R = np.eye(3)
    for axis, deg in enumerate(rot_deg):
        c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
        i, j = [k for k in range(3) if k != axis]
        Q = np.eye(3)
        Q[i, i], Q[i, j], Q[j, i], Q[j, j] = c, -s, s, c
        R = R @ Q
    return np.hstack([R, np.array(t)[:, None]]).astype(np.float32)


def _color():
    c = np.full((480, 640, 3), 40, np.uint8)
    c[180:300, 250:400] = (200, 120, 60)
    return c


def _context(capi, synth, poses, texture=(), region=False, cameras=None, camera_w2c=(W2C,), renderers=None, plane=True,
             **tex):
    """Depth (+ region) bodies on the prism at `poses` in front of a depth plane at 0.53 m (an empty depth frame without
    `plane`). Body b is seen by camera cameras[b] (default 0). Each body of `texture` gets a texture modality whose
    silhouette renderer is renderers[b] = (renderer, geometry bodies, referenced bodies), by default a renderer of its
    own over its own geometry."""
    n = len(poses)
    cameras = list(cameras) if cameras is not None else [0] * n
    intr = synth.default_color_intrinsics()
    ctx = capi.Context(0, max_bodies=n + 1, max_cameras=len(camera_w2c), max_models=1)
    for c, w2c in enumerate(camera_w2c):
        ctx.set_color_camera(c, intr, w2c)
        ctx.set_depth_camera(c, intr, w2c, 0.001)
        ctx.upload_depth(c, np.full((480, 640), 530 if plane else 0, np.uint16))
        if region:
            ctx.upload_color(c, _color())
    tri, diam = synth.prism_triangles()
    for b in range(n):
        ctx.set_body_geometry(b, tri, W2C, diam, True, body_id=b + 1, region_id=b + 1)
    mp = capi.model_params(n_divides=1, n_points=40, image_size=200)
    ctx.generate_depth_model(0, 0, params=mp)
    if region:
        ctx.generate_region_model(0, 0, params=mp)
    op = capi.OptimizerParams(1000.0, 30000.0)
    for b in range(n):
        ctx.set_body(b, capi.region_params() if region else None, capi.depth_params(), op, region_model=0,
                     depth_model=0, color_camera=cameras[b], depth_camera=cameras[b])
    ctx.set_poses(np.stack(poses))
    params = capi.texture_params_default()
    for k, v in tex.items():
        setattr(params, k, v)
    made = set()
    for k, b in enumerate(texture):
        rid, geometry, referenced = renderers[b] if renderers else (k, [b], [b])
        if rid not in made:
            ctx.set_focused_renderer(rid, "color", cameras[b], geometry, referenced, 200, id_type="body")
            made.add(rid)
        ctx.set_texture_modality(b, params, cameras[b])
        ctx.attach_renderer(b, "texture_silhouette", rid)
    return ctx, params


def _chain(synth, bodies=(0, 1, 2), constrained=False):
    """Root with 6 DoF, two revolute children 3 cm apart along x (about z, then about y); `constrained` adds a hard
    constraint between the root and the last link and an active soft constraint between the two children."""
    I = synth.identity_pose
    links = [synth.LinkSpec(body=bodies[0], parent=-1, body2joint=I(), joint2parent=I()),
             synth.LinkSpec(body=bodies[1], parent=0, body2joint=I(), joint2parent=synth.translation_pose(0.03),
                            free_directions=(0, 0, 1, 0, 0, 0)),
             synth.LinkSpec(body=bodies[2], parent=1, body2joint=I(), joint2parent=synth.translation_pose(0.03),
                            free_directions=(0, 1, 0, 0, 0, 0))]
    cons = []
    if constrained:
        cons = [synth.ConstraintSpec(link1=0, link2=2, body12joint1=I(), body22joint2=synth.translation_pose(0.06),
                                     directions=(1, 0, 0, 0, 0, 0)),
                synth.ConstraintSpec(link1=1, link2=2, body12joint1=I(), body22joint2=synth.translation_pose(0.032),
                                     directions=(1, 1, 1, 1, 1, 1), soft=True, max_distance_rotation=0.001,
                                     max_distance_translation=0.0005, standard_deviation_rotation=0.05,
                                     standard_deviation_translation=0.01)]
    return synth.StructureSpec(links=links, constraints=cons, tikhonov_rotation=1000.0, tikhonov_translation=30000.0)


CHAIN_POSES = [_pose(t=(-0.03, 0.0, 0.5)), _pose(t=(0.0, 0.0, 0.5)), _pose(t=(0.03, 0.0, 0.5))]
MOTION = _pose((1.0, -1.0, 0.5), (0.003, -0.002, 0.003))  # world-frame motion of the whole object to the next frame


def _b2c(pose, w2c=W2C):
    return tr.pose_mul(w2c, pose)


def _start(ctx, bodies, n=200):
    """Seeded features in each body's focus region, StartModality; returns {body: keyframe}."""
    roi, scale, valid = ctx.get_texture_focus()
    xy = {}
    for b in bodies:
        assert valid[b]
        rng = np.random.default_rng(100 + b)
        x, y, w, h = roi[b]
        pts = np.stack([rng.uniform(x, x + w, n), rng.uniform(y, y + h, n)], 1).astype(np.float32)
        crop = ((pts - np.array([x, y], np.float32)) * np.float32(scale[b])).astype(np.float32)
        desc = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        ctx.upload_texture_features(b, crop, desc, x, y, scale[b])
        xy[b] = (tr.crop_to_image(crop, x, y, scale[b]), desc)
    ctx.start_modalities(0)
    return {b: ctx.get_texture_keyframes(b) for b in bodies}, xy


def _next_frame(ctx, kfs, motion=MOTION, cameras=None, camera_w2c=(W2C,)):
    """Each body's keyframe points seen after `motion` with a few descriptor bits flipped, plus distractors; returns
    {body: (image xy, descriptors)}."""
    roi, scale, _ = ctx.get_texture_focus()
    poses = ctx.get_poses()
    out = {}
    for b, kf in kfs.items():
        rng = np.random.default_rng(200 + b)
        w2c = camera_w2c[cameras[b] if cameras else 0]
        proj = tr.project(_b2c(tr.pose_mul(motion, poses[b]), w2c), INTR, kf["points"])
        x, y = roi[b][:2].astype(np.float32)
        crop = ((proj - np.array([x, y], np.float32)) * scale[b]).astype(np.float32)
        desc = kf["descriptors"].copy()
        for r in range(len(desc)):
            for bit in rng.choice(256, 12, replace=False):
                desc[r, bit // 8] ^= np.uint8(1 << (bit % 8))
        nx = np.stack([rng.uniform(x, x + roi[b][2], 40), rng.uniform(y, y + roi[b][3], 40)], 1).astype(np.float32)
        crop = np.vstack([crop, ((nx - np.array([x, y], np.float32)) * scale[b]).astype(np.float32)])
        desc = np.vstack([desc, rng.integers(0, 256, (40, 32), dtype=np.uint8)])
        ctx.upload_texture_features(b, crop, desc, roi[b][0], roi[b][1], scale[b])
        out[b] = (tr.crop_to_image(crop, roi[b][0], roi[b][1], scale[b]), desc)
    return out


def _oracle(oracle, spec, state, g, H):
    """orc_optimize_structure from the device's state and per-body sums: (theta, ok, link2world, joint poses)."""
    L = oracle.lib()
    so = oracle.OracleStructure(sr.with_joint_poses(spec, state.body2joint[:, :3], state.joint2parent[:, :3]))
    S = so.as_struct()
    gl, Hl = sr.link_gradients(spec, g, H)
    l2w = np.ascontiguousarray(state.link2world[:, :3].reshape(-1, 12), np.float32)
    theta = np.zeros(sr.n_unknowns(spec), np.float32)
    ok = L.orc_optimize_structure(S, oracle.ptr(gl.astype(np.float32)), oracle.ptr(Hl.reshape(-1, 36).astype(np.float32)),
                                  oracle.ROTATION_LINEAR, oracle.EXP_RODRIGUES, oracle.ptr(l2w), oracle.ptr(theta))
    return theta, ok, l2w, so.joint_poses()


def _fine_iteration(ctx, oracle, spec, params, corr, keyframes, frame, matches, region=False, cameras=None,
                    camera_w2c=(W2C,), stale=None):
    """One correspondence iteration through the fine-grained calls, every step held to the restatements. matches
    (filled at corr 0) holds each texture body's data points; stale receives the pose of each body's last gradient
    pass."""
    nl = len(spec.links)
    nb = ctx.n_bodies
    if region:
        ctx.region_correspondences(1, corr)
    ctx.depth_correspondences(1, corr)
    ctx.texture_correspondences(1, corr)
    poses = ctx.get_poses()
    for b, kf in keyframes.items():
        w2c = camera_w2c[cameras[b] if cameras else 0]
        if corr == 0:
            matches[b] = tr.match([(kf["points"], kf["descriptors"])], *frame[b], params.descriptor_distance_threshold)
        cb, cc = matches[b]
        assert len(cb) > 20, b
        got = ctx.get_texture_points(b)
        assert np.array_equal(got["center_f_body"].view(np.uint32), cb.view(np.uint32))
        assert np.array_equal(got["correspondence_center"].view(np.uint32), cc.view(np.uint32))
        assert np.array_equal(got["center"].view(np.uint32), tr.project(_b2c(poses[b], w2c), INTR, cb).view(np.uint32))
    sd = params.standard_deviations[min(corr, params.n_standard_deviations - 1)]
    for upd in range(N_UPDATE):
        poses = ctx.get_poses()
        b2j, j2p, l2w = ctx.get_link_poses(0, nl)
        g = np.zeros((3, nb, 6), np.float32)
        H = np.zeros((3, nb, 6, 6), np.float32)
        if region:
            g[0], H[0] = ctx.region_gradient_hessian(1, corr, upd)
        g[1], H[1] = ctx.depth_gradient_hessian(1, corr, upd)
        g[2], H[2] = ctx.texture_gradient_hessian(1, corr, upd)
        for b in range(nb):
            if b not in keyframes:
                assert not g[2, b].any()
                continue
            w2c = camera_w2c[cameras[b] if cameras else 0]
            eg, eH = tr.gradient_hessian(_b2c(poses[b], w2c), INTR, *matches[b], sd, params.tukey_norm_constant)
            scale = np.abs(eH).max()
            assert scale > 0
            assert np.abs(g[2, b] - eg).max() <= 1e-5 * scale and np.abs(H[2, b] - eH).max() <= 1e-5 * scale, b
            if stale is not None:
                stale[b] = poses[b].copy()
        state = sr.State.from_arrays(l2w.reshape(nl, 12), b2j.reshape(nl, 12), j2p.reshape(nl, 12))
        theta_o, ok, l2w_o, (ob2j, oj2p) = _oracle(oracle, spec, state, g, H)
        ctx.calculate_optimization(1, corr, upd)
        theta_g, updated = ctx.get_structure_theta(0)
        assert ok == 1 and updated and len(theta_g) == len(theta_o)
        assert np.abs(theta_g - theta_o).max() <= 2e-4 * np.abs(theta_o).max() + 1e-7, (corr, upd)
        b2j, j2p, lw = ctx.get_link_poses(0, nl)
        assert np.abs(lw.reshape(nl, 12) - l2w_o).max() < 5e-6, (corr, upd)
        assert np.abs(b2j.reshape(nl, 12) - np.reshape(ob2j, (nl, 12))).max() < 5e-6
        assert np.abs(j2p.reshape(nl, 12) - np.reshape(oj2p, (nl, 12))).max() < 5e-6
        for l, link in enumerate(spec.links):  # the link's pose is written to its body and to its extra bodies
            for b in (link.body,) + tuple(link.extra_bodies):
                assert np.array_equal(ctx.get_poses()[b].reshape(12), lw[l].reshape(12))


@pytest.mark.parametrize("region,constrained", [(False, False), (True, False), (False, True)])
def test_textured_chain_fine_grained_fused_and_step(capi, oracle, synth, region, constrained):
    """Root (6 DoF) + two revolute children, each with depth (+ region) + texture: the fine-grained calls against the
    restatements at every update; corr_iteration and tracking_step against the fine-grained path."""
    spec = _chain(synth, constrained=constrained)
    ctxs = []
    for _ in range(3):
        ctx, params = _context(capi, synth, CHAIN_POSES, texture=(0, 1, 2), region=region)
        ctx.set_structure(0, spec)
        kfs, _ = _start(ctx, (0, 1, 2))
        frame = _next_frame(ctx, kfs)
        ctxs.append((ctx, kfs, frame))
    (fine, kfs, frame), (fused, _, _), (step, _, _) = ctxs
    start = fine.get_poses().copy()
    target = np.stack([tr.pose_mul(MOTION, p).reshape(3, 4) for p in start])
    matches = {}
    for corr in range(2):
        _fine_iteration(fine, oracle, spec, params, corr, kfs, frame, matches, region=region)
        before = fused.launch_count
        fused.corr_iteration(1, corr, N_UPDATE)
        assert fused.last_launch()["kernel"] == "k_track"
        # one k_render, k_texture_match at iteration 0 only, then k_track + k_structure per update
        assert fused.launch_count - before == 1 + (corr == 0) + 2 * N_UPDATE, corr
        assert np.abs(fused.get_poses() - fine.get_poses()).max() < 1e-4, corr
    step.tracking_step(1, 2, N_UPDATE)
    assert step.last_launch()["kernel"] == "k_track"
    assert np.abs(step.get_poses() - fine.get_poses()).max() < 1e-4
    # without the depth plane, which pulls the chain towards itself, the step moves every link towards the position
    # its features were seen at (as in the rigid test, the translation: for the flat prism a small rotation about an
    # axis in the image plane looks much like a translation)
    alone, _ = _context(capi, synth, CHAIN_POSES, texture=(0, 1, 2), region=region, plane=False)
    alone.set_structure(0, spec)
    _next_frame(alone, _start(alone, (0, 1, 2))[0])
    alone.tracking_step(1, 2, N_UPDATE)
    for b in range(3):
        moved = np.abs(alone.get_poses()[b][:, 3] - target[b][:, 3]).max()
        assert moved < 0.5 * np.abs(start[b][:, 3] - target[b][:, 3]).max(), b


def test_link_seen_by_two_cameras(capi, oracle, synth):
    """One object seen by two cameras: body 0 (camera 0) is the link's body, body 1 (camera 1, shifted 3 cm) its extra
    body, each with its own texture modality, silhouette renderer and features. Both carry bit-equal poses after every
    update, the solve matches the oracle fed both sets' sums, and the result differs from set A's texture alone."""
    w2c1 = W2C.copy()
    w2c1[:, 3] = (-0.03, 0.01, 0.0)
    cams = dict(cameras=(0, 1), camera_w2c=(W2C, w2c1))
    spec = synth.StructureSpec(links=[synth.LinkSpec(body=0, parent=-1, body2joint=synth.identity_pose(),
                                                     joint2parent=synth.identity_pose(), extra_bodies=(1,))])
    finals = []
    for texture in ((0, 1), (0,)):
        ctxs = []
        for _ in range(2):
            ctx, params = _context(capi, synth, [_pose(), _pose()], texture=texture, **cams)
            ctx.set_structure(0, spec)
            kfs, _ = _start(ctx, texture)
            ctxs.append((ctx, kfs, _next_frame(ctx, kfs, **cams)))
        (ctx, kfs, frame), (fused, _, _) = ctxs
        matches = {}
        for corr in range(2):
            _fine_iteration(ctx, oracle, spec, params, corr, kfs, frame, matches, **cams)
            # the fused step: both sets' texture terms through k_track -> gh_link -> k_structure
            fused.corr_iteration(1, corr, N_UPDATE)
            assert np.abs(fused.get_poses() - ctx.get_poses()).max() < 1e-4, (texture, corr)
            assert np.array_equal(fused.get_poses()[0], fused.get_poses()[1])
        finals.append(ctx.get_poses()[0].reshape(12).copy())
    assert np.abs(finals[0] - finals[1]).max() > 1e-5


def test_keyframes_of_links_sharing_a_silhouette_renderer(capi, oracle, synth):
    """Two links in one BODY-id silhouette renderer, the second partly in front of the first: each link's keyframe
    holds only the keypoints on its own body's pixels. With max_keyframe_age = 0, CalculateResults after a fused step
    reconstructs with the pose of the last gradient pass."""
    I = synth.identity_pose
    spec = synth.StructureSpec(links=[
        synth.LinkSpec(body=0, parent=-1, body2joint=I(), joint2parent=I()),
        synth.LinkSpec(body=1, parent=0, body2joint=I(), joint2parent=synth.translation_pose(0.03, 0.0, -0.05),
                       free_directions=(0, 0, 1, 0, 0, 0))])
    poses = [_pose(), _pose(t=(0.03, 0.0, 0.45))]
    shared = {0: (0, [0, 1], [0, 1]), 1: (0, [0, 1], [0, 1])}
    ctxs = []
    for _ in range(2):
        ctx, params = _context(capi, synth, poses, texture=(0, 1), renderers=shared, max_keyframe_age=0)
        ctx.set_structure(0, spec)
        kfs, xy = _start(ctx, (0, 1), n=400)
        ctxs.append((ctx, kfs, xy))
    fused, kfs, xy = ctxs[0]
    rend = fused.get_rendering(0)
    for b in (0, 1):
        c2b = tr.pose_inverse(_b2c(fused.get_poses()[b]))
        idx, pts = tr.reconstruct(xy[b][0], rend, INTR, c2b, b + 1)
        other, _ = tr.reconstruct(xy[b][0], rend, INTR, c2b, 2 - b)
        assert len(idx) > 20 and len(other) > 0, b  # some of the body's keypoints lie on the other body's pixels
        assert np.array_equal(kfs[b]["points"].view(np.uint32), pts.view(np.uint32))
        assert np.array_equal(kfs[b]["descriptors"], xy[b][1][idx])
    fine, fkfs, _ = ctxs[1]
    frames = [_next_frame(c, k) for c, k, _ in ctxs]
    fused.tracking_step(1, 2, N_UPDATE)
    stale, matches = {}, {}
    for corr in range(2):
        _fine_iteration(fine, oracle, spec, params, corr, fkfs, frames[1], matches, stale=stale)
    assert np.abs(fused.get_poses() - fine.get_poses()).max() < 1e-4
    fused.calculate_results(1)
    rend = fused.get_rendering(0)
    for b in (0, 1):
        idx, pts = tr.reconstruct(frames[0][b][0], rend, INTR, tr.pose_inverse(_b2c(stale[b])), b + 1)
        kf = fused.get_texture_keyframes(b)
        assert kf["age"] == 0
        new = kf["points"][-kf["sizes"][-1]:]
        assert len(new) == len(idx) > 10 and np.abs(new - pts).max() < 1e-3, b


def _mixed(capi, synth, textured_rigid, with_chain):
    """Body 0 a rigid body (textured or not), bodies 1..3 an untextured depth-only chain when with_chain."""
    poses = [_pose(t=(-0.08, 0.0, 0.5))] + (CHAIN_POSES if with_chain else [])
    poses = poses[:1] + [tr.pose_mul(_pose(t=(0.04, 0.0, 0.0)), p).reshape(3, 4) for p in poses[1:]]
    ctx, _ = _context(capi, synth, poses, texture=(0,) if textured_rigid else ())
    if with_chain:
        ctx.set_structure(0, _chain(synth, bodies=(1, 2, 3)))
    if textured_rigid:
        kfs, _ = _start(ctx, (0,))
        _next_frame(ctx, kfs)
    else:
        ctx.start_modalities(0)
    return ctx


def test_mixed_contexts(capi, synth):
    """A textured rigid body next to an untextured chain tracks as without the chain, the chain as without the texture;
    a chain context without texture launches k_track + k_structure per update and nothing else."""
    both = _mixed(capi, synth, True, True)
    rigid = _mixed(capi, synth, True, False)
    chain = _mixed(capi, synth, False, True)
    for frame in range(1, 3):
        counts = []
        for c in (both, rigid, chain):
            before = c.launch_count
            c.tracking_step(frame, 2, N_UPDATE)
            counts.append(c.launch_count - before)
        assert both.last_launch()["kernel"] == "k_track"
        if frame > 1:  # the first step may also make the new structure's poses consistent
            assert counts[2] == 2 * 2 * N_UPDATE
        assert np.abs(both.get_poses()[0] - rigid.get_poses()[0]).max() < 1e-4, frame
        assert np.abs(both.get_poses()[1:] - chain.get_poses()[1:]).max() < 1e-4, frame
    assert np.abs(rigid.get_poses()[0] - _pose(t=(-0.08, 0.0, 0.5))).max() > 1e-4  # the texture term moved it


def test_removed_link_texture_leaves_no_stale_term(capi, synth):
    """m3tb_set_texture_modality(link body, NULL) after a texture gradient pass leaves that body's row of texture sums
    behind: the later link solves carry no texture term of it and equal those of a context that never had texture on
    that body."""
    spec = _chain(synth)
    ctxs = []
    for texture in ((0, 1, 2), (0, 2)):
        ctx, _ = _context(capi, synth, CHAIN_POSES, texture=texture)
        ctx.set_structure(0, spec)
        kfs, _ = _start(ctx, texture)
        _next_frame(ctx, kfs)
        ctxs.append(ctx)
    had, never = ctxs
    for c in ctxs:
        c.texture_correspondences(1, 0)
    g = [c.texture_gradient_hessian(1, 0, 0)[0] for c in ctxs]
    assert np.abs(g[0][1]).max() > 0 and not g[1][1].any()
    start = had.get_poses().copy()
    had.set_texture_modality(1, None)
    for c in ctxs:  # the solve reads the texture sums left by the gradient pass above
        c.depth_correspondences(1, 0)
        c.depth_gradient_hessian(1, 0, 0)
        c.calculate_optimization(1, 0, 0)
    assert np.array_equal(had.get_poses(), never.get_poses())
    assert np.abs(had.get_poses() - start).max() > 1e-5
    for c in ctxs:
        c.corr_iteration(1, 1, N_UPDATE)
    assert np.abs(had.get_poses() - never.get_poses()).max() < 1e-6


def test_textured_structure_without_silhouette_renderer_is_refused(capi, synth):
    """TextureModality::SetUp's conditions hold in the structure step too: a texture modality whose silhouette renderer
    was detached refuses the step (M3TB_ERR_NOT_SET_UP) instead of tracking without its texture term, also where the
    cluster-fused chain path would otherwise take the step."""
    ctx, _ = _context(capi, synth, CHAIN_POSES, texture=(0, 1, 2))
    ctx.set_structure(0, _chain(synth))
    _start(ctx, (0, 1, 2))
    for b in range(3):
        ctx.attach_renderer(b, "texture_silhouette", -1)
    for step in (lambda: ctx.corr_iteration(1, 0, N_UPDATE), lambda: ctx.tracking_step(1, 2, 0)):
        with pytest.raises(capi.M3TBError, match="status -4"):
            step()
