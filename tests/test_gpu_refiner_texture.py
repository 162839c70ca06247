"""m3tb_refine_poses_orb = Refiner::RefinePoses with ORB texture bodies (refiner.cpp:98-139, texture_modality.cpp:314-332):
device detection, a new keyframe and the start renders before every correspondence iteration, the texture match at
correspondence iteration 0, the texture term in every update.

Gates: refining every body is the composition texture_detect_orb + start_modalities + corr_iteration bit for bit
(poses, keyframes, data points, detections, histograms, lines, points), rigid and for a textured chain; a refined
subset leaves every other body bit for bit as it was, and later tracking moves them as in a twin that never refined;
at a fixed pose the deque and the data points are the restatement's (tests/texture_reference.py) of the device's own
detection and rendering; refusals launch nothing; the launch count follows the documented sequence.
"""
import ctypes as C

import numpy as np
import pytest

import texture_reference as tr
from test_gpu_texture_device_front_end import CHAIN_POSES, FIX, FIX_FRAME, W2C, _intr
from test_gpu_texture_structures import _chain

pytestmark = pytest.mark.gpu

OK, ERR_INVALID, ERR_CUDA, ERR_UNSUPPORTED, ERR_NOT_SET_UP = 0, -1, -2, -3, -4
ORB = (300, 1.2, 3)
N_BINS = 16


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _scene(capi, synth, poses, texture, region=(), chain=None, upload=True, descriptor=None, n_keyframes=None,
           max_bodies=None):
    """Depth bodies on the prism at `poses` in the cv2-golden frame; the bodies of `region` also have a region
    modality, those of `texture` a texture modality (ORB unless `descriptor`). Every body has a renderer of its own
    (renderer b) that draws only itself. chain: the bodies of _chain(synth, chain[0], constrained=chain[1])."""
    n = len(poses)
    intr = _intr(capi, synth)
    ctx = capi.Context(0, max_bodies=max_bodies or n, max_cameras=1, max_models=1)
    ctx.set_color_camera(0, intr, W2C)
    ctx.set_depth_camera(0, intr, W2C, 0.001)
    ctx.upload_depth(0, np.zeros((intr.height, intr.width), np.uint16))
    if upload:
        ctx.upload_color(0, FIX_FRAME)
    tri, diam = synth.prism_triangles()
    for b in range(n):
        ctx.set_body_geometry(b, tri, W2C, diam, True, body_id=b + 1, region_id=b + 1)
    mp = capi.model_params(n_divides=1, n_points=40, image_size=200)
    ctx.generate_depth_model(0, 0, params=mp)
    if region:
        ctx.generate_region_model(0, 0, params=mp)
    op = capi.OptimizerParams(1000.0, 30000.0)
    rp = capi.region_params()
    rp.n_histogram_bins = N_BINS
    for b in range(n):
        ctx.set_body(b, rp if b in region else None, capi.depth_params(), op, region_model=0, depth_model=0,
                     color_camera=0, depth_camera=0)
    ctx.set_poses(np.stack(poses))
    params = capi.texture_params_default()
    params.descriptor_type = capi.DESCRIPTOR_ORB if descriptor is None else descriptor
    params.focused_image_size = int(FIX["focused_image_size"])
    if n_keyframes is not None:
        params.n_keyframes = n_keyframes
    for b in range(n):
        ctx.set_focused_renderer(b, "color", 0, [b], [b], 200, id_type="body")
    for b in texture:
        ctx.set_texture_modality(b, params, 0)
        ctx.attach_renderer(b, "texture_silhouette", b)
    if chain is not None:
        ctx.set_structure(0, _chain(synth, chain[0], constrained=chain[1]))
    return ctx, params


def _state(ctx, b, texture, region):
    """Everything of body b that a refinement and the composition must agree on."""
    s = dict(pose=_bits(ctx.get_poses()[b]).tobytes(), points=ctx.get_depth_points(b, 64).tobytes(),
             detections=int(ctx.get_texture_detections()[b]))
    if b in region:
        hf, hb = ctx.get_histograms(b, N_BINS)
        s.update(hf=_bits(hf).tobytes(), hb=_bits(hb).tobytes(), lines=ctx.get_region_lines(b, 256).tobytes())
    if b in texture:  # renderer b is the texture modality's silhouette renderer
        rend = ctx.get_rendering(b)
        s.update(depth_image=rend["depth"].tobytes(), silhouette_image=rend["silhouette"].tobytes())
        kf = ctx.get_texture_keyframes(b)
        s.update(kf_sizes=kf["sizes"].tobytes(), kf_points=_bits(kf["points"]).tobytes(),
                 kf_desc=kf["descriptors"].tobytes(), kf_age=kf["age"], kf_orientation=_bits(kf["orientation"]).tobytes(),
                 tex_points=ctx.get_texture_points(b).tobytes())
        orb = ctx.get_texture_orb_keypoints(b)
        s.update({"orb_" + k: np.asarray(v).tobytes() for k, v in orb.items()})
    return s


def _assert_same(x, y, bodies):
    for b in bodies:
        for k in x[b]:
            assert x[b][k] == y[b][k], (b, k)


def _composition(ctx, texture, n_corr, n_update, orb=ORB, structures=False):
    """What refining every body does, from the fine-grained calls: Refiner::CalculateConsistentPoses, then per
    correspondence iteration DetectAndComputeCorrKeypoints + StartModalities + CalculateCorrespondences + updates."""
    if structures:
        ctx.calculate_consistent_poses()
    for corr in range(n_corr):
        ctx.texture_detect_orb(list(texture), orb)
        ctx.start_modalities(0)
        ctx.corr_iteration(0, corr, n_update)


RIGID_POSES = [FIX["poses"][i] for i in (1, 9, 4, 3)]


def test_refine_every_rigid_body_is_the_composition(capi, synth, monkeypatch):
    texture, region = (0, 1, 2), (0, 1, 3)
    a, params = _scene(capi, synth, RIGID_POSES, texture, region)
    monkeypatch.setenv("M3TB_KERNEL", "1")
    b, _ = _scene(capi, synth, RIGID_POSES, texture, region)
    monkeypatch.delenv("M3TB_KERNEL")
    a.refine_poses_orb(range(4), (), 7, 2, orb_params=ORB)
    _composition(b, texture, 7, 2)
    assert b.last_launch()["kernel"] == "k_track" and a.last_launch()["kernel"] == "k_track"
    sa = {x: _state(a, x, texture, region) for x in range(4)}
    sb = {x: _state(b, x, texture, region) for x in range(4)}
    _assert_same(sa, sb, range(4))
    for x in texture:  # the refinement did move the bodies and kept what the reference keeps
        assert len(a.get_texture_keyframes(x)["sizes"]) == params.n_keyframes
        assert len(a.get_texture_points(x)) > 0 and a.get_texture_detections()[x] > 0
    assert not np.array_equal(a.get_poses()[0], np.float32(RIGID_POSES[0]))
    a.close()
    b.close()


@pytest.mark.parametrize("constrained", [False, True])
def test_refine_textured_chain_is_the_composition(capi, synth, monkeypatch, constrained):
    texture = region = (0, 1, 2)
    a, _ = _scene(capi, synth, list(CHAIN_POSES), texture, region, chain=((0, 1, 2), constrained))
    b, _ = _scene(capi, synth, list(CHAIN_POSES), texture, region, chain=((0, 1, 2), constrained))
    a.refine_poses_orb((), [0], 7, 2)  # default ORB settings
    _composition(b, texture, 7, 2, orb=None, structures=True)
    sa = {x: _state(a, x, texture, region) for x in range(3)}
    sb = {x: _state(b, x, texture, region) for x in range(3)}
    _assert_same(sa, sb, range(3))
    for x, y in zip(a.get_link_poses(0, 3), b.get_link_poses(0, 3)):
        assert np.array_equal(_bits(x), _bits(y))
    a.close()
    b.close()


MIXED_POSES = [FIX["poses"][i] for i in (1, 9, 4, 3, 0)] + list(CHAIN_POSES)
MIXED_TEXTURE, MIXED_REGION = (0, 1, 2, 5, 6, 7), (0, 1, 3, 5, 6, 7)


def _mixed(capi, synth):
    """Rigid ORB bodies 0, 1, 2 (region on 0, 1), plain bodies 3 (region + depth) and 4 (depth), the textured chain
    5-6-7; started and one tracking step behind them, so every body has state of its own."""
    ctx, _ = _scene(capi, synth, MIXED_POSES, MIXED_TEXTURE, MIXED_REGION, chain=((5, 6, 7), False))
    ctx.texture_detect_orb(list(MIXED_TEXTURE), ORB)
    ctx.start_modalities(0)
    ctx.tracking_step(0, 2, 2)
    ctx.calculate_results(0)
    ctx.synchronize()
    return ctx


def test_refine_subset_leaves_the_others(capi, synth):
    refined, others = [0, 3], [1, 2, 4]
    state = lambda c, bodies: {x: _state(c, x, MIXED_TEXTURE, MIXED_REGION) for x in bodies}
    a, twin, every = _mixed(capi, synth), _mixed(capi, synth), _mixed(capi, synth)
    before = state(a, others)
    a.refine_poses_orb(refined, [0], 7, 2, orb_params={0: ORB})
    _assert_same(before, state(a, others), others)
    # the refined bodies are those of a refinement of every body
    every.refine_poses_orb([0, 1, 2, 3, 4], [0], 7, 2, orb_params=ORB)
    _assert_same(state(every, refined + [5, 6, 7]), state(a, refined + [5, 6, 7]), refined + [5, 6, 7])
    # the next frame moves the others exactly as in a twin that never refined
    for c in (a, twin):
        c.texture_detect_orb(list(MIXED_TEXTURE), ORB)
        c.start_modalities(1)
        c.tracking_step(1, 2, 2)
        c.calculate_results(1)
    _assert_same(state(twin, others), state(a, others), others)
    for c in (a, twin, every):
        c.close()


def test_fixed_pose_deque_and_matches_follow_the_restatement(capi, synth):
    """n_update 0: every iteration detects at the same pose, so the deque holds n_keyframes copies of the reconstruction
    of that detection, and the data points are the corr-0 match against the one keyframe the deque then held."""
    ctx, params = _scene(capi, synth, [FIX["poses"][1]], (0,), (0,), n_keyframes=2)
    ctx.refine_poses_orb([0], (), 3, 0, orb_params=ORB)
    pose = ctx.get_poses()[0]
    assert np.array_equal(_bits(pose), _bits(FIX["poses"][1]))
    roi, scale, valid = ctx.get_texture_focus()
    assert valid[0]
    orb = ctx.get_texture_orb_keypoints(0)
    assert len(orb["xy"]) > 20
    xy = tr.crop_to_image(orb["xy"], roi[0][0], roi[0][1], scale[0])
    intr = dict(zip(("fu", "fv", "ppu", "ppv", "width", "height"), (float(v) for v in FIX["intrinsics"])))
    intr["width"], intr["height"] = int(intr["width"]), int(intr["height"])
    b2c = tr.pose_mul(W2C, pose)
    idx, pts = tr.reconstruct(xy, ctx.get_rendering(0), intr, tr.pose_inverse(b2c), 1)
    assert len(idx) > 10
    kf = ctx.get_texture_keyframes(0)
    assert list(kf["sizes"]) == [len(idx), len(idx)] and kf["age"] == 0
    for k in range(2):
        block = slice(k * len(idx), (k + 1) * len(idx))
        assert np.array_equal(_bits(kf["points"][block]), _bits(pts))
        assert np.array_equal(kf["descriptors"][block], orb["descriptors"][idx])
    assert np.array_equal(_bits(kf["orientation"]), _bits(tr.orientation(b2c)))
    cb, cc = tr.match([(pts, orb["descriptors"][idx])], xy, orb["descriptors"], params.descriptor_distance_threshold)
    got = ctx.get_texture_points(0)
    assert len(cb) > 10
    assert np.array_equal(_bits(got["center_f_body"]), _bits(cb))
    assert np.array_equal(_bits(got["correspondence_center"]), _bits(cc))
    ctx.close()


def _call(capi, ctx, bodies, structures=(), n_corr=7, n_update=2, orb=None):
    b = (C.c_int * max(1, len(bodies)))(*bodies)
    s = (C.c_int * max(1, len(structures)))(*structures)
    arr = None
    if orb is not None:
        arr = (capi.OrbParams * ctx.n_bodies)(*([capi.OrbParams(*orb)] * ctx.n_bodies))
    return capi.lib().m3tb_refine_poses_orb(ctx.h, b, len(bodies), s, len(structures), n_corr, n_update, arr)


def test_refusals_launch_nothing(capi, synth):
    ctx, _ = _scene(capi, synth, MIXED_POSES, MIXED_TEXTURE, MIXED_REGION, chain=((5, 6, 7), False))
    ctx.synchronize()
    poses, n0 = ctx.get_poses(), ctx.launch_count
    cases = [(ERR_INVALID, dict(bodies=[8])), (ERR_INVALID, dict(bodies=[0, 0])), (ERR_INVALID, dict(bodies=[5])),
             (ERR_INVALID, dict(bodies=[0], n_corr=-1)), (ERR_INVALID, dict(bodies=[0], n_update=-1)),
             (ERR_INVALID, dict(bodies=[], structures=[1])),
             (ERR_INVALID, dict(bodies=[0], orb=(0, 1.2, 3))), (ERR_INVALID, dict(bodies=[0], orb=(300, 1.0, 3))),
             (ERR_INVALID, dict(bodies=[], structures=[0], orb=(300, float("nan"), 3))),
             (ERR_UNSUPPORTED, dict(bodies=[1], orb=(300, 1.2, 9))), (ERR_UNSUPPORTED, dict(bodies=[2], orb=(1 << 25, 1.2, 3)))]
    for code, kw in cases:
        assert _call(capi, ctx, **kw) == code, kw
    # only the refined bodies' settings are read: body 4 has no texture modality
    assert ctx.launch_count == n0 and np.array_equal(_bits(ctx.get_poses()), _bits(poses))
    # m3tb_refine_poses keeps its refusal
    L = capi.lib()
    assert L.m3tb_refine_poses(ctx.h, (C.c_int * 1)(0), 1, (C.c_int * 1)(), 0, 7, 2) == ERR_UNSUPPORTED
    assert ctx.launch_count == n0
    ctx.close()
    for descriptor in (capi.DESCRIPTOR_SIFT, capi.DESCRIPTOR_DAISY):
        ctx, _ = _scene(capi, synth, RIGID_POSES[:2], (1,), (0, 1), descriptor=descriptor)
        n0 = ctx.launch_count
        assert _call(capi, ctx, [0, 1]) == ERR_UNSUPPORTED
        assert ctx.launch_count == n0
        ctx.refine_poses_orb([0], (), 1, 1)  # body 0 has no texture modality
        ctx.close()
    ctx, _ = _scene(capi, synth, RIGID_POSES[:2], (0, 1), (), upload=False)
    n0 = ctx.launch_count
    assert _call(capi, ctx, [1]) == ERR_NOT_SET_UP
    assert ctx.launch_count == n0
    ctx.close()


def test_selection_without_texture_is_refine_poses(capi, synth):
    out = []
    for orb in (False, True):
        ctx, _ = _scene(capi, synth, MIXED_POSES, MIXED_TEXTURE, MIXED_REGION, chain=((5, 6, 7), False))
        ctx.synchronize()
        n0 = ctx.launch_count
        (ctx.refine_poses_orb if orb else ctx.refine_poses)([3, 4], (), 7, 2)
        out.append((ctx.launch_count - n0, _bits(ctx.get_poses()).tobytes(), ctx.get_histograms(3, N_BINS)[0].tobytes()))
        ctx.close()
    assert out[0] == out[1]


def test_allocation_failure_of_the_detection_scratch(capi, synth):
    """Body 0's focus is cut by the image border, so its crop is smaller than body 1's: refining body 1 after body 0
    has to grow the detection scratch at its first detection, before anything of the call is launched."""
    ctx, _ = _scene(capi, synth, [FIX["poses"][5], FIX["poses"][1], FIX["poses"][3]], (0, 1), (0, 1, 2))
    ctx.refine_poses_orb([0], (), 1, 1)
    ctx.start_modalities(0)  # renders body 1's renderer, whose image is part of its state
    ctx.synchronize()
    state = {x: _state(ctx, x, (0, 1), (0, 1, 2)) for x in range(3)}
    n0, live = ctx.launch_count, capi.debug_resources()
    capi.debug_resources(1)
    try:
        rc = _call(capi, ctx, [1])
    finally:
        capi.debug_resources(0)
    assert rc == ERR_CUDA
    assert capi.debug_resources() == live and ctx.launch_count == n0
    _assert_same(state, {x: _state(ctx, x, (0, 1), (0, 1, 2)) for x in range(3)}, range(3))
    ctx.refine_poses_orb([1], (), 7, 2)
    assert ctx.launch_count > n0 and ctx.get_texture_detections()[1] > 0
    ctx.close()


def test_launch_count(capi, synth):
    """Per correspondence iteration: crop + ORB, the start renders, k_histogram, k_texture_keyframe, (the
    correspondence renders: none, a texture modality has no correspondence renderer), k_texture_match at iteration 0,
    k_track; two crop + ORB pairs for more than 128 texture bodies."""
    ctx, _ = _scene(capi, synth, [FIX["poses"][1]], (0,), (0,))
    n0 = ctx.launch_count
    ctx.refine_poses_orb([0], (), 7, 2)
    assert ctx.launch_count - n0 == 7 * 6 + 1
    ctx.close()
    n = 130
    ctx, _ = _scene(capi, synth, [FIX["poses"][1]] * n, tuple(range(n)), ())
    n0 = ctx.launch_count
    ctx.refine_poses_orb(range(n), (), 1, 0)
    # 2 x (crop + ORB), start renders, k_texture_keyframe, k_texture_match, k_track (depth only: no k_histogram)
    assert ctx.launch_count - n0 == 4 + 1 + 1 + 1 + 1
    assert len(ctx.get_texture_keyframes(129)["sizes"]) == 1
    ctx.close()


def test_cpp_mirror_refines_texture_bodies(pkg, tmp_path):
    """examples/texture_refiner_mirror.cpp: a rigid ORB body and a textured 3-link chain refined through the mirror's
    Refiner::RefinePoses, against the same refinement through m3tb_refine_poses_orb with the modalities' ORB settings:
    equal poses and texture points, bit for bit."""
    import json
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg._build.build_cuda()
    pkg._build.build_synth()
    csrc = os.path.join(root, "3dobjecttracking_b200", "csrc")
    synth_dir = os.path.join(root, "3dobjecttracking_b200", "synth")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = str(tmp_path / "texture_refiner_mirror")
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-I", os.path.join(root, "include"), "-I",
           os.path.join(root, "3dobjecttracking_b200", "host"), "-I", synth_dir, "-I", os.path.join(cuda, "include"),
           os.path.join(root, "examples", "texture_refiner_mirror.cpp"), "-o", exe, "-L", csrc, "-L", synth_dir,
           "-L", os.path.join(cuda, "lib64"), "-lm3t_b200", "-lm3t_synth", "-lcudart", "-Wl,-rpath," + csrc,
           "-Wl,-rpath," + synth_dir, "-Wl,-rpath," + os.path.join(cuda, "lib64"), "-fopenmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, "1", "400"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    out = json.loads(r.stdout.strip().split("\n")[-1])
    assert out["orb_n_features"] == 400
    assert min(out["texture_points_mirror"]) > 10 and out["texture_points_equal"]
    assert out["texture_points_mirror"] == out["texture_points_cabi"]
    mirror, cabi, start = (np.array(out[k], np.float32).reshape(-1, 12) for k in ("mirror", "cabi", "start"))
    assert np.array_equal(_bits(mirror), _bits(cabi))
    assert not np.array_equal(_bits(mirror), _bits(start))  # the refinement moved the bodies
