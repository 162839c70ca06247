"""m3tb_refine_poses = Refiner::RefinePoses (refiner.cpp:76-117) for a subset of a context's optimisers, against the
oracle's per-body start / correspondence / update functions run on the same subset.

Gates, as elsewhere: per-line and per-point state bit-exact at every correspondence iteration (ROTATION_LINEAR /
EXP_RODRIGUES oracle, no pose update in between), the pose within 1e-4 m / 1e-4 rad of the reference-faithful oracle
(polar rotation(), Pade exp). Every body and structure that is not named keeps its state bit for bit.
"""
import ctypes as C

import numpy as np
import pytest

from helpers import assert_lines_bit_equal, assert_points_bit_equal, pose_error

pytestmark = pytest.mark.gpu

TOL_POSE_M = 1e-4
TOL_POSE_RAD = 1e-4
OK, ERR_INVALID, ERR_CUDA, ERR_UNSUPPORTED = 0, -1, -2, -3  # m3tb_status


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _workload(synth, n=6, seed=31, **kw):
    return synth.make_workload("c2", n_bodies=n, n_lines=200, n_points=200, n_divides=3, seed=seed, **kw)


def _oracle_refine(oracle, orc, bodies, n_corr, n_update):
    """Refiner::ExecuteRefinementStep on the oracle for the rigid bodies `bodies`: the per-body functions run on a
    compact copy of those bodies (a shared histogram object then sees only the refined members), copied back after."""
    L = orc.L
    sub = (oracle.Body * len(bodies))()
    for i, b in enumerate(bodies):
        sub[i] = orc.bodies[b]
    for corr in range(n_corr):
        L.orc_start_modalities(sub, len(bodies), 0, orc.rotation_mode, 1)
        L.orc_tracking_step(sub, len(bodies), 0, corr, corr + 1, n_update, orc.rotation_mode, orc.exp_mode, 1, None)
    for i, b in enumerate(bodies):
        orc.bodies[b] = sub[i]
    orc._mirror_shared_histograms()


def _state(ctx, wl, b):
    """Everything of body b that a refinement of other bodies must leave alone."""
    nb = wl.region.n_histogram_bins
    hf, hb = ctx.get_histograms(b, nb)
    return dict(pose=_bits(ctx.get_poses()[b]), hf=_bits(hf), hb=_bits(hb),
                lines=ctx.get_region_lines(b, wl.lines_per_body).tobytes(),
                points=ctx.get_depth_points(b, wl.points_per_body).tobytes(),
                views=ctx.get_closest_views(b))


def _assert_same_state(before, after, bodies):
    for b in bodies:
        for k in before[b]:
            x, y = before[b][k], after[b][k]
            same = np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y
            assert same, (b, k)


def _tracked_context(capi, wl):
    """A context whose bodies carry state of their own: started and one tracking step behind them."""
    ctx = capi.context_from_workload(wl)
    ctx.start_modalities(0)
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    ctx.synchronize()
    return ctx


def test_refine_subset_follows_oracle_and_leaves_others(capi, oracle, synth):
    wl = _workload(synth)
    refined, others = [1, 3], [0, 2, 4, 5]
    ctx = _tracked_context(capi, wl)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_POLAR, exp_mode=oracle.EXP_PADE)
    orc.set_poses(ctx.get_poses())
    before = {b: _state(ctx, wl, b) for b in others}
    ctx.refine_poses(refined, (), 7, 2)
    _oracle_refine(oracle, orc, refined, 7, 2)
    dt, dr = pose_error(ctx.get_poses()[refined], orc.get_poses()[refined])
    assert dt.max() < TOL_POSE_M and dr.max() < TOL_POSE_RAD, (dt, dr)
    assert ctx.last_launch()["kernel"] == "k_track"
    _assert_same_state(before, {b: _state(ctx, wl, b) for b in others}, others)
    ctx.close()


@pytest.mark.parametrize("n_corr", [1, 3, 5])
def test_refine_state_bit_exact_per_corr_iteration(capi, oracle, synth, n_corr):
    """Without pose updates every correspondence iteration starts from the same pose on both sides: the histograms
    and the lines / points of the last iteration (its scale and standard deviations) are bit-exact."""
    wl = _workload(synth)
    refined = [1, 3]
    ctx = capi.context_from_workload(wl)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    ctx.refine_poses(refined, (), n_corr, 0)
    _oracle_refine(oracle, orc, refined, n_corr, 0)
    nb = wl.region.n_histogram_bins
    for b in refined:
        hf, hb = ctx.get_histograms(b, nb)
        assert np.array_equal(_bits(hf), _bits(orc.hist_f[b])) and np.array_equal(_bits(hb), _bits(orc.hist_b[b])), b
        B = orc.bodies[b]
        assert ctx.get_closest_views(b) == (B.region_view, B.depth_view)
        assert_lines_bit_equal(ctx.get_region_lines(b, wl.lines_per_body), orc.lines[b][:B.n_lines])
        assert_points_bit_equal(ctx.get_depth_points(b, wl.points_per_body), orc.points[b][:B.n_points])
    ctx.close()


def test_refine_leaves_no_trace_on_the_others(capi, synth):
    """After a refinement of {1, 3}, tracking and a histogram update of the whole context move the other bodies exactly
    as in a twin context that never refined. With measured occlusion handling from 3 iterations after the start on, a
    first_iteration written for another body would switch that body's handling on at iteration 11."""
    from test_oracle_occlusion import occluded_workload
    wl = occluded_workload(n_bodies=6, n_unoccluded_iterations=3)
    wl.depth.n_unoccluded_iterations = 3
    twins = [capi.context_from_workload(wl) for _ in range(2)]
    for ctx in twins:
        ctx.start_modalities(10)
        ctx.tracking_step(10, wl.n_corr_iterations, wl.n_update_iterations)
        ctx.calculate_results(10)
    a, b = twins
    a.refine_poses([1, 3], (), 7, 2)
    for ctx in twins:
        ctx.tracking_step(11, wl.n_corr_iterations, wl.n_update_iterations)
        ctx.calculate_results(11)
    others = [0, 2, 4, 5]
    for body in others:
        sa, sb = _state(a, wl, body), _state(b, wl, body)
        _assert_same_state({body: sa}, {body: sb}, [body])
    assert not np.array_equal(_bits(a.get_poses()[[1, 3]]), _bits(b.get_poses()[[1, 3]]))
    a.close()
    b.close()


def test_refine_all_bodies_matches_the_start_and_corr_composition(capi, synth, monkeypatch):
    """Refining every body is the composition start_modalities + corr_iteration per correspondence iteration: bit for
    bit when the composition runs k_track too, within the pose gate against its k_track2 path (both from a tracked
    state, where no closest-view switch or line truncation separates the two kernels' last bits)."""
    wl = _workload(synth)

    def composition(ctx):
        for corr in range(7):
            ctx.start_modalities(0)
            ctx.corr_iteration(0, corr, 2)

    a = capi.context_from_workload(wl)
    monkeypatch.setenv("M3TB_KERNEL", "1")
    b = capi.context_from_workload(wl)
    monkeypatch.delenv("M3TB_KERNEL")
    a.refine_poses(range(wl.n_bodies), (), 7, 2)
    composition(b)
    assert b.last_launch()["kernel"] == "k_track"
    assert np.array_equal(_bits(a.get_poses()), _bits(b.get_poses()))
    a.close()
    b.close()
    a, b = _tracked_context(capi, wl), _tracked_context(capi, wl)
    a.refine_poses(range(wl.n_bodies), (), 7, 2)
    composition(b)
    assert b.last_launch()["kernel"] == "k_track2"
    dt, dr = pose_error(a.get_poses(), b.get_poses())
    assert dt.max() < TOL_POSE_M and dr.max() < TOL_POSE_RAD, (dt, dr)
    a.close()
    b.close()


def test_refine_one_of_two_chains(capi, oracle, synth):
    """Chain 0 of two follows the oracle's structure refinement, one correspondence iteration per call on identical
    inputs (the oracle starts each call from the device's body and joint poses: a chain's first iterations expand
    last-bit differences, so free-running trajectories are no gate); chain 1 keeps its state bit for bit."""
    wl = synth.make_chain_workload(n_chains=2, n_links=4, n_lines=200, n_points=200, n_divides=3, seed=8)
    ctx = capi.context_from_workload(wl)
    assert ctx.n_structures() == 2
    ctx.start_modalities(0)
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    other = [4, 5, 6, 7]
    before = {b: _state(ctx, wl, b) for b in other}
    links_before = [x.copy() for x in ctx.get_link_poses(1, 4)]
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_POLAR, exp_mode=oracle.EXP_PADE)
    L, S = orc.L, C.pointer(orc.structures[0])
    sub = (oracle.Body * 4)()
    for step in range(3):
        poses0 = ctx.get_poses()
        b2j, j2p, _ = ctx.get_link_poses(0, 4)
        for k in range(4):
            orc.structure_objs[0].links[k].body2joint[:] = b2j[k].reshape(12).tolist()
            orc.structure_objs[0].links[k].joint2parent[:] = j2p[k].reshape(12).tolist()
        ctx.refine_poses((), [0], 1, 2)
        # oracle: CalculateConsistentPoses, start modalities of the chain, one structure step at correspondence iteration 0
        l2w = np.ascontiguousarray(poses0[:4].reshape(4, 12))
        L.orc_structure_consistent_poses(S, orc.exp_mode, oracle.ptr(l2w))
        orc.set_poses(np.concatenate([l2w.reshape(4, 3, 4), poses0[4:]]))
        for i in range(4):
            sub[i] = orc.bodies[i]
        L.orc_start_modalities(sub, 4, 0, orc.rotation_mode, 1)
        for i in range(4):
            orc.bodies[i] = sub[i]
        L.orc_tracking_step_structures(orc.bodies, S, 1, 0, 0, 1, 2, orc.rotation_mode, orc.exp_mode, 1,
                                       oracle.ptr(orc.bodyless), orc.max_links)
        dt, dr = pose_error(ctx.get_poses()[:4], orc.get_poses()[:4])
        assert dt.max() < TOL_POSE_M and dr.max() < TOL_POSE_RAD, (step, dt, dr)
    ctx.refine_poses((), [0], 7, 2)
    _assert_same_state(before, {b: _state(ctx, wl, b) for b in other}, other)
    for x, y in zip(links_before, ctx.get_link_poses(1, 4)):
        assert np.array_equal(_bits(x), _bits(y))
    ctx.close()


def test_refine_one_member_of_a_shared_histogram_object(capi, oracle, synth):
    wl = _workload(synth)
    wl.histogram_owner = np.array([0, 0, 0, -1, -1, -1], np.int32)
    ctx = _tracked_context(capi, wl)
    orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    orc.set_poses(ctx.get_poses())
    nb = wl.region.n_histogram_bins
    h_alone_before = ctx.get_histograms(3, nb)
    ctx.refine_poses([1], (), 1, 0)
    _oracle_refine(oracle, orc, [1], 1, 0)
    ref_f, ref_b = orc.hist_f[0], orc.hist_b[0]  # the object, from body 1's line pixels only
    for b in (0, 1, 2):
        hf, hb = ctx.get_histograms(b, nb)
        assert np.array_equal(_bits(hf), _bits(ref_f)) and np.array_equal(_bits(hb), _bits(ref_b)), b
    h3 = ctx.get_histograms(3, nb)
    assert np.array_equal(_bits(h3[0]), _bits(h_alone_before[0]))
    # what the three members together would give is different
    o3 = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
    o3.set_poses(ctx.get_poses())
    _oracle_refine(oracle, o3, [0, 1, 2], 1, 0)
    assert not np.array_equal(_bits(o3.hist_f[0]), _bits(ref_f))
    ctx.close()


def test_refine_with_pinned_and_pageable_frames(capi, synth):
    import torch
    wl = _workload(synth)
    pin_c = torch.from_numpy(wl.color_frames.copy()).pin_memory()
    pin_d = torch.from_numpy(wl.depth_frames.view(np.uint8).reshape(wl.n_bodies, wl.depth_frames.shape[1], -1).copy()).pin_memory()
    out = []
    for pinned in (False, True):
        ctx = capi.context_from_workload(wl, upload_frames=not pinned)
        if pinned:
            ctx.upload_batch_ptr(True, 0, wl.n_bodies, pin_c.data_ptr(), pin_c.stride(0), pin_c.stride(1))
            ctx.upload_batch_ptr(False, 0, wl.n_bodies, pin_d.data_ptr(), pin_d.stride(0), pin_d.stride(1))
        ctx.refine_poses([2, 4], (), 7, 2)
        p_refined = ctx.get_poses()
        ctx.start_modalities(0)  # the other bodies' rectangles are fetched by the next launch over the context
        ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
        hf, hb = ctx.get_histograms(4, wl.region.n_histogram_bins)
        out.append((p_refined, ctx.get_poses(), hf, hb))
        ctx.close()
    for x, y in zip(out[0], out[1]):
        assert np.array_equal(_bits(x), _bits(y))


def test_refusals_empty_selection_and_allocation_failure(capi, synth):
    wl = _workload(synth, n=4)
    ctx = capi.context_from_workload(wl)
    ctx.start_modalities(0)
    ctx.synchronize()
    poses = ctx.get_poses()
    n0 = ctx.launch_count
    ctx.refine_poses((), (), 7, 2)
    assert ctx.launch_count == n0
    L = capi.lib()
    for bodies, structures, nc, nu in (([4], [], 7, 2), ([-1], [], 7, 2), ([1, 1], [], 7, 2), ([1], [], -1, 2),
                                       ([1], [], 7, -1), ([], [0], 7, 2)):
        b = (C.c_int * max(1, len(bodies)))(*bodies)
        s = (C.c_int * max(1, len(structures)))(*structures)
        rc = L.m3tb_refine_poses(ctx.h, b, len(bodies), s, len(structures), nc, nu)
        assert rc == ERR_INVALID, (bodies, structures, nc, nu, rc)
    assert ctx.launch_count == n0
    # an injected allocation failure (the device list is made by the first refinement) leaves the context as it was
    live = capi.debug_resources()
    capi.debug_resources(1)
    try:
        rc = L.m3tb_refine_poses(ctx.h, (C.c_int * 1)(1), 1, (C.c_int * 1)(), 0, 7, 2)
    finally:
        capi.debug_resources(0)
    assert rc == ERR_CUDA
    assert capi.debug_resources() == live and ctx.launch_count == n0
    assert np.array_equal(_bits(ctx.get_poses()), _bits(poses))
    ctx.refine_poses([1], (), 7, 2)
    assert ctx.launch_count > n0
    ctx.close()


def test_refusals_for_links_and_texture_bodies(capi, synth):
    wl = synth.make_chain_workload(n_chains=2, n_links=2, n_lines=64, n_points=64, n_divides=2, seed=3)
    ctx = capi.context_from_workload(wl)
    L = capi.lib()
    rc = L.m3tb_refine_poses(ctx.h, (C.c_int * 1)(1), 1, (C.c_int * 1)(), 0, 7, 2)
    assert rc == ERR_INVALID  # a link's body: the structure has to be named
    rc = L.m3tb_refine_poses(ctx.h, (C.c_int * 1)(), 0, (C.c_int * 2)(1, 1), 2, 7, 2)
    assert rc == ERR_INVALID
    rc = L.m3tb_refine_poses(ctx.h, (C.c_int * 1)(), 0, (C.c_int * 1)(2), 1, 7, 2)
    assert rc == ERR_INVALID  # structure ids are 0 and 1
    tri, _ = synth.prism_triangles()
    ctx.set_body_geometry(3, tri)
    ctx.set_texture_modality(3, capi.texture_params_default(), 3)
    n0 = ctx.launch_count
    rc = L.m3tb_refine_poses(ctx.h, (C.c_int * 1)(), 0, (C.c_int * 1)(1), 1, 7, 2)
    assert rc == ERR_UNSUPPORTED  # body 3 is a link of chain 1
    assert ctx.launch_count == n0
    ctx.refine_poses((), [0], 1, 1)  # chain 0 has no texture body
    ctx.close()
    wl = _workload(synth, n=3)
    ctx = capi.context_from_workload(wl)
    ctx.set_body_geometry(2, tri)
    ctx.set_texture_modality(2, capi.texture_params_default(), 2)
    rc = L.m3tb_refine_poses(ctx.h, (C.c_int * 2)(0, 2), 2, (C.c_int * 1)(), 0, 7, 2)
    assert rc == ERR_UNSUPPORTED
    ctx.close()


def test_refine_with_device_renderers_and_modeled_occlusion(capi, oracle, synth):
    """Device renderers with modeled occlusion, region checking and silhouette checking (renderer 2b: body b's colour
    camera, 2b + 1: its depth camera, each drawing bodies b and b + 1). Each refinement call of one correspondence
    iteration follows the oracle fed the CPU restatement of the renderings at the pose it starts from; the refined
    bodies' renderers hold exactly those images afterwards, and the renderers of the other bodies keep their last
    image bit for bit, as does the other bodies' state."""
    import copy
    import render_reference as rr
    from test_gpu_device_renderers import _device_context, _scene, _workload
    wl = _workload(synth)
    ctx = _device_context(capi, synth, wl)
    ctx.start_modalities(0)
    ctx.tracking_step(0, wl.n_corr_iterations, wl.n_update_iterations)
    refined, others = [1, 3], [0, 2, 4]
    geometry, renderers = _scene(synth, wl)
    before = {b: _state(ctx, wl, b) for b in others}
    images_before = {k: ctx.get_rendering(k) for k, r in enumerate(renderers) if r["body"] in others}

    def cpu_renderings(poses):
        pd = {b: poses[b] for b in range(wl.n_bodies)}
        out, images = {}, {}
        for k, r in enumerate(renderers):
            m = "region" if r["kind"] == "color" else "depth"
            intr = wl.color_intrinsics if m == "region" else wl.depth_intrinsics
            w2c = wl.color_world2camera if m == "region" else wl.depth_world2camera
            o = rr.render_focused(intr, w2c, pd, geometry, r["geometry"], r["referenced"], id_type=r["id_type"])
            images[k] = o
            common = (float(o["corner_u"]), float(o["corner_v"]), float(o["scale"]))
            vis = bool(o["visible"][0])
            sid = 7 if m == "region" else r["body"] + 1
            per = out.setdefault(r["body"], {})
            per[f"{m}_depth"] = synth.Rendering(o["depth"], *common, float(o["projection_term_a"]),
                                                float(o["projection_term_b"]), 0, vis)
            per[f"{m}_silhouette"] = synth.Rendering(o["silhouette"], *common, 0.0, 0.0, sid, vis)
        return out, images

    for step in range(3):
        start = ctx.get_poses()
        rendered, images = cpu_renderings(start)
        ctx.refine_poses(refined, (), 1, 2)
        fed = copy.copy(wl)
        fed.renderings = rendered
        orc = oracle.OracleTracker(fed, rotation_mode=oracle.ROTATION_POLAR, exp_mode=oracle.EXP_PADE)
        orc.set_poses(start)
        _oracle_refine(oracle, orc, refined, 1, 2)
        dt, dr = pose_error(ctx.get_poses()[refined], orc.get_poses()[refined])
        assert dt.max() < TOL_POSE_M and dr.max() < TOL_POSE_RAD, (step, dt, dr)
        for k, r in enumerate(renderers):
            if r["body"] in refined:  # drawn at the pose this call started from
                got = ctx.get_rendering(k)
                assert np.array_equal(got["depth"], images[k]["depth"]), (step, k)
                assert np.array_equal(got["silhouette"], images[k]["silhouette"]), (step, k)
                assert _bits(got["scale"]) == _bits(images[k]["scale"]), (step, k)
    for k, old in images_before.items():
        new = ctx.get_rendering(k)
        for key in old:
            assert np.array_equal(np.asarray(old[key]), np.asarray(new[key])), (k, key)
    _assert_same_state(before, {b: _state(ctx, wl, b) for b in others}, others)
    assert ctx.last_launch()["occ"] == 1
    ctx.close()
