"""The state a context carries from one frame to the next, held to the mirror oracle over frame sequences.

One context tracks a sequence of frames whose ground truth moves a few mm and degrees per frame. Each frame reaches it by
one of the upload paths of PATHS, and the schedule also changes the histogram resolution, jumps bodies after their ROI
was fetched and refines a subset of bodies between frames. After every launch the camera's bin-index image (the source
of k_track2's TMA colour tiles, m3tb_debug_bin_image) must equal the restatement of ColorHistograms' bin index
(color_histograms.cpp:97-99) wherever its state says it is valid, and every correspondence iteration must be
bit-exact against the oracle. A twin context that gets each frame by a plain pageable copy, and the stateful context's
histograms, must give bit-identical results whenever it runs the same kernel: any difference is stale state."""
import ctypes as C

import numpy as np
import pytest

from helpers import assert_lines_bit_equal, assert_points_bit_equal, pose_error, record, rel_to_max
from test_lut_slot import lut_slot

# How a frame reaches the context:
#   pageable        per-camera upload_color / upload_depth from pageable memory (Upload's copy branch)
#   batch           one pageable upload_*_batch into the pooled frames
#   device          per-camera m3tb_upload_*_device from device memory
#   pinned_packed   pinned batch, rows 3 W bytes apart. IngestColorRect unpacks 16 pixels at a time (Bins16) when the
#                   host rows are 16-byte aligned: at 644 px (1932-byte rows) they are not, and every rectangle takes the
#                   scalar path; at 640 / 1280 px (1920 / 3840-byte rows) they are, and it takes Bins16
#   pinned_aligned  pinned batch, rows padded to 16 bytes: Bins16 at every size (colour rectangles are always 16-px
#                   aligned, BoxRect / RoiRect)
#   prefetch        pinned (packed) batch, then prefetch_frames: the ingest runs on the side stream into the other pool
#   detach          pinned (packed) batch, detach_frames after the first consumer: the rest of the frame reads the full copy
#   undistorted     pageable batch through an undistortion map (k_undistort); the oracle gets the rectified frame
PATHS = ("pageable", "batch", "device", "pinned_packed", "pinned_aligned", "prefetch", "detach", "undistorted")
PINNED = ("pinned_packed", "pinned_aligned", "prefetch", "detach")
FULL = ("pageable", "batch", "device", "undistorted")
BIN_CYCLE = (16, 8, 32, 2, 64, 16)  # the histogram resolutions the schedule moves through, in this order
SIZES = {"640x480": (614.0, 614.5, 321.3, 238.9, 640, 480),
         "644x480": (614.0, 614.5, 322.8, 238.9, 644, 480),  # width a multiple of 4 but not of 16
         "1280x720": (912.0, 912.5, 640.3, 359.6, 1280, 720)}

# One sequence per row: frame size, upload path of each frame, histogram bins of each frame, and the frames after whose
# tracking some bodies jump (JUMP_BODIES, beyond the ingest's motion margin) and before whose tracking some bodies are
# refined (REFINE_BODIES). The first eight rows keep one resolution of <= 32 bins, so that every frame-to-frame
# transition can show a bin-index image kept stale across it (a resolution change or 64 bins rebuilds or drops the image
# anyway); their paths, joined, walk every ordered pair of distinct paths once. The last row moves through BIN_CYCLE.
SCHEDULE = [
    dict(size="640x480", bins=(16,) * 8, jump=(4,), refine=(),
         paths=("pageable", "undistorted", "detach", "undistorted", "prefetch", "undistorted", "pinned_aligned", "undistorted")),
    dict(size="644x480", bins=(8,) * 8, jump=(1,), refine=(),
         paths=("undistorted", "pinned_packed", "undistorted", "device", "undistorted", "batch", "undistorted", "pageable")),
    dict(size="1280x720", bins=(32,) * 8, jump=(), refine=(6,),
         paths=("pageable", "detach", "prefetch", "detach", "pinned_aligned", "detach", "pinned_packed", "detach")),
    dict(size="640x480", bins=(2,) * 8, jump=(6,), refine=(),
         paths=("detach", "device", "detach", "batch", "detach", "pageable", "prefetch", "pinned_aligned")),
    dict(size="644x480", bins=(16,) * 8, jump=(5,), refine=(2,),
         paths=("pinned_aligned", "prefetch", "pinned_packed", "prefetch", "device", "prefetch", "batch", "prefetch")),
    dict(size="1280x720", bins=(16,) * 8, jump=(2,), refine=(3,),
         paths=("prefetch", "pageable", "pinned_aligned", "pinned_packed", "pinned_aligned", "device", "pinned_aligned", "batch")),
    dict(size="640x480", bins=(16,) * 8, jump=(3,), refine=(1,),
         paths=("batch", "pinned_aligned", "pageable", "pinned_packed", "device", "pinned_packed", "batch", "pinned_packed")),
    dict(size="644x480", bins=(32,) * 8, jump=(), refine=(),
         paths=("pinned_packed", "pageable", "device", "batch", "device", "pageable", "batch", "pageable")),
    dict(size="640x480", bins=BIN_CYCLE, jump=(), refine=(),
         paths=("pinned_aligned", "batch", "prefetch", "pinned_packed", "pageable", "detach")),
]
# One colour (and depth) camera per object, each object tracked by two bodies: bins[0] is the resolution of the first
# body on every camera, bins[1] of the second. path None: the resolution changes on the frame the cameras already hold.
# Bodies of different resolutions write one bin-index image with different bit shifts, so its state must say none.
SHARED_STEPS = (
    dict(path="pinned_aligned", bins=(16, 32)),  # mixed at the ingest (NoteIngestBins sees the bodies disagree)
    dict(path=None, bins=(16, 16)),              # unified on that pinned frame: its image still holds mixed shifts
    dict(path="pinned_aligned", bins=(16, 16)),  # a fresh pinned frame at one resolution: valid over the rectangles
    dict(path="batch", bins=(8, 32)),            # mixed on a full copy: no k_bin
    dict(path=None, bins=(32, 32)),              # unified on that full copy: k_bin rebuilds the whole image
)
JUMP_BODIES = (0, 1, 2, 3)       # mid-edge bodies 20 px inside the frame: jumped towards its centre
JUMP_PX = 35.0                   # > kIngestMotionMarginPx (8 px): the jumped lines reach outside the fetched rectangle
REFINE_BODIES = (1, 3, 5)
N_CORR = 7


def _bitshift(n_bins):
    return 8 - int(np.log2(n_bins))  # color_histograms.cpp:131-159


def restated_bins(frame, width, n_bins):
    """Lookup-table slot of every pixel of a BGR frame [H, >= 3 W] at `n_bins` bins (color_histograms.cpp:97-99)."""
    s, nb = _bitshift(n_bins), n_bins
    px = np.asarray(frame)[:, :3 * width].reshape(frame.shape[0], width, 3).astype(np.int64)
    return lut_slot(((px[..., 0] >> s) * nb + (px[..., 1] >> s)) * nb + (px[..., 2] >> s)).astype(np.uint16)


def _roi_mask(info):
    """Pixels of a pinned frame whose device copy (and bin indices) the current ingest fetched."""
    m = np.zeros((info["height"], info["width"]), bool)
    for r in info["rois"]:
        if r["generation"] == info["generation"]:
            m[r["y0"]:r["y1"], r["x0"]:r["x1"]] = True
    return m


def check_bin_images(ctx, wl, expect_state=None, cache=None, n_cameras=None):
    """The bin-index image of every camera equals the restatement wherever its state says it is valid. expect_state:
    the state every camera must report; cache: restatements of the current frames by (camera, state); camera k shows
    wl.color_frames[k] (n_cameras of them, default one per body)."""
    cache = {} if cache is None else cache
    for cam in range(wl.n_bodies if n_cameras is None else n_cameras):
        img, info = ctx.debug_bin_image(cam)
        if expect_state is not None:
            assert info["state"] == expect_state, (cam, info["state"], expect_state)
        if info["state"] < 0 or img is None:
            continue
        W = wl.color_intrinsics.width
        key = (cam, info["state"])
        if key not in cache:
            cache[key] = restated_bins(wl.color_frames[cam], W, 2 ** (8 - info["state"]))
        ref = cache[key]
        if info["pinned"]:
            mask = _roi_mask(info)
            assert mask.any(), (cam, info)
            bad = np.argwhere(mask & (img != ref))
        else:
            bad = np.argwhere(img != ref)
        assert len(bad) == 0, (cam, info["state"], info["pinned"], len(bad), bad[:4].tolist())


def _oracle_refine(oracle, orc, bodies, n_corr):
    """Refiner::RefinePoses without pose updates on the oracle: every correspondence iteration starts the modalities."""
    L = orc.L
    sub = (oracle.Body * len(bodies))()
    for i, b in enumerate(bodies):
        sub[i] = orc.bodies[b]
    for corr in range(n_corr):
        L.orc_start_modalities(sub, len(bodies), 0, orc.rotation_mode, 1)
        L.orc_tracking_step(sub, len(bodies), 0, corr, corr + 1, 0, orc.rotation_mode, orc.exp_mode, 1, None)
    for i, b in enumerate(bodies):
        orc.bodies[b] = sub[i]


def _stale_samples(line_rec, roi, scale, W, H):
    """Lines one of whose end samples lies inside the frame but outside the fetched rectangle."""
    h = 0.5 * 19 * scale
    n = 0
    for e in (-h, h):
        u = line_rec["center_u"] + e * line_rec["normal_u"]
        v = line_rec["center_v"] + e * line_rec["normal_v"]
        inside = (u >= 0) & (u < W) & (v >= 0) & (v < H)
        outside_roi = (u < roi["x0"]) | (u >= roi["x1"]) | (v < roi["y0"]) | (v >= roi["y1"])
        n += int((inside & outside_roi).sum())
    return n


def test_schedule_covers_every_path_pair_and_resolution_change():
    """Every upload path runs at least twice and follows every other path at least once between two frames of one
    resolution of <= 32 bins (where only the upload paths decide whether the bin-index image is rebuilt); every
    resolution change of BIN_CYCLE happens; the scalar ingest path (packed 644 px rows at <= 32 bins) runs; jumps land on
    pinned frames at <= 32 bins and refinements on fresh pinned frames; the shared-camera steps mix resolutions on a
    pinned and on a full-copy frame and unify them on each."""
    counts = {p: 0 for p in PATHS}
    pairs, changes = set(), set()
    scalar = False
    for seq in SCHEDULE:
        assert seq["size"] in SIZES and len(seq["paths"]) == len(seq["bins"]) and 6 <= len(seq["paths"]) <= 8
        for i, p in enumerate(seq["paths"]):
            counts[p] += 1
            scalar |= seq["size"] == "644x480" and p in ("pinned_packed", "prefetch", "detach") and seq["bins"][i] <= 32
            if i:
                if seq["bins"][i] == seq["bins"][i - 1] <= 32:
                    pairs.add((seq["paths"][i - 1], p))
                if seq["bins"][i] != seq["bins"][i - 1]:
                    changes.add((seq["bins"][i - 1], seq["bins"][i]))
        for f in seq["jump"]:
            assert seq["paths"][f] in ("pinned_packed", "pinned_aligned", "prefetch") and seq["bins"][f] <= 32, seq
        for f in seq["refine"]:
            assert f > 0 and seq["paths"][f] in ("pinned_packed", "pinned_aligned") and seq["bins"][f] == seq["bins"][f - 1], seq
    assert all(c >= 2 for c in counts.values()), counts
    missing = {(a, b) for a in PATHS for b in PATHS if a != b} - pairs
    assert not missing, sorted(missing)
    assert set(zip(BIN_CYCLE, BIN_CYCLE[1:])) <= changes, changes
    assert {s["size"] for s in SCHEDULE} == set(SIZES)
    assert scalar
    assert any(s["jump"] for s in SCHEDULE) and any(s["refine"] for s in SCHEDULE)
    kinds = set()
    for i, st in enumerate(SHARED_STEPS):
        mixed = len(set(st["bins"])) > 1
        frame = st["path"] if st["path"] is not None else SHARED_STEPS[i - 1]["path"]
        kinds.add((mixed, frame in PINNED, st["path"] is None))
        assert st["path"] is not None or i > 0
    # mixed on a fresh pinned / full-copy frame, then unified on that same frame
    assert {(True, True, False), (False, True, True), (True, False, False), (False, False, True)} <= kinds, kinds


def test_bin_restatement_matches_the_index_order():
    """restated_bins is ColorHistograms' index (B, G, R memory order, the blue bin most significant) through LutSlot."""
    frame = np.array([[10, 200, 255, 0, 0, 0]], np.uint8)
    out = restated_bins(frame, 2, 16)
    assert out[0, 0] == lut_slot(((10 >> 4) * 16 + (200 >> 4)) * 16 + (255 >> 4)) and out[0, 1] == 0
    assert restated_bins(frame, 2, 2)[0, 0] == lut_slot(0 * 4 + 1 * 2 + 1)


# ---- GPU ---------------------------------------------------------------------------------------------------------------

class _Sequence:
    """One stateful context, one twin, one mirror oracle over the frames of one SCHEDULE row."""

    def __init__(self, capi, oracle, synth, seq, seed):
        import torch
        self.capi, self.oracle, self.synth, self.seq, self.seed = capi, oracle, synth, seq, seed
        ci = synth.Intrinsics(*SIZES[seq["size"]])
        wl = synth.make_edge_workload("border", "region+depth", n_divides=2, seed=seed, color_intrinsics=ci)
        wl.region.n_histogram_bins = seq["bins"][0]
        self.wl = wl
        self.W, self.H = ci.width, ci.height
        self.gt = wl.gt_body2world.copy()
        self.ctx = capi.context_from_workload(wl, upload_frames=False)
        self.twin = capi.context_from_workload(wl, upload_frames=False)
        self.orc = oracle.OracleTracker(wl, rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
        nb, H, W = wl.n_bodies, self.H, self.W
        self.pin_packed = torch.empty((nb, H, 3 * W), dtype=torch.uint8).pin_memory()
        self.pin_aligned = torch.empty(tuple(wl.color_frames.shape), dtype=torch.uint8).pin_memory()
        self.pin_depth = torch.empty((nb, wl.depth_intrinsics.height, 2 * wl.depth_intrinsics.width), dtype=torch.uint8).pin_memory()
        self.rec = dict(worst_m=[], worst_rad=[], launches=set(), stale_samples=0, twin_compared=0, discrete_events=[])

    def close(self):
        self.ctx.close()
        self.twin.close()

    # -- frames --
    def render(self, f):
        wl, s = self.wl, self.synth
        if f == 0:
            return
        for b in range(wl.n_bodies):
            self.gt[b] = s.perturb_pose(self.seed * 131 + f, b, 1.5, 0.003, self.gt[b])
            s.render_color(wl.color_intrinsics, s.pose_mul(wl.color_world2camera, self.gt[b]), self.seed * 7919 + 97 * f + b,
                           out=wl.color_frames[b])
            s.render_depth(wl.depth_intrinsics, s.pose_mul(wl.depth_world2camera, self.gt[b]), self.seed * 7919 + 97 * f + b,
                           depth_scale=wl.depth_scale, out=wl.depth_frames[b])

    def upload(self, path):
        import torch
        ctx, wl, nb, W = self.ctx, self.wl, self.wl.n_bodies, self.W
        dview = wl.depth_frames.view(np.uint8).reshape(self.pin_depth.shape)
        if path == "pageable":
            for b in range(nb):
                ctx.upload_color(b, wl.color_frames[b])
                ctx.upload_depth(b, wl.depth_frames[b])
        elif path == "batch":
            ctx.upload_color_batch(0, wl.color_frames)
            ctx.upload_depth_batch(0, wl.depth_frames)
        elif path == "device":
            dc = torch.from_numpy(wl.color_frames).cuda()
            dd = torch.from_numpy(wl.depth_frames.view(np.int16)).cuda()
            torch.cuda.synchronize()
            for b in range(nb):
                ctx._ck(ctx.L.m3tb_upload_color_device(ctx.h, b, C.c_void_p(dc[b].data_ptr()), dc.stride(1)))
                ctx._ck(ctx.L.m3tb_upload_depth_device(ctx.h, b, C.c_void_p(dd[b].data_ptr()), 2 * dd.stride(1)))
            ctx.synchronize()
            del dc, dd
        elif path == "undistorted":
            raw = wl.color_frames.copy()
            m = self.capi.undistortion_map(wl.color_intrinsics, np.array([0.05, -0.01, 5e-4, -5e-4, 2e-3, 0.03, -0.01, 1e-3],
                                                                         np.float32), wl.color_intrinsics)
            for b in range(nb):
                ctx.set_camera_undistortion("color", b, m, 3)
            ctx.upload_color_batch(0, raw)
            ctx.upload_depth_batch(0, wl.depth_frames)
            for b in range(nb):  # the oracle and the twin see the rectified frame
                wl.color_frames[b, :, :3 * W] = ctx.get_camera_image("color", b, W, self.H).reshape(self.H, 3 * W)
                ctx.set_camera_undistortion("color", b, None, 3)
        else:
            if path == "pinned_aligned":
                pin = self.pin_aligned
                pin.numpy()[:] = wl.color_frames
            else:
                pin = self.pin_packed
                pin.numpy()[:] = wl.color_frames[:, :, :3 * W]
            self.pin_depth.numpy()[:] = dview
            ctx.upload_batch_ptr(True, 0, nb, pin.data_ptr(), pin.stride(0), pin.stride(1))
            ctx.upload_batch_ptr(False, 0, nb, self.pin_depth.data_ptr(), self.pin_depth.stride(0), self.pin_depth.stride(1))
            if path == "prefetch":
                ctx.prefetch_frames()
        self.twin.upload_color_batch(0, wl.color_frames)
        self.twin.upload_depth_batch(0, wl.depth_frames)

    def set_bins(self, n_bins):
        wl, capi = self.wl, self.capi
        wl.region.n_histogram_bins = n_bins
        rp, dp = capi.region_params(wl.region), capi.depth_params(wl.depth)
        op = capi.OptimizerParams(wl.tikhonov_rotation, wl.tikhonov_translation)
        for c in (self.ctx, self.twin):
            for b in range(wl.n_bodies):
                c.set_body(b, rp, dp, op, 0, 0, b, b)
        poses = self.orc.get_poses()
        self.orc = self.oracle.OracleTracker(wl, rotation_mode=self.oracle.ROTATION_LINEAR, exp_mode=self.oracle.EXP_RODRIGUES)
        self.orc.set_poses(poses)

    # -- checks --
    def histograms_exact(self, stage):
        nb = self.wl.region.n_histogram_bins
        for b in range(self.wl.n_bodies):
            hf, hb = self.ctx.get_histograms(b, nb)
            assert np.array_equal(hf.view(np.uint32), self.orc.hist_f[b].view(np.uint32)), (stage, b)
            assert np.array_equal(hb.view(np.uint32), self.orc.hist_b[b].view(np.uint32)), (stage, b)

    def give_twin_histograms(self):
        nb = self.wl.region.n_histogram_bins
        for b in range(self.wl.n_bodies):
            self.twin.set_histograms(b, *self.ctx.get_histograms(b, nb))

    def expect_tma(self):
        return self.wl.region.n_histogram_bins <= 32

    def corr_pass(self, f, path, extras, started, stale_bodies=()):
        """N_CORR correspondence iterations, each from the mirror oracle's pose on both contexts; extras[c]: the launches
        besides the tracking kernel that iteration c must make (k_ingest, k_bin)."""
        ctx, twin, orc, wl = self.ctx, self.twin, self.orc, self.wl
        deltas, worst = [], [0.0, 0.0]
        scales = list(wl.region.scales)
        for corr in range(N_CORR):
            start = orc.get_poses()
            ctx.set_poses(start)
            twin.set_poses(start)
            n0 = ctx.launch_count
            ctx.corr_iteration(0, corr, wl.n_update_iterations)
            deltas.append(ctx.launch_count - n0)
            launch = ctx.last_launch()
            self.rec["launches"].add((launch["kernel"], launch["tma_mode"]))
            if self.expect_tma():
                assert launch["kernel"] == "k_track2" and launch["tma_mode"] != 0, (f, path, corr, launch)
                check_bin_images(ctx, wl, expect_state=_bitshift(wl.region.n_histogram_bins), cache=self.bins_cache)
            else:
                assert launch["kernel"] == "k_track", (f, path, corr, launch)
                check_bin_images(ctx, wl, cache=self.bins_cache)
            gpu = ctx.get_poses()
            twin.corr_iteration(0, corr, wl.n_update_iterations)
            same_kernel = twin.last_launch()["kernel"] == launch["kernel"]
            if same_kernel:
                assert np.array_equal(twin.get_poses().view(np.uint32), gpu.view(np.uint32)), (f, path, corr)
                self.rec["twin_compared"] += 1
            ogh = []
            for b in range(wl.n_bodies):
                n, view = orc.region_correspondences(b, 0, corr)
                og_r, oH_r = orc.region_gradient_hessian(b, corr, 0)
                lines = ctx.get_region_lines(b, wl.lines_per_body)
                assert ctx.get_closest_views(b)[0] == view, (f, path, corr, b)
                assert_lines_bit_equal(lines, orc.lines[b][:n])
                n, view = orc.depth_correspondences(b, 0, corr)
                assert ctx.get_closest_views(b)[1] == view, (f, path, corr, b)
                pts = ctx.get_depth_points(b, wl.points_per_body)
                assert_points_bit_equal(pts, orc.points[b][:n])
                ogh.append((og_r, oH_r) + orc.depth_gradient_hessian(b, corr))
                if same_kernel:
                    assert_lines_bit_equal(twin.get_region_lines(b, wl.lines_per_body), lines)
                    assert_points_bit_equal(twin.get_depth_points(b, wl.points_per_body), pts)
                if b in stale_bodies:
                    _, info = ctx.debug_bin_image(b)
                    self.rec["stale_samples"] += _stale_samples(lines, info["rois"][0], scales[min(corr, len(scales) - 1)],
                                                                self.W, self.H)
            orc.tracking_step(0, n_corr=corr + 1, corr_begin=corr)
            dt, dr = pose_error(gpu, orc.get_poses())
            split = (dt >= 1e-5) | (dr >= 1e-5)
            if split.any():
                # The second update iteration takes integer decisions (the local-mode bin pair) from the pose the first
                # one produced, so a last-bit difference of the g / H sums can flip one of them. Such a discrete event
                # is accepted only where the first update's g / H (the fine-grained calls, from the same start pose)
                # meet per_iteration_parity's bars, and within a bound; a sequence may hold one
                ctx.set_poses(start)
                ctx.region_correspondences(0, corr)
                ctx.depth_correspondences(0, corr)
                g_r, H_r = ctx.region_gradient_hessian(0, corr, 0)
                g_d, H_d = ctx.depth_gradient_hessian(0, corr, 0)
                for b in np.flatnonzero(split):
                    og_r, oH_r, og_d, oH_d = ogh[b]
                    e = (rel_to_max(H_r[b], oH_r), rel_to_max(g_r[b], og_r), rel_to_max(H_d[b], oH_d), rel_to_max(g_d[b], og_d))
                    assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 1e-5 and e[3] < 1e-4, (f, path, corr, b, e)
                    assert dt[b] < 1e-3 and dr[b] < 1e-2, (f, path, corr, b, dt[b], dr[b])
                    self.rec["discrete_events"].append(dict(frame=f, corr=corr, body=int(b), m=float(f"{dt[b]:.2e}"),
                                                            rad=float(f"{dr[b]:.2e}")))
            dense = ~split
            if dense.any():
                worst = [max(worst[0], dt[dense].max()), max(worst[1], dr[dense].max())]
            if path == "detach" and corr == 0 and not started:
                ctx.detach_frames()  # after the first consumer: the rest of the frame reads the full copy
        assert worst[0] < 1e-5 and worst[1] < 1e-5, (f, path, worst)
        if extras is not None:
            base = deltas[-1]
            assert [d - base for d in deltas] == extras, (f, path, deltas, extras)
        return worst

    def run(self):
        seq = self.seq
        ctx, wl = self.ctx, self.wl
        for f, path in enumerate(seq["paths"]):
            self.render(f)
            n_bins = seq["bins"][f]
            changed = f > 0 and n_bins != seq["bins"][f - 1]
            if changed:
                self.set_bins(n_bins)
            self.upload(path)
            self.bins_cache = {}
            started = f == 0 or changed
            if started:  # the reference's SetUp / StartModalities after a resolution change
                ctx.start_modalities(0)
                self.twin.start_modalities(0)
                self.orc.start_modalities(0)
                self.histograms_exact("start")
                if path == "detach":
                    ctx.detach_frames()
            check_bin_images(ctx, wl, cache=self.bins_cache)
            if f in seq["refine"]:
                ctx.refine_poses(REFINE_BODIES, (), N_CORR, 0)
                _oracle_refine(self.oracle, self.orc, REFINE_BODIES, N_CORR)
                for b in REFINE_BODIES:
                    B = self.orc.bodies[b]
                    assert_lines_bit_equal(ctx.get_region_lines(b, wl.lines_per_body), self.orc.lines[b][:B.n_lines])
                    assert ctx.get_closest_views(b)[0] == B.region_view
                self.histograms_exact("refine")
                # a refinement fetches its bodies' rectangles only: the bin images wait for the next full ingest
                for b in REFINE_BODIES:
                    assert ctx.debug_bin_image(b)[1]["state"] == self.capi.BINS_AT_INGEST
                check_bin_images(ctx, wl, cache=self.bins_cache)
            # launches besides the tracking kernel: the pinned frame's ingest at its first consumer, k_bin after a full
            # copy (or the detach) when the batch stages TMA tiles
            extras = [0] * N_CORR
            if path in ("pinned_packed", "pinned_aligned", "detach") and not started:
                extras[0] += 1
            if self.expect_tma() and (path in FULL or (path == "detach" and started)):
                extras[0] += 1
            if self.expect_tma() and path == "detach" and not started:
                extras[1] += 1
            self.give_twin_histograms()
            worst = self.corr_pass(f, path, extras, started)
            if path in PINNED:
                assert ctx.last_ingest_bytes() > 0, (f, path)
            if f in seq["jump"]:
                poses = self.orc.get_poses().copy()
                R = np.asarray(wl.color_world2camera, np.float64)[:, :3]
                for b in JUMP_BODIES:
                    c = R @ poses[b][:, 3] + np.asarray(wl.color_world2camera, np.float64)[:, 3]
                    u = c[0] / c[2] * wl.color_intrinsics.fu + wl.color_intrinsics.ppu
                    v = c[1] / c[2] * wl.color_intrinsics.fv + wl.color_intrinsics.ppv
                    d = np.array([0.5 * (self.W - 1) - u, 0.5 * (self.H - 1) - v])
                    d *= JUMP_PX / max(np.linalg.norm(d), 1e-9)
                    shift_cam = np.array([d[0] / wl.color_intrinsics.fu * c[2], d[1] / wl.color_intrinsics.fv * c[2], 0.0])
                    poses[b][:, 3] = (poses[b][:, 3] + R.T @ shift_cam).astype(np.float32)
                self.orc.set_poses(poses)
                n_before = self.rec["stale_samples"]
                w2 = self.corr_pass(f, path, [0] * N_CORR, True, stale_bodies=JUMP_BODIES)
                worst = [max(worst[0], w2[0]), max(worst[1], w2[1])]
                assert self.rec["stale_samples"] > n_before, (f, path)
            final = self.orc.get_poses()
            ctx.set_poses(final)
            self.twin.set_poses(final)
            self.give_twin_histograms()
            ctx.calculate_results(0)
            self.twin.calculate_results(0)
            self.orc.calculate_results(0)
            self.histograms_exact("results")
            check_bin_images(ctx, wl, cache=self.bins_cache)
            nb = wl.region.n_histogram_bins
            for b in range(wl.n_bodies):
                for x, y in zip(self.twin.get_histograms(b, nb), ctx.get_histograms(b, nb)):
                    assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), (f, path, b)
            self.rec["worst_m"].append(float(f"{worst[0]:.2e}"))
            self.rec["worst_rad"].append(float(f"{worst[1]:.2e}"))


@pytest.mark.gpu
@pytest.mark.parametrize("index", range(len(SCHEDULE)))
def test_frame_sequence_follows_oracle(capi, oracle, synth, index):
    seq = SCHEDULE[index]
    s = _Sequence(capi, oracle, synth, seq, seed=11 + index)
    try:
        s.run()
    finally:
        s.close()
    r = s.rec
    record(f"frame_sequence_{index}", size=seq["size"], paths="/".join(seq["paths"]), bins=list(seq["bins"]),
           worst_m=r["worst_m"], worst_rad=r["worst_rad"], launches=sorted(map(str, r["launches"])),
           stale_roi_samples=r["stale_samples"], twin_compared=r["twin_compared"], discrete_events=r["discrete_events"])
    assert len(r["discrete_events"]) <= 1, r["discrete_events"]
    assert r["twin_compared"] > 0


@pytest.mark.gpu
def test_shared_camera_with_mixed_resolutions(capi, oracle, synth):
    """Two bodies of different histogram resolutions on one camera, on pinned and full-copy frames, and then unified on
    the same frame: the bin-index state says none while the shifts disagree and while the image holds the rectangles of
    a mixed ingest, no launch stages TMA tiles from it then, and once the state is a shift again the image matches."""
    import dataclasses
    import torch
    base = synth.make_workload("c2", n_bodies=2, n_lines=200, n_points=200, n_divides=2, seed=41)
    n_obj, W, H = base.n_bodies, base.color_intrinsics.width, base.color_intrinsics.height
    gt = base.gt_body2world.copy()
    # one mirror oracle per body group: group g holds body g of every camera (the oracle has one resolution per tracker)
    subs = [dataclasses.replace(base, region=dataclasses.replace(base.region)) for _ in range(2)]
    orcs = [None, None]
    ctx = capi.Context(max_bodies=2 * n_obj, max_cameras=n_obj, max_models=1)
    ctx.set_region_model(0, base.region_model)
    ctx.set_depth_model(0, base.depth_model)
    for k in range(n_obj):
        ctx.set_color_camera(k, base.color_intrinsics, base.color_world2camera)
        ctx.set_depth_camera(k, base.depth_intrinsics, base.depth_world2camera, base.depth_scale)
    dp = capi.depth_params(base.depth)
    op = capi.OptimizerParams(base.tikhonov_rotation, base.tikhonov_translation)
    pin_c = torch.empty(tuple(base.color_frames.shape), dtype=torch.uint8).pin_memory()
    pin_d = torch.empty((n_obj, H, 2 * W), dtype=torch.uint8).pin_memory()
    body = lambda k, g: 2 * k + g  # noqa: E731
    bins = (None, None)
    try:
        for step, st in enumerate(SHARED_STEPS):
            if st["path"] is not None and step:  # a new frame: the objects moved
                for k in range(n_obj):
                    gt[k] = synth.perturb_pose(4100 + step, k, 1.5, 0.003, gt[k])
                    synth.render_color(base.color_intrinsics, synth.pose_mul(base.color_world2camera, gt[k]), 4200 + 10 * step + k,
                                       out=base.color_frames[k])
                    synth.render_depth(base.depth_intrinsics, synth.pose_mul(base.depth_world2camera, gt[k]), 4200 + 10 * step + k,
                                       depth_scale=base.depth_scale, out=base.depth_frames[k])
            for g in range(2):
                if st["bins"][g] != bins[g]:
                    subs[g].region.n_histogram_bins = st["bins"][g]
                    rp = capi.region_params(subs[g].region)
                    for k in range(n_obj):
                        ctx.set_body(body(k, g), rp, dp, op, 0, 0, k, k)
                    poses = orcs[g].get_poses() if orcs[g] is not None else base.start_body2world
                    orcs[g] = oracle.OracleTracker(subs[g], rotation_mode=oracle.ROTATION_LINEAR, exp_mode=oracle.EXP_RODRIGUES)
                    orcs[g].set_poses(poses)
            changed = st["bins"] != bins
            bins = st["bins"]
            if step == 0:
                ctx.set_poses(np.stack([orcs[g].get_poses()[k] for k in range(n_obj) for g in range(2)]))
            if st["path"] == "batch":
                ctx.upload_color_batch(0, base.color_frames)
                ctx.upload_depth_batch(0, base.depth_frames)
            elif st["path"] == "pinned_aligned":
                pin_c.numpy()[:] = base.color_frames
                pin_d.numpy()[:] = base.depth_frames.view(np.uint8).reshape(n_obj, H, 2 * W)
                ctx.upload_batch_ptr(True, 0, n_obj, pin_c.data_ptr(), pin_c.stride(0), pin_c.stride(1))
                ctx.upload_batch_ptr(False, 0, n_obj, pin_d.data_ptr(), pin_d.stride(0), pin_d.stride(1))
            mixed = bins[0] != bins[1]
            pinned = (st["path"] or SHARED_STEPS[step - 1]["path"]) in PINNED
            # the state after this step's launches: a shift only where one resolution wrote (or k_bin rebuilt) it all
            trusted = not mixed and st["path"] is not None or not mixed and not pinned
            expect_state = _bitshift(bins[0]) if trusted else capi.BINS_NONE
            if changed:
                ctx.start_modalities(0)
                for o in orcs:
                    o.start_modalities(0)
            worst = [0.0, 0.0]
            for corr in range(N_CORR):
                start = [o.get_poses() for o in orcs]
                ctx.set_poses(np.stack([start[g][k] for k in range(n_obj) for g in range(2)]))
                ctx.corr_iteration(0, corr, base.n_update_iterations)
                launch = ctx.last_launch()
                if trusted:
                    assert launch["kernel"] == "k_track2" and launch["tma_mode"] != 0, (step, corr, launch)
                else:
                    assert launch["kernel"] == "k_track" or launch["tma_mode"] == 0, (step, corr, launch)
                check_bin_images(ctx, base, expect_state=expect_state, n_cameras=n_obj)
                gpu = ctx.get_poses()
                for k in range(n_obj):
                    for g in range(2):
                        b, o = body(k, g), orcs[g]
                        n, view = o.region_correspondences(k, 0, corr)
                        assert ctx.get_closest_views(b)[0] == view, (step, corr, b)
                        assert_lines_bit_equal(ctx.get_region_lines(b, base.lines_per_body), o.lines[k][:n])
                        n, view = o.depth_correspondences(k, 0, corr)
                        assert_points_bit_equal(ctx.get_depth_points(b, base.points_per_body), o.points[k][:n])
                for o in orcs:
                    o.tracking_step(0, n_corr=corr + 1, corr_begin=corr)
                dt, dr = pose_error(gpu, np.stack([orcs[g].get_poses()[k] for k in range(n_obj) for g in range(2)]))
                worst = [max(worst[0], dt.max()), max(worst[1], dr.max())]
            assert worst[0] < 1e-5 and worst[1] < 1e-5, (step, worst)
            ctx.set_poses(np.stack([orcs[g].get_poses()[k] for k in range(n_obj) for g in range(2)]))
            ctx.calculate_results(0)
            for o in orcs:
                o.calculate_results(0)
            for k in range(n_obj):
                for g in range(2):
                    hf, hb = ctx.get_histograms(body(k, g), bins[g])
                    assert np.array_equal(hf.view(np.uint32), orcs[g].hist_f[k].view(np.uint32)), (step, k, g)
                    assert np.array_equal(hb.view(np.uint32), orcs[g].hist_b[k].view(np.uint32)), (step, k, g)
            record(f"shared_camera_step_{step}", path=st["path"], bins=list(bins), state=expect_state,
                   launch=(launch["kernel"], launch["tma_mode"]), worst_m=float(f"{worst[0]:.2e}"),
                   worst_rad=float(f"{worst[1]:.2e}"))
    finally:
        ctx.close()
