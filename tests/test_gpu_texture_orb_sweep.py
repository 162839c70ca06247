"""cv::ORB on the device (m3tb_texture_detect_orb, k_texture_orb) against the NumPy restatement
(tests/texture_orb_reference.py, which tests/test_texture_orb_reference.py holds to cv2) on the device's own crops,
across crop sizes from 1 to 640 px (clipped at the frame border into shapes such as 63 x 156), every detector setting of
R.SWEEP and frames of texture, noise, 0 / 255 noise, a constant grey, dots and a checkerboard: all five read-back fields
bit-equal in the canonical order, the count equal to R's. The sweep reaches per-level counts of 0, ties kept at both cuts,
candidate lists longer than one 512-thread chunk, kept keypoints with a Harris response <= 0, levels emptied by the
31-pixel border, pyramids with an empty level (no keypoints at all, as cv::ORB) and crops without keypoints. Also: mixed
settings and sizes in one call and in more than one launch, the n_features_max boundary at F and F - 1, scratch reused
after a larger detection, and tracking from the device's feature slot against the host upload of the read-back."""
import time

import numpy as np
import pytest

import texture_orb_reference as R
from test_gpu_texture_device_front_end import FIX, FIX_FRAME, _crop, _same, _scene

pytestmark = pytest.mark.gpu

FIELDS = ("xy", "angle", "response", "octave", "descriptors")
PATTERN = R.bit_pattern()
SIZES = (1, 7, 62, 63, 64, 65, 100, 200, 369, 640)  # focused_image_size
N_MAX = 4096  # n_features_max of every body: a body that keeps more is compared by its count alone
WIDE_BODY = 2  # golden body 2's focus region is mostly margin: its crop is 1.85 focused_image_size wide


def _pose(x, y, z):
    return np.hstack([np.eye(3), [[x], [y], [z]]]).astype(np.float32)


# near the frame border, so the focus region is clipped: at focused_image_size 200 the crops are 63 x 156, 62 x 156,
# 195 x 64, 191 x 63, 2 x 137 and 64 x 59
BORDER_POSES = np.stack([_pose(-0.2605, 0.0, 0.3), _pose(-0.261, 0.0, 0.3), _pose(0.05, -0.1535, 0.3),
                         _pose(-0.03, 0.1535, 0.3), _pose(0.2615, 0.01, 0.25), _pose(-0.26, -0.15, 0.3)])
POSES = np.concatenate([FIX["poses"], BORDER_POSES]).astype(np.float32)


def _frames():
    h, w = 540, 960
    return [("golden", FIX_FRAME), ("textured", R.as_frame(R.textured(h, w, 21))),
            ("textured_block16", R.as_frame(R.textured(h, w, 22, block=16))), ("noise", R.as_frame(R.noise(h, w, 23))),
            ("binary_noise", R.as_frame(R.binary_noise(h, w, 24))), ("constant", R.as_frame(np.full((h, w), 90, np.uint8))),
            ("dots", R.dot_frame()), ("checkerboard", R.as_frame(R.checkerboard(h, w, cell=5)))]


FRAMES = _frames()


def _assignment(fi, n_bodies=len(POSES)):
    """Frame fi's focused_image_size and setting per body: every size and 17 of the settings in each frame, every
    setting over the frames. Golden body 2 stays below 640 (1181 px would take R seconds per setting)."""
    sizes = [SIZES[(b + fi) % len(SIZES)] for b in range(n_bodies)]
    sizes = [369 if b % len(POSES) == WIDE_BODY and s == 640 else s for b, s in enumerate(sizes)]
    settings = [R.SWEEP[(3 * b + 5 * fi) % len(R.SWEEP)] for b in range(n_bodies)]
    return sizes, settings


def _params(capi, size, n_max=N_MAX):
    p = capi.texture_params_default()
    p.descriptor_type = capi.DESCRIPTOR_ORB
    p.focused_image_size = size
    p.n_features_max = n_max
    return p


def _context(capi, synth, frame, sizes, poses=POSES):
    ctx = _scene(capi, synth, poses=poses, upload=False)
    ctx.upload_color(0, frame)
    for b, s in enumerate(sizes):
        ctx.set_texture_modality(b, _params(capi, s), 0)
    return ctx


class Stats:
    """What the comparisons reached: keypoints compared field by field or by count, and the branches of k_texture_orb."""

    def __init__(self):
        self.compared = self.counted = self.bodies = 0
        self.reached = set()
        self.crop_sides = set()
        self.level_shapes = set()
        self.scales = []

    def add(self, st, res, w, h, scale, full):
        self.bodies += 1
        self.crop_sides.update((w, h))
        self.scales.append(scale)
        n = len(res["angle"])
        if st["empty_pyramid"]:
            self.reached.add("empty pyramid")
            return
        if n == 0:
            self.reached.add("no keypoints")
        if not full:
            return
        for level, img in enumerate(st["levels"]):
            lh, lw = img.shape
            want = st["per_level"][level]
            self.level_shapes.add((lw, lh))
            if want == 0 and st["n_fast"][level] > 0:
                self.reached.add("per-level count 0")
            if want > 0 and st["n_first_cut"][level] > 2 * want:
                self.reached.add("first cut keeps ties")
            if want > 0 and st["n_second_cut"][level] > want:
                self.reached.add("second cut keeps ties")
            if st["n_fast"][level] > 512:
                self.reached.add("more than 512 candidates")
            if min(lw, lh) <= 2 * R.EDGE_THRESHOLD and st["n_corners"][level] > 0:
                self.reached.add("level emptied by the border")
        if (res["response"] <= 0).any():
            self.reached.add("Harris response <= 0")


def _check(ctx, bodies, settings, stats, cap=1200, detect=True):
    """Detects `bodies` in that order with `settings` (unless `detect` is false: the caller has), reads their crops back
    (m3tb_texture_crop) and holds each body's count and read-back to R.orb of its crop; returns R's results by body."""
    if detect:
        ctx.texture_detect_orb(bodies, settings)
    found = ctx.get_texture_detections()
    out, roi, scale, size, valid = _crop(ctx, bodies, (cap, cap))
    host = out.cpu().numpy()
    del out
    results = {}
    for k, b in enumerate(bodies):
        got = ctx.get_texture_orb_keypoints(b)
        if not valid[k]:  # no focus, or a crop of 0 pixels: no keypoints
            assert found[b] == 0 and len(got["angle"]) == 0, b
            results[b] = None
            continue
        w, h = (int(v) for v in size[k])
        st = {}
        mine = R.orb(host[k, :h, :w], *settings[k], pattern=PATTERN, stages=st)
        n = len(mine["angle"])
        assert found[b] == n, (b, (w, h), settings[k], int(found[b]), n)
        full = n <= N_MAX
        if full:
            for f in FIELDS:
                assert _same(got[f], mine[f]), (b, (w, h), settings[k], f)
            stats.compared += n
        else:  # more than n_features_max: the count is reported, the body gets no features
            assert len(got["angle"]) == 0, b
            stats.counted += n
        stats.add(st, mine, w, h, float(scale[k]), full)
        results[b] = mine
    return results


def test_device_detection_equals_the_restatement_across_the_sweep(capi, synth):
    start = time.perf_counter()
    stats = Stats()
    order = [int(b) for b in np.random.default_rng(5).permutation(len(POSES))]
    for fi, (name, frame) in enumerate(FRAMES):
        ctx = _context(capi, synth, frame, _assignment(fi)[0])
        for a in (fi, fi + len(FRAMES)):  # two assignments per frame; the second reuses the first's scratch
            sizes, settings = _assignment(a)
            for b, s in enumerate(sizes):
                ctx.set_texture_modality(b, _params(capi, s), 0)
            # one call, mixed settings and crop sizes; the largest crop (which sets the scratch pitch) is not first
            call = order[:]
            while sizes[call[0]] == max(sizes):
                call = call[1:] + call[:1]
            _check(ctx, call, [settings[b] for b in call], stats)
        ctx.close()
    assert set(stats.reached) >= {"per-level count 0", "first cut keeps ties", "second cut keeps ties",
                                  "more than 512 candidates", "Harris response <= 0", "level emptied by the border",
                                  "empty pyramid", "no keypoints"}, stats.reached
    assert {1, 2, 7, 62, 63, 64, 65} <= stats.crop_sides, sorted(stats.crop_sides)
    assert any(62 in s and max(s) > 62 for s in stats.level_shapes)  # no interior
    assert any(63 in s and max(s) > 63 for s in stats.level_shapes)  # one interior row or column
    assert min(stats.scales) < 0.5 and any(0.9 < s < 1.1 for s in stats.scales) and max(stats.scales) > 2.0
    print(f"sweep: {stats.bodies} crops, {stats.compared} keypoints compared field by field, {stats.counted} by count, "
          f"{time.perf_counter() - start:.1f} s")
    assert stats.compared >= 25000


def test_more_bodies_than_one_launch_takes(capi, synth):
    """131 bodies of mixed crop sizes and settings in one call: two crop and two detection launches."""
    n = 131
    poses = POSES[[b % len(POSES) for b in range(n)]]
    sizes = [(100, 200, 369, 65, 7)[b % 5] for b in range(n)]
    large = [s for s in R.SWEEP if s[0] in (1000, 4096)]
    settings = [large[(3 * b) % len(large)] for b in range(n)]
    ctx = _context(capi, synth, FRAMES[1][1], sizes, poses=poses)
    order = [int(b) for b in np.random.default_rng(9).permutation(n)]
    before = ctx.launch_count
    ctx.texture_detect_orb(order, [settings[b] for b in order])
    assert ctx.launch_count == before + 4  # a crop and a detection launch per 128 bodies
    stats = Stats()
    _check(ctx, order, [settings[b] for b in order], stats, cap=700, detect=False)
    print(f"{n} bodies: {stats.compared} keypoints compared field by field, {stats.counted} by count")
    assert stats.compared >= 60000
    ctx.close()


def test_empty_pyramid_gives_the_body_no_keypoints(capi, synth):
    """At (300, 2.5, 8) level 7 of every golden crop but crop 2 has a side of 0 pixels: cv::ORB detects nothing there
    (cv::resize throws while it builds the pyramid), so every body gets a count of 0, no read-back and no features,
    while the earlier levels do have keypoints. Crop 2's pyramid is whole, and it has no keypoints. Another body of the
    same call, at (300, 1.2, 3), keeps its own."""
    n = len(FIX["poses"])
    ctx = _scene(capi, synth)
    ctx.texture_detect_orb(list(range(n)), (300, 2.5, 8))
    assert list(ctx.get_texture_detections()) == [0] * n
    host = _crop(ctx, list(range(n)))[0].cpu().numpy()
    for i in range(n):
        w, h = FIX["sizes"][i]
        assert len(ctx.get_texture_orb_keypoints(i)["angle"]) == 0
        assert R.empty_pyramid(w, h, 2.5, 8) == (i != 2)
        assert len(R.orb(host[i, :h, :w], 300, 2.5, 8, pattern=PATTERN)["angle"]) == 0
        if i != 2:  # the levels before the first empty one have keypoints
            whole = next(k for k in range(1, 8) if R.empty_pyramid(w, h, 2.5, k + 1))
            assert len(R.orb(host[i, :h, :w], 300, 2.5, whole, pattern=PATTERN)["angle"]) > 0, i
    ctx.start_modalities(0)
    assert all(int(ctx.get_texture_keyframes(i)["sizes"].sum()) == 0 for i in range(n))
    ctx.close()
    ctx = _scene(capi, synth, bodies=[0, 3])
    ctx.texture_detect_orb([0, 1], [(300, 2.5, 8), (300, 1.2, 3)])
    ref = R.orb(np.ascontiguousarray(FIX["crops"][3, :FIX["sizes"][3][1], :FIX["sizes"][3][0]]), 300, 1.2, 3,
                pattern=PATTERN)
    assert list(ctx.get_texture_detections()) == [0, len(ref["angle"])]
    got = ctx.get_texture_orb_keypoints(1)
    assert all(_same(got[f], ref[f]) for f in FIELDS)
    ctx.start_modalities(0)
    assert int(ctx.get_texture_keyframes(0)["sizes"].sum()) == 0 < int(ctx.get_texture_keyframes(1)["sizes"].sum())
    ctx.close()


def test_capacity_boundary(capi, synth):
    """A crop that keeps F keypoints, 512 < F <= 4096: kept whole at n_features_max F, dropped at F - 1 with the count
    F still reported."""
    body, setting = 4, (1000, 1.3, 4)  # golden body 4 at focused_image_size 200: a 220 px crop at scale 1
    ctx = _context(capi, synth, FRAMES[1][1], [200], poses=POSES[[body]])
    stats = Stats()
    ref = _check(ctx, [0], [setting], stats)[0]
    f = len(ref["angle"])
    assert 512 < f <= 4096
    for n_max, kept in ((f, True), (f - 1, False)):
        ctx.set_texture_modality(0, _params(capi, 200, n_max), 0)
        ctx.texture_detect_orb([0], setting)
        assert list(ctx.get_texture_detections()) == [f]
        got = ctx.get_texture_orb_keypoints(0)
        if kept:
            assert all(_same(got[k], ref[k]) for k in FIELDS)
        else:
            assert len(got["angle"]) == 0
        ctx.start_modalities(0)
        assert (int(ctx.get_texture_keyframes(0)["sizes"].sum()) > 0) == kept
    ctx.close()


def test_scratch_reused_after_a_larger_detection(capi, synth):
    """A 704 px noise crop at (2^24, 1.2, 3), 47,247 keypoints, then a 110 px textured crop in the same context: the
    second detection equals a fresh context's and R's."""
    body = 4
    ctx = _context(capi, synth, FRAMES[3][1], [640], poses=POSES[[body]])
    ctx.texture_detect_orb([0], (1 << 24, 1.2, 3))
    assert list(ctx.get_texture_detections()) == [47247]
    fresh = _context(capi, synth, FRAMES[1][1], [100], poses=POSES[[body]])
    ctx.upload_color(0, FRAMES[1][1])
    ctx.set_texture_modality(0, _params(capi, 100), 0)
    stats = Stats()
    setting = (300, 1.2, 3)
    ref = _check(ctx, [0], [setting], stats)[0]
    assert len(ref["angle"]) > 50
    fresh.texture_detect_orb([0], setting)
    assert list(fresh.get_texture_detections()) == list(ctx.get_texture_detections())
    a, b = ctx.get_texture_orb_keypoints(0), fresh.get_texture_orb_keypoints(0)
    assert all(_same(a[k], b[k]) for k in FIELDS)
    ctx.close()
    fresh.close()


@pytest.mark.parametrize("fi", [0, 1], ids=[FRAMES[0][0], FRAMES[1][0]])
def test_feature_slot_equals_the_host_upload_of_the_read_back(capi, synth, fi):
    """The sweep's poses on one frame at focused_image_size 200, with the sweep settings of 300 to 4096 features:
    keyframes from the device detection's feature slot, and one tracking step, equal to a context fed the read-back
    through m3tb_upload_texture_features."""
    name, frame = FRAMES[fi]
    sizes = [200] * len(POSES)
    subset = [s for s in R.SWEEP if 300 <= s[0] <= 4096]
    settings = [subset[(b + fi) % len(subset)] for b in range(len(POSES))]
    ctx_d = _context(capi, synth, frame, sizes)
    ctx_h = _context(capi, synth, frame, sizes)
    roi, scale, valid = ctx_d.get_texture_focus()
    bodies = [b for b in range(len(POSES)) if valid[b]]
    assert len(bodies) >= 12

    def detect_and_feed():
        ctx_d.texture_detect_orb(bodies, [settings[b] for b in bodies])
        for b in bodies:
            got = ctx_d.get_texture_orb_keypoints(b)
            ctx_h.upload_texture_features(b, got["xy"], got["descriptors"], roi[b][0], roi[b][1], scale[b])

    detect_and_feed()
    for ctx in (ctx_d, ctx_h):
        ctx.start_modalities(0)
    total = 0
    for b in bodies:
        kd, kh = ctx_d.get_texture_keyframes(b), ctx_h.get_texture_keyframes(b)
        assert _same(kd["sizes"], kh["sizes"]) and _same(kd["points"], kh["points"]), b
        assert _same(kd["descriptors"], kh["descriptors"]), b
        total += int(kd["sizes"].sum())
    assert total >= 50, total
    for ctx in (ctx_d, ctx_h):
        ctx.upload_color(0, frame)
    detect_and_feed()
    for ctx in (ctx_d, ctx_h):
        ctx.tracking_step(1, 2, 2)
        ctx.calculate_results(1)
    assert _same(ctx_d.get_poses(), ctx_h.get_poses())
    for b in bodies:
        assert _same(ctx_d.get_texture_points(b), ctx_h.get_texture_points(b)), b
    ctx_d.close()
    ctx_h.close()
