"""Hand-made scenes that put region lines and depth points on the integer and tie decisions of the correspondence
search (tests/correspondence_reference.py counts them).

Exact projection: identity camera and body poses, fu = fv = 128, principal point (0, 0), every model point at a dyadic
position, so that a line centre lands exactly on the pixel coordinate it was built for (integers, halves, quarters).
Depth samples use depth_scale = 2^-10, so raw * depth_scale is exact as well.

Region lines: centres on integers and halves (delta_r ties at odd and even scales), normals along
both axes in both directions, the four diagonals (|nu| == |nv|) and two slanted ones; lines whose start truncates from
(-1, 0) to 0, that leave the frame at either end of the major axis, and that sit on rows / columns 0, 1, size - 2 and
size - 1 (the minor_f_end margins) or slant out of the frame on the minor axis. The colour frame is a one-pixel
checkerboard of a foreground-only and a background-only colour on the left half (every segment of two or more pixels
multiplies a 0 into both products: the 0.5 / 0.5 fallback) and a colour in both histograms on the right.

Depth points: two pairs of equidistant samples (the first in row-major order wins), a sample at
exactly the upper raw bound next to one inside, a point 1 / 32 m away whose considered distance exceeds its depth (raw
0 admitted, a window clipped on every side, stride above 1) and points in two corners of the frame.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32
W, H, F = 640, 480, 128.0
DEPTH_SCALE = 2.0 ** -10
WHITE, BLACK, GREY = (255, 255, 255), (0, 0, 0), (128, 128, 128)
S = float(f32(np.sqrt(f32(0.5))))
NORMALS = [(1.0, 0.0), (-1.0, 0.0), (0.0, 1.0), (0.0, -1.0), (S, S), (-S, S), (S, -S), (-S, -S), (0.8, 0.6), (-0.6, 0.8)]
CENTRES = [(300.0, 220.0), (300.5, 260.25), (340.0, 220.0), (340.5, 260.5), (310.25, 240.0), (330.0, 240.5)]
COMPACT_Z, COMPACT_T = 4.0, (10.0, 7.5, 4.0)   # the compact body's origin projects to (320, 240)
G = (2.0 / np.sqrt(5.0), 1.0 / np.sqrt(5.0))
EDGE_LINES = [
    (8.25, 240.0, 1.0, 0.0),       # scale 1: start 8.25 - 8.5 = -0.25 truncates to 0
    (27.25, 240.0, 1.0, 0.0),      # scale 3: start 27.25 - 27.5 = -0.25
    (5.0, 240.0, 1.0, 0.0),        # starts left of the frame
    (635.0, 240.0, -1.0, 0.0),     # ends right of the frame
    (320.0, 0.25, 1.0, 0.0),       # int(minor_f_end) = 0
    (320.0, 1.0, 1.0, 0.0),        # int(minor_f_end) = 1
    (320.0, 478.0, 1.0, 0.0),      # int(minor_f_end) = height - 2
    (320.0, 478.625, 1.0, 0.0),    # int(minor_f_end) = height - 1
    (0.25, 240.0, 0.0, 1.0),
    (1.0, 240.0, 0.0, 1.0),
    (638.0, 240.0, 0.0, -1.0),
    (638.625, 240.0, 0.0, 1.0),
    (320.0, 2.0, G[0], G[1]),      # slants above row 0 at the start
    (320.0, 477.0, G[0], -G[1]),   # slants below the last row at the start
]


def _intrinsics(synth):
    return synth.Intrinsics(F, F, 0.0, 0.0, W, H)


def _point(u, v, z, compact):
    """Body coordinates of the point that projects to pixel (u, v) at depth z (exact: dyadic values)."""
    x, y = u * z / F, v * z / F
    if compact:
        return (x - COMPACT_T[0], y - COMPACT_T[1], z - COMPACT_T[2])
    return (x, y, z)


def _region_model(synth, compact):
    lines = ([(cu, cv, nu, nv) for cu, cv in CENTRES for nu, nv in NORMALS] if compact else EDGE_LINES)
    z = COMPACT_Z if compact else 1.0
    pts = np.zeros((1, len(lines), 38), f32)
    for i, (cu, cv, nu, nv) in enumerate(lines):
        pts[0, i, 0:3] = _point(cu, cv, z, compact)
        pts[0, i, 3:6] = (nu, nv, 0.0)
        pts[0, i, 6:8] = (1.0, 1.0)
    return synth.Model("region", np.array([[0.0, 0.0, 1.0]], f32), np.ones(1, f32), pts)


def _color_frame():
    img = np.zeros((H, W, 3), np.uint8)
    img[:, W // 2:] = GREY
    uu, vv = np.meshgrid(np.arange(W // 2), np.arange(H))
    img[:, :W // 2][(uu + vv) % 2 == 0] = WHITE
    return img.reshape(H, 3 * W)


def histograms(n_bins):
    """White only in the foreground histogram, black only in the background one, grey in both."""
    shift = {2: 7, 4: 6, 8: 5, 16: 4, 32: 3, 64: 2}[n_bins]
    idx = lambda c: ((c[0] >> shift) * n_bins + (c[1] >> shift)) * n_bins + (c[2] >> shift)
    hf, hb = np.zeros(n_bins ** 3, f32), np.zeros(n_bins ** 3, f32)
    hf[idx(WHITE)] = hf[idx(GREY)] = 0.5
    hb[idx(BLACK)] = hb[idx(GREY)] = 0.5
    return hf, hb


# (u, v, z) of each depth point and the raw samples {(u, v): raw} placed for it: the compact body's, then the others
COMPACT_POINTS = [
    ((310.5, 230.0, 4.0), {(310, 230): 4096, (311, 230): 4096}),     # equidistant along u (4096 * 2^-10 = 4 m)
    ((320.0, 250.5, 4.0), {(320, 250): 4096, (320, 251): 4096}),     # equidistant along v
    ((330.0, 230.0, 4.0), {(330, 230): 4160, (332, 230): 4100}),     # 4160 = (z + 1/16) / 2^-10: refused
]
EDGE_POINTS = [
    ((300.0, 100.0, 1.0), {(300, 100): 1088, (302, 100): 1040}),     # 1088 = (z + 1/16) / 2^-10: refused
    ((400.0, 200.0, 1.0 / 32.0), {}),                                # raw 0 at its centre is the closest sample
    ((636.0, 476.0, 1.0), {(636, 476): 1030}),
    ((2.0, 2.0, 1.0), {(3, 2): 1020}),
]


def _depth_model_and_frame(synth, compact):
    points = COMPACT_POINTS if compact else EDGE_POINTS
    pts = np.zeros((1, len(points), 36), f32)
    frame = np.zeros((H, W), np.uint16)
    for i, ((u, v, z), samples) in enumerate(points):
        pts[0, i, 0:3] = _point(u, v, z, compact)
        pts[0, i, 3:6] = (0.0, 0.0, -1.0)
        for (su, sv), raw in samples.items():
            frame[sv, su] = raw
    return synth.Model("depth", np.array([[0.0, 0.0, 1.0]], f32), np.ones(1, f32), pts), frame


def decision_scenes(synth, scales=(6, 4, 2, 1), n_bins=16, region=True, depth=True):
    """Two one-body workloads carrying the lines and / or points above (n_corr_iterations = len(scales)): the compact
    body 4 m in front of the camera, whose projected bounding sphere is small enough for the ROI tiles (its lines and
    windows take the tile paths where they fit), and the body at the frame's borders, whose origin is at the camera
    (no tile: every line and window takes the out-of-tile paths)."""
    out = []
    for compact in (True, False):
        eye = np.eye(4, dtype=f32)[:3]
        pose = eye.copy()
        if compact:
            pose[:, 3] = COMPACT_T
        intr = _intrinsics(synth)
        rs = ds = rm = dm = frame = None
        if region:
            rm = _region_model(synth, compact)
            rs = synth.RegionSettings(n_lines_max=rm.n_points, scales=tuple(scales),
                                      standard_deviations=(15.0, 5.0, 3.5, 1.5), n_histogram_bins=n_bins,
                                      min_continuous_distance=0.0)
        if depth:
            dm, frame = _depth_model_and_frame(synth, compact)
            ds = synth.DepthSettings(n_points_max=dm.n_points, stride_length=2.0 ** -9,
                                     considered_distances=(2.0 ** -4, 2.0 ** -5), standard_deviations=(0.05, 0.03))
        out.append(synth.Workload(
            name="decisions", n_bodies=1, region=rs, depth=ds, tikhonov_rotation=1000.0, tikhonov_translation=30000.0,
            n_corr_iterations=len(scales), n_update_iterations=1, color_intrinsics=intr, depth_intrinsics=intr,
            color_world2camera=eye, depth_world2camera=eye, depth_scale=DEPTH_SCALE, region_model=rm, depth_model=dm,
            color_frames=_color_frame()[None] if region else None, depth_frames=frame[None] if depth else None,
            gt_body2world=pose[None], start_body2world=pose[None]))
    return out


def gh_shifts(wl, corr):
    """Pose offsets (camera x, metres) at which the local-mode gradient is evaluated: 5 and 6 line steps of the
    iteration's scale, so that dist_idx_upper reaches 11 / 12 on lines with normal_u = 1 and 1 / 0 on normal_u = -1."""
    scale = wl.region.scales[min(corr, len(wl.region.scales) - 1)]
    z = float(wl.start_body2world[0][2, 3]) or 1.0     # the lines' depth: COMPACT_Z or 1
    return [5.0 * scale * z / F, 6.0 * scale * z / F]


REGION_COUNTERS = ("delta_r_ties", "ties_nu_nv", "start_truncated", "rejected_major_lo", "rejected_major_hi",
                   "rejected_minor_lo", "rejected_minor_hi", "rejected_end_lo", "rejected_end_hi", "end_at_1",
                   "end_at_minor_m2", "horizontal", "vertical", "forward", "reverse")
DEPTH_COUNTERS = ("equal_ties", "raw_at_min", "raw_at_max", "raw0_admitted", "clipped_left", "clipped_top",
                  "clipped_right", "clipped_bottom", "stride_1", "stride_above_1")


def reached(st, region=True, depth=True, local=True, fallbacks=True):
    """The counters the scene was built to reach that stayed at 0."""
    keys = list(REGION_COUNTERS if region else ()) + list(DEPTH_COUNTERS if depth else ())
    if region and local:
        keys += ["upper_0", "upper_1", "upper_11", "upper_12"]
    if region and fallbacks:
        keys += ["segment_fallbacks"]
    return [k for k in keys if not st[k] > 0]


def screen_scene(synth, depth_scale=1e-3, fu=365.0):
    """A depth-only body about 30 m away, off axis near the top-left corner of a 640 x 480 frame (depth scaling, every
    pixel of the window sampled; its points lie within 40 px of the body's origin, so the depth tile holds their
    windows). For each point the frame holds two samples: B, the closest, and A, earlier in row-major order, whose
    squared distance lies between B's and B's reciprocal-screen value minus 1e-6 m^2. The strict test takes A, then B;
    the earlier fixed-margin screen rejected B and kept A."""
    import correspondence_reference as ref
    from occlusion_reference import apply
    intr = synth.Intrinsics(fu, fu, 320.0, 240.0, W, H)
    eye = np.eye(4, dtype=f32)[:3]
    ds = synth.DepthSettings(n_points_max=6, stride_length=0.00125, considered_distances=(0.05,),
                             standard_deviations=(0.05,), use_depth_scaling=True)

    class It:
        pass
    it = It()
    it.fu = it.fv = f32(fu)
    it.ppu, it.ppv = f32(320.0), f32(240.0)
    it.depth_scale = f32(depth_scale)
    pose = eye.copy()
    pose[:, 3] = ((80.0 - 320.0) * 30.0 / fu, (80.0 - 240.0) * 30.0 / fu, 30.0)
    frame = np.zeros((H, W), np.uint16)
    model = []
    for u_c, v_c, z in ((45.0, 45.0, 28.0), (115.0, 45.0, 30.0), (45.0, 115.0, 32.0), (115.0, 115.0, 30.0),
                        (80.0, 50.0, 29.0), (80.0, 110.0, 31.0)):
        target = ((u_c - 320.0) * z / fu, (v_c - 240.0) * z / fu, z)
        X = np.array([target[k] - pose[k, 3] for k in range(3)], f32)
        x, y, z = (f32(c) for c in apply(pose, X))
        cd = f32(0.05) * z
        uu, vv, rr = np.meshgrid(np.arange(int(u_c) - 15, int(u_c) + 16), np.arange(int(v_c) - 15, int(v_c) + 16),
                                 np.arange(int(z / it.depth_scale) - 60, int(z / it.depth_scale) + 61), indexing="ij")
        uu, vv, rr = uu.ravel(), vv.ravel(), rr.ravel()
        _, _, _, d2 = ref.exact_distance2(uu, vv, rr, x, y, z, it)
        depth = rr.astype(f32) * it.depth_scale
        ax = (uu.astype(f32) - it.ppu) * depth * (f32(1) / it.fu) - x
        ay = (vv.astype(f32) - it.ppv) * depth * (f32(1) / it.fv) - y
        dz = depth - z
        s = ax * ax + ay * ay + dz * dz
        order = vv * W + uu
        found = None
        for b in np.argsort(-(s - d2))[:400]:
            if not (s[b] - d2[b] > f32(2e-6) and d2[b] < cd * cd):
                continue
            band = (order < order[b]) & (d2 > d2[b]) & (d2 < s[b] - f32(1e-6)) & (rr != rr[b])
            if band.any():
                found = (int(np.nonzero(band)[0][0]), int(b))
                break
        assert found is not None, (u_c, v_c, z)
        for i in found:
            frame[vv[i], uu[i]] = rr[i]
        model.append(X)
    pts = np.zeros((1, len(model), 36), f32)
    for i, X in enumerate(model):
        pts[0, i, 0:3] = X
        pts[0, i, 3:6] = (0.0, 0.0, -1.0)
    dm = synth.Model("depth", np.array([[0.0, 0.0, 1.0]], f32), np.ones(1, f32), pts)
    return synth.Workload(name="screen", n_bodies=1, region=None, depth=ds, tikhonov_rotation=1000.0,
                          tikhonov_translation=30000.0, n_corr_iterations=1, n_update_iterations=1,
                          color_intrinsics=intr, depth_intrinsics=intr, color_world2camera=eye, depth_world2camera=eye,
                          depth_scale=depth_scale, region_model=None, depth_model=dm, color_frames=None,
                          depth_frames=frame[None], gt_body2world=pose[None], start_body2world=pose[None])
