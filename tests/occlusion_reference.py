"""Restatement of the checks that decide whether a region line or a depth point survives, written from M3T's
region_modality.cpp / depth_modality.cpp rather than from the oracle (SURVEY row f4):

- IsLineUnoccludedMeasured / IsLineUnoccludedModeled (region_modality.cpp:1343-1431);
- IsDynamicLineRegionSufficient (:1293-1341) and DynamicRegionDistance (:1157-1223);
- IsPointUnoccludedMeasured / IsPointUnoccludedModeled and IsPointOnValidSilhouette (depth_modality.cpp:728-824);
- the depth-offset selections (region_modality.cpp:965-991, depth_modality.cpp:669-693);
- the n_unoccluded_iterations gate and the two-pass rule of CalculateCorrespondences (region_modality.cpp:435-463,
  depth_modality.cpp:295-313);
- AddLinePixelColorsToTempHistograms' choice of lines and sampled lengths (region_modality.cpp:1025-1155).

Everything is float32 in the reference's order of operations. int() is truncation; for NaN and out-of-range values it
follows the device's conversion (saturation, NaN -> 0), which is what a scan of a non-finite item would meet there.
ushort(x) is truncation followed by reduction modulo 2^16. FocusedDepthRenderer::Depth is a / (b - value).

The rule the reference leaves undefined: a window whose diameter is not finite or is negative would get a stride of 0
(a scan that never ends) or none at all; it scans nothing and counts as unoccluded. `parent_rule=True` restates the
earlier guards instead (z <= 0 as the only projection test, no diameter test, region depth-offset ids not limited to
the table): a scan that would not end is then reported in stats["stride0_scans"] rather than looped.

What is not restated here: the closest view; the line's segment probabilities and the depth point's correspondence
search are restated in tests/correspondence_reference.py. `geometric_valid` (an item's validity with every check off,
from a run without them) and `view` come from the caller; the predicted valid flag is geometric_valid and the checks.
"""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32
K_MAX_N_OCCLUSION_STRIDES = 5   # region_modality.h:145, depth_modality.h:113
K_N_REGION_STRIDE = 5           # region_modality.h:146
K_REGION_OFFSET = f32(2.0)      # region_modality.h:147
N_DEPTH_OFFSETS = 30            # DataPoint::depth_offsets
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1

STAT_KEYS = ("windows", "clipped_left", "clipped_top", "clipped_right", "clipped_bottom", "empty_windows",
             "wrapped_bounds", "stride_above_1", "all_background", "top_ids", "region_id_mismatch", "fallbacks",
             "stride0_scans", "refused_ids", "zero_pixels", "occluded", "walk_outside", "handled_passes",
             "unhandled_passes")


def new_stats():
    """Counters of the edges the checks met, and the depth-offset ids they selected ("offset_ids")."""
    st = {k: 0 for k in STAT_KEYS}
    st["offset_ids"] = set()
    return st


def trunc(x) -> int:
    """int(x) of a float32 as the device converts it (cvt.rzi.s32.f32: saturating, NaN -> 0)."""
    x = float(x)
    if math.isnan(x):
        return 0
    if x >= 2.0 ** 31:
        return INT_MAX
    if x < -2.0 ** 31:
        return INT_MIN
    return int(x)


def i32(n: int) -> int:
    """Two's-complement wrap of an int product (the device's int arithmetic)."""
    return (n + 2 ** 31) % 2 ** 32 - 2 ** 31


def pose_mul(a, b):
    a, b = np.asarray(a, f32).reshape(3, 4), np.asarray(b, f32).reshape(3, 4)
    r = np.zeros((3, 4), f32)
    for i in range(3):
        for j in range(3):
            r[i, j] = a[i, 0] * b[0, j] + a[i, 1] * b[1, j] + a[i, 2] * b[2, j]
        r[i, 3] = a[i, 0] * b[0, 3] + a[i, 1] * b[1, 3] + a[i, 2] * b[2, 3] + a[i, 3]
    return r


def apply(p, x):
    return tuple(p[i, 0] * x[0] + p[i, 1] * x[1] + p[i, 2] * x[2] + p[i, 3] for i in range(3))


def normal2(p, n):
    """(body2camera rotation_xy * normal_f_body).normalized() with the pose's linear block (as the device and the
    mirror oracle take it)."""
    nu = p[0, 0] * n[0] + p[0, 1] * n[1] + p[0, 2] * n[2]
    nv = p[1, 0] * n[0] + p[1, 1] * n[1] + p[1, 2] * n[2]
    zz = nu * nu + nv * nv
    if zz > f32(0):
        s = f32(np.sqrt(zz))
        nu, nv = nu / s, nv / s
    return f32(nu), f32(nv)


# ---- the strided window scans ----------------------------------------------------------------------------------------
def _window(center_u, center_v, diameter, w_m1, h_m1, stats, parent_rule):
    """Limits of the strided window (region_modality.cpp:1356-1371): (u_min, v_min, u_max, v_max, stride), or None when
    the window is not scanned."""
    if not parent_rule and not (diameter >= f32(0) and not np.isinf(diameter)):
        return None
    stride = trunc(diameter / f32(K_MAX_N_OCCLUSION_STRIDES) + f32(1))
    if stride == 0:  # the reference's loop would never advance (unless the window is empty)
        n_strides, rd = 0, 0
    else:
        n_strides = trunc(diameter / f32(stride) + f32(0.5))
        rd = i32(n_strides * stride)
    rr = f32(0.5) * f32(rd)
    u_min, v_min = trunc(center_u - rr + f32(0.5)), trunc(center_v - rr + f32(0.5))
    u_max, v_max = i32(u_min + rd), i32(v_min + rd)
    if stats is not None:
        stats["windows"] += 1
        stats["clipped_left"] += u_min < 0
        stats["clipped_top"] += v_min < 0
        stats["clipped_right"] += u_max > w_m1
        stats["clipped_bottom"] += v_max > h_m1
        stats["stride_above_1"] += stride > 1
    u_min, v_min, u_max, v_max = max(u_min, 0), max(v_min, 0), min(u_max, w_m1), min(v_max, h_m1)
    empty = u_min > u_max or v_min > v_max
    if stats is not None:
        stats["empty_windows"] += empty
    if stride == 0 and not empty:
        if stats is not None:
            stats["stride0_scans"] += 1
        return None
    return u_min, v_min, u_max, v_max, stride


def window_unoccluded(image, center_u, center_v, diameter, min_depth_value, stats=None, parent_rule=False):
    """The measured scan (region_modality.cpp:1355-1388, depth_modality.cpp:739-775): False if a valid depth sample
    inside the window lies in front of ushort(min_depth_value)."""
    h, w = image.shape
    win = _window(f32(center_u), f32(center_v), f32(diameter), w - 1, h - 1, stats, parent_rule)
    if win is None:
        return True
    u0, v0, u1, v1, stride = win
    t = trunc(min_depth_value)
    min_depth = t & 0xFFFF
    if stats is not None and min_depth != t:
        stats["wrapped_bounds"] += 1
    if stride < 0:
        return True
    block = image[v0:v1 + 1:stride, u0:u1 + 1:stride].astype(np.int64)
    occluded = bool(((block > 0) & (block < min_depth)).any())
    if stats is not None:
        stats["zero_pixels"] += int((block == 0).sum())
        stats["occluded"] += occluded
    return not occluded


def modeled_window_unoccluded(r, center_u, center_v, diameter, min_allowed_depth, stats=None, parent_rule=False):
    """The modeled scan (region_modality.cpp:1394-1430, depth_modality.cpp:780-823) in the focused depth image `r`
    (synth.Rendering)."""
    sc = f32(r.scale)
    fcu = (f32(center_u) - f32(r.corner_u)) * sc
    fcv = (f32(center_v) - f32(r.corner_v)) * sc
    S = r.image.shape[0]
    win = _window(fcu, fcv, f32(diameter), S - 1, S - 1, stats, parent_rule)
    if win is None:
        return True
    u0, v0, u1, v1, stride = win
    mv = 65535
    if stride > 0:
        block = r.image[v0:v1 + 1:stride, u0:u1 + 1:stride]
        if block.size:
            mv = int(block.min())
    if stats is not None and mv == 65535:
        stats["all_background"] += 1
    min_depth = f32(r.projection_term_a) / (f32(r.projection_term_b) - f32(mv))
    unoccluded = bool(min_depth > f32(min_allowed_depth))
    if stats is not None:
        stats["occluded"] += not unoccluded
    return unoccluded


# ---- depth-offset selection ------------------------------------------------------------------------------------------
def region_offset_id(radius, model, stats=None, parent_rule=False):
    """measured_ / modeled_depth_offset_id_ (region_modality.cpp:965-991). None: refused. The reference refuses only a
    radius above max_radius; an id of 30 or more (max_radius / stride in [29.5, 30)) is refused as well."""
    if f32(radius) > f32(model.max_radius_depth_offset):
        return None
    i = trunc(f32(radius) / f32(model.stride_depth_offset) + f32(0.5))
    if stats is not None:
        stats["top_ids"] += i == N_DEPTH_OFFSETS - 1
        stats["offset_ids"].add(i)
    if i >= N_DEPTH_OFFSETS and not parent_rule:
        if stats is not None:
            stats["refused_ids"] += 1
        return None
    return i


def depth_offset_id(radius, depth, use_depth_scaling, stride, stats=None):
    """CalculateBasicPointData's selection (depth_modality.cpp:669-693): an id past the table takes the last entry."""
    radius = f32(radius)
    if use_depth_scaling:
        radius = radius * f32(depth)
    i = trunc(radius / f32(stride) + f32(0.5))
    if stats is not None:
        stats["offset_ids"].add(min(i, N_DEPTH_OFFSETS - 1))
    if i >= N_DEPTH_OFFSETS - 1:
        if stats is not None:
            stats["top_ids"] += 1
        i = N_DEPTH_OFFSETS - 1
    return i


# ---- renderer-image checks -------------------------------------------------------------------------------------------
def silhouette_at(r, v, u):
    return int(r.image[v, u])


def dynamic_line_region_sufficient(r, min_continuous_distance, fscale, center_u, center_v, normal_u, normal_v,
                                   stats=None):
    """IsDynamicLineRegionSufficient (region_modality.cpp:1293-1341). A foreground sample outside the focused image
    (undefined in the reference) counts as 'not this region'."""
    region_id = int(r.id) & 0xFF
    fsize = f32(r.image.shape[0])
    sc = f32(r.scale)
    fmcd = f32(min_continuous_distance) * f32(fscale) * sc
    fstride = max(f32((fmcd - K_REGION_OFFSET) / f32(K_N_REGION_STRIDE)), f32(0))
    su, sv = fstride * f32(normal_u), fstride * f32(normal_v)
    ou, ov = K_REGION_OFFSET * f32(normal_u), K_REGION_OFFSET * f32(normal_v)
    fcu = f32(0.5) + (f32(center_u) - f32(r.corner_u)) * sc
    fcv = f32(0.5) + (f32(center_v) - f32(r.corner_v)) * sc
    u, v = f32(fcu - ou), f32(fcv - ov)
    for _ in range(K_N_REGION_STRIDE + 1):
        if u >= fsize or u < 0 or v >= fsize or v < 0:
            if stats is not None:
                stats["walk_outside"] += 1
            return False
        if silhouette_at(r, trunc(v), trunc(u)) != region_id:
            if stats is not None:
                stats["region_id_mismatch"] += 1
            return False
        u, v = f32(u - su), f32(v - sv)
    u, v = f32(fcu + ou), f32(fcv + ov)
    for _ in range(K_N_REGION_STRIDE + 1):
        if u >= fsize or u < 0 or v >= fsize or v < 0:
            if stats is not None:
                stats["walk_outside"] += 1
            break
        if silhouette_at(r, trunc(v), trunc(u)) == region_id:
            return False
        u, v = f32(u + su), f32(v + sv)
    return True


def dynamic_region_distance(r, max_considered_line_length, unconsidered_line_length, center_u, center_v, normal_u,
                            normal_v, length_f, length_b):
    """DynamicRegionDistance (region_modality.cpp:1157-1223), including :1218, where a background sample of the own
    region overwrites the foreground distance. Returns (length_f, length_b)."""
    region_id = int(r.id) & 0xFF
    fsize = f32(r.image.shape[0])
    sc = f32(r.scale)
    stride = f32(max_considered_line_length) / f32(K_N_REGION_STRIDE)
    fstride = stride * sc
    fsu, fsv = fstride * f32(normal_u), fstride * f32(normal_v)
    delta_start = K_REGION_OFFSET / sc - f32(unconsidered_line_length)
    i_start = max(trunc(delta_start / stride + f32(1)), 0)
    offset = f32(unconsidered_line_length) + f32(i_start) * stride
    fo = offset * sc
    fou, fov = fo * f32(normal_u), fo * f32(normal_v)
    fcu = f32(0.5) + (f32(center_u) - f32(r.corner_u)) * sc
    fcv = f32(0.5) + (f32(center_v) - f32(r.corner_v)) * sc
    u, v = f32(fcu - fou), f32(fcv - fov)
    for i in range(i_start, K_N_REGION_STRIDE + 1):
        if u >= fsize or u < 0 or v >= fsize or v < 0:
            length_f = f32(stride * f32(i))
            break
        if silhouette_at(r, trunc(v), trunc(u)) != region_id:
            length_f = f32(0) if i == i_start else f32(stride * f32(i))
            break
        u, v = f32(u - fsu), f32(v - fsv)
    u, v = f32(fcu + fou), f32(fcv + fov)
    for i in range(i_start, K_N_REGION_STRIDE + 1):
        if u >= fsize or u < 0 or v >= fsize or v < 0:
            length_b = f32(max_considered_line_length)
            break
        if silhouette_at(r, trunc(v), trunc(u)) == region_id:
            if i == i_start:
                length_b = f32(0)
            else:
                length_f = f32(stride * f32(i))
            break
        u, v = f32(u + fsu), f32(v + fsv)
    return length_f, length_b


def point_on_valid_silhouette(r, i_center_u, i_center_v, stats=None):
    """IsPointOnValidSilhouette (depth_modality.cpp:728-734) via FocusedSilhouetteRenderer::SilhouetteValue; a pixel
    outside the focused image (read out of bounds by the reference) counts as another body's."""
    sc = f32(r.scale)
    su = trunc((f32(i_center_u) - f32(r.corner_u)) * sc + f32(0.5))
    sv = trunc((f32(i_center_v) - f32(r.corner_v)) * sc + f32(0.5))
    S = r.image.shape[0]
    if su < 0 or su >= S or sv < 0 or sv >= S:
        return False
    if silhouette_at(r, sv, su) != (int(r.id) & 0xFF):
        if stats is not None:
            stats["region_id_mismatch"] += 1
        return False
    return True


# ---- per-body drivers ------------------------------------------------------------------------------------------------
def _camera(wl, b, which):
    intr = wl.color_intrinsics if which == "color" else wl.depth_intrinsics
    per = getattr(wl, f"{which}_world2camera_per_body", None)
    w2c = getattr(wl, f"{which}_world2camera") if per is None else per[b]
    return intr, np.asarray(w2c, f32).reshape(3, 4)


def _rendering(wl, b, key, enabled):
    r = (getattr(wl, "renderings", None) or {}).get(b, {}).get(key)
    return r if enabled and r is not None and r.visible else None


def _scale(rp, corr):
    s = rp.scales
    return int(s[corr] if corr < len(s) else s[-1])


def region_valid(wl, b, pose, view, n_lines, geometric_valid, iteration, first_iteration, corr_iteration,
                 stats=None, parent_rule=False):
    """Predicted `valid` of body b's region lines [0, n_lines) after CalculateCorrespondences (region_modality.cpp:
    390-465): the first pass handles occlusions once (iteration - first_iteration) >= n_unoccluded_iterations, and if
    fewer than min_n_unoccluded_lines survive it, the second pass repeats without occlusion handling."""
    rp, model = wl.region, wl.region_model
    intr, w2c = _camera(wl, b, "color")
    fu, fv, ppu, ppv = (f32(getattr(intr, k)) for k in ("fu", "fv", "ppu", "ppv"))
    w_m1, h_m1 = intr.width - 1, intr.height - 1
    b2c = pose_mul(w2c, pose)
    fscale = f32(_scale(rp, corr_iteration))
    measured = rp.measure_occlusions and wl.depth_frames is not None
    if measured:
        dintr, dw2c = _camera(wl, b, "depth")
        b2d = pose_mul(dw2c, pose)
        offset_id = region_offset_id(rp.measured_depth_offset_radius, model, stats, parent_rule)
    dr = _rendering(wl, b, "region_depth", rp.model_occlusions)
    sr = _rendering(wl, b, "region_silhouette", rp.use_region_checking)
    modeled_id = region_offset_id(rp.modeled_depth_offset_radius, model, stats, parent_rule) if dr is not None else 0
    first = 8
    pts = model.points[view]

    def checks(i, handle):
        dp = pts[i]
        X = dp[0:3].astype(f32)
        x, y, z = apply(b2c, X)
        if min(f32(dp[7]), f32(dp[6])) * fu / (z * fscale) < f32(rp.min_continuous_distance):
            return False
        if parent_rule:
            if z <= f32(0):
                return False
        elif not z > f32(0):
            return False
        cu, cv = x * fu / z + ppu, y * fv / z + ppv
        icu, icv = trunc(cu + f32(0.5)), trunc(cv + f32(0.5))
        if icu < 0 or icu > w_m1 or icv < 0 or icv > h_m1:
            return False
        if sr is not None:
            nu, nv = normal2(b2c, dp[3:6].astype(f32))
            if not dynamic_line_region_sufficient(sr, rp.min_continuous_distance, fscale, cu, cv, nu, nv, stats):
                return False
        if handle and measured:
            xd, yd, zd = apply(b2d, X)
            dfu = f32(dintr.fu)
            du, dv = xd * dfu / zd + f32(dintr.ppu), yd * f32(dintr.fv) / zd + f32(dintr.ppv)
            diameter = f32(2) * f32(rp.measured_occlusion_radius) * (dfu / zd)
            off = f32(dp[first + offset_id])
            bound = (zd - off - f32(rp.measured_occlusion_threshold)) / f32(wl.depth_scale)
            if not window_unoccluded(wl.depth_frames[b], du, dv, diameter, bound, stats, parent_rule):
                return False
        if handle and dr is not None:
            diameter = f32(2) * f32(rp.modeled_occlusion_radius) * ((fu / z) * f32(dr.scale))
            off = f32(dp[first + modeled_id])
            if not modeled_window_unoccluded(dr, cu, cv, diameter, z - off - f32(rp.modeled_occlusion_threshold),
                                             stats, parent_rule):
                return False
        return True

    geometric_valid = np.asarray(geometric_valid[:n_lines]) != 0
    handle = (iteration - first_iteration) >= rp.n_unoccluded_iterations
    occ = handle and (measured or dr is not None)
    if stats is not None:
        stats["handled_passes" if occ else "unhandled_passes"] += 1
    valid = np.array([bool(geometric_valid[i]) and checks(i, occ) for i in range(n_lines)], bool)
    if occ and valid.sum() < rp.min_n_unoccluded_lines:
        if stats is not None:
            stats["fallbacks"] += 1
        valid = np.array([bool(geometric_valid[i]) and checks(i, False) for i in range(n_lines)], bool)
    return valid


def depth_valid(wl, b, pose, view, n_points, geometric_valid, iteration, first_iteration, stats=None,
                parent_rule=False):
    """Predicted `valid` of body b's depth points [0, n_points) after CalculateCorrespondences (depth_modality.cpp:
    255-313), with silhouette checking in both passes."""
    dp_, model = wl.depth, wl.depth_model
    intr, w2c = _camera(wl, b, "depth")
    fu, fv, ppu, ppv = (f32(getattr(intr, k)) for k in ("fu", "fv", "ppu", "ppv"))
    w_m1, h_m1 = intr.width - 1, intr.height - 1
    b2c = pose_mul(w2c, pose)
    dr = _rendering(wl, b, "depth_depth", dp_.model_occlusions)
    sr = _rendering(wl, b, "depth_silhouette", dp_.use_silhouette_checking)
    scaling = bool(dp_.use_depth_scaling)
    stride = model.stride_depth_offset
    first = 6
    pts = model.points[view]

    def checks(i, handle):
        dp = pts[i]
        x, y, z = apply(b2c, dp[0:3].astype(f32))
        cu, cv = x * fu / z + ppu, y * fv / z + ppv
        if parent_rule:
            if z <= f32(0):
                return False
        elif not z > f32(0):
            return False
        icu, icv = trunc(cu + f32(0.5)), trunc(cv + f32(0.5))
        if icu < 0 or icu > w_m1 or icv < 0 or icv > h_m1:
            return False
        if sr is not None and not point_on_valid_silhouette(sr, icu, icv, stats):
            return False
        if handle and dp_.measure_occlusions:
            off = f32(dp[first + depth_offset_id(dp_.measured_depth_offset_radius, z, scaling, stride, stats)])
            diameter = f32(2) * f32(dp_.measured_occlusion_radius) * fu
            if not scaling:
                diameter = diameter / z
            threshold = f32(dp_.measured_occlusion_threshold)
            if scaling:
                threshold = threshold * z
            bound = (z - off - threshold) / f32(wl.depth_scale)
            if not window_unoccluded(wl.depth_frames[b], cu, cv, diameter, bound, stats, parent_rule):
                return False
        if handle and dr is not None:
            off = f32(dp[first + depth_offset_id(dp_.modeled_depth_offset_radius, z, scaling, stride, stats)])
            m2p = fu * f32(dr.scale)
            if not scaling:
                m2p = m2p / z
            diameter = f32(2) * f32(dp_.modeled_occlusion_radius) * m2p
            threshold = f32(dp_.modeled_occlusion_threshold)
            if scaling:
                threshold = threshold * z
            if not modeled_window_unoccluded(dr, cu, cv, diameter, z - off - threshold, stats, parent_rule):
                return False
        return True

    geometric_valid = np.asarray(geometric_valid[:n_points]) != 0
    handle = (iteration - first_iteration) >= dp_.n_unoccluded_iterations
    occ = handle and (dp_.measure_occlusions or dr is not None)
    if stats is not None:
        stats["handled_passes" if occ else "unhandled_passes"] += 1
    valid = np.array([bool(geometric_valid[i]) and checks(i, occ) for i in range(n_points)], bool)
    if occ and valid.sum() < dp_.min_n_unoccluded_points:
        if stats is not None:
            stats["fallbacks"] += 1
        valid = np.array([bool(geometric_valid[i]) and checks(i, False) for i in range(n_points)], bool)
    return valid


def _bin(bgr, n_bins):
    shift = {2: 7, 4: 6, 8: 5, 16: 4, 32: 3, 64: 2}[n_bins]
    return ((int(bgr[0]) >> shift) * n_bins + (int(bgr[1]) >> shift)) * n_bins + (int(bgr[2]) >> shift)


def histogram_counts(wl, b, pose, view, n_lines, handle_occlusions, stats=None, parent_rule=False):
    """AddLinePixelColorsToTempHistograms (region_modality.cpp:1025-1155): per-bin pixel counts (foreground,
    background) the body's lines add, with occlusion handling as StartModality / CalculateResults ask for it."""
    with np.errstate(over="ignore", invalid="ignore"):   # the background distance of a model point may be huge
        return _histogram_counts(wl, b, pose, view, n_lines, handle_occlusions, stats, parent_rule)


def _histogram_counts(wl, b, pose, view, n_lines, handle_occlusions, stats, parent_rule):
    rp, model = wl.region, wl.region_model
    nb = rp.n_histogram_bins
    cnt_f = np.zeros(nb ** 3, np.int64)
    cnt_b = np.zeros(nb ** 3, np.int64)
    intr, w2c = _camera(wl, b, "color")
    fu, fv, ppu, ppv = (f32(getattr(intr, k)) for k in ("fu", "fv", "ppu", "ppv"))
    w_m1, h_m1 = intr.width - 1, intr.height - 1
    b2c = pose_mul(w2c, pose)
    measured = handle_occlusions and rp.measure_occlusions and wl.depth_frames is not None
    if measured:
        dintr, dw2c = _camera(wl, b, "depth")
        b2d = pose_mul(dw2c, pose)
        offset_id = region_offset_id(rp.measured_depth_offset_radius, model, stats, parent_rule)
    dr = _rendering(wl, b, "region_depth", handle_occlusions and rp.model_occlusions)
    sr = _rendering(wl, b, "region_silhouette", rp.use_region_checking)
    modeled_id = region_offset_id(rp.modeled_depth_offset_radius, model, stats, parent_rule) if dr is not None else 0
    img = wl.color_frames[b]
    ul = f32(rp.unconsidered_line_length)
    mcl = f32(rp.max_considered_line_length)
    for i in range(n_lines):
        dp = model.points[view][i]
        X = dp[0:3].astype(f32)
        x, y, z = apply(b2c, X)
        if parent_rule:
            if z <= f32(0):
                continue
        elif not z > f32(0):
            continue
        cu, cv = x * fu / z + ppu, y * fv / z + ppv
        icu, icv = trunc(cu + f32(0.5)), trunc(cv + f32(0.5))
        if icu < 0 or icu > w_m1 or icv < 0 or icv > h_m1:
            continue
        if dr is not None:
            diameter = f32(2) * f32(rp.modeled_occlusion_radius) * ((fu / z) * f32(dr.scale))
            if not modeled_window_unoccluded(dr, cu, cv, diameter, z - f32(dp[8 + modeled_id]) -
                                             f32(rp.modeled_occlusion_threshold), stats, parent_rule):
                continue
        if measured:
            xd, yd, zd = apply(b2d, X)
            dfu = f32(dintr.fu)
            du, dv = xd * dfu / zd + f32(dintr.ppu), yd * f32(dintr.fv) / zd + f32(dintr.ppv)
            diameter = f32(2) * f32(rp.measured_occlusion_radius) * (dfu / zd)
            bound = (zd - f32(dp[8 + offset_id]) - f32(rp.measured_occlusion_threshold)) / f32(wl.depth_scale)
            if not window_unoccluded(wl.depth_frames[b], du, dv, diameter, bound, stats, parent_rule):
                continue
        nu, nv = normal2(b2c, dp[3:6].astype(f32))
        length_f = length_b = mcl
        if sr is not None:
            length_f, length_b = dynamic_region_distance(sr, mcl, ul, cu, cv, nu, nv, length_f, length_b)
        length_f = min(length_f, f32(f32(dp[6]) * fu / z - f32(2) * ul))
        length_b = min(length_b, f32(f32(dp[7]) * fu / z - f32(2) * ul))
        anu, anv = abs(nu), abs(nv)
        if anu > anv:
            us, vs = f32(np.sign(nu)), nv / anu
            plf, plb = trunc(length_f * anu + f32(0.5)), trunc(length_b * anu + f32(0.5))
        else:
            us, vs = nu / anv, f32(np.sign(nv))
            plf, plb = trunc(length_f * anv + f32(0.5)), trunc(length_b * anv + f32(0.5))
        for sign, pl, cnt in ((-1, plf, cnt_f), (1, plb, cnt_b)):
            u = f32(cu - nu * ul + f32(0.5)) if sign < 0 else f32(cu + nu * ul + f32(0.5))
            v = f32(cv - nv * ul + f32(0.5)) if sign < 0 else f32(cv + nv * ul + f32(0.5))
            for _ in range(pl):
                iu, iv = trunc(u), trunc(v)
                if iu < 0 or iu > w_m1 or iv < 0 or iv > h_m1:
                    break
                cnt[_bin(img[iv, 3 * iu:3 * iu + 3], nb)] += 1
                u, v = (f32(u - us), f32(v - vs)) if sign < 0 else (f32(u + us), f32(v + vs))
    return cnt_f, cnt_b
