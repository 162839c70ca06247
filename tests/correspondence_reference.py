"""Restatement of the region line's segment probabilities and the depth point's correspondence search, with the
gradient / Hessian terms that consume them, written from M3T's region_modality.cpp / depth_modality.cpp rather than
from the oracle:

Region (region_modality.cpp):
- PrecalculateFunctionLookup / PrecalculateDistributionVariables (:910-936), PrecalculateIterationDependentVariables
  (:1011-1023);
- CalculateBasicLineData (:1231-1250) and the geometric part of IsLineValid (:1256-1267);
- CalculateSegmentProbabilities (:1433-1573), MultiplyPixelColorProbability (:1575-1598) from the body's histograms,
  CalculateDistribution (:1600-1637) and CalculateDistributionMoments (:1639-1658);
- CalculateGradientAndHessian (:485-558), global and local.

Depth (depth_modality.cpp):
- PrecalculateIterationDependentVariables (:648-654), CalculateBasicPointData (:656-666) and IsPointValid's
  projection test (:701-709);
- FindCorrespondence (:826-884), including the std::min(0, ...) lower depth bound (:851-852) that admits raw-0 pixels
  once the considered distance exceeds the point's depth;
- CalculateGradientAndHessian (:333-381).

Everything is float32 with one rounding per operation in the reference's order. int() is truncation and follows the
device's conversion for NaN and out-of-range values (occlusion_reference.trunc). std::round rounds halves away from
zero; std::max(a, b) is `a < b ? b : a`, so a NaN first argument is kept. powf(x, 2.0f) is the rounded square x * x.
The projection test is `!(z > 0)` (the reference's `z <= 0` lets a NaN depth through to an undefined int()). tanh,
atanh and powf of the function lookup and the minimum expected variance come from the C library, as on the host.

The closest view and the number of items are inputs, as in occlusion_reference; the checks on depth and renderer
images are not applied here (the occlusion_reference restates them).

`stats` (new_stats()) counts the decisions the cases were built to reach; see STAT_KEYS. The device's reciprocal screen
of the depth search (m3t_b200_kernels.cuh, DepthPoint) is emulated in the kernel's order of operations:
stats["screen_misses"] counts samples the exact test accepts and the screen would reject (must stay 0), and
stats["parent_screen_misses"] the same for the earlier fixed 1e-6 m^2 margin.
"""
from __future__ import annotations

import ctypes
import ctypes.util
import math

import numpy as np

from occlusion_reference import apply, normal2, pose_mul, trunc

f32 = np.float32
K_FUNCTION_LENGTH = 8        # region_modality.h:104
K_DISTRIBUTION_LENGTH = 12   # region_modality.h:105
K_SEGMENTS = K_FUNCTION_LENGTH + K_DISTRIBUTION_LENGTH - 1

STAT_KEYS = (
    # region lines
    "lines", "horizontal", "vertical", "ties_nu_nv", "forward", "reverse", "delta_r_ties", "start_truncated",
    "rejected_major_lo", "rejected_major_hi", "rejected_minor_lo", "rejected_minor_hi", "rejected_end_lo",
    "rejected_end_hi", "end_at_1", "end_at_minor_m2", "segment_fallbacks", "zero_areas", "subnormal_areas",
    "zero_entries", "nan_variances", "upper_0", "upper_1", "upper_11", "upper_12", "valid_lines",
    # depth points
    "points", "clipped_left", "clipped_top", "clipped_right", "clipped_bottom", "stride_1", "stride_above_1",
    "equal_ties", "raw_at_min", "raw_at_max", "raw0_admitted", "screen_misses", "parent_screen_misses",
    "samples", "valid_points")


def new_stats():
    return {k: 0 for k in STAT_KEYS}


_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
for _name, _n in (("tanhf", 1), ("atanhf", 1), ("powf", 2)):
    getattr(_libm, _name).restype = ctypes.c_float
    getattr(_libm, _name).argtypes = [ctypes.c_float] * _n


def std_max(a, b):
    return b if a < b else a


def std_round(x) -> float:
    """std::round of a float32: halves away from zero (exact in float64)."""
    x = float(x)
    t = math.trunc(x)
    if abs(x - t) >= 0.5:
        t += 1 if x > 0 else -1
    return float(t)


def last_valid(values, i):
    """LastValidValue (common.h:170-176)."""
    return values[min(i, len(values) - 1)]


# ---- region -----------------------------------------------------------------------------------------------------------
def function_lookup(rp):
    """(lookup_f, lookup_b, min_expected_variance) of PrecalculateFunctionLookup / PrecalculateDistributionVariables."""
    amp, slope = f32(rp.function_amplitude), f32(rp.function_slope)
    lf = np.zeros(K_FUNCTION_LENGTH, f32)
    for i in range(K_FUNCTION_LENGTH):
        x = f32(i) - f32(K_FUNCTION_LENGTH - 1) / f32(2)
        if slope == f32(0):
            lf[i] = f32(0.5) - amp * f32(int(f32(0) < x) - int(x < f32(0)))
        else:
            lf[i] = f32(0.5) - amp * f32(_libm.tanhf(float(x / (f32(2) * slope))))
    lb = (f32(1) - lf).astype(f32)
    laplace = f32(1) / (f32(2) * f32(_libm.powf(_libm.atanhf(float(f32(2) * amp)), 2.0)))
    return lf, lb, std_max(f32(laplace), slope)


class RegionIteration:
    """The iteration-dependent variables of one correspondence iteration (:1011-1023) and the camera's."""

    def __init__(self, wl, b, pose, corr):
        rp = wl.region
        intr = wl.color_intrinsics
        per = getattr(wl, "color_world2camera_per_body", None)
        w2c = np.asarray(wl.color_world2camera if per is None else per[b], f32).reshape(3, 4)
        self.b2c = pose_mul(w2c, pose)
        self.fu, self.fv, self.ppu, self.ppv = (f32(getattr(intr, k)) for k in ("fu", "fv", "ppu", "ppv"))
        self.w_m1, self.h_m1, self.w_m2, self.h_m2 = intr.width - 1, intr.height - 1, intr.width - 2, intr.height - 2
        self.scale = int(last_valid(rp.scales, corr))
        self.fscale = f32(self.scale)
        ll = K_SEGMENTS * self.scale
        self.ll_m1 = ll - 1
        self.ll_m1_half = f32(ll - 1) * f32(0.5)
        self.ll_half_m1 = f32(ll) * f32(0.5) - f32(1)
        sd = f32(last_valid(rp.standard_deviations, corr))
        self.variance = sd * sd
        self.lf, self.lb, self.min_expected_variance = function_lookup(rp)
        self.min_continuous_distance = f32(rp.min_continuous_distance)
        self.n_bins = rp.n_histogram_bins
        self.shift = {2: 7, 4: 6, 8: 5, 16: 4, 32: 3, 64: 2}[rp.n_histogram_bins]


def _pixel_probability(img, u, v, it, hist_f, hist_b):
    """GetProbabilities (color_histograms.cpp:94-102) and the normalisation of MultiplyPixelColorProbability."""
    px = img[v, 3 * u:3 * u + 3]
    nb, s = it.n_bins, it.shift
    idx = ((int(px[0]) >> s) * nb + (int(px[1]) >> s)) * nb + (int(px[2]) >> s)
    pf, pb = f32(hist_f[idx]), f32(hist_b[idx])
    if pf != 0 or pb != 0:
        total = pf + pb
        return pf / total, pb / total
    return f32(0.5), f32(0.5)


def region_line(it, img, hist_f, hist_b, point, stats=None):
    """One DataLine: a dict with the record's fields (REGION_LINE_DTYPE names) and `valid`."""
    st = stats if stats is not None else new_stats()
    st["lines"] += 1
    X = point[0:3].astype(f32)
    x, y, z = apply(it.b2c, X)
    nu, nv = normal2(it.b2c, point[3:6].astype(f32))
    cu = x * it.fu / z + it.ppu
    cv = y * it.fv / z + it.ppv
    rec = dict(valid=0, center_f_body=X, center_u=f32(cu), center_v=f32(cv), normal_u=nu, normal_v=nv,
               delta_r=f32(0), normal_component_to_scale=f32(0), distribution=np.zeros(K_DISTRIBUTION_LENGTH, f32),
               mean=f32(0), measured_variance=f32(0))
    continuous_distance = min(f32(point[7]), f32(point[6])) * it.fu / (z * it.fscale)
    if continuous_distance < it.min_continuous_distance or not z > f32(0):
        return rec
    icu, icv = trunc(cu + f32(0.5)), trunc(cv + f32(0.5))
    if icu < 0 or icu > it.w_m1 or icv < 0 or icv > it.h_m1:
        return rec
    # CalculateSegmentProbabilities
    if abs(nu) == abs(nv):
        st["ties_nu_nv"] += 1
    horizontal = abs(nv) < abs(nu)
    st["horizontal" if horizontal else "vertical"] += 1
    c_major, c_minor = (cu, cv) if horizontal else (cv, cu)
    n_major, n_minor = (nu, nv) if horizontal else (nv, nu)
    major_m1, minor_m1, minor_m2 = (it.w_m1, it.h_m1, it.h_m2) if horizontal else (it.h_m1, it.w_m1, it.w_m2)
    step = n_minor / n_major
    start = c_major - it.ll_half_m1
    major = trunc(start)
    if f32(-1) < start < f32(0):
        st["start_truncated"] += 1
    major_end = major + it.ll_m1
    minor_f = c_minor + step * (f32(major) - c_major) + f32(0.5)
    minor_f_end = minor_f + step * f32(it.ll_m1)
    for failed, key in ((major < 0, "major_lo"), (major_end > major_m1, "major_hi"),
                        (trunc(minor_f) < 0, "minor_lo"), (trunc(minor_f) > minor_m1, "minor_hi"),
                        (trunc(minor_f_end) < 1, "end_lo"), (trunc(minor_f_end) > minor_m2, "end_hi")):
        if failed:
            st["rejected_" + key] += 1
            return rec
    st["end_at_1"] += trunc(minor_f_end) == 1
    st["end_at_minor_m2"] += trunc(minor_f_end) == minor_m2
    forward = n_major > f32(0)
    st["forward" if forward else "reverse"] += 1
    sf = np.ones(K_SEGMENTS, f32)
    sb = np.ones(K_SEGMENTS, f32)
    for k in range(it.ll_m1 + 1):
        s = k // it.scale if forward else K_SEGMENTS - 1 - k // it.scale
        minor = trunc(minor_f)
        u, v = (major, minor) if horizontal else (minor, major)
        pf, pb = _pixel_probability(img, u, v, it, hist_f, hist_b)
        sf[s] = sf[s] * pf
        sb[s] = sb[s] * pb
        major += 1
        minor_f = minor_f + step
    ncts = abs(n_major) / it.fscale
    r = c_major - it.ll_m1_half
    if abs(float(r) - math.trunc(float(r))) == 0.5:
        st["delta_r_ties"] += 1
    delta_r = (f32(std_round(r)) + it.ll_m1_half - c_major) / n_major
    if it.scale > 1:
        for s in range(K_SEGMENTS):
            if sf[s] != 0 or sb[s] != 0:
                total = sf[s] + sb[s]
                sf[s], sb[s] = sf[s] / total, sb[s] / total
            else:
                st["segment_fallbacks"] += 1
                sf[s] = sb[s] = f32(0.5)
    # CalculateDistribution
    dist = np.zeros(K_DISTRIBUTION_LENGTH, f32)
    area = f32(0)
    for d in range(K_DISTRIBUTION_LENGTH):
        val = f32(1)
        for k in range(K_FUNCTION_LENGTH):
            val = val * (sf[d + k] * it.lf[k] + sb[d + k] * it.lb[k])
        dist[d] = val
        st["zero_entries"] += val == 0
        area = area + val
    st["zero_areas"] += area == 0
    st["subnormal_areas"] += bool(0 < area < np.finfo(f32).tiny)
    with np.errstate(invalid="ignore", divide="ignore"):
        dist = (dist / area).astype(f32)
    # CalculateDistributionMoments
    mfb = f32(0)
    for d in range(K_DISTRIBUTION_LENGTH):
        mfb = mfb + f32(d) * dist[d]
    var = f32(0)
    for d in range(K_DISTRIBUTION_LENGTH):
        dd = f32(d) - mfb
        var = var + (dd * dd) * dist[d]
    st["nan_variances"] += bool(np.isnan(var))
    st["valid_lines"] += 1
    rec.update(valid=1, delta_r=f32(delta_r), normal_component_to_scale=f32(ncts), distribution=dist,
               mean=f32(mfb - (f32(K_DISTRIBUTION_LENGTH) - f32(1)) / f32(2)),
               measured_variance=f32(std_max(var, it.min_expected_variance)))
    return rec


def region_lines(wl, b, pose, view, n, hist_f, hist_b, corr, stats=None, dtype=None):
    """Body b's lines [0, n) of the closest view `view` as a structured array (dtype: REGION_LINE_DTYPE)."""
    it = RegionIteration(wl, b, pose, corr)
    img = wl.color_frames[b]
    pts = wl.region_model.points[view]
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        recs = [region_line(it, img, hist_f, hist_b, pts[i], stats) for i in range(n)]
    out = np.zeros(n, dtype)
    for i, r in enumerate(recs):
        out[i]["model_index"] = i
        for k, v in r.items():
            out[i][k] = v
    return out


def region_gradient_hessian(wl, b, pose, lines, corr, opt, stats=None):
    """CalculateGradientAndHessian (:485-558) over the valid lines, float32 in the reference's order. (g, H [6, 6])."""
    st = stats if stats is not None else new_stats()
    it = RegionIteration(wl, b, pose, corr)
    rp = wl.region
    R = it.b2c[:, :3]
    g = np.zeros(6, f32)
    H = np.zeros((6, 6), f32)
    dl_plus_1_half = (f32(K_DISTRIBUTION_LENGTH) + f32(1)) / f32(2)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        for L in lines:
            if not L["valid"]:
                continue
            cb = L["center_f_body"].astype(f32)
            x, y, z = apply(it.b2c, cb)
            fu_z, fv_z = it.fu / z, it.fv / z
            xfu_z, yfv_z = x * fu_z, y * fv_z
            nu, nv, ncts = L["normal_u"], L["normal_v"], L["normal_component_to_scale"]
            delta_cs = (nu * (xfu_z + it.ppu - L["center_u"]) + nv * (yfv_z + it.ppv - L["center_v"]) -
                        L["delta_r"]) * ncts
            if opt < rp.n_global_iterations:
                dll = (L["mean"] - delta_cs) / L["measured_variance"]
            else:
                upper = trunc(delta_cs + dl_plus_1_half)
                for k in (0, 1, 11, 12):
                    st[f"upper_{k}"] += upper == k
                if upper <= 0 or upper >= K_DISTRIBUTION_LENGTH:
                    continue
                dist = L["distribution"]
                dll = (np.log(dist[upper]) - np.log(dist[upper - 1])) * f32(rp.learning_rate) / L["measured_variance"]
            dc = (ncts * nu * fu_z, ncts * nv * fv_z, ncts * (-nu * xfu_z - nv * yfv_z) / z)
            dt = [dc[0] * R[0, j] + dc[1] * R[1, j] + dc[2] * R[2, j] for j in range(3)]
            J = (cb[1] * dt[2] - cb[2] * dt[1], cb[2] * dt[0] - cb[0] * dt[2], cb[0] * dt[1] - cb[1] * dt[0],
                 dt[0], dt[1], dt[2])
            weight = it.min_expected_variance / (ncts * ncts * it.variance)
            wg, wh = weight * dll, weight / L["measured_variance"]
            for i in range(6):
                g[i] = g[i] + wg * J[i]
                for j in range(i + 1):
                    H[i, j] = H[i, j] - (wh * J[i]) * J[j]
    return g, np.tril(H) + np.tril(H, -1).T


# ---- depth ------------------------------------------------------------------------------------------------------------
class DepthIteration:
    def __init__(self, wl, b, pose, corr):
        dp = wl.depth
        intr = wl.depth_intrinsics
        per = getattr(wl, "depth_world2camera_per_body", None)
        w2c = np.asarray(wl.depth_world2camera if per is None else per[b], f32).reshape(3, 4)
        self.b2c = pose_mul(w2c, pose)
        self.fu, self.fv, self.ppu, self.ppv = (f32(getattr(intr, k)) for k in ("fu", "fv", "ppu", "ppv"))
        self.w_m1, self.h_m1 = intr.width - 1, intr.height - 1
        self.depth_scale = f32(wl.depth_scale)
        self.considered_distance = f32(last_valid(dp.considered_distances, corr))
        self.max_n_strides = trunc(self.considered_distance / f32(dp.stride_length) + f32(0.5))
        self.standard_deviation = f32(last_valid(dp.standard_deviations, corr))
        self.use_depth_scaling = bool(dp.use_depth_scaling)


def screen_bound(x, y):
    """The additive term of the screen for a point at camera coordinates (x, y): 2^-33 (|x| + |y|)^2 + 2^-126."""
    q = np.abs(np.asarray(x, f32)) + np.abs(np.asarray(y, f32))
    return f32(2.0 ** -33) * (q * q) + f32(2.0 ** -126)


def screen_passes(u, v, raw, x, y, z, best, it, bound=None):
    """The device's tests before its exact evaluation (DepthPoint's tile path), in the kernel's order: True where the
    sample is evaluated with the reference's expression. Arrays broadcast. bound: screen_bound() of the point; None:
    the earlier fixed margin, s > best + 1e-6 m^2."""
    rfu, rfv = f32(1) / it.fu, f32(1) / it.fv
    depth = np.asarray(raw, f32) * it.depth_scale
    dz0 = depth - f32(z)
    dz2 = dz0 * dz0
    ux = np.asarray(u, f32) - it.ppu
    vy = np.asarray(v, f32) - it.ppv
    ax = ux * depth * rfu - f32(x)
    ay = vy * depth * rfv - f32(y)
    s = ax * ax + ay * ay + dz2
    best = np.asarray(best, f32)
    screen = best + f32(1e-6) if bound is None else best * f32(1 + 2.0 ** -8) + bound
    return (dz2 < best) & ~(s > screen)


def exact_distance2(u, v, raw, x, y, z, it):
    """(tx, ty, depth, d2) of FindCorrespondence (:869-875) for arrays of samples."""
    depth = np.asarray(raw, f32) * it.depth_scale
    tx = (np.asarray(u, f32) - it.ppu) * depth / it.fu
    ty = (np.asarray(v, f32) - it.ppv) * depth / it.fv
    dx, dy, dz = tx - f32(x), ty - f32(y), depth - f32(z)
    return tx, ty, depth, dx * dx + dy * dy + dz * dz


def depth_point(it, image, point, stats=None):
    st = stats if stats is not None else new_stats()
    st["points"] += 1
    X = point[0:3].astype(f32)
    x, y, z = apply(it.b2c, X)
    rec = dict(valid=0, center_f_body=X, normal_f_body=point[3:6].astype(f32),
               correspondence_center_f_camera=np.zeros(3, f32))
    cu = x * it.fu / z + it.ppu
    cv = y * it.fv / z + it.ppv
    if not z > f32(0):
        return rec
    icu, icv = trunc(cu + f32(0.5)), trunc(cv + f32(0.5))
    if icu < 0 or icu > it.w_m1 or icv < 0 or icv > it.h_m1:
        return rec
    # FindCorrespondence
    cd = it.considered_distance
    if it.use_depth_scaling:
        cd = cd * z
    meter_to_pixel = it.fu / z
    diameter = f32(2) * cd * meter_to_pixel
    stride = trunc(diameter / f32(it.max_n_strides) + f32(1))
    n_strides = trunc(diameter / f32(stride) + f32(0.5))
    rd = n_strides * stride
    rr = f32(0.5) * f32(rd)
    u_min, v_min = trunc(cu - rr + f32(0.5)), trunc(cv - rr + f32(0.5))
    u_max, v_max = u_min + rd, v_min + rd
    st["clipped_left"] += u_min < 0
    st["clipped_top"] += v_min < 0
    st["clipped_right"] += u_max > it.w_m1
    st["clipped_bottom"] += v_max > it.h_m1
    st["stride_1" if stride == 1 else "stride_above_1"] += 1
    u_min, v_min, u_max, v_max = max(u_min, 0), max(v_min, 0), min(u_max, it.w_m1), min(v_max, it.h_m1)
    min_depth_value = min(f32(0), (z - cd) / it.depth_scale)   # std::min(0.0f, ...): the first argument on ties
    max_depth_value = (z + cd) / it.depth_scale
    best0 = cd * cd
    us = np.arange(u_min, u_max + 1, stride)
    vs = np.arange(v_min, v_max + 1, stride)
    if len(us) == 0 or len(vs) == 0:
        return rec
    vv, uu = np.meshgrid(vs, us, indexing="ij")
    raw = image[vv, uu].astype(f32)
    inside = (raw > min_depth_value) & (raw < max_depth_value)
    st["samples"] += int(inside.sum())
    st["raw_at_min"] += int((raw == min_depth_value).sum())
    st["raw_at_max"] += int((raw == max_depth_value).sum())
    st["raw0_admitted"] += int((inside & (raw == 0)).sum())
    tx, ty, depth, d2 = exact_distance2(uu, vv, raw, x, y, z, it)
    d2 = np.where(inside, d2, f32(np.inf)).ravel()
    # the running best before each sample in row-major order, and the samples the strict test takes
    before = np.minimum.accumulate(np.concatenate(([best0], d2[:-1]))).astype(f32)
    accepted = d2 < before
    for bound, key in ((screen_bound(x, y), "screen_misses"), (None, "parent_screen_misses")):
        ok = screen_passes(uu.ravel(), vv.ravel(), raw.ravel(), x, y, z, before, it, bound)
        st[key] += int((accepted & ~ok).sum())
    if not accepted.any():
        return rec
    i = int(np.argmin(d2))    # the first of equal minima wins: a later equal value is not < best
    st["equal_ties"] += int((d2 == d2[i]).sum() > 1)
    rec.update(valid=1, correspondence_center_f_camera=np.array([tx.ravel()[i], ty.ravel()[i], depth.ravel()[i]], f32))
    st["valid_points"] += 1
    return rec


def depth_points(wl, b, pose, view, n, corr, stats=None, dtype=None):
    """Body b's points [0, n) of the closest view `view` as a structured array (dtype: DEPTH_POINT_DTYPE)."""
    it = DepthIteration(wl, b, pose, corr)
    pts = wl.depth_model.points[view]
    out = np.zeros(n, dtype)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore", under="ignore"):
        for i in range(n):
            r = depth_point(it, wl.depth_frames[b], pts[i], stats)
            out[i]["model_index"] = i
            for k, v in r.items():
                out[i][k] = v
    return out


def depth_gradient_hessian(wl, b, pose, points, corr):
    """CalculateGradientAndHessian (:333-381) over the valid points. (g, H [6, 6])."""
    it = DepthIteration(wl, b, pose, corr)
    R, t = it.b2c[:, :3], it.b2c[:, 3]
    c2b = np.zeros((3, 4), f32)      # camera2body as the device and the oracle take it: [R^T | -R^T t]
    c2b[:, :3] = R.T
    for i in range(3):
        c2b[i, 3] = -(R[0, i] * t[0] + R[1, i] * t[1] + R[2, i] * t[2])
    g = np.zeros(6, f32)
    H = np.zeros((6, 6), f32)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        for P in points:
            if not P["valid"]:
                continue
            y = apply(c2b, P["correspondence_center_f_camera"].astype(f32))
            n = P["normal_f_body"].astype(f32)
            c = P["center_f_body"].astype(f32)
            eps = n[0] * (c[0] - y[0]) + n[1] * (c[1] - y[1]) + n[2] * (c[2] - y[2])
            cx = (y[1] * n[2] - y[2] * n[1], y[2] * n[0] - y[0] * n[2], y[0] * n[1] - y[1] * n[0])
            w = f32(1) / (it.standard_deviation * f32(P["correspondence_center_f_camera"][2]))
            sw = w * w
            v = [w * cx[0], w * cx[1], w * cx[2], w * n[0], w * n[1], w * n[2]]
            se = sw * eps
            for r in range(3):
                g[r] = g[r] - se * cx[r]
                g[3 + r] = g[3 + r] - se * n[r]
            for r in range(6):
                for q in range(r, 6):
                    H[r, q] = H[r, q] - v[r] * v[q]
    return g, np.triu(H) + np.triu(H, 1).T
