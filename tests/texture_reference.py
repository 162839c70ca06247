"""CPU restatement of the texture modality (M3T TextureModality, texture_modality.cpp) as the device computes it:
focus region, keyframe reconstruction from a focused silhouette rendering, brute-force Hamming kNN (k = 2) with the
ratio test, the Tukey-weighted reprojection gradient / Hessian, the keyframe rule of CalculateResults, and one
Optimizer step. Scalar float32 arithmetic in the order the kernels write it, so that integer truncations and
comparisons come out the same; the gradient sums are float64 (compared within a tolerance)."""
import numpy as np

f32 = np.float32
FLT_MIN = f32(1.17549435e-38)
ROI_MARGIN = 10


def pose_mul(a, b):
    """PoseMul: float[12] row-major 3x4, a * b, in the kernels' summation order."""
    a = np.asarray(a, f32).reshape(12)
    b = np.asarray(b, f32).reshape(12)
    o = np.zeros(12, f32)
    for i in range(3):
        for j in range(3):
            o[4 * i + j] = a[4 * i] * b[j] + a[4 * i + 1] * b[4 + j] + a[4 * i + 2] * b[8 + j]
        o[4 * i + 3] = a[4 * i] * b[3] + a[4 * i + 1] * b[7] + a[4 * i + 2] * b[11] + a[4 * i + 3]
    return o


def pose_inverse(p):
    """PoseInverse: cofactor inverse of the 3x3 part, translation -inv * t."""
    p = np.asarray(p, f32).reshape(12)
    m = [p[0], p[1], p[2], p[4], p[5], p[6], p[8], p[9], p[10]]

    def cof(i, j):
        return (m[3 * ((i + 1) % 3) + (j + 1) % 3] * m[3 * ((i + 2) % 3) + (j + 2) % 3] -
                m[3 * ((i + 1) % 3) + (j + 2) % 3] * m[3 * ((i + 2) % 3) + (j + 1) % 3])
    c00, c10, c20 = cof(0, 0), cof(1, 0), cof(2, 0)
    det = c00 * m[0] + c10 * m[3] + c20 * m[6]
    invdet = f32(1.0) / det
    inv = [c00 * invdet, c10 * invdet, c20 * invdet, cof(0, 1) * invdet, cof(1, 1) * invdet, cof(2, 1) * invdet,
           cof(0, 2) * invdet, cof(1, 2) * invdet, cof(2, 2) * invdet]
    o = np.zeros(12, f32)
    for i in range(3):
        o[4 * i:4 * i + 3] = inv[3 * i:3 * i + 3]
        o[4 * i + 3] = (-inv[3 * i]) * p[3] + (-inv[3 * i + 1]) * p[7] + (-inv[3 * i + 2]) * p[11]
    return o


def apply(p, v):
    return (p[0] * v[0] + p[1] * v[1] + p[2] * v[2] + p[3], p[4] * v[0] + p[5] * v[1] + p[6] * v[2] + p[7],
            p[8] * v[0] + p[9] * v[1] + p[10] * v[2] + p[11])


def tukey_norm(error, c):
    """TextureModality::TukeyNorm (texture_modality.cpp:1231-1237)."""
    error, c = f32(error), f32(c)
    if abs(error) <= c:
        return f32(c ** f32(2) / f32(6) * (f32(1) - (f32(1) - (error / c) ** f32(2)) ** f32(3)))
    return f32(c ** f32(2) / f32(6))


def focus(intr, b2c, radius, focused_image_size):
    """CalculateScaleAndRegionOfInterest (texture_modality.cpp:890-931): ((x, y, w, h), scale) or None."""
    fu, fv, ppu, ppv = (f32(intr[k]) for k in ("fu", "fv", "ppu", "ppv"))
    r = f32(radius)
    x, y, z = f32(b2c[3]), f32(b2c[7]), f32(b2c[11])
    if z < r * f32(1.5):
        return None
    x2, y2, z2, r2, rz = x * x, y * y, z * z, r * r, r * z
    z2_r2 = z2 - r2
    z3_zr2 = z2_r2 * z
    r_u = fu * (abs(x) * r2 + rz * np.sqrt(z2_r2 + x2)) / z3_zr2
    r_v = fv * (abs(y) * r2 + rz * np.sqrt(z2_r2 + y2)) / z3_zr2
    cu, cv = x * fu / z + ppu, y * fv / z + ppv
    m = f32(ROI_MARGIN)
    u_min, u_max = int(cu - r_u - m + f32(0.5)), int(cu + r_u + m + f32(0.5))
    v_min, v_max = int(cv - r_v - m + f32(0.5)), int(cv + r_v + m + f32(0.5))
    u_min, v_min = max(u_min, 0), max(v_min, 0)
    u_max, v_max = min(u_max, int(intr["width"]) - 1), min(v_max, int(intr["height"]) - 1)
    if u_min >= u_max or v_min >= v_max:
        return None
    return (u_min, v_min, u_max - u_min, v_max - v_min), f32(f32(focused_image_size) / max(f32(2) * r_u, f32(2) * r_v))


def crop_to_image(xy_crop, roi_x, roi_y, scale):
    """DetectAndComputeCorrKeypoints' focus offset (texture_modality.cpp:884-887)."""
    xy = np.asarray(xy_crop, f32).reshape(-1, 2)
    return np.stack([f32(roi_x) + xy[:, 0] / f32(scale), f32(roi_y) + xy[:, 1] / f32(scale)], 1).astype(f32)


def orientation(b2c):
    """R^T normalize(t) of a body2camera pose, as the device computes orientation_last_keyframe_."""
    p = np.asarray(b2c, f32).reshape(12)
    n2 = p[3] * p[3] + p[7] * p[7] + p[11] * p[11]
    t = (p[3], p[7], p[11])
    if n2 > 0:  # Eigen's normalized() leaves a zero vector zero
        n = np.sqrt(n2)
        t = (p[3] / n, p[7] / n, p[11] / n)
    return np.array([p[i] * t[0] + p[4 + i] * t[1] + p[8 + i] * t[2] for i in range(3)], f32)


def keyframe_fires(b2c_stale, last_orientation, age, max_rotation, max_age):
    """CalculateResults' rule (texture_modality.cpp:456-472) with the pose of the last gradient pass:
    (fires, new age)."""
    o = orientation(b2c_stale)
    d = f32(o[0] * last_orientation[0] + o[1] * last_orientation[1] + o[2] * last_orientation[2])
    with np.errstate(invalid="ignore"):
        diff = f32(np.arccos(d))
    age += 1
    return bool(diff > f32(max_rotation) or age > max_age), age


def _scanned(diameter):
    """A window whose diameter is not finite or is negative scans nothing and counts as unoccluded (its stride would be
    0 or negative)."""
    return bool(diameter >= f32(0)) and not np.isinf(diameter)


def _window(center_u, center_v, diameter, w_m1, h_m1):
    stride = int(diameter / f32(5) + f32(1))  # kMaxNOcclusionStrides
    n_strides = int(diameter / f32(stride) + f32(0.5))
    rd = n_strides * stride
    rr = f32(0.5) * f32(rd)
    u_min, v_min = int(center_u - rr + f32(0.5)), int(center_v - rr + f32(0.5))
    u_max, v_max = u_min + rd, v_min + rd
    return max(u_min, 0), max(v_min, 0), min(u_max, w_m1), min(v_max, h_m1), stride


def unoccluded_measured(X, m):
    """IsPointUnoccludedMeasured (texture_modality.cpp:1035-1085); m = dict(image (u16), intr, depth_scale, b2d,
    radius, threshold)."""
    intr = m["intr"]
    fu, fv, ppu, ppv = (f32(intr[k]) for k in ("fu", "fv", "ppu", "ppv"))
    x, y, z = apply(m["b2d"], X)
    cu, cv = x * fu / z + ppu, y * fv / z + ppv
    diameter = f32(2) * f32(m["radius"]) * (fu / z)
    if not _scanned(diameter):
        return True
    u0, v0, u1, v1, stride = _window(cu, cv, diameter, int(intr["width"]) - 1, int(intr["height"]) - 1)
    min_depth = int((z - f32(m["threshold"])) / f32(m["depth_scale"])) & 0xFFFF
    img = m["image"]
    for v in range(v0, v1 + 1, stride):
        for u in range(u0, u1 + 1, stride):
            d = int(img[v, u])
            if 0 < d < min_depth:
                return False
    return True


def unoccluded_modeled(X, m):
    """IsPointUnoccludedModeled (texture_modality.cpp:1087-1127); m = dict(rendering (focused depth image + corner /
    scale / projection terms), intr, b2c, radius, threshold)."""
    r, intr = m["rendering"], m["intr"]
    fu, fv, ppu, ppv = (f32(intr[k]) for k in ("fu", "fv", "ppu", "ppv"))
    x, y, z = apply(m["b2c"], X)
    sc = f32(r["scale"])
    diameter = f32(2) * f32(m["radius"]) * ((fu / z) * sc)
    if not _scanned(diameter):
        return True
    cu, cv = x * fu / z + ppu, y * fv / z + ppv
    fcu, fcv = (cu - f32(r["corner_u"])) * sc, (cv - f32(r["corner_v"])) * sc
    S = r["depth"].shape[0]
    u0, v0, u1, v1, stride = _window(fcu, fcv, diameter, S - 1, S - 1)
    mv = 65535
    for v in range(v0, v1 + 1, stride):
        for u in range(u0, u1 + 1, stride):
            mv = min(mv, int(r["depth"][v, u]))
    min_depth = f32(r["projection_term_a"]) / (f32(r["projection_term_b"]) - f32(mv))
    return bool(min_depth > z - f32(m["threshold"]))


def reconstruct(xy, rendering, intr, c2b, body_id, measured=None, modeled=None):
    """Reconstruct3DPoint (texture_modality.cpp:987-1023) + IsPointValid for every keypoint: (indexes, points [n, 3]).
    measured / modeled: the arguments of unoccluded_measured / unoccluded_modeled, None when the check is off."""
    sil, depth = rendering["silhouette"], rendering["depth"]
    S = sil.shape[0]
    cu0, cv0, sc = f32(rendering["corner_u"]), f32(rendering["corner_v"]), f32(rendering["scale"])
    a, b = f32(rendering["projection_term_a"]), f32(rendering["projection_term_b"])
    fu, fv, ppu, ppv = (f32(intr[k]) for k in ("fu", "fv", "ppu", "ppv"))
    idx, pts = [], []
    for i, (x, y) in enumerate(np.asarray(xy, f32)):
        us, vs = int((x - cu0) * sc + f32(0.5)), int((y - cv0) * sc + f32(0.5))
        if us < 0 or us > S - 1 or vs < 0 or vs > S - 1 or sil[vs, us] != body_id:
            continue
        d = a / (b - f32(depth[vs, us]))
        c = (d * (x - ppu) / fu, d * (y - ppv) / fv, d)
        X = apply(c2b, c)
        if measured is not None and not unoccluded_measured(X, measured):
            continue
        if modeled is not None and not unoccluded_modeled(X, modeled):
            continue
        idx.append(i)
        pts.append(X)
    return np.array(idx, np.int64), np.array(pts, f32).reshape(-1, 3)


def hamming(a, b):
    return int(np.unpackbits(np.bitwise_xor(a, b)).sum())


def knn2(queries, train):
    """cv::BFMatcher(NORM_HAMMING).knnMatch(k = 2): per query [(train_idx, distance), ...] (at most 2, best first; a
    strictly smaller distance enters, ties keep the earlier train index)."""
    out = []
    for q in np.asarray(queries, np.uint8).reshape(-1, 32):
        best = []
        for j, t in enumerate(np.asarray(train, np.uint8).reshape(-1, 32)):
            d = hamming(q, t)
            if len(best) < 2 or d < best[1][1]:
                k = len(best) if len(best) < 2 else 1
                while k > 0 and best[k - 1][1] > d:
                    k -= 1
                best.insert(k, (j, d))
                best = best[:2]
        out.append(best)
    return out


def match(keyframes, frame_xy, frame_desc, threshold):
    """CalculateCorrespondences at corr_iteration 0: keyframes = [(points [n, 3], descriptors [n, 32])] front to back.
    Returns (center_f_body [m, 3], correspondence_center [m, 2])."""
    cb, cc = [], []
    for pts, desc in keyframes:
        if len(desc) == 0 or len(frame_desc) == 0:
            continue
        for q, m in enumerate(knn2(desc, frame_desc)):
            if len(m) < 2:
                continue
            with np.errstate(invalid="ignore", divide="ignore"):
                if f32(m[0][1]) / f32(m[1][1]) >= f32(threshold):
                    continue
            cb.append(pts[q])
            cc.append(frame_xy[m[0][0]])
    return np.array(cb, f32).reshape(-1, 3), np.array(cc, f32).reshape(-1, 2)


def project(b2c, intr, cb):
    fu, fv, ppu, ppv = (f32(intr[k]) for k in ("fu", "fv", "ppu", "ppv"))
    out = np.zeros((len(cb), 2), f32)
    for i, p in enumerate(np.asarray(cb, f32)):
        x, y, z = apply(b2c, p)
        out[i] = (x * fu / z + ppu, y * fv / z + ppv)
    return out


def gradient_hessian(b2c, intr, cb, cc, standard_deviation, tukey_c):
    """CalculateGradientAndHessian (texture_modality.cpp:397-444): gradient [6], Hessian [6, 6] (float64 sums)."""
    fu, fv, ppu, ppv = (np.float64(intr[k]) for k in ("fu", "fv", "ppu", "ppv"))
    p = np.asarray(b2c, np.float64).reshape(3, 4)
    R = p[:, :3]
    variance = np.float64(standard_deviation) ** 2
    g, H = np.zeros(6), np.zeros((6, 6))
    b2c32 = np.asarray(b2c, f32).reshape(12)
    for X, X32, c, c32 in zip(np.asarray(cb, np.float64), np.asarray(cb, f32), np.asarray(cc, np.float64),
                              np.asarray(cc, f32)):
        # the residual in float32 as the device forms it (it cancels: pixel coordinates of a few hundred)
        x32, y32, z32 = apply(b2c32, X32)
        diff = np.array([x32 * f32(fu) / z32 + f32(ppu) - c32[0], y32 * f32(fv) / z32 + f32(ppv) - c32[1]], np.float64)
        x, y, z = R @ X + p[:, 3]
        e2 = float(diff @ diff)
        e = np.sqrt(e2)
        w = 1.0 / variance
        if e > FLT_MIN:
            w = (float(tukey_norm(e, tukey_c)) / e2) / variance
        dx_dX = np.array([[fu / z, 0, -x * fu / z ** 2], [0, fv / z, -y * fv / z ** 2]])
        dt = dx_dX @ R
        J = np.hstack([-dt @ skew(X), dt])
        g -= w * diff @ J
        H -= w * J.T @ J
    return g, H


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def optimize(body2world, g, H, tikhonov_rotation=1000.0, tikhonov_translation=30000.0):
    """Optimizer::CalculateOptimization + Link::UpdatePoses for one rigid body (float64)."""
    from scipy.linalg import expm
    a = -np.asarray(H, np.float64) + np.diag([tikhonov_rotation] * 3 + [tikhonov_translation] * 3)
    theta = np.linalg.solve(a, np.asarray(g, np.float64))
    T = np.eye(4)
    T[:3, :] = np.asarray(body2world, np.float64).reshape(3, 4)
    V = np.eye(4)
    V[:3, :3] = expm(skew(theta[:3]))
    V[:3, 3] = theta[3:]
    return (T @ V)[:3, :].astype(f32)
