"""CPU restatement of region-model generation (DESIGN.md §3 "k_region_contours / k_region_points"), operation for
operation in float32 like the kernels built with -fmad=false, so that contour lists, silhouettes, contour lengths and
points are compared bit for bit. Rasterisation is model_generation_reference.raster (one z-buffer per renderer, the
silhouette value is the id of the winning draw); border following restates cv::findContours(RETR_LIST,
CHAIN_APPROX_NONE) (Suzuki & Abe 1985 as OpenCV implements it) and is itself checked against cv2; the sampler replays
std::mt19937{7}. Test infrastructure only."""
import numpy as np

import model_generation_reference as mg
import render_reference as rr

f32 = np.float32
BACKGROUND_ID, MAIN_BODY_ID, DIFFERENT_BODY_ID = 0, 255, 120
CONTOUR_NORMAL_APPROX_RADIUS = 3
MIN_CONTOUR_LENGTH = 15
MAX_POINT_SAMPLING_TRIES = 100
MAX_SURFACE_GRADIENT = f32(10)
FLT_MAX = np.finfo(np.float32).max
POINT_FLOATS = 38

# 8-neighbour chain codes of the border follower: 0 = +x, counter-clockwise in image orientation (y down)
_DX = (1, 1, 0, -1, -1, -1, 0, 1)
_DY = (0, -1, -1, -1, 0, 1, 1, 1)


def _trace(lab, x0, y0, hole):
    """One border from (x0, y0) of the padded label image (icvFetchContour with nbd 2): visited pixels become 2,
    right-bound pixels -126. Returns the points in padded coordinates."""
    s = s_end = 0 if hole else 4
    while True:
        s = (s - 1) & 7
        x1, y1 = x0 + _DX[s], y0 + _DY[s]
        if lab[y1, x1] != 0 or s == s_end:
            break
    if s == s_end and lab[y1, x1] == 0:  # single pixel
        lab[y0, x0] = -126
        return [(x0, y0)]
    pts = []
    x3, y3 = x0, y0
    while True:
        s_end = s
        while s < 15:
            s += 1
            x4, y4 = x3 + _DX[s & 7], y3 + _DY[s & 7]
            if lab[y4, x4] != 0:
                break
        s &= 7
        if 0 <= s - 1 < s_end:
            lab[y3, x3] = -126
        elif lab[y3, x3] == 1:
            lab[y3, x3] = 2
        pts.append((x3, y3))
        if (x4, y4) == (x0, y0) and (x3, y3) == (x1, y1):
            break
        x3, y3 = x4, y4
        s = (s + 4) & 7
    return pts


def find_contours(mask):
    """cv::findContours(mask != 0, RETR_LIST, CHAIN_APPROX_NONE): a list of [n, 2] int32 (x, y) arrays. The image is
    zero-padded by one pixel; the raster scan starts an outer border at a 0 -> 1 step and a hole border at a step from
    a pixel marked 1 or 2 to 0; the list is in reverse order of discovery."""
    m = np.asarray(mask) != 0
    H, W = m.shape
    lab = np.zeros((H + 2, W + 2), np.int8)
    lab[1:-1, 1:-1] = m
    found = []
    for y in range(1, H + 1):
        row = lab[y] != 0
        for x in np.nonzero(row[1:W + 1] != row[0:W])[0] + 1:
            p, prev = lab[y, x], lab[y, x - 1]
            if prev == 0 and p == 1:
                found.append(_trace(lab, x, y, False))
            elif p == 0 and prev >= 1:
                found.append(_trace(lab, x - 1, y, True))
    return [np.array(c, np.int32).reshape(-1, 2) - 1 for c in reversed(found)]


def valid_contours(mask):
    """RegionModel::GenerateValidContours: the contours of the main body's silhouette, shorter ones dropped."""
    return [c for c in find_contours(mask == MAIN_BODY_ID) if len(c) >= MIN_CONTOUR_LENGTH]


def hypotf(a, b):
    """glibc's hypotf: the exact sum of the double squares, one double sqrt, rounded to float."""
    a, b = np.float64(f32(a)), np.float64(f32(b))
    return f32(np.sqrt(a * a + b * b))


class Setup:
    """Model::SetUpRenderer / AddBodiesToRenderer for RegionModel::GenerateModel. `groups` holds the associated bodies
    (rr.Geometry) as (fixed, fixed same-region, movable, movable same-region), each in insertion order. Renderers in
    the order main, same-region, occlusion, foreground, background (each only if used), as draw lists (body, id)."""

    def __init__(self, body, groups, sphere_radius, image_size):
        fixed, fixed_sr, movable, movable_sr = (list(g) for g in groups)
        B, M = BACKGROUND_ID, MAIN_BODY_ID
        self.body, self.r, self.S = body, f32(sphere_radius), int(image_size)
        self.renderers = {"main": [(body, M)] + [(g, DIFFERENT_BODY_ID) for g in fixed]}
        if fixed_sr or movable_sr:
            self.renderers["same_region"] = [(body, B)] + [(g, B) for g in fixed] + [(g, M) for g in fixed_sr + movable_sr]
        if movable:
            self.renderers["occlusion"] = [(body, B)] + [(g, B) for g in fixed] + [(g, M) for g in movable]
        if movable or fixed_sr or movable_sr:
            self.renderers["foreground"] = ([(body, M)] + [(g, B) for g in fixed] + [(g, B) for g in movable] +
                                            [(g, M) for g in fixed_sr])
            self.renderers["background"] = ([(body, M)] + [(g, B) for g in fixed] + [(g, M) for g in fixed_sr] +
                                            [(g, M) for g in movable_sr])
        rad = mg.HALF_D(body)
        self.fu = f32(0.5) * f32(self.S - mg.IMAGE_SIZE_SAFETY_BOUNDARY) / mg._libm_f("tanf", mg._libm_f("asinf", rad / self.r))
        self.pp = f32(self.S) / f32(2)
        self.ranges = {}
        for name, draws in self.renderers.items():
            lo, hi = self.r - rad, self.r + rad
            for g, _ in draws:
                lo, hi = min(self.r - mg.HALF_D(g), lo), max(self.r + mg.HALF_D(g), hi)
            self.ranges[name] = (lo, hi)
        lo, hi = self.ranges["main"]
        self.projection_term_a = hi * lo * f32(65535) / (hi - lo)
        self.projection_term_b = hi * f32(65535) / (hi - lo)

    def render(self, camera2body):
        """dict(name -> silhouette [S,S] u8) and the main renderer's depth image [S,S] u16."""
        S = self.S
        fS = f32(S)
        P00 = f32(2) * self.fu / fS
        P02 = f32(2) * (self.pp + f32(0.5)) / fS - f32(1)
        w2c = mg.pose_inverse(camera2body)
        sils, depth = {}, None
        for name, draws in self.renderers.items():
            lo, hi = self.ranges[name]
            P22 = (hi + lo) / (hi - lo)
            P23 = f32(-2) * hi * lo / (hi - lo)
            z = np.full((S, S), mg.CLEAR, np.uint64)
            for d, (g, _) in enumerate(draws):
                T = rr.pose_mul(w2c, g.geometry2body)
                M = np.zeros(16, f32)
                for c in range(4):
                    M[c] = P00 * T[c] + P02 * T[8 + c]
                    M[4 + c] = P00 * T[4 + c] + P02 * T[8 + c]
                    M[8 + c] = P22 * T[8 + c]
                    M[12 + c] = T[8 + c]
                M[11] = M[11] + P23
                mg.raster(M, g.triangles, g.enable_culling, S, d, z)
            ids = np.array([i for _, i in draws] + [0], np.uint8)
            draw = np.where(z == mg.CLEAR, len(draws), (z >> np.uint64(32)) & np.uint64(0xFFFF)).astype(np.int64)
            sils[name] = ids[draw]
            if name == "main":
                depth = (z >> np.uint64(48)).astype(np.uint16)
        return sils, depth


def view_points(st: Setup, camera2body, sils, depth, n_points, stride_depth_offset, max_radius_depth_offset, seed=7,
                stats=None):
    """RegionModel::GeneratePointData for one view -> ([n_points, 38] f32, contour_length, contours). `stats` (a dict)
    counts the contour points each validity rule rejects ('same_region', 'occlusion', 'fixed_depth'), the points next
    to a fixed body that pass ('fixed_kept'), and views that give up sampling ('exhausted')."""
    stats = {} if stats is None else stats
    S = st.S
    out = np.zeros((n_points, POINT_FLOATS), f32)
    main = sils["main"]
    contours = valid_contours(main)
    if not contours:
        return out, f32(0), contours
    a, b = st.projection_term_a, st.projection_term_b

    def dep(x, y):
        return a / (b - f32(depth[y, x]))

    px = st.r / st.fu
    max_dd = px * MAX_SURFACE_GRADIENT
    same, occ = sils.get("same_region"), sils.get("occlusion")
    valid = []
    for c in contours:  # IsContourPointValid
        for x, y in c:
            nb = ((x, y + 1), (x, y - 1), (x + 1, y), (x - 1, y))
            if same is not None and any(same[v, u] != BACKGROUND_ID for u, v in nb):
                stats["same_region"] = stats.get("same_region", 0) + 1
                continue
            if occ is not None and occ[y, x] != BACKGROUND_ID:
                stats["occlusion"] = stats.get("occlusion", 0) + 1
                continue
            s, n = f32(0), 0
            for u, v in nb:
                if main[v, u] == DIFFERENT_BODY_ID:
                    s = s + dep(u, v)
                    n += 1
            if n > 0 and s / f32(n) < dep(x, y) - max_dd:
                stats["fixed_depth"] = stats.get("fixed_depth", 0) + 1
                continue
            if n > 0:
                stats["fixed_kept"] = stats.get("fixed_kept", 0) + 1
            valid.append((x, y))
    contour_length = f32(len(valid)) * px
    if contour_length == 0:
        return out, contour_length, contours
    fg_img, bg_img = (sils["foreground"], sils["background"]) if "foreground" in sils else (main, main)
    flat = np.concatenate(contours, 0)
    fx, fy = flat[:, 0].astype(f32), flat[:, 1].astype(f32)

    def closest(u, v):  # FindClosestContourPoint: strict <, the first minimum wins
        du, dv = (fx - f32(u)).astype(np.float64), (fy - f32(v)).astype(np.float64)
        d = np.sqrt(du * du + dv * dv).astype(f32)
        return flat[int(np.argmin(d))]

    T = np.asarray(camera2body, f32).reshape(3, 4)
    stride_m = f32(stride_depth_offset)
    n_values = int(f32(max_radius_depth_offset) / stride_m + f32(1))
    gen = mg.mt19937_stream(seed)
    k, tries = 0, 0
    while k < n_points:
        if tries > MAX_POINT_SAMPLING_TRIES:
            stats["exhausted"] = stats.get("exhausted", 0) + 1
            out[k:] = 0
            return out, f32(0), contours
        tries += 1
        cx, cy = valid[next(gen) % len(valid)]
        seg = None
        for c in contours:  # CalculateContourSegment: the first contour and index holding the centre
            hit = np.nonzero((c[:, 0] == cx) & (c[:, 1] == cy))[0]
            if len(hit):
                i, n = int(hit[0]), len(c)
                seg = (c[(i - CONTOUR_NORMAL_APPROX_RADIUS) % n], c[(i + CONTOUR_NORMAL_APPROX_RADIUS) % n])
                break
        ddx, ddy = int(seg[1][0] - seg[0][0]), int(seg[1][1] - seg[0][1])
        if not hypotf(f32(ddx), f32(ddy)) > f32(CONTOUR_NORMAL_APPROX_RADIUS):
            continue
        vx, vy = -f32(ddy), f32(ddx)  # ApproximateNormalVector: -float(dy) (a zero dy gives -0), v / sqrt(squaredNorm)
        s = np.sqrt(vx * vx + vy * vy)
        nx, ny = vx / s, vy / s
        d = dep(cx, cy)  # FullDepthRenderer::PointVector on the main depth image
        c3 = (d * (f32(cx) - st.pp) / st.fu, d * (f32(cy) - st.pp) / st.fu, d)
        for r in range(3):
            out[k, r] = T[r, 0] * c3[0] + T[r, 1] * c3[1] + T[r, 2] * c3[2] + T[r, 3]
            out[k, 3 + r] = T[r, 0] * nx + T[r, 1] * ny + T[r, 2] * f32(0)
        ptm = c3[2] / st.fu
        out[k, 8:] = mg.depth_offsets(depth, cx, cy, ptm, stride_m, n_values, a, b)
        # CalculateLineDistances
        if abs(ny) < abs(nx):
            us, vs = f32(np.sign(nx)), ny / abs(nx)
        else:
            us, vs = nx / abs(ny), f32(np.sign(ny))
        u, v = f32(cx) + f32(0.5), f32(cy) + f32(0.5)
        while True:
            u, v = u - us, v - vs
            iu, iv = int(u), int(v)
            if not (0 <= iu < S and 0 <= iv < S) or fg_img[iv, iu] != MAIN_BODY_ID:
                e = closest(u + us - f32(0.5), v + vs - f32(0.5))
                out[k, 6] = ptm * hypotf(f32(int(e[0]) - cx), f32(int(e[1]) - cy))
                break
        u, v = f32(cx) + f32(0.5), f32(cy) + f32(0.5)
        while True:
            u, v = u + us, v + vs
            iu, iv = int(u), int(v)
            if iu < 0 or iu >= S or iv < 0 or iv >= S:
                out[k, 7] = FLT_MAX
                break
            if bg_img[iv, iu] == MAIN_BODY_ID:
                e = closest(u - f32(0.5), v - f32(0.5))
                out[k, 7] = ptm * hypotf(f32(int(e[0]) - cx), f32(int(e[1]) - cy))
                break
        k += 1
        tries = 0
    return out, contour_length, contours


def generate(body, groups=((), (), (), ()), sphere_radius=0.8, n_divides=4, n_points=200, max_radius_depth_offset=0.05,
             stride_depth_offset=0.002, image_size=2000, views=None, stats=None):
    """The whole model: (camera2body [nv,3,4], orientations [nv,3], contour lengths [nv], points [nv,n_points,38])."""
    st = Setup(body, groups, sphere_radius, image_size)
    poses = mg.geodesic_poses(n_divides, sphere_radius)
    sel = range(poses.shape[0]) if views is None else views
    pts, lengths = [], []
    for v in sel:
        sils, depth = st.render(poses[v])
        p, cl, _ = view_points(st, poses[v], sils, depth, n_points, stride_depth_offset, max_radius_depth_offset,
                               stats=stats)
        pts.append(p)
        lengths.append(cl)
    return (poses, poses[:, :, 2].copy(), np.array(lengths, f32),
            np.array(pts, f32).reshape(len(lengths), n_points, POINT_FLOATS))
