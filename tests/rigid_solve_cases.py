"""Systems for the rigid-body solve (Optimizer::CalculateOptimization of one free root link, then Link::UpdatePoses),
shared by the CPU and GPU tests of that solve: per case the region / depth / texture gradients and Hessians, the two
Tikhonov parameters and the start pose, all float32 and deterministic.

The device builds the system in float32 as a(lower) = (0 - H) + diag(tikhonov), b = 0 + g, with
H = (0 + H_region + H_depth) (+ H_texture), g likewise (PH_LOAD_GH of k_track, SumAndSolve of k_track2); the oracle's
orc_optimize_rigid does the same from the same sums. `system()` restates that, bit for bit.

Groups (Case.group): regular, pivot, singular, nonfinite, exp, sum. Tags (Case.tags) name the branch a case is there to
reach; the CPU test checks that every branch is reached.
"""
from dataclasses import dataclass, field
from itertools import permutations

import numpy as np

F32 = np.float32
TOLERANCE32 = F32(1.0) / F32(3.402823466e38)   # Eigen's 1 / highest() in float (a denormal)
SINF_FAST_LIMIT = 105615.0                     # |x| above which CUDA's sinf leaves its fast reduction
TIK_DEFAULT = (1000.0, 30000.0)


@dataclass
class Case:
    name: str
    group: str
    g: np.ndarray                  # [3, 6]    region, depth, texture
    H: np.ndarray                  # [3, 6, 6]
    tikhonov: tuple                # (rotation, translation)
    pose: np.ndarray               # [3, 4]
    texture: bool = False          # the body has a texture modality (its terms are added)
    knife_edge: bool = False       # float32 rounding alone decides the outcome: judged against the float32 oracle only
    a_direct: np.ndarray = None    # a system the modality sums cannot produce (a -0.0 diagonal): the test aid only
    tags: set = field(default_factory=set)

    def sums(self):
        """(g, H) as the device and the oracle sum them: 0 + region + depth (+ texture), float32"""
        with np.errstate(invalid="ignore", over="ignore"):
            g = (F32(0.0) + self.g[0]) + self.g[1]
            H = (F32(0.0) + self.H[0]) + self.H[1]
            if self.texture:
                g, H = g + self.g[2], H + self.H[2]
        return g.astype(F32), H.astype(F32)

    def system(self):
        """(a [6, 6] lower triangle meaningful, b [6]) in float32, as the kernels build them"""
        g, H = self.sums()
        with np.errstate(invalid="ignore", over="ignore"):
            a = np.tril(F32(0.0) - H)
            for i in range(6):
                a[i, i] = a[i, i] + F32(self.tikhonov[0] if i < 3 else self.tikhonov[1])
            b = F32(0.0) + g
        if self.a_direct is not None:
            a = np.tril(self.a_direct.astype(F32))
        return a.astype(F32), b.astype(F32)

    def finite_inputs(self):
        g, H = self.sums()
        return bool(np.isfinite(g).all() and np.isfinite(H).all())


def _pose(rng, angle=0.5, trans=0.3):
    rv = rng.normal(size=3)
    rv *= rng.uniform(0, angle) / np.linalg.norm(rv)
    t = float(np.linalg.norm(rv))
    K = np.array([[0, -rv[2], rv[1]], [rv[2], 0, -rv[0]], [-rv[1], rv[0], 0]])
    R = np.eye(3) + (np.sin(t) / t) * K + ((1 - np.cos(t)) / t ** 2) * K @ K
    p = np.zeros((3, 4), F32)
    p[:, :3] = R
    p[:, 3] = rng.normal(size=3) * trans + np.array([0, 0, 0.8])
    return p


def _spd(rng, scale=1.0):
    """-H of tracking scale: rotation block 1e2 - 1e4, translation block 1e5 - 1e7 (as test_ldlt_solve_spd)"""
    w = np.concatenate([10 ** rng.uniform(1, 2, 3), 10 ** rng.uniform(2.5, 3.5, 3)])
    A = rng.normal(size=(6, 6)) * w[:, None]
    return (A @ A.T) / 6.0 * scale


def _grad(rng, scale=1.0):
    return rng.normal(size=6) * np.array([3, 3, 3, 300, 300, 300]) * scale


def _case(name, group, a=None, b=None, tik=(0.0, 0.0), pose=None, rng=None, **kw):
    """a case whose region modality carries -a (so that a = (0 - H) + tik) and whose gradient is b"""
    g = np.zeros((3, 6), F32)
    H = np.zeros((3, 6, 6), F32)
    if a is not None:
        with np.errstate(invalid="ignore", over="ignore"):
            H[0] = -np.asarray(a, np.float64)
    if b is not None:
        g[0] = b
    p = pose if pose is not None else _pose(rng)
    return Case(name, group, g, H, (F32(tik[0]), F32(tik[1])), np.asarray(p, F32), **kw)


def _theta_system(theta):
    """a = I, b = theta: the solve returns theta exactly"""
    return np.eye(6), np.asarray(theta, F32)


def _t2(w):
    w = np.asarray(w, F32)
    return (w[0] * w[0] + w[1] * w[1]) + w[2] * w[2]


def _rotation_for_t2(target):
    """theta_r whose float32 t2 = w0^2 + w1^2 + w2^2 (ExpSkew's order) equals `target` exactly"""
    target = F32(target)
    x0 = F32(np.sqrt(np.float64(target) * 0.98))
    for _ in range(4000):
        x0 = np.nextafter(x0, F32(1.0), dtype=F32)
        xx = x0 * x0
        rest = target - xx
        if rest <= 0:
            break
        y = F32(np.sqrt(np.float64(rest)))
        for cand in (y, np.nextafter(y, F32(0), dtype=F32), np.nextafter(y, F32(1), dtype=F32)):
            w = np.array([x0, cand, 0.0], F32)
            if _t2(w) == target:
                return w
    raise AssertionError(f"no theta_r with t2 == {target!r}")


def regular(rng):
    out = []
    for k in range(24):
        a = _spd(rng)
        out.append(_case(f"spd{k}", "regular", a, _grad(rng), tik=TIK_DEFAULT if k % 2 else (0.0, 0.0), rng=rng,
                         tags={"regular"}))
    for s in (1e-30, 1e-20, 1e-10, 1e10, 1e20, 1e30):
        a = _spd(rng) * s
        out.append(_case(f"scaled{s:.0e}", "regular", a, _grad(rng, s), tik=(1000.0 * s, 30000.0 * s), rng=rng,
                         tags={"regular", "scaled"}))
    return out


def pivot(rng):
    out = []
    mags = np.array([1.0, 2.0, 4.0, 8.0, 16.0, 32.0]) * 1e3
    off = rng.normal(size=(6, 6)) * 20.0
    off = off + off.T
    np.fill_diagonal(off, 0.0)
    b = _grad(rng, 0.1)
    for k, perm in enumerate(permutations(range(6))):
        a = off + np.diag(mags[list(perm)] * np.where(np.arange(6) % 2, 1.0, -1.0) ** k)
        out.append(_case(f"order{k}", "pivot", a, b, rng=rng, tags={"order"}))
    for k, diag in enumerate(([5e3] * 6, [5e3, 5e3, 1e3, 1e3, 5e3, 5e3], [1e3, 7e3, 7e3, 2e3, 7e3, 1e3])):
        out.append(_case(f"tie{k}", "pivot", off + np.diag(diag), b, rng=rng, tags={"tie"}))
    for k, diag in enumerate(([5e3, -5e3, 5e3, -5e3, 5e3, -5e3], [-3e3, 3e3, 1e3, -1e3, 3e3, -3e3])):
        out.append(_case(f"opposite{k}", "pivot", off + np.diag(diag), b, rng=rng, tags={"opposite_signs"}))
    for k, zeros in enumerate(((-0.0, 0.0), (0.0, -0.0))):
        d = np.array([1e3, zeros[0], 2e3, zeros[1], 3e3, 0.0])
        a = (off * 0.01 + np.diag(np.zeros(6))).astype(F32)
        np.fill_diagonal(a, d.astype(F32))
        c = _case(f"signed_zero{k}", "pivot", None, b, rng=rng, tags={"signed_zero"}, knife_edge=True)
        c.a_direct = a
        out.append(c)
    return out


def singular(rng):
    out = []
    for r in range(6):
        V = rng.integers(-3, 4, size=(6, r)).astype(np.float64) * np.array([10, 10, 10, 300, 300, 300])[:, None]
        out.append(_case(f"rank{r}", "singular", V @ V.T, _grad(rng), rng=rng, knife_edge=r > 0,
                         tags={"rank"} | ({"zero_exit"} if r == 0 else set())))
    off = rng.normal(size=(6, 6)) * 50.0
    off = off + off.T
    np.fill_diagonal(off, 0.0)
    out.append(_case("zero_diagonal", "singular", off, _grad(rng), rng=rng, tags={"zero_exit"}))
    out.append(_case("all_zero", "singular", np.zeros((6, 6)), _grad(rng), rng=rng, tags={"zero_exit"}))
    for k in range(3):
        out.append(_case(f"negative_tikhonov{k}", "singular", _spd(rng), _grad(rng), tik=(-1000.0 * (k + 1), -3e4 * (k + 1)),
                         rng=rng, tags={"negative_tikhonov"}))
    # pivots D at Eigen's tolerance 1 / FLT_MAX (a denormal): above it divides, at or below it gives 0
    up = np.nextafter(TOLERANCE32, F32(1), dtype=F32)
    down = np.nextafter(TOLERANCE32, F32(0), dtype=F32)
    for name, d, tag in (("tolerance_above", up, "tolerance_divides"), ("tolerance_at", TOLERANCE32, "tolerance_zero"),
                         ("tolerance_below", down, "tolerance_zero")):
        diag = np.array([4.0, 3.0, 2.0, 1.0, 0.5, float(d)])
        bb = np.array([0.1, -0.1, 0.05, 0.01, -0.02, float(d) * 0.75])
        out.append(_case(name, "singular", np.diag(diag), bb, rng=rng, knife_edge=True, tags={tag}))
    return out


def nonfinite(rng):
    out = []
    base = _spd(rng)
    b = _grad(rng)
    nan, inf = np.nan, np.inf
    for i in range(6):
        bb = b.copy()
        bb[i] = nan
        out.append(_case(f"nan_g{i}", "nonfinite", base, bb, tik=TIK_DEFAULT, rng=rng, tags={f"nan_g{i}"}))
    for i in range(6):
        a = base.copy()
        a[i, i] = nan
        out.append(_case(f"nan_diag{i}", "nonfinite", a, b, tik=TIK_DEFAULT, rng=rng, tags={f"nan_diag{i}"}))
    for i in range(6):
        for j in range(i):
            a = base.copy()
            a[i, j] = a[j, i] = nan
            out.append(_case(f"nan_off{i}{j}", "nonfinite", a, b, tik=TIK_DEFAULT, rng=rng, tags={"nan_off"}))
    for i in range(6):
        a = base.copy()
        a[i, :] = nan
        a[:, i] = nan
        out.append(_case(f"nan_rowcol{i}", "nonfinite", a, b, tik=TIK_DEFAULT, rng=rng, tags={"nan_rowcol"}))
    for i in range(6):
        for s in (1.0, -1.0):
            a = base.copy()
            a[i, i] = s * inf
            out.append(_case(f"inf_diag{i}{'+' if s > 0 else '-'}", "nonfinite", a, b, tik=TIK_DEFAULT, rng=rng,
                             tags={"inf_diag"}))
    for i in range(6):
        bb = b.copy()
        bb[i] = inf if i % 2 else -inf
        out.append(_case(f"inf_g{i}", "nonfinite", base, bb, tik=TIK_DEFAULT, rng=rng, tags={"inf_g"}))
    for tik in ((nan, 3e4), (1e3, nan), (nan, nan), (inf, 3e4), (1e3, inf), (-inf, -inf), (inf, nan)):
        out.append(_case(f"tikhonov_{tik[0]}_{tik[1]}", "nonfinite", base, b, tik=tik, rng=rng,
                         tags={"nonfinite_tikhonov"}))
    # the zero-matrix exit through a NaN first pivot, other diagonal entries finite and non-zero
    a = base.copy()
    a[0, 0] = nan
    out.append(_case("nan_first_pivot_offdiag_zero", "nonfinite", np.diag(np.diag(a)), b, rng=rng,
                     tags={"nan_diag0", "zero_exit"}))
    return out


def exp_map(rng):
    out = []
    t01 = F32(0.01)
    for name, target in (("t2_at_branch", t01), ("t2_ulp_below", np.nextafter(t01, F32(0), dtype=F32)),
                         ("t2_ulp_above", np.nextafter(t01, F32(1), dtype=F32))):
        w = _rotation_for_t2(target)
        th = np.concatenate([w, [0.01, -0.02, 0.03]])
        tag = "exp_series" if target < t01 else "exp_closed"
        out.append(_case(name, "exp", *_theta_system(th), rng=rng, tags={tag, "t2_branch_point"}))
    for m in (0.1, 1.0, np.pi, 2 * np.pi, 10.0, 1e3, 1e5, 2e5, 1e6, 1e10):
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        th = np.concatenate([d * m, rng.normal(size=3) * 0.05])
        tags = {"exp_closed" if _t2(th[:3]) >= t01 else "exp_series"}
        if float(np.sqrt(np.float64(_t2(th[:3])))) > SINF_FAST_LIMIT:
            tags.add("sinf_large_argument")
        out.append(_case(f"theta_r{m:.3g}", "exp", *_theta_system(th), rng=rng, tags=tags))
    out.append(_case("theta_zero", "exp", *_theta_system(np.zeros(6)), rng=rng, tags={"exp_series", "theta_zero"}))
    for k, th in enumerate(([0.0, 0.05, 0.0, 0.01, 0.0, 0.0], [0.0, 0.0, 1.5, 0.0, 0.0, 0.2],
                            [0.3, 0.0, 0.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.1, 0.2, 0.3])):
        out.append(_case(f"theta_zero_components{k}", "exp", *_theta_system(th), rng=rng, tags={"theta_zero_components"}))
    for k in range(4):  # start poses drifted from orthonormal
        p = _pose(rng)
        p[:, :3] += rng.normal(size=(3, 3)).astype(F32) * F32(10.0 ** -(3 + k))
        out.append(_case(f"drifted{k}", "exp", _spd(rng), _grad(rng), tik=TIK_DEFAULT, pose=p,
                         tags={"drifted_pose"}))
    return out


def modality_sum(rng):
    """region, depth and texture terms that cancel: the float32 result depends on the order of the sum"""
    out = []
    for k in range(6):
        a = _spd(rng)
        big = _spd(rng) * 1e3
        gbig = _grad(rng, 1e5)
        g = np.zeros((3, 6), F32)
        H = np.zeros((3, 6, 6), F32)
        g[0], g[1] = gbig, -gbig + _grad(rng)
        H[0], H[1] = -big, big - a
        texture = k % 2 == 0
        if texture:  # texture carries the rest of what region and depth cancelled
            g[2] = _grad(rng, 1e-3)
            H[2] = -_spd(rng, 1e-3)
        out.append(Case(f"sum{k}", "sum", g, H, (F32(1000.0), F32(30000.0)), _pose(rng), texture=texture,
                        tags={"modality_sum"}))
    return out


def all_cases(seed=20261017):
    rng = np.random.default_rng(seed)
    return regular(rng) + pivot(rng) + singular(rng) + nonfinite(rng) + exp_map(rng) + modality_sum(rng)
