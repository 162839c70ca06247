"""Optimizer::CalculateOptimization of a kinematic structure restated in float64 NumPy (link.cpp, constraint.cpp,
soft_constraint.cpp, optimizer.cpp), independent of the CUDA kernel and of the float32 oracle's summation order.

Poses are 4x4 float64 matrices. Transform3fA::rotation() is taken as the linear block of the pose, as on the device and
in the oracle's ROTATION_LINEAR mode: the inputs are float32 poses, orthonormal to float32 rounding, and the polar
factor differs from the linear block by that rounding only.

Every product that the reference forms is formed here too, element by element (no BLAS, which may skip zero
factors): with an inf or a NaN in an input, 0 * inf = NaN spreads exactly as in the reference's small fixed-size
products. Eigen's triangular solves skip a column whose right-hand-side entry is exactly zero inside a panel of 8;
with finite factors that changes nothing, so it is not restated.

The second half builds the structure shapes that the structure tests share (limit shapes, degenerate systems).
"""
import copy
from dataclasses import dataclass, field

import numpy as np

_ERR = dict(invalid="ignore", over="ignore", divide="ignore")


# ---------------------------------------------------------------------------------------------------------------
# small Lie-group helpers
# ---------------------------------------------------------------------------------------------------------------
def T4(p):
    """[3,4] (or [12]) pose -> 4x4 float64"""
    m = np.eye(4)
    m[:3] = np.asarray(p, np.float64).reshape(3, 4)
    return m


def inv4(m):
    """rigid-transform inverse [R^T, -R^T t] (Transform3fA::inverse of an isometry)"""
    out = np.eye(4)
    out[:3, :3] = m[:3, :3].T
    out[:3, 3] = -(m[:3, :3].T @ m[:3, 3])
    return out


def skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def adjoint(m):
    """Link::Adjoint (link.cpp:341-348): [[R, 0], [skew(t) R, R]]"""
    R, t = m[:3, :3], m[:3, 3]
    a = np.zeros((6, 6))
    a[:3, :3] = R
    a[3:, :3] = skew(t) @ R
    a[3:, 3:] = R
    return a


def exp_so3(w):
    """Vector2Skewsymmetric(w).exp(): Rodrigues' formula in float64"""
    t = float(np.sqrt(np.dot(w, w)))
    K = skew(w)
    if t < 1e-8:
        return np.eye(3) + K + 0.5 * K @ K
    return np.eye(3) + (np.sin(t) / t) * K + ((1.0 - np.cos(t)) / (t * t)) * K @ K


def angle_axis(R):
    """Eigen::AngleAxis(Eigen::Quaternion(R)): Shepperd's quaternion of the matrix, then angle = 2 atan2(|v|, |w|)
    and the axis sign chosen so that the angle lies in [0, pi] (constraint.cpp:177)."""
    q = np.zeros(4)  # x, y, z, w
    t = R[0, 0] + R[1, 1] + R[2, 2]
    if t > 0.0:
        t = np.sqrt(t + 1.0)
        q[3] = 0.5 * t
        t = 0.5 / t
        q[0], q[1], q[2] = (R[2, 1] - R[1, 2]) * t, (R[0, 2] - R[2, 0]) * t, (R[1, 0] - R[0, 1]) * t
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        q[i] = 0.5 * t
        t = 0.5 / t
        q[3] = (R[k, j] - R[j, k]) * t
        q[j] = (R[j, i] + R[i, j]) * t
        q[k] = (R[k, i] + R[i, k]) * t
    n = float(np.sqrt(q[0] ** 2 + q[1] ** 2 + q[2] ** 2))
    if n == 0.0:
        return 0.0, np.array([1.0, 0.0, 0.0])
    angle = 2.0 * np.arctan2(n, abs(q[3]))
    if q[3] < 0.0:
        n = -n
    return angle, q[:3] / n


def xcotx(x):
    """x cot(x) (common.h:73-77), 1 at 0"""
    return 1.0 if x == 0.0 else x / np.tan(x)


def _dot(a, b, axis):
    """sum of the element-wise products (every product formed)"""
    with np.errstate(**_ERR):
        return (a * b).sum(axis=axis)


# ---------------------------------------------------------------------------------------------------------------
# the structure's state and the pieces of Optimizer::CalculateOptimization
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class State:
    """Link poses (link2world) and joint poses of every link, 4x4 float64 each, in the structure's link order."""
    link2world: np.ndarray   # [n_links, 4, 4]
    body2joint: np.ndarray
    joint2parent: np.ndarray

    @staticmethod
    def from_arrays(link2world, body2joint, joint2parent):
        f = lambda a: np.stack([T4(p) for p in np.asarray(a, np.float64).reshape(-1, 12)])
        return State(f(link2world), f(body2joint), f(joint2parent))

    def copy(self):
        return State(self.link2world.copy(), self.body2joint.copy(), self.joint2parent.copy())


def free_dirs(link):
    return [d for d in range(6) if link.free_directions[d]]


def dof_of(spec):
    return sum(len(free_dirs(l)) for l in spec.links)


def rows_of(c):
    return [d for d in range(6) if c.directions[d]]


def n_unknowns(spec):
    return dof_of(spec) + sum(len(rows_of(c)) for c in spec.constraints if not c.soft)


def link_jacobians(spec, state):
    """Link::CalculateJacobian (link.cpp:159-182): J_l [6, dof], the body-frame twist of link l per unknown. A child
    takes its parent's Jacobian through Adjoint((joint2parent body2joint)^-1) and adds its own joint columns
    Adjoint(body2joint^-1)[:, d] for its free directions d."""
    dof = dof_of(spec)
    J = np.zeros((len(spec.links), 6, dof))
    first = 0
    for l, link in enumerate(spec.links):
        if link.parent >= 0:
            ad = adjoint(inv4(state.joint2parent[l] @ state.body2joint[l]))
            J[l] = _dot(ad[:, :, None], J[link.parent][None, :, :], 1)
        own = adjoint(inv4(state.body2joint[l]))
        for k, d in enumerate(free_dirs(link)):
            J[l][:, first + k] = own[:, d]
        first += len(free_dirs(link))
    return J


def link_gradients(spec, g, H):
    """Link::CalculateGradientAndHessian (link.cpp:184-193): the sum over the link's modality sets (its body, then its
    extra bodies) of the region and depth gradients / Hessians. g [2, n_bodies, 6], H [2, n_bodies, 6, 6] (modality 0
    region, 1 depth). Links without a body have none."""
    g = np.asarray(g, np.float64)
    H = np.asarray(H, np.float64).reshape(g.shape[0], g.shape[1], 6, 6)
    gl = np.zeros((len(spec.links), 6))
    Hl = np.zeros((len(spec.links), 6, 6))
    with np.errstate(**_ERR):
        for l, link in enumerate(spec.links):
            if link.body < 0:
                continue
            for b in (link.body,) + tuple(getattr(link, "extra_bodies", ()) or ()):
                for m in range(g.shape[0]):
                    gl[l] += g[m, b]
                    Hl[l] += H[m, b]
    return gl, Hl


@dataclass
class JointGeometry:
    body22joint1: np.ndarray
    joint22joint1: np.ndarray
    angle: float
    axis: np.ndarray
    rotation_vector: np.ndarray
    translation_vector: np.ndarray


def joint_geometry(c, state):
    """The required poses of Constraint / SoftConstraint (constraint.cpp:88-92): joint 2 in joint 1, its angle-axis."""
    b22j1 = T4(c.body12joint1) @ inv4(state.link2world[c.link1]) @ state.link2world[c.link2]
    j22j1 = b22j1 @ inv4(T4(c.body22joint2))
    angle, axis = angle_axis(j22j1[:3, :3])
    return JointGeometry(b22j1, j22j1, angle, axis, angle * axis, j22j1[:3, 3].copy())


def unprojected_jacobian(jg, body2joint1, directions, rotation_rows=True, translation_rows=True):
    """Constraint::UnprojectedConstraintJacobian (constraint.cpp:205-274): d(rotation vector, translation) of joint 2
    in joint 1 per body-frame twist of the body whose pose in joint 1 is body2joint1, rows of the selected
    directions. Rotation rows: the inverse right Jacobian of SO(3) at the residual rotation times R(body2joint1);
    translation rows: [joint2 -> body translation x r_d, r_d]."""
    body2joint2 = inv4(jg.joint22joint1) @ body2joint1
    jt = inv4(body2joint2)[:3, 3]
    r1 = body2joint1[:3, :3]
    h = 0.5 * jg.angle
    xc = xcotx(h)
    a = jg.axis
    var = xc * np.eye(3) - h * skew(a) + (1.0 - xc) * np.outer(a, a)
    rows = []
    for d in range(6):
        if not directions[d] or (d < 3 and not rotation_rows) or (d >= 3 and not translation_rows):
            continue
        row = np.zeros(6)
        if d < 3:
            row[:3] = var[d] @ r1
        else:
            rr = r1[d - 3]
            row[:3] = np.cross(jt, rr)
            row[3:] = rr
        rows.append(row)
    return np.array(rows).reshape(-1, 6)


def constraint_residual_jacobian(c, state, J):
    """Constraint::CalculateResidualAndConstraintJacobian (constraint.cpp:81-103): residual [nr] (rotation vector /
    translation of joint 2 in joint 1, selected directions) and its Jacobian [nr, dof] = U2 J_link2 - U1 J_link1."""
    jg = joint_geometry(c, state)
    full = np.concatenate([jg.rotation_vector, jg.translation_vector])
    res = full[rows_of(c)]
    u2 = unprojected_jacobian(jg, jg.body22joint1, c.directions)
    u1 = unprojected_jacobian(jg, T4(c.body12joint1), c.directions)
    cj = _dot(u2[:, :, None], J[c.link2][None], 1) - _dot(u1[:, :, None], J[c.link1][None], 1)
    return res, cj


def soft_constraint_terms(c, state):
    """SoftConstraint::AddGradientsAndHessiansToLinks (soft_constraint.cpp:113-131, 220-270). Per part (rotation,
    translation) with selected components r: inactive while |r| <= max_distance; else the energy
    (|r| - d_max)^2 / (2 sd^2) gives g -= sign / sd^2 U^T (r - d_max r/|r|) and
    H -= 1 / sd^2 U^T (I - d_max / |r| (I - u u^T)) U, sign -1 for link 1 and +1 for link 2.
    Returns ((g1, H1), (g2, H2)) and [(part, |r|, max_distance, active)]."""
    jg = joint_geometry(c, state)
    out = []
    parts = []
    for li, (b2j1, sign) in enumerate(((T4(c.body12joint1), -1.0), (jg.body22joint1, 1.0))):
        g = np.zeros(6)
        H = np.zeros((6, 6))
        for part in range(2):
            sel = [d for d in range(3) if c.directions[d + 3 * part]]
            if not sel:
                continue
            vec = (jg.rotation_vector if part == 0 else jg.translation_vector)[sel]
            max_d = c.max_distance_rotation if part == 0 else c.max_distance_translation
            sd = c.standard_deviation_rotation if part == 0 else c.standard_deviation_translation
            dist = float(np.sqrt(np.dot(vec, vec)))
            active = dist > max_d
            if li == 0:
                parts.append((part, dist, float(max_d), active))
            if not active:
                continue
            U = unprojected_jacobian(jg, b2j1, c.directions, part == 0, part == 1)
            unit = vec / dist if dist > 0.0 else vec
            inv_var = 1.0 / (sd * sd)
            g -= sign * inv_var * (U.T @ (vec - unit * max_d))
            W = np.eye(len(sel)) - (max_d / dist) * (np.eye(len(sel)) - np.outer(unit, unit))
            H -= inv_var * (U.T @ W @ U)
        out.append((g, H))
    return tuple(out), parts


@dataclass
class System:
    a: np.ndarray            # [n, n], lower triangle meaningful (symmetric)
    b: np.ndarray            # [n]
    dof: int
    jacobians: np.ndarray    # [n_links, 6, dof]
    soft_parts: list = field(default_factory=list)   # (constraint, part, |r|, max_distance, active)


def build_system(spec, state, gl, Hl, drop_soft=None, drop_row=None, drop_tikhonov=None):
    """Optimizer::CalculateOptimization up to the solve (optimizer.cpp:144-159, 283-332): soft-constraint terms added to
    the links (constraint order), b = sum_l J_l^T g_l, a = -sum_l J_l^T H_l J_l, hard-constraint rows [C, 0] with
    b = residual, tikhonov_vector_ on the diagonal of the unknowns.
    drop_soft / drop_row / drop_tikhonov: leave out one soft constraint (its index in spec.constraints), zero one hard
    row (its index among the rows) or skip the Tikhonov term of one unknown - used to show the tests' gates are
    tight enough to notice a missing term."""
    dof = dof_of(spec)
    n = n_unknowns(spec)
    J = link_jacobians(spec, state)
    gl = np.array(gl, np.float64)
    Hl = np.array(Hl, np.float64)
    soft_parts = []
    with np.errstate(**_ERR):
        for ci, c in enumerate(spec.constraints):
            if not c.soft or ci == drop_soft:
                continue
            ((g1, H1), (g2, H2)), parts = soft_constraint_terms(c, state)
            gl[c.link1] += g1
            Hl[c.link1] += H1
            gl[c.link2] += g2
            Hl[c.link2] += H2
            soft_parts += [(ci,) + p for p in parts]
        a = np.zeros((n, n))
        b = np.zeros(n)
        for l in range(len(spec.links)):
            b[:dof] += _dot(J[l], gl[l][:, None], 0)
            jh = _dot(J[l][:, :, None], Hl[l][:, None, :], 0)        # [dof, 6]: (J^T H)[i, q]
            a[:dof, :dof] -= _dot(jh[:, :, None], J[l][None, :, :], 1)
        row = dof
        for c in spec.constraints:
            if c.soft:
                continue
            res, cj = constraint_residual_jacobian(c, state, J)
            for r in range(len(res)):
                if row - dof != drop_row:
                    b[row] = res[r]
                    a[row, :dof] = -cj[r]
                    a[:dof, row] = -cj[r]
                row += 1
        di = 0
        for link in spec.links:
            for d in free_dirs(link):
                if di != drop_tikhonov:
                    a[di, di] += spec.tikhonov_rotation if d < 3 else spec.tikhonov_translation
                di += 1
    return System(a, b, dof, J, soft_parts)


# Eigen::LDLT<MatrixXd, Lower>::_solve_impl replaces 1 / D_i by 0 where |D_i| <= tolerance. The tolerance followed is
# that of Eigen 3.3.2 (the oldest release the reference accepts), 1 / NumTraits<Scalar>::highest(); the device uses
# its float counterpart 1 / FLT_MAX. Later Eigen releases use numeric_limits<Scalar>::min() instead; either way an
# exactly zero pivot gives an exact zero.
LDLT_TOLERANCE = 1.0 / np.finfo(np.float64).max


@dataclass
class Factorization:
    mat: np.ndarray          # strictly lower: L; diagonal: D
    transpositions: np.ndarray
    zero_matrix: bool


def ldlt_factor(a):
    """Eigen's ldlt_inplace<Lower>::unblocked: at step k the largest |diagonal| of the not-yet-factorised tail is
    pivoted in (maxCoeff: the tail's first entry, replaced only by a strictly greater one, so the first maximum wins and
    a leading NaN stays); the diagonal of the tail is the original one - the left-looking update touches column k only.
    Column k is updated with the factored columns (temp = D_j L_kj), then divided by a valid (non-zero) pivot. A zero
    first pivot means the whole diagonal is zero: identity transpositions, stop (k == 0 && !pivot_is_valid). n <= 1:
    nothing to factorise."""
    n = a.shape[0]
    mat = np.tril(np.array(a, np.float64))
    trans = np.arange(n)
    if n <= 1:
        return Factorization(mat, trans, False)
    with np.errstate(**_ERR):
        for k in range(n):
            tail = np.abs(np.diag(mat)[k:])
            big, best = 0, tail[0]
            for i in range(1, len(tail)):
                if tail[i] > best:
                    big, best = i, tail[i]
            big += k
            trans[k] = big
            if big != k:  # symmetric swap of row / column k and big inside the lower triangle
                mat[[k, big], :k] = mat[[big, k], :k]
                mat[big + 1:, [k, big]] = mat[big + 1:, [big, k]]
                mat[k, k], mat[big, big] = mat[big, big], mat[k, k]
                for i in range(k + 1, big):
                    mat[i, k], mat[big, i] = mat[big, i], mat[i, k]
            if k > 0:
                temp = np.diag(mat)[:k] * mat[k, :k]
                mat[k, k] -= _dot(mat[k, :k], temp, 0)
                mat[k + 1:, k] -= _dot(mat[k + 1:, :k], temp[None, :], 1)
            akk = mat[k, k]
            valid = abs(akk) > 0.0
            if k == 0 and not valid:
                return Factorization(mat, np.arange(n), True)
            if valid:
                mat[k + 1:, k] /= akk
    return Factorization(mat, trans, False)


def ldlt_solve(a, b, factorization=None):
    """LDLT::_solve_impl: x = P^T L^-T D^+ L^-1 P b, D^+ the pseudo-inverse (0 for |D_i| <= LDLT_TOLERANCE)."""
    f = ldlt_factor(a) if factorization is None else factorization
    n = len(b)
    mat, trans = f.mat, f.transpositions
    x = np.array(b, np.float64)
    with np.errstate(**_ERR):
        for k in range(n):
            x[k], x[trans[k]] = x[trans[k]], x[k]
        for j in range(n):
            x[j + 1:] -= mat[j + 1:, j] * x[j]
        for i in range(n):
            d = mat[i, i]
            x[i] = x[i] / d if abs(d) > LDLT_TOLERANCE else 0.0
        for j in range(n - 1, -1, -1):
            x[:j] -= mat[j, :j] * x[j]
        for k in range(n - 1, -1, -1):
            x[k], x[trans[k]] = x[trans[k]], x[k]
    return x


def update_poses(spec, state, theta):
    """Link::UpdatePoses of every link in pre-order (optimizer.cpp:334-346, link.cpp:205-241). The variation of a link
    is [exp(skew(theta_r)), theta_t] over its free directions. A child moves its joint: joint2parent *= variation
    (fixed_body2joint_pose) or body2joint = variation * body2joint, then link2world = parent2world joint2parent
    body2joint. The root moves about its joint: link2world = link2world body2joint^-1 variation body2joint."""
    s = state.copy()
    theta = np.asarray(theta, np.float64)
    idx = 0
    for l, link in enumerate(spec.links):
        th = np.zeros(6)
        for d in free_dirs(link):
            th[d] = theta[idx]
            idx += 1
        var = np.eye(4)
        var[:3, :3] = exp_so3(th[:3])
        var[:3, 3] = th[3:]
        if link.parent >= 0:
            if link.fixed_body2joint_pose:
                s.joint2parent[l] = s.joint2parent[l] @ var
            else:
                s.body2joint[l] = var @ s.body2joint[l]
            s.link2world[l] = s.link2world[link.parent] @ s.joint2parent[l] @ s.body2joint[l]
        else:
            s.link2world[l] = s.link2world[l] @ inv4(s.body2joint[l]) @ var @ s.body2joint[l]
    return s


@dataclass
class Result:
    theta: np.ndarray
    updated: bool
    state: State             # after the update (the input state when the NaN guard refused it)
    system: System
    factorization: Factorization


def calculate_optimization(spec, state, g, H, **drop):
    """Optimizer::CalculateOptimization: g [2, n_bodies, 6], H [2, n_bodies, 6, 6] of the two modalities per body."""
    gl, Hl = link_gradients(spec, g, H)
    sysm = build_system(spec, state, gl, Hl, **drop)
    f = ldlt_factor(sysm.a)
    theta = ldlt_solve(sysm.a, sysm.b, f)
    if np.isnan(theta).any():   # optimizer.cpp:165
        return Result(theta, False, state.copy(), sysm, f)
    return Result(theta, True, update_poses(spec, state, theta), sysm, f)


def theta_blocks(theta, dof):
    """the joint variations theta[:dof] and the constraint multipliers theta[dof:]: different units and, with hard
    constraints, magnitudes orders apart, so every accuracy bar is taken per block"""
    theta = np.asarray(theta, np.float64)
    return [theta[:dof], theta[dof:]]


def theta_gates(theta_o32, theta64, dof):
    """The bar of a float32 solve, per block: max(4 |theta_oracle32 - theta64|inf, 1e-6 |theta64|inf) - no less accurate
    than the float32 reference arithmetic."""
    return [max(4.0 * np.abs(o - r).max(initial=0.0), 1e-6 * np.abs(r).max(initial=0.0))
            for o, r in zip(theta_blocks(theta_o32, dof), theta_blocks(theta64, dof))]


def theta_deviations(theta, theta64, dof):
    return [np.abs(t - r).max(initial=0.0) for t, r in zip(theta_blocks(theta, dof), theta_blocks(theta64, dof))]


def oracle_optimize(oracle, spec, state, g, H):
    """orc_optimize_structure (float32, the device's summation order, ROTATION_LINEAR / EXP_RODRIGUES) from the same
    state and the same per-body g / H: (theta, status)"""
    L = oracle.lib()
    so = oracle.OracleStructure(with_joint_poses(spec, state.body2joint[:, :3], state.joint2parent[:, :3]))
    S = so.as_struct()
    with np.errstate(**_ERR):
        gl, Hl = link_gradients(spec, g, H)
        gl, Hl = gl.astype(np.float32), Hl.reshape(-1, 36).astype(np.float32)
    l2w = np.ascontiguousarray(state.link2world[:, :3].reshape(-1, 12), np.float32)
    theta = np.zeros(n_unknowns(spec), np.float32)
    ok = L.orc_optimize_structure(S, oracle.ptr(gl), oracle.ptr(Hl), oracle.ROTATION_LINEAR, oracle.EXP_RODRIGUES,
                                  oracle.ptr(l2w), oracle.ptr(theta))
    return theta, ok


def struct_smem_bytes(n_links, dof, n, n_constraints):
    """k_structure's dynamic shared memory for one structure (StructSmemFloats, m3t_b200_structures.cuh): link poses,
    gradients, Hessians, two adjoints, variations (138 floats per link), the link Jacobians, 84 floats per constraint,
    the n x (n | 1) system, five vectors of n and 16 floats of padding."""
    lda = n | 1
    floats = n_links * 138 + n_links * 6 * max(dof, 1) + max(n_constraints, 1) * 84 + n * lda + 5 * n + 16
    return 4 * floats


def spec_smem_bytes(spec):
    return struct_smem_bytes(len(spec.links), dof_of(spec), n_unknowns(spec), len(spec.constraints))


# ---------------------------------------------------------------------------------------------------------------
# structure shapes shared by the structure tests
# ---------------------------------------------------------------------------------------------------------------
def rand_pose(rng, angle=1.0, trans=0.1):
    """random [3,4] float32 pose: rotation angle uniform in [0, angle], translation N(0, trans)"""
    rv = rng.normal(size=3)
    rv *= rng.uniform(0, angle) / np.linalg.norm(rv)
    p = np.zeros((3, 4), np.float32)
    p[:, :3] = exp_so3(rv)
    p[:, 3] = rng.normal(size=3) * trans
    return p


def tree16(synth, rng, bodies):
    """16-link branching tree (children of 0, 1, 2, 5, ...), free directions from one revolute axis to all six, some
    links moving body2joint (fixed_body2joint_pose = False), non-identity body2joint, one hard and one soft constraint."""
    parents = [-1, 0, 1, 1, 0, 4, 5, 5, 2, 8, 0, 10, 11, 11, 6, 3]
    frees = [(1, 1, 1, 1, 1, 1), (1, 0, 0, 0, 0, 0), (0, 1, 0, 0, 0, 0), (0, 0, 1, 1, 0, 0), (1, 1, 1, 0, 0, 0),
             (0, 0, 0, 1, 1, 1), (1, 0, 1, 0, 1, 0), (0, 1, 0, 0, 0, 1), (1, 1, 1, 1, 1, 1), (0, 0, 1, 0, 0, 0)]
    links = []
    for i, p in enumerate(parents):
        links.append(synth.LinkSpec(body=bodies[i], parent=p, body2joint=rand_pose(rng, 0.3, 0.02),
                                    joint2parent=synth.identity_pose() if p < 0 else rand_pose(rng, 0.6, 0.04),
                                    free_directions=frees[i % len(frees)], fixed_body2joint_pose=(i % 4 != 2)))
    cons = [synth.ConstraintSpec(link1=7, link2=12, body12joint1=rand_pose(rng, 0.5, 0.03),
                                 body22joint2=rand_pose(rng, 0.5, 0.03), directions=(1, 0, 0, 0, 1, 1)),
            synth.ConstraintSpec(link1=9, link2=15, body12joint1=rand_pose(rng, 0.5, 0.03),
                                 body22joint2=rand_pose(rng, 0.5, 0.03), directions=(1, 1, 1, 1, 1, 1), soft=True,
                                 max_distance_rotation=0.02, max_distance_translation=0.005,
                                 standard_deviation_rotation=0.1, standard_deviation_translation=0.02)]
    return synth.StructureSpec(links=links, constraints=cons, tikhonov_rotation=300.0, tikhonov_translation=3000.0)


def dof96_rows32(synth, rng, bodies):
    """16 six-DoF links (chain of four-link branches), 6 hard constraints between disjoint link pairs with 32 rows
    (96 + 32 = 128 unknowns), the other 26 of the 32 constraints soft: even ones with a max_distance far beyond any
    violation here (inside, no term), odd ones with a small max_distance (outside, active)."""
    I = synth.identity_pose
    links = [synth.LinkSpec(body=bodies[0], parent=-1, body2joint=rand_pose(rng, 0.2, 0.01), joint2parent=I())]
    for i in range(1, 16):
        links.append(synth.LinkSpec(body=bodies[i], parent=(i - 1) if i % 4 else 0, body2joint=rand_pose(rng, 0.2, 0.01),
                                    joint2parent=rand_pose(rng, 0.5, 0.04), fixed_body2joint_pose=(i % 5 != 3)))
    cons = []
    for k, dirs in enumerate([(1,) * 6, (1,) * 6, (0, 1, 1, 1, 1, 1), (1, 1, 1, 1, 1, 0), (1, 0, 1, 1, 1, 1),
                              (1, 1, 1, 0, 1, 1)]):
        l1, l2 = 2 * k + 1, 2 * k + 2
        cons.append(synth.ConstraintSpec(link1=l1, link2=l2, body12joint1=rand_pose(rng, 0.3, 0.03),
                                         body22joint2=rand_pose(rng, 0.3, 0.03), directions=dirs))
    for k in range(26):
        l1 = k % 16
        l2 = (l1 + 3 + k // 16) % 16
        inside = k % 2 == 0
        dirs = [(1, 1, 1, 1, 1, 1), (1, 1, 0, 0, 1, 1), (0, 0, 1, 1, 0, 0), (1, 0, 1, 0, 1, 0)][k % 4]
        cons.append(synth.ConstraintSpec(link1=l1, link2=l2, body12joint1=rand_pose(rng, 0.5, 0.05),
                                         body22joint2=rand_pose(rng, 0.5, 0.05), directions=dirs, soft=True,
                                         max_distance_rotation=100.0 if inside else 0.01,
                                         max_distance_translation=100.0 if inside else 0.002,
                                         standard_deviation_rotation=0.2, standard_deviation_translation=0.05))
    return synth.StructureSpec(links=links, constraints=cons, tikhonov_rotation=500.0, tikhonov_translation=5000.0)


def extra3(synth, rng, bodies):
    """3-link chain whose first two links carry 3 extra bodies each (Link::modality_ptrs of one physical body seen by
    four camera pairs)."""
    links = [synth.LinkSpec(body=bodies[0], parent=-1, body2joint=rand_pose(rng, 0.2, 0.01),
                            joint2parent=synth.identity_pose(), extra_bodies=tuple(bodies[3:6])),
             synth.LinkSpec(body=bodies[1], parent=0, body2joint=rand_pose(rng, 0.2, 0.01),
                            joint2parent=rand_pose(rng, 0.5, 0.04), free_directions=(1, 1, 0, 0, 0, 1),
                            extra_bodies=tuple(bodies[6:9])),
             synth.LinkSpec(body=bodies[2], parent=1, body2joint=synth.identity_pose(),
                            joint2parent=rand_pose(rng, 0.5, 0.04))]
    return synth.StructureSpec(links=links, tikhonov_rotation=200.0, tikhonov_translation=2000.0)


def bodyless_mid(synth, rng, bodies):
    """A link without a body below the root (its pose lives in the link, it gets no modality terms), with children
    that carry bodies and a soft constraint through it."""
    links = [synth.LinkSpec(body=bodies[0], parent=-1, body2joint=synth.identity_pose(), joint2parent=synth.identity_pose()),
             synth.LinkSpec(body=-1, parent=0, body2joint=rand_pose(rng, 0.2, 0.01), joint2parent=rand_pose(rng, 0.5, 0.04),
                            free_directions=(1, 1, 1, 0, 0, 0)),
             synth.LinkSpec(body=bodies[1], parent=1, body2joint=synth.identity_pose(), joint2parent=rand_pose(rng, 0.5, 0.04)),
             synth.LinkSpec(body=bodies[2], parent=1, body2joint=rand_pose(rng, 0.2, 0.01),
                            joint2parent=rand_pose(rng, 0.5, 0.04), free_directions=(0, 0, 1, 0, 0, 0))]
    cons = [synth.ConstraintSpec(link1=1, link2=3, body12joint1=rand_pose(rng, 0.3, 0.02),
                                 body22joint2=rand_pose(rng, 0.3, 0.02), directions=(1, 1, 1, 1, 1, 1), soft=True,
                                 max_distance_rotation=0.01, max_distance_translation=0.002,
                                 standard_deviation_rotation=0.1, standard_deviation_translation=0.02)]
    return synth.StructureSpec(links=links, constraints=cons, tikhonov_rotation=300.0, tikhonov_translation=3000.0)


def one_unknown(synth, rng, bodies):
    """One link with one free direction: n == 1 (Eigen's LDLT does not factorise)."""
    return synth.StructureSpec(links=[synth.LinkSpec(body=bodies[0], parent=-1, body2joint=rand_pose(rng, 0.3, 0.02),
                                                     joint2parent=synth.identity_pose(), free_directions=(0, 0, 1, 0, 0, 0))],
                               tikhonov_rotation=100.0, tikhonov_translation=1000.0)


def seven_unknowns(synth, rng, bodies):
    """Two links, 6 + 1 unknowns."""
    return synth.StructureSpec(links=[
        synth.LinkSpec(body=bodies[0], parent=-1, body2joint=synth.identity_pose(), joint2parent=synth.identity_pose()),
        synth.LinkSpec(body=bodies[1], parent=0, body2joint=rand_pose(rng, 0.2, 0.01), joint2parent=rand_pose(rng, 0.5, 0.04),
                       free_directions=(0, 0, 0, 1, 0, 0))], tikhonov_rotation=100.0, tikhonov_translation=1000.0)


def constrained83(synth, rng, bodies):
    """optimization_time.cpp's constrained shape: the root and 7 six-DoF children of it, consecutive links tied by
    7 x 5 constraint rows (48 + 35 = 83 unknowns)."""
    I = synth.identity_pose
    links = [synth.LinkSpec(body=bodies[0], parent=-1, body2joint=I(), joint2parent=I())]
    cons = []
    for j in range(1, 8):
        links.append(synth.LinkSpec(body=bodies[j], parent=0, body2joint=I(), joint2parent=rand_pose(rng, 0.5, 0.05)))
        cons.append(synth.ConstraintSpec(link1=j - 1, link2=j, body12joint1=synth.translation_pose(-0.01),
                                         body22joint2=I(), directions=(0, 1, 1, 1, 1, 1)))
    return synth.StructureSpec(links=links, constraints=cons, tikhonov_rotation=100.0, tikhonov_translation=1000.0)


# name -> (builder, number of bodies it uses)
LIMIT_SHAPES = {
    "tree16": (tree16, 16),
    "dof96_rows32": (dof96_rows32, 16),
    "extra3": (extra3, 9),
    "bodyless_mid": (bodyless_mid, 3),
    "one_unknown": (one_unknown, 1),
}


def implicit_structure(synth, body, tikhonov_rotation, tikhonov_translation):
    """The one-link structure the device gives a body that no structure references: a free root link with identity
    joint poses (the rigid-body optimiser)."""
    return synth.StructureSpec(links=[synth.LinkSpec(body=body, parent=-1, body2joint=synth.identity_pose(),
                                                     joint2parent=synth.identity_pose())],
                               tikhonov_rotation=tikhonov_rotation, tikhonov_translation=tikhonov_translation)


def random_gh(rng, n_bodies, scale=1.0):
    """Per-body gradients [2, n_bodies, 6] and symmetric negative definite Hessians [2, n_bodies, 6, 6] of the two
    modalities, float32, at the magnitudes of real region / depth terms."""
    g = np.zeros((2, n_bodies, 6), np.float32)
    H = np.zeros((2, n_bodies, 6, 6), np.float32)
    w = np.array([30, 30, 30, 300, 300, 300])
    for m in range(2):
        for b in range(n_bodies):
            A = rng.normal(size=(6, 6)) * w[:, None] * scale
            Hm = -(A @ A.T)
            H[m, b] = (0.5 * (Hm + Hm.T)).astype(np.float32)
            g[m, b] = rng.normal(size=6) * np.array([3, 3, 3, 30, 30, 30]) * scale
    return g, H


def start_state(spec, world_poses):
    """The state Optimizer::SetUp leaves: link poses from the bodies' poses (link2world for body-less links), joint
    poses from the spec, then CalculateConsistentPoses (UpdatePoses with theta = 0)."""
    l2w = np.stack([np.asarray(world_poses[l.body] if l.body >= 0 else (l.link2world if l.link2world is not None
                                                                         else np.eye(4)[:3]), np.float64).reshape(12)
                    for l in spec.links])
    s = State.from_arrays(l2w, [l.body2joint for l in spec.links], [l.joint2parent for l in spec.links])
    return update_poses(spec, s, np.zeros(dof_of(spec)))


def with_joint_poses(spec, body2joint, joint2parent):
    """A copy of spec whose links start from the given joint poses (the device's current ones)."""
    out = copy.deepcopy(spec)
    for k, l in enumerate(out.links):
        l.body2joint = np.asarray(body2joint[k], np.float32).reshape(3, 4)
        l.joint2parent = np.asarray(joint2parent[k], np.float32).reshape(3, 4)
    return out
