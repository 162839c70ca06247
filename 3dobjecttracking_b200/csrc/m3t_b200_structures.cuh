// m3t_b200_structures.cuh — Optimizer::CalculateOptimization for kinematic structures (SURVEY §8 a13-a16).
//
//   k_structure : one CTA per Optimizer (= one Link tree with its Constraints / SoftConstraints).
//     Link::CalculateJacobian                      (M3T/src/link.cpp:159-182, Adjoint :341-348)
//     SoftConstraint::AddGradientsAndHessiansToLinks (M3T/src/soft_constraint.cpp:113-131,220-349)
//     Constraint::CalculateResidualAndConstraintJacobian (M3T/src/constraint.cpp:81-103,176-274)
//     Optimizer::AddProjectedGradientsAndHessians / AddResidualsAndConstraintJacobians / tikhonov
//                                                  (M3T/src/optimizer.cpp:144-167,308-332)
//     Eigen::LDLT<MatrixXf, Lower> of the (DoF + nc)^2 system, NaN guard, Link::UpdatePoses (link.cpp:205-241)
//
// The per-link gradients / Hessians come from k_track (PH_STORE_LINK_GH). Summation orders are those of the
// CPU oracle (oracle/m3t_oracle.cpp, "Kinematic structures"), so that both agree to rounding of the
// transcendental functions only. All state that changes per update (joint poses, link poses) lives in global
// memory in LinkDev / the pose array, so the kernel is re-entrant per update iteration.
#pragma once

#include "m3t_b200_device.cuh"

namespace m3tb {

// index of (i, j), i >= j, in the packed lower triangle
__host__ __device__ __forceinline__ constexpr int Tri(int i, int j) { return i * (i + 1) / 2 + j; }

constexpr int kMaxLinks = 16;        // links per structure
constexpr int kMaxStructDof = 96;    // 16 x 6
constexpr int kMaxSystem = 128;      // DoF + constraint rows
constexpr int kMaxStructConstraints = 32;
constexpr int kStructThreads = 128;

struct LinkDev {
  int body, parent;          // body index or -1; parent link (index inside the structure) or -1
  int first_index, dof;      // first_jacobian_index_, DegreesOfFreedom()
  int free_directions[6];
  int fixed_body2joint;
  int level;                 // depth in the tree (root 0)
  float body2joint[12], joint2parent[12];
  float link2world[12];      // links without a body
  int n_extra, extra[3];     // further modality sets (bodies) of the same physical body: summed into the link, poses written back
};

struct ConstraintDev {
  int link1, link2;          // indices inside the structure
  int soft, n_rows, first_row, pad;
  int directions[6];
  float body12joint1[12], body22joint2[12];
  float max_distance_rotation, max_distance_translation, sd_rotation, sd_translation;
};

struct StructureDev {
  int first_link, n_links, first_constraint, n_constraints;
  int dof, n_rows;           // unknowns, hard-constraint rows
  float tikhonov_rotation, tikhonov_translation;
};

struct StructArgs {
  const StructureDev* structures;
  LinkDev* links;
  const ConstraintDev* constraints;
  float* poses;              // [n_bodies][12] body2world
  const float* gh_link;      // [n_bodies][27]: g[6], H lower[21] summed over the body's modalities, or null:
  const float* gh_region;    //   then 0 + gh_region + gh_depth (+ gh_texture) (Link::CalculateGradientAndHessian,
  const float* gh_depth;     //   link.cpp:184-193)
  const float* gh_texture;   // null when no body has a texture modality; else added for bodies with has_texture
  const BodyDev* bodies;
  int mode;                  // 0: CalculateOptimization, 1: CalculateConsistentPoses (UpdatePoses with theta = 0)
  float* theta_out;          // optional [n_structures][kMaxSystem]
  int* status;               // [n_structures]: 1 updated, 0 NaN guard
  const int* list;           // optional: CTA i handles structure list[i] (m3tb_refine_poses), null: structure i
};

__device__ __forceinline__ void Skew3(const float* v, float* m) {
  m[0] = 0.0f; m[1] = -v[2]; m[2] = v[1];
  m[3] = v[2]; m[4] = 0.0f; m[5] = -v[0];
  m[6] = -v[1]; m[7] = v[0]; m[8] = 0.0f;
}

// Link::Adjoint: [[R, 0], [skew(t) R, R]] (rotation() taken as the linear block, as everywhere on the device)
__device__ inline void AdjointDev(const float* pose, float* m) {
  float r[9], s[9], sr[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r[3 * i + j] = pose[4 * i + j];
  const float t[3] = {pose[3], pose[7], pose[11]};
  Skew3(t, s);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) sr[3 * i + j] = s[3 * i] * r[j] + s[3 * i + 1] * r[3 + j] + s[3 * i + 2] * r[6 + j];
  for (int k = 0; k < 36; ++k) m[k] = 0.0f;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      m[6 * i + j] = r[3 * i + j];
      m[6 * (i + 3) + j] = sr[3 * i + j];
      m[6 * (i + 3) + j + 3] = r[3 * i + j];
    }
}

// Eigen::Quaternionf(Matrix3f) followed by AngleAxisf = Quaternionf (constraint.cpp:177)
__device__ inline void AngleAxisDev(const float* m, float& angle, float* axis) {
  float q[4];
  float t = m[0] + m[4] + m[8];
  if (t > 0.0f) {
    t = sqrtf(t + 1.0f);
    q[3] = 0.5f * t;
    t = 0.5f / t;
    q[0] = (m[7] - m[5]) * t;
    q[1] = (m[2] - m[6]) * t;
    q[2] = (m[3] - m[1]) * t;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[4 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrtf(m[4 * i] - m[4 * j] - m[4 * k] + 1.0f);
    q[i] = 0.5f * t;
    t = 0.5f / t;
    q[3] = (m[3 * k + j] - m[3 * j + k]) * t;
    q[j] = (m[3 * j + i] + m[3 * i + j]) * t;
    q[k] = (m[3 * k + i] + m[3 * i + k]) * t;
  }
  float n = sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  if (n < 1.1920929e-7f) {
    const double sx = q[0], sy = q[1], sz = q[2];
    n = float(sqrt(sx * sx + sy * sy + sz * sz));
  }
  if (n != 0.0f) {
    angle = 2.0f * atan2f(n, fabsf(q[3]));
    if (q[3] < 0.0f) n = -n;
    axis[0] = q[0] / n; axis[1] = q[1] / n; axis[2] = q[2] / n;
  } else {
    angle = 0.0f;
    axis[0] = 1.0f; axis[1] = 0.0f; axis[2] = 0.0f;
  }
}

__device__ inline float XcotxDev(float x) {  // common.h:73-77 (including its behaviour just above pi/2)
  const float tf = tanf(x);
  if (tf <= 1.17549435e-38f) return 1.0f;
  if (tf >= 3.40282347e+38f) return 0.0f;
  return float(double(x) / tan(double(x)));
}

struct JointGeometryDev {
  float body22joint1[12], joint22joint1[12];
  float angle, axis[3], rotation_vector[3], translation_vector[3];
};

__device__ inline void CalcJointGeometryDev(const float* body12joint1, const float* body22joint2, const float* l1,
                                            const float* l2, JointGeometryDev& jg) {
  float inv1[12], tmp[12], inv22[12], rot[9];
  PoseInverse(l1, inv1);
  PoseMul(body12joint1, inv1, tmp);
  PoseMul(tmp, l2, jg.body22joint1);
  PoseInverse(body22joint2, inv22);
  PoseMul(jg.body22joint1, inv22, jg.joint22joint1);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) rot[3 * i + j] = jg.joint22joint1[4 * i + j];
  AngleAxisDev(rot, jg.angle, jg.axis);
  for (int i = 0; i < 3; ++i) {
    jg.rotation_vector[i] = jg.angle * jg.axis[i];
    jg.translation_vector[i] = jg.joint22joint1[4 * i + 3];
  }
}

// Constraint::UnprojectedConstraintJacobian for the selected directions, rows[nr][6]
__device__ inline int UnprojectedJacobianDev(const JointGeometryDev& jg, const float* body2joint1, const int* directions,
                                             bool rotation_rows, bool translation_rows, float* rows) {
  float inv_j[12], body2joint2[12], inv_b[12], r1[9];
  PoseInverse(jg.joint22joint1, inv_j);
  PoseMul(inv_j, body2joint1, body2joint2);
  PoseInverse(body2joint2, inv_b);
  const float jt[3] = {inv_b[3], inv_b[7], inv_b[11]};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r1[3 * i + j] = body2joint1[4 * i + j];
  const float angle_half = 0.5f * jg.angle;
  const float xc = XcotxDev(angle_half);
  float sk[9], var[9];
  Skew3(jg.axis, sk);
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      var[3 * i + j] = (xc * (i == j ? 1.0f : 0.0f) - angle_half * sk[3 * i + j]) + ((1.0f - xc) * jg.axis[i]) * jg.axis[j];
  int idx = 0;
  for (int d = 0; d < 6; ++d) {
    if (!directions[d]) continue;
    if (d < 3 && !rotation_rows) continue;
    if (d >= 3 && !translation_rows) continue;
    float* row = rows + 6 * idx;
    for (int k = 0; k < 6; ++k) row[k] = 0.0f;
    if (d < 3) {
      for (int j = 0; j < 3; ++j) row[j] = var[3 * d] * r1[j] + var[3 * d + 1] * r1[3 + j] + var[3 * d + 2] * r1[6 + j];
    } else {
      const float* rr = r1 + 3 * (d - 3);
      row[0] = jt[1] * rr[2] - jt[2] * rr[1];
      row[1] = jt[2] * rr[0] - jt[0] * rr[2];
      row[2] = jt[0] * rr[1] - jt[1] * rr[0];
      row[3] = rr[0]; row[4] = rr[1]; row[5] = rr[2];
    }
    idx++;
  }
  return idx;
}

// SoftConstraint::AddGradientsAndHessiansToLink: out[0..5] gradient, out[6..41] hessian of this constraint for one link
__device__ inline void SoftLinkTermsDev(const ConstraintDev& c, const JointGeometryDev& jg, const float* body2joint1,
                                        float sign, float* out) {
  for (int k = 0; k < 42; ++k) out[k] = 0.0f;
  for (int part = 0; part < 2; ++part) {
    int n = 0;
    float vec[3];
    for (int d = 0; d < 3; ++d)
      if (c.directions[d + 3 * part]) vec[n++] = part == 0 ? jg.rotation_vector[d] : jg.translation_vector[d];
    if (!n) continue;
    const float max_d = part == 0 ? c.max_distance_rotation : c.max_distance_translation;
    const float sd = part == 0 ? c.sd_rotation : c.sd_translation;
    float sq = 0.0f;
    for (int i = 0; i < n; ++i) sq += vec[i] * vec[i];
    const float dist = sqrtf(sq);
    if (!(dist > max_d)) continue;
    float rows[18];
    UnprojectedJacobianDev(jg, body2joint1, c.directions, part == 0, part == 1, rows);
    float unit[3] = {0.0f, 0.0f, 0.0f};
    for (int i = 0; i < n; ++i) unit[i] = vec[i];
    if (sq > 0.0f)
      for (int i = 0; i < n; ++i) unit[i] = vec[i] / dist;
    const float inv_var = 1.0f / (sd * sd);
    float e[3];
    for (int i = 0; i < n; ++i) e[i] = vec[i] - unit[i] * max_d;
    for (int k = 0; k < 6; ++k) {
      float acc = 0.0f;
      for (int i = 0; i < n; ++i) acc += rows[6 * i + k] * e[i];
      out[k] -= (sign * inv_var) * acc;
    }
    float w[9];
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) {
        const float id = i == j ? 1.0f : 0.0f;
        w[3 * i + j] = id - (max_d / dist) * (id - unit[i] * unit[j]);
      }
    for (int a = 0; a < 6; ++a)
      for (int b = 0; b < 6; ++b) {
        float acc = 0.0f;
        for (int i = 0; i < n; ++i) {
          float jw = 0.0f;
          for (int k = 0; k < n; ++k) jw += rows[6 * k + a] * w[3 * k + i];
          acc += jw * rows[6 * i + b];
        }
        out[6 + 6 * a + b] -= inv_var * acc;
      }
  }
}

// Shared-memory carve-up of one structure (floats unless noted); sizes depend on (n_links, dof, n, n_constraints)
struct StructSmem {
  float *l2w, *g, *H, *ad, *adj, *jac, *var, *cdata, *a, *b, *dst, *temp, *absdiag;
  int* trans;
  int lda;
};
__host__ __device__ inline size_t StructSmemFloats(int n_links, int dof, int n, int n_constraints) {
  const int lda = n | 1;
  return size_t(n_links) * (12 + 6 + 36 + 36 + 36 + 12) + size_t(n_links) * 6 * (dof > 0 ? dof : 1) +
         size_t(n_constraints > 0 ? n_constraints : 1) * 84 + size_t(n) * lda + size_t(n) * 5 + 16;
}
__device__ inline StructSmem CarveStructSmem(float* base, int nl, int dof, int n, int nc) {
  StructSmem s;
  float* p = base;
  s.l2w = p; p += nl * 12;
  s.g = p; p += nl * 6;
  s.H = p; p += nl * 36;
  s.ad = p; p += nl * 36;
  s.adj = p; p += nl * 36;
  s.var = p; p += nl * 12;
  s.jac = p; p += size_t(nl) * 6 * (dof > 0 ? dof : 1);
  s.cdata = p; p += size_t(nc > 0 ? nc : 1) * 84;
  s.lda = n | 1;
  s.a = p; p += size_t(n) * s.lda;
  s.b = p; p += n;
  s.dst = p; p += n;
  s.temp = p; p += n;
  s.absdiag = p; p += n;
  s.trans = reinterpret_cast<int*>(p);
  return s;
}

// The solver's barriers over the first T threads of a CTA (T a multiple of 32; k_structure passes its whole CTA).
// Named barrier 1 keeps them independent of any other warps of the CTA.
__device__ __forceinline__ void StructSync(int T) { asm volatile("bar.sync 1, %0;" ::"r"(T) : "memory"); }
__device__ __forceinline__ int StructSyncOr(int T, int pred) {
  int out;
  asm volatile(
      "{\n"
      ".reg .pred p, q;\n"
      "setp.ne.s32 p, %1, 0;\n"
      "bar.red.or.pred q, 1, %2, p;\n"
      "selp.s32 %0, 1, 0, q;\n"
      "}\n"
      : "=r"(out)
      : "r"(pred), "r"(T)
      : "memory");
  return out;
}

// Link::UpdatePoses for every link (optimizer.cpp:334-346, link.cpp:205-241); theta in s.dst. The new link poses are
// left in s.l2w (the caller publishes the bodies' poses), joint poses go to the links' global records.
__device__ inline void UpdatePosesBlock(const StructSmem& s, LinkDev* links, int nl, int tid, int T) {
  // ---- Link::UpdatePoses: pose variations in parallel, then the chain products in pre-order ----
  if (tid < nl) {
    const LinkDev& link = links[tid];
    float th[6];
    int idx = link.first_index;
    for (int d = 0; d < 6; ++d) th[d] = link.free_directions[d] ? s.dst[idx++] : 0.0f;
    float e[9];
    ExpSkew(th, e);
    float* var = s.var + 12 * tid;
    var[0] = e[0]; var[1] = e[1]; var[2] = e[2]; var[3] = th[3];
    var[4] = e[3]; var[5] = e[4]; var[6] = e[5]; var[7] = th[4];
    var[8] = e[6]; var[9] = e[7]; var[10] = e[8]; var[11] = th[5];
  }
  StructSync(T);
  if (tid == 0) {
    for (int l = 0; l < nl; ++l) {
      LinkDev& link = links[l];
      const float* var = s.var + 12 * l;
      float* l2w = s.l2w + 12 * l;
      float tmp[12], tmp2[12], out[12];
      if (link.parent >= 0) {
        if (link.fixed_body2joint) {
          PoseMul(link.joint2parent, var, tmp);
          for (int k = 0; k < 12; ++k) link.joint2parent[k] = tmp[k];
          PoseMul(s.l2w + 12 * link.parent, tmp, tmp2);
          PoseMul(tmp2, link.body2joint, out);
        } else {
          PoseMul(var, link.body2joint, tmp);
          for (int k = 0; k < 12; ++k) link.body2joint[k] = tmp[k];
          PoseMul(s.l2w + 12 * link.parent, link.joint2parent, tmp2);
          PoseMul(tmp2, tmp, out);
        }
      } else {
        float inv[12];
        PoseInverse(link.body2joint, inv);
        PoseMul(l2w, inv, tmp);
        PoseMul(tmp, var, tmp2);
        PoseMul(tmp2, link.body2joint, out);
      }
      for (int k = 0; k < 12; ++k) l2w[k] = out[k];
      if (link.body < 0)
        for (int k = 0; k < 12; ++k) link.link2world[k] = out[k];
    }
  }
}

// Optimizer::CalculateOptimization for one structure, executed by the first T threads of one CTA (tid < T). In: s.l2w (link poses),
// s.g / s.H (the links' summed modality gradients / Hessians), the links' joint poses in global memory. Out: s.l2w,
// joint poses, theta_out[n] (optional). Returns false when the NaN guard (optimizer.cpp:165) skipped the update.
// Not inlined: this rarely executed, latency-bound code is kept out of its caller's register allocation.
static __device__ __noinline__ bool StructureSolveBlock(const StructureDev& st, LinkDev* links, const ConstraintDev* cons,
                                                 const StructSmem& s, float* theta_out, int tid, int T) {
  const int nl = st.n_links, dof = st.dof, nc = st.n_constraints, n = st.dof + st.n_rows;
  const int lda = s.lda;
  StructSync(T);
  // ---- Link::CalculateJacobian, part 1: the two adjoints of every link (independent of the parent) ----
  if (tid < nl) {
    const LinkDev& link = links[tid];
    float prod[12], inv[12];
    if (link.parent >= 0) {
      PoseMul(link.joint2parent, link.body2joint, prod);
      PoseInverse(prod, inv);
      AdjointDev(inv, s.ad + 36 * tid);
    }
    PoseInverse(link.body2joint, inv);
    AdjointDev(inv, s.adj + 36 * tid);
  }
  for (int e = tid; e < n * lda; e += T) s.a[e] = 0.0f;
  for (int e = tid; e < n; e += T) s.b[e] = 0.0f;
  StructSync(T);
  // part 2: parent Jacobian pushed through the adjoint, then the link's own joint columns (pre-order = list order)
  for (int l = 0; l < nl; ++l) {
    const LinkDev& link = links[l];
    float* J = s.jac + size_t(l) * 6 * dof;
    const float* Jp = link.parent >= 0 ? s.jac + size_t(link.parent) * 6 * dof : nullptr;
    for (int e = tid; e < 6 * dof; e += T) {
      const int i = e / dof, c = e - i * dof;
      float v = 0.0f;
      if (Jp) {
        float acc = 0.0f;
        for (int k = 0; k < 6; ++k) acc += s.ad[36 * l + 6 * i + k] * Jp[size_t(k) * dof + c];
        v = acc;
      }
      if (c >= link.first_index && c < link.first_index + link.dof) {
        int d = 0, seen = c - link.first_index;  // the (c - first)-th free direction
        for (; d < 6; ++d)
          if (link.free_directions[d]) { if (seen == 0) break; --seen; }
        v = s.adj[36 * l + 6 * i + d];
      }
      J[e] = v;
    }
    StructSync(T);
  }
  // ---- constraints: one thread each (soft: the two links' terms, hard: residual + unprojected Jacobians) ----
  if (tid < nc) {
    const ConstraintDev& c = cons[tid];
    JointGeometryDev jg;
    CalcJointGeometryDev(c.body12joint1, c.body22joint2, s.l2w + 12 * c.link1, s.l2w + 12 * c.link2, jg);
    float* out = s.cdata + 84 * tid;
    if (c.soft) {
      SoftLinkTermsDev(c, jg, c.body12joint1, -1.0f, out);
      SoftLinkTermsDev(c, jg, jg.body22joint1, 1.0f, out + 42);
    } else {
      int idx = 0;
      for (int d = 0; d < 6; ++d)
        if (c.directions[d]) out[idx++] = d < 3 ? jg.rotation_vector[d] : jg.translation_vector[d - 3];
      UnprojectedJacobianDev(jg, jg.body22joint1, c.directions, true, true, out + 6);
      UnprojectedJacobianDev(jg, c.body12joint1, c.directions, true, true, out + 42);
    }
  }
  StructSync(T);
  // SoftConstraint terms are added to the links in constraint order (optimizer.cpp:283-288)
  for (int e = tid; e < nl * 42; e += T) {
    const int l = e / 42, k = e - 42 * l;
    float* dst = k < 6 ? &s.g[6 * l + k] : &s.H[36 * l + k - 6];
    float v = *dst;
    for (int c = 0; c < nc; ++c) {
      if (!cons[c].soft) continue;
      if (cons[c].link1 == l) v += s.cdata[84 * c + k];
      if (cons[c].link2 == l) v += s.cdata[84 * c + 42 + k];
    }
    *dst = v;
  }
  StructSync(T);
  // ---- AddProjectedGradientsAndHessians: b += J^T g, a(lower) -= J^T H J, links in pre-order ----
  for (int e = tid; e < dof * (dof + 1) / 2; e += T) {
    int i = int((sqrtf(8.0f * float(e) + 1.0f) - 1.0f) * 0.5f);
    while (i * (i + 1) / 2 > e) --i;
    while ((i + 1) * (i + 2) / 2 <= e) ++i;
    const int j = e - i * (i + 1) / 2;
    float aij = 0.0f, bi = 0.0f;
    for (int l = 0; l < nl; ++l) {
      const float* J = s.jac + size_t(l) * 6 * dof;
      const float* Hl = s.H + 36 * l;
      if (i == j) {
        float acc = 0.0f;
        for (int k = 0; k < 6; ++k) acc += J[size_t(k) * dof + i] * s.g[6 * l + k];
        bi += acc;
      }
      float t = 0.0f;
      for (int q = 0; q < 6; ++q) {
        float jh = 0.0f;
        for (int k = 0; k < 6; ++k) jh += J[size_t(k) * dof + i] * Hl[6 * k + q];
        t += jh * J[size_t(q) * dof + j];
      }
      aij -= t;
    }
    s.a[i * lda + j] = aij;
    if (i == j) s.b[i] = bi;
  }
  // ---- AddResidualsAndConstraintJacobians ----
  for (int c = 0; c < nc; ++c) {
    if (cons[c].soft) continue;
    const int nr = cons[c].n_rows, row0 = dof + cons[c].first_row;
    const float* out = s.cdata + 84 * c;
    const float* J2 = s.jac + size_t(cons[c].link2) * 6 * dof;
    const float* J1 = s.jac + size_t(cons[c].link1) * 6 * dof;
    for (int e = tid; e < nr * dof; e += T) {
      const int r = e / dof, col = e - r * dof;
      float a2 = 0.0f, a1 = 0.0f;
      for (int k = 0; k < 6; ++k) a2 += out[6 + 6 * r + k] * J2[size_t(k) * dof + col];
      for (int k = 0; k < 6; ++k) a1 += out[42 + 6 * r + k] * J1[size_t(k) * dof + col];
      s.a[(row0 + r) * lda + col] = -(a2 - a1);
    }
    if (tid < nr) s.b[row0 + tid] = out[tid];
  }
  StructSync(T);
  // tikhonov_vector_ on the diagonal of the unknowns
  for (int l = tid; l < nl; l += T) {
    int di = links[l].first_index;
    for (int d = 0; d < 6; ++d)
      if (links[l].free_directions[d]) {
        s.a[di * lda + di] += d < 3 ? st.tikhonov_rotation : st.tikhonov_translation;
        di++;
      }
  }
  StructSync(T);

  // ---- Eigen::LDLT<Lower>: the transposition sequence follows from the original diagonal (left-looking) ----
  for (int e = tid; e < n; e += T) s.absdiag[e] = fabsf(s.a[e * lda + e]);
  StructSync(T);
  if (tid < 32) {
    for (int k = 0; k < n; ++k) {
      float best = -1.0f;
      int bi = n;
      for (int i = k + tid; i < n; i += 32) {
        const float v = s.absdiag[i];
        if (v > best) { best = v; bi = i; }
      }
      for (int off = 16; off >= 1; off >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
      }
      if (tid == 0) {
        // Eigen's maxCoeff starts from the first entry of the tail and only takes strictly greater ones: a NaN there
        // is kept (and a NaN further down never wins). Without this a tail of NaNs left bi = n, out of range.
        if (!(s.absdiag[k] == s.absdiag[k])) bi = k;
        s.trans[k] = bi;
        const float tmp = s.absdiag[k];
        s.absdiag[k] = s.absdiag[bi];
        s.absdiag[bi] = tmp;
      }
      __syncwarp();
    }
  }
  StructSync(T);
  bool zero_matrix = false;
  if (n > 1) {
    for (int k = 0; k < n; ++k) {
      const int big = s.trans[k];
      if (k != big) {  // symmetric row/column swap restricted to the lower triangle
        for (int j = tid; j < k; j += T) { const float t = s.a[k * lda + j]; s.a[k * lda + j] = s.a[big * lda + j]; s.a[big * lda + j] = t; }
        for (int i = big + 1 + tid; i < n; i += T) { const float t = s.a[i * lda + k]; s.a[i * lda + k] = s.a[i * lda + big]; s.a[i * lda + big] = t; }
        for (int i = k + 1 + tid; i < big; i += T) { const float t = s.a[i * lda + k]; s.a[i * lda + k] = s.a[big * lda + i]; s.a[big * lda + i] = t; }
        if (tid == 0) { const float t = s.a[k * lda + k]; s.a[k * lda + k] = s.a[big * lda + big]; s.a[big * lda + big] = t; }
        StructSync(T);
      }
      if (k > 0) {
        for (int j = tid; j < k; j += T) s.temp[j] = s.a[j * lda + j] * s.a[k * lda + j];
        StructSync(T);
        for (int i = k + tid; i < n; i += T) {
          float acc = 0.0f;
          for (int j = 0; j < k; ++j) acc += s.a[i * lda + j] * s.temp[j];
          s.a[i * lda + k] -= acc;
        }
        StructSync(T);
      }
      const float akk = s.a[k * lda + k];
      const bool pivot_is_valid = fabsf(akk) > 0.0f;
      if (k == 0 && !pivot_is_valid) { zero_matrix = true; break; }
      if (pivot_is_valid)
        for (int i = k + 1 + tid; i < n; i += T) s.a[i * lda + k] /= akk;
      StructSync(T);
    }
  }
  if (zero_matrix || n == 1)
    for (int e = tid; e < n; e += T) s.trans[e] = (zero_matrix || n == 1) ? e : s.trans[e];
  StructSync(T);
  // ---- solve: P b, L^-1, D^-1, L^-T, P^T (Eigen LDLT::_solve_impl) ----
  if (tid == 0) {
    for (int k = 0; k < n; ++k) s.dst[k] = s.b[k];
    for (int k = 0; k < n; ++k) { const float t = s.dst[k]; s.dst[k] = s.dst[s.trans[k]]; s.dst[s.trans[k]] = t; }
  }
  StructSync(T);
  for (int j = 0; j < n; ++j) {
    const float dj = s.dst[j];
    for (int i = j + 1 + tid; i < n; i += T) s.dst[i] -= s.a[i * lda + j] * dj;
    StructSync(T);
  }
  for (int i = tid; i < n; i += T) {
    const float d = s.a[i * lda + i];
    s.dst[i] = fabsf(d) > (1.0f / 3.40282347e+38f) ? s.dst[i] / d : 0.0f;
  }
  StructSync(T);
  for (int j = n - 1; j >= 0; --j) {
    const float dj = s.dst[j];
    for (int i = tid; i < j; i += T) s.dst[i] -= s.a[j * lda + i] * dj;
    StructSync(T);
  }
  if (tid == 0)
    for (int k = n - 1; k >= 0; --k) { const float t = s.dst[k]; s.dst[k] = s.dst[s.trans[k]]; s.dst[s.trans[k]] = t; }
  StructSync(T);
  // theta = dst; NaN guard (optimizer.cpp:165)
  int has_nan = 0;
  for (int i = tid; i < n; i += T) has_nan |= (s.dst[i] != s.dst[i]) ? 1 : 0;
  has_nan = StructSyncOr(T, has_nan);
  if (theta_out)
    for (int i = tid; i < n; i += T) theta_out[i] = s.dst[i];
  if (has_nan) return false;
  UpdatePosesBlock(s, links, nl, tid, T);
  StructSync(T);
  return true;
}

#ifndef M3TB_TRACK_TU
__global__ void __launch_bounds__(kStructThreads) k_structure(const StructArgs args) {
  extern __shared__ __align__(16) float smem_f[];
  const int si = args.list ? args.list[blockIdx.x] : int(blockIdx.x);
  const StructureDev st = args.structures[si];
  LinkDev* links = args.links + st.first_link;
  const ConstraintDev* cons = args.constraints + st.first_constraint;
  const int nl = st.n_links, dof = st.dof, nc = st.n_constraints, n = st.dof + st.n_rows;
  const int tid = threadIdx.x, T = blockDim.x;
  StructSmem s = CarveStructSmem(smem_f, nl, dof, n, nc);
  const int lda = s.lda;

  // ---- load link poses and link gradients / Hessians (Link::CalculateGradientAndHessian result) ----
  // one modality set's sum in Link::modality_ptrs order: region, depth, then texture where the body has one (its
  // table row may be stale after the modality was removed, so the body's flag decides, not the row)
  auto modalities = [&](int b, int src) {
    float sum = 0.0f + args.gh_region[27 * b + src] + args.gh_depth[27 * b + src];
    if (args.gh_texture && args.bodies[b].has_texture) sum = sum + args.gh_texture[27 * b + src];
    return sum;
  };
  for (int e = tid; e < nl * 12; e += T) {
    const int l = e / 12, k = e - 12 * l;
    const int body = links[l].body;
    s.l2w[e] = body >= 0 ? args.poses[12 * body + k] : links[l].link2world[k];
  }
  for (int e = tid; e < nl * 42; e += T) {
    const int l = e / 42, k = e - 42 * l;
    const int body = links[l].body;
    float v = 0.0f;
    if (body >= 0) {
      int src = k;
      if (k >= 6) {
        const int i = (k - 6) / 6, j = (k - 6) - 6 * i;
        src = 6 + (i >= j ? Tri(i, j) : Tri(j, i));
      }
      v = args.gh_link ? args.gh_link[27 * body + src] : modalities(body, src);
      for (int x = 0; x < links[l].n_extra; ++x) {  // Link::CalculateGradientAndHessian over all modalities (link.cpp:184-193)
        const int eb = links[l].extra[x];
        v += args.gh_link ? args.gh_link[27 * eb + src] : modalities(eb, src);
      }
    }
    if (k < 6) s.g[6 * l + k] = v; else s.H[36 * l + k - 6] = v;
  }
  if (args.mode == 1) {
    for (int e = tid; e < n; e += T) s.dst[e] = 0.0f;
    __syncthreads();
    UpdatePosesBlock(s, links, nl, tid, T);
    __syncthreads();
  } else {
    const bool updated = StructureSolveBlock(st, links, cons, s, args.theta_out ? args.theta_out + size_t(si) * kMaxSystem : nullptr, tid, T);
    if (tid == 0) args.status[si] = updated ? 1 : 0;
    if (!updated) return;
  }
  // Body::set_body2world_pose of every link that carries a body
  for (int e = tid; e < nl * 12; e += T) {
    const int l = e / 12, k = e - 12 * l;
    const int body = links[l].body;
    if (body >= 0) {
      args.poses[12 * body + k] = s.l2w[e];
      for (int x = 0; x < links[l].n_extra; ++x) args.poses[12 * links[l].extra[x] + k] = s.l2w[e];
    }
  }
}

#endif  // M3TB_TRACK_TU

}  // namespace m3tb
