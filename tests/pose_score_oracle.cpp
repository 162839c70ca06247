// pose_score_oracle.cpp — CPU restatement of the evaluators' pose scoring (test infrastructure only): strict IEEE
// float32 in the reference's evaluation order when built with -ffp-contract=off, which the device results are held to
// bit for bit (the rotation error up to acosf's ulp bound). The same source built with -O3 -march=native -fopenmp is
// the CPU baseline of scripts/pose_score_timing.py.
//   GenderateReducedVertices      ycb_evaluator.cpp:1222-1248 (the same in opt_ / rtb_evaluator.cpp)
//   CalculatePoseResults          ycb_evaluator.cpp:803-848, rtb_evaluator.cpp:930-989, opt_evaluator.cpp:462-488,
//                                 rbot_evaluator.cpp:416-433
//   CalculateDiameters            opt_evaluator.cpp:580-599
// The k-d tree of the reference is replaced by a brute-force search with nanoflann's result-set rules: the distance
// starts at numeric_limits<float>::max() (KNNResultSet::init) and a point is taken only when dist < worst_dist
// (searchLevel). The result is the minimum over all vertices; a query whose distances are all NaN or infinite (a NaN or
// infinite pose) keeps FLT_MAX.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <random>
#include <vector>

namespace {

constexpr int kNCurveValues = 100;

// Transform3fA * Transform3fA, poses row-major 3x4
void PoseMul(const float* a, const float* b, float* o) {
  float r[12];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) r[4 * i + j] = a[4 * i + 0] * b[j] + a[4 * i + 1] * b[4 + j] + a[4 * i + 2] * b[8 + j];
    r[4 * i + 3] = a[4 * i + 0] * b[3] + a[4 * i + 1] * b[7] + a[4 * i + 2] * b[11] + a[4 * i + 3];
  }
  std::memcpy(o, r, sizeof(r));
}

// Transform3fA::inverse() (Affine): Eigen's cofactor 3x3 inverse, translation = -inv * t
void PoseInverse(const float* p, float* o) {
  const float m[9] = {p[0], p[1], p[2], p[4], p[5], p[6], p[8], p[9], p[10]};
  auto cof = [&](int i, int j) {
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    return m[3 * i1 + j1] * m[3 * i2 + j2] - m[3 * i1 + j2] * m[3 * i2 + j1];
  };
  const float c00 = cof(0, 0), c10 = cof(1, 0), c20 = cof(2, 0);
  const float det = c00 * m[0] + c10 * m[3] + c20 * m[6];
  const float invdet = 1.0f / det;
  const float inv[9] = {c00 * invdet, c10 * invdet, c20 * invdet, cof(0, 1) * invdet, cof(1, 1) * invdet,
                        cof(2, 1) * invdet, cof(0, 2) * invdet, cof(1, 2) * invdet, cof(2, 2) * invdet};
  float r[12];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) r[4 * i + j] = inv[3 * i + j];
    r[4 * i + 3] = (-inv[3 * i + 0]) * p[3] + (-inv[3 * i + 1]) * p[7] + (-inv[3 * i + 2]) * p[11];
  }
  std::memcpy(o, r, sizeof(r));
}

void Apply(const float* p, const float* v, float* o) {
  o[0] = p[0] * v[0] + p[1] * v[1] + p[2] * v[2] + p[3];
  o[1] = p[4] * v[0] + p[5] * v[1] + p[6] * v[2] + p[7];
  o[2] = p[8] * v[0] + p[9] * v[1] + p[10] * v[2] + p[11];
}

// Transform3fA::rotation() as the polar factor: Newton's iteration X <- (X + X^-T) / 2 in double, rounded to float
void PolarRotation(const float* p, float* r) {
  double x[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) x[3 * i + j] = double(p[4 * i + j]);
  for (int it = 0; it < 12; ++it) {
    double c[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        c[3 * i + j] = x[3 * i1 + j1] * x[3 * i2 + j2] - x[3 * i1 + j2] * x[3 * i2 + j1];
      }
    const double det = c[0] * x[0] + c[1] * x[1] + c[2] * x[2];
    double delta = 0.0;
    for (int k = 0; k < 9; ++k) {
      const double nx = 0.5 * (x[k] + c[k] / det);
      delta = std::max(delta, std::fabs(nx - x[k]));
      x[k] = nx;
    }
    if (delta < 1e-15) break;
  }
  for (int k = 0; k < 9; ++k) r[k] = float(x[k]);
}

}  // namespace

extern "C" {

// GenderateReducedVertices: all vertices for n_evaluation <= 0 or >= n, else n_evaluation draws of std::mt19937{7}
// (out: [max(n_evaluation, n)][3]); returns the size of the reduced set
int orc_reduce_vertices(const float* vertices, int n, int n_evaluation, float* out) {
  if (n_evaluation <= 0 || n_evaluation >= n) {
    std::memcpy(out, vertices, sizeof(float) * 3 * size_t(n));
    return n;
  }
  std::mt19937 generator{7};
  for (int k = 0; k < n_evaluation; ++k) {
    const int idx = int(generator() % n);
    std::memcpy(out + 3 * size_t(k), vertices + 3 * size_t(idx), sizeof(float) * 3);
  }
  return n_evaluation;
}

// One body: result[7] = add_error, adds_error, add_auc, adds_auc, translation_error, rotation_error, tracking_success
// (m3tb_pose_score order); curves [2][100] (add, adds). geometry2body may be NULL.
void orc_score_pose(const float* reduced, int n_reduced, const float* full, int n_full, const float* body2world,
                    const float* gt, const float* geometry2body, float threshold_max, float curve_scale,
                    float auc_scale, float translation_threshold, float rotation_threshold, float* result,
                    float* curves) {
  float delta[12], inv[12];
  if (geometry2body) {
    float p[12], t[12];
    PoseMul(body2world, geometry2body, p);
    PoseInverse(p, inv);
    PoseMul(inv, gt, t);
    PoseMul(t, geometry2body, delta);
  } else {
    PoseInverse(body2world, inv);
    PoseMul(inv, gt, delta);
  }
  float add_error = 0.0f, adds_error = 0.0f;
  for (int i = 0; i < n_reduced; ++i) {
    const float* v = reduced + 3 * size_t(i);
    float w[3];
    Apply(delta, v, w);
    const float dx = v[0] - w[0], dy = v[1] - w[1], dz = v[2] - w[2];
    add_error += std::sqrt(dx * dx + dy * dy + dz * dz);
    float best = std::numeric_limits<float>::max();
    for (int j = 0; j < n_full; ++j) {
      const float* u = full + 3 * size_t(j);
      float d = 0.0f;  // nanoflann L2_Adaptor: ((0 + dx²) + dy²) + dz²
      for (int k = 0; k < 3; ++k) {
        const float diff = w[k] - u[k];
        d += diff * diff;
      }
      if (d < best) best = d;
    }
    adds_error += std::sqrt(best);
  }
  add_error /= float(n_reduced);
  adds_error /= float(n_reduced);
  const float errors[2] = {add_error, adds_error};
  const float step = threshold_max / float(kNCurveValues);
  const float threshold = curve_scale * threshold_max;
  for (int c = 0; c < 2; ++c) {
    float* curve = curves + c * kNCurveValues;
    std::fill(curve, curve + kNCurveValues, 1.0f);
    for (int i = 0; i < kNCurveValues; ++i) {
      if (errors[c] < curve_scale * (step * (0.5f + float(i)))) break;
      curve[i] = 0.0f;
    }
    result[2 + c] = auc_scale * (1.0f - std::min(errors[c] / threshold, 1.0f));
  }
  result[0] = add_error;
  result[1] = adds_error;
  const float tx = body2world[3] - gt[3], ty = body2world[7] - gt[7], tz = body2world[11] - gt[11];
  result[4] = std::sqrt(tx * tx + ty * ty + tz * tz);
  float r[9], rg[9];
  PolarRotation(body2world, r);
  PolarRotation(gt, rg);
  float trace = 0.0f;
  for (int i = 0; i < 3; ++i) {
    const float d = r[i] * rg[i] + r[3 + i] * rg[3 + i] + r[6 + i] * rg[6 + i];
    trace = i == 0 ? d : trace + d;
  }
  result[5] = std::acos((trace - 1.0f) / 2.0f);
  result[6] = (result[4] > translation_threshold || result[5] > rotation_threshold) ? 0.0f : 1.0f;
}

// CalculateDiameters: the largest (v_i - v_j).norm() over all pairs
float orc_diameter(const float* vertices, int n) {
  const long long size = n, size_squared = size * size;
  float d_max = 0.0f;
#pragma omp parallel
  {
    float d_max_thread = 0.0f;
#pragma omp for
    for (long long i = 0; i < size_squared; ++i) {
      const float* a = vertices + 3 * (i / size);
      const float* b = vertices + 3 * (i % size);
      const float dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
      d_max_thread = std::max(d_max_thread, std::sqrt(dx * dx + dy * dy + dz * dz));
    }
#pragma omp critical
    d_max = std::max(d_max, d_max_thread);
  }
  return d_max;
}

// n bodies at once (the timing baseline parallelises over bodies, as parameter_study_* runs evaluators in parallel):
// body q uses reduced / full set model[q] (offsets into the packed sets), results [n][7], curves [n][2][100]
void orc_score_poses(int n, const int* model, const float* reduced, const int* reduced_offset, const int* n_reduced,
                     const float* full, const int* full_offset, const int* n_full, const float* body2world,
                     const float* gt, const float* geometry2body, const int* has_geometry2body, float threshold_max,
                     float curve_scale, float auc_scale, float translation_threshold, float rotation_threshold,
                     float* results, float* curves) {
#pragma omp parallel for schedule(dynamic)
  for (int q = 0; q < n; ++q) {
    const int m = model[q];
    orc_score_pose(reduced + 3 * size_t(reduced_offset[m]), n_reduced[m], full + 3 * size_t(full_offset[m]), n_full[m],
                   body2world + 12 * size_t(q), gt + 12 * size_t(q),
                   has_geometry2body[q] ? geometry2body + 12 * size_t(q) : nullptr, threshold_max, curve_scale,
                   auc_scale, translation_threshold, rotation_threshold, results + 7 * size_t(q),
                   curves + 2 * kNCurveValues * size_t(q));
  }
}

}  // extern "C"
