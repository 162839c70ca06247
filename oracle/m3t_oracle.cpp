// m3t_oracle.cpp — CPU oracle (TEST INFRASTRUCTURE ONLY, see m3t_oracle.h).
//
// Scalar float32 restatement of the reference's pose-optimisation hot path. Every function cites the
// reference file:line (relative to /root/reference/M3T/) it follows. Compile with
// -ffp-contract=off so that each float operation rounds once, in the order written here; the CUDA
// path is compiled with -fmad=false for the same reason, which makes the per-line state comparable
// bit for bit (ORC_ROTATION_LINEAR / ORC_EXP_RODRIGUES modes).
#include "m3t_oracle.h"

#include <algorithm>
#include <chrono>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <limits>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

// ---------------------------------------------------------------------------------------------
// Small fixed-size helpers (stand-ins for Eigen::Transform<float,3,Affine> / Matrix3f / Vector3f)
// Pose layout: float[12] row-major 3x4, p[4*i+j]; p[4*i+3] = translation.
// ---------------------------------------------------------------------------------------------
inline float R_(const float* p, int i, int j) { return p[4 * i + j]; }
inline float T_(const float* p, int i) { return p[4 * i + 3]; }

// Transform3fA * Transform3fA (Affine x Affine): res.affine() = lhs.affine() * rhs.matrix()
void PoseMul(const float* a, const float* b, float* out) {
  float r[12];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j)
      r[4 * i + j] = R_(a, i, 0) * R_(b, 0, j) + R_(a, i, 1) * R_(b, 1, j) + R_(a, i, 2) * R_(b, 2, j);
    r[4 * i + 3] = R_(a, i, 0) * T_(b, 0) + R_(a, i, 1) * T_(b, 1) + R_(a, i, 2) * T_(b, 2) + T_(a, i);
  }
  std::memcpy(out, r, sizeof(r));
}

// Transform3fA * Vector3f : linear * v + translation
inline void PoseApply(const float* p, const float* v, float* out) {
  float x = R_(p, 0, 0) * v[0] + R_(p, 0, 1) * v[1] + R_(p, 0, 2) * v[2] + T_(p, 0);
  float y = R_(p, 1, 0) * v[0] + R_(p, 1, 1) * v[1] + R_(p, 1, 2) * v[2] + T_(p, 1);
  float z = R_(p, 2, 0) * v[0] + R_(p, 2, 1) * v[1] + R_(p, 2, 2) * v[2] + T_(p, 2);
  out[0] = x; out[1] = y; out[2] = z;
}

// Eigen 3x3 inverse (compute_inverse_size3_helper): cofactors, det from first column, * (1/det).
// m, out: row-major 3x3.
void Inverse3(const float* m, float* out) {
  auto M = [&](int i, int j) { return m[3 * i + j]; };
  auto cof = [&](int i, int j) {
    int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    return M(i1, j1) * M(i2, j2) - M(i1, j2) * M(i2, j1);
  };
  float c00 = cof(0, 0), c10 = cof(1, 0), c20 = cof(2, 0);
  float det = c00 * M(0, 0) + c10 * M(1, 0) + c20 * M(2, 0);
  float invdet = 1.0f / det;
  out[0] = c00 * invdet; out[1] = c10 * invdet; out[2] = c20 * invdet;
  out[3] = cof(0, 1) * invdet; out[4] = cof(1, 1) * invdet; out[5] = cof(2, 1) * invdet;
  out[6] = cof(0, 2) * invdet; out[7] = cof(1, 2) * invdet; out[8] = cof(2, 2) * invdet;
}

// Transform3fA::inverse() for Affine mode: linear().inverse(), translation = -inv * t.
void PoseInverse(const float* p, float* out) {
  float m[9], inv[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) m[3 * i + j] = R_(p, i, j);
  Inverse3(m, inv);
  float r[12];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) r[4 * i + j] = inv[3 * i + j];
    // res.translation() = -res.linear() * translation()
    r[4 * i + 3] = (-inv[3 * i + 0]) * T_(p, 0) + (-inv[3 * i + 1]) * T_(p, 1) + (-inv[3 * i + 2]) * T_(p, 2);
  }
  std::memcpy(out, r, sizeof(r));
}

// Transform3fA::rotation(): for an Affine transform Eigen computes the rotation factor of the
// linear block via JacobiSVD (R = U V^T, computeRotationScaling). Restated as the polar factor,
// evaluated in double with Newton's iteration X <- (X + X^-T)/2 and rounded once to float.
void PoseRotation(const float* p, int rotation_mode, float* r /*row-major 3x3*/) {
  if (rotation_mode == ORC_ROTATION_LINEAR) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) r[3 * i + j] = R_(p, i, j);
    return;
  }
  double x[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) x[3 * i + j] = double(R_(p, i, j));
  for (int it = 0; it < 12; ++it) {
    auto X = [&](int i, int j) { return x[3 * i + j]; };
    double c[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        c[3 * i + j] = X(i1, j1) * X(i2, j2) - X(i1, j2) * X(i2, j1);
      }
    double det = c[0] * x[0] + c[1] * x[1] + c[2] * x[2];
    double delta = 0.0;
    for (int k = 0; k < 9; ++k) {
      double nx = 0.5 * (x[k] + c[k] / det);  // X^-T = cofactor matrix / det
      delta = std::max(delta, std::fabs(nx - x[k]));
      x[k] = nx;
    }
    if (delta < 1e-15) break;
  }
  for (int k = 0; k < 9; ++k) r[k] = float(x[k]);
}

// Eigen's Vector::normalized(): v / sqrt(squaredNorm) if squaredNorm > 0.
inline void Normalize3(float* v) {
  float z = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  if (z > 0.0f) {
    float n = std::sqrt(z);
    v[0] /= n; v[1] /= n; v[2] /= n;
  }
}
inline void Normalize2(float* v) {
  float z = v[0] * v[0] + v[1] * v[1];
  if (z > 0.0f) {
    float n = std::sqrt(z);
    v[0] /= n; v[1] /= n;
  }
}

// common.h:170-176
template <typename T>
inline T LastValidValue(const T* values, int n, int idx) {
  return idx < n ? values[idx] : values[n - 1];
}

// common.h:48-56
inline float sgnf(float v) { return v < 0.0f ? -1.0f : (v > 0.0f ? 1.0f : 0.0f); }

inline int Bitshift(int n_bins) {  // color_histograms.cpp:131-159
  switch (n_bins) {
    case 2: return 7;
    case 4: return 6;
    case 8: return 5;
    case 16: return 4;
    case 32: return 3;
    case 64: return 2;
    default: return -1;
  }
}

inline int HistIndex(int n_bins, int bitshift, const uint8_t* px) {  // color_histograms.cpp:97-99
  return (px[0] >> bitshift) * n_bins * n_bins + (px[1] >> bitshift) * n_bins + (px[2] >> bitshift);
}

// ---------------------------------------------------------------------------------------------
// Region modality precalculated variables
// ---------------------------------------------------------------------------------------------
struct RegionVars {
  // PrecalculateFunctionLookup / PrecalculateDistributionVariables (region_modality.cpp:910-936)
  float lookup_f[8], lookup_b[8];
  int line_length_in_segments;
  float dl_minus_1_half, dl_plus_1_half;
  float min_expected_variance;
  // PrecalculateCameraVariables (:945-966)
  float fu, fv, ppu, ppv;
  int w_m1, h_m1, w_m2, h_m2;
  // PrecalculatePoseVariables (:1000-1009)
  float body2camera[12];
  float rot[9];  // body2camera_rotation_
  // PrecalculateIterationDependentVariables (:1011-1023)
  int scale;
  float fscale;
  int line_length, line_length_minus_1;
  float line_length_minus_1_half, line_length_half_minus_1;
  float variance;
  int n_bins, bitshift;
};

void FunctionLookup(const orc_region_params* p, float* lf, float* lb, float* min_expected_variance) {
  // region_modality.cpp:910-923
  for (int i = 0; i < p->function_length; ++i) {
    float x = float(i) - float(p->function_length - 1) / 2.0f;
    if (p->function_slope == 0.0f)
      lf[i] = 0.5f - p->function_amplitude * float((0.0f < x) - (x < 0.0f));
    else
      lf[i] = 0.5f - p->function_amplitude * std::tanh(x / (2.0f * p->function_slope));
    lb[i] = 1.0f - lf[i];
  }
  // region_modality.cpp:925-936
  float laplace = 1.0f / (2.0f * powf(atanhf(2.0f * p->function_amplitude), 2.0f));
  float gaussian = p->function_slope;
  *min_expected_variance = std::max(laplace, gaussian);
}

void RegionPrecalc(const orc_region_params* p, const orc_color_frame* c, const float* body2world,
                   int corr_iteration, int rotation_mode, RegionVars* v) {
  FunctionLookup(p, v->lookup_f, v->lookup_b, &v->min_expected_variance);
  v->line_length_in_segments = p->function_length + p->distribution_length - 1;
  v->dl_minus_1_half = (float(p->distribution_length) - 1.0f) / 2.0f;
  v->dl_plus_1_half = (float(p->distribution_length) + 1.0f) / 2.0f;
  v->fu = c->intrinsics.fu; v->fv = c->intrinsics.fv;
  v->ppu = c->intrinsics.ppu; v->ppv = c->intrinsics.ppv;
  v->w_m1 = c->intrinsics.width - 1; v->h_m1 = c->intrinsics.height - 1;
  v->w_m2 = c->intrinsics.width - 2; v->h_m2 = c->intrinsics.height - 2;
  PoseMul(c->world2camera, body2world, v->body2camera);
  PoseRotation(v->body2camera, rotation_mode, v->rot);
  v->scale = LastValidValue(p->scales, p->n_scales, corr_iteration);
  v->fscale = float(v->scale);
  v->line_length = v->line_length_in_segments * v->scale;
  v->line_length_minus_1 = v->line_length - 1;
  v->line_length_minus_1_half = float(v->line_length - 1) * 0.5f;
  v->line_length_half_minus_1 = float(v->line_length) * 0.5f - 1.0f;
  float sd = LastValidValue(p->standard_deviations, p->n_standard_deviations, corr_iteration);
  v->variance = sd * sd;  // powf(sd, 2.0f)
  v->n_bins = p->n_histogram_bins;
  v->bitshift = Bitshift(p->n_histogram_bins);
}

// RegionModel::GetClosestView (region_model.cpp:105-130) / DepthModel::GetClosestView (depth_model.cpp:81-106)
int ClosestView(const orc_model* m, const float* body2camera, int rotation_mode) {
  float t[3] = {T_(body2camera, 0), T_(body2camera, 1), T_(body2camera, 2)};
  float norm = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
  if (norm == 0.0f) return 0;
  Normalize3(t);
  float o[3];
  if (rotation_mode == ORC_ROTATION_POLAR) {
    float r[9], inv[9];
    PoseRotation(body2camera, rotation_mode, r);
    Inverse3(r, inv);  // rotation().inverse()
    for (int i = 0; i < 3; ++i) o[i] = inv[3 * i + 0] * t[0] + inv[3 * i + 1] * t[1] + inv[3 * i + 2] * t[2];
  } else {
    for (int j = 0; j < 3; ++j) o[j] = R_(body2camera, 0, j) * t[0] + R_(body2camera, 1, j) * t[1] + R_(body2camera, 2, j) * t[2];
  }
  float closest_dot = -1.0f;
  int best = 0;  // reference leaves the pointer untouched if no dot > -1; views_[0] is our stand-in
  for (int v = 0; v < m->n_views; ++v) {
    const float* vo = m->orientations + 3 * v;
    float dot = o[0] * vo[0] + o[1] * vo[1] + o[2] * vo[2];
    if (dot > closest_dot) {
      best = v;
      closest_dot = dot;
    }
  }
  return best;
}

// n_lines / n_points selection (region_modality.cpp:414-430, depth_modality.cpp:281-293)
int AdaptiveCount(int n_max, int use_adaptive, float reference, float view_scalar, float max_scalar, int n_model) {
  int n = n_max;
  if (use_adaptive) {
    if (reference > 0.0f)
      n = int(float(n_max) * std::min(1.0f, view_scalar / reference));
    else
      n = int(float(n_max) * view_scalar / max_scalar);
  }
  if (n > n_model) n = n_model;
  return n;
}

// MultiplyPixelColorProbability (region_modality.cpp:1575-1598) + GetProbabilities (color_histograms.cpp:94-102)
inline void MultiplyPixel(const RegionVars& v, const float* hist_f, const float* hist_b, const uint8_t* px,
                          float* pf_acc, float* pb_acc) {
  int idx = HistIndex(v.n_bins, v.bitshift, px);
  float pf = hist_f[idx];
  float pb = hist_b[idx];
  if (pf || pb) {
    float sum = pf;
    sum += pb;
    pf /= sum;
    pb /= sum;
  } else {
    pf = 0.5f;
    pb = 0.5f;
  }
  *pf_acc *= pf;
  *pb_acc *= pb;
}

// CalculateSegmentProbabilities (region_modality.cpp:1433-1573)
bool SegmentProbabilities(const RegionVars& v, const orc_color_frame* c, const float* hist_f, const float* hist_b,
                          float center_u, float center_v, float normal_u, float normal_v, float* sf, float* sb,
                          float* normal_component_to_scale, float* delta_r) {
  const int n_seg = v.line_length_in_segments;
  const uint8_t* img = c->bgr;
  const size_t pitch = c->pitch;
  if (std::fabs(normal_v) < std::fabs(normal_u)) {
    float v_step = normal_v / normal_u;
    int u = int(center_u - v.line_length_half_minus_1);
    int u_end = u + v.line_length_minus_1;
    float v_f = center_v + v_step * (float(u) - center_u) + 0.5f;
    float v_f_end = v_f + v_step * float(v.line_length_minus_1);
    if (u < 0 || u_end > v.w_m1 || int(v_f) < 0 || int(v_f) > v.h_m1 || int(v_f_end) < 1 || int(v_f_end) > v.h_m2)
      return false;
    int seg = normal_u > 0 ? 0 : n_seg - 1;
    int dir = normal_u > 0 ? 1 : -1;
    sf[seg] = 1.0f; sb[seg] = 1.0f;
    int segment_idx = 0;
    for (; u <= u_end; ++u, v_f += v_step, ++segment_idx) {
      if (segment_idx == v.scale) {
        seg += dir;
        sf[seg] = 1.0f; sb[seg] = 1.0f;
        segment_idx = 0;
      }
      MultiplyPixel(v, hist_f, hist_b, img + size_t(int(v_f)) * pitch + 3 * size_t(u), &sf[seg], &sb[seg]);
    }
    *normal_component_to_scale = std::fabs(normal_u) / v.fscale;
    *delta_r = (std::round(center_u - v.line_length_minus_1_half) + v.line_length_minus_1_half - center_u) / normal_u;
  } else {
    float u_step = normal_u / normal_v;
    int vv = int(center_v - v.line_length_half_minus_1);
    int v_end = vv + v.line_length_minus_1;
    float u_f = center_u + u_step * (float(vv) - center_v) + 0.5f;
    float u_f_end = u_f + u_step * float(v.line_length_minus_1);
    if (vv < 0 || v_end > v.h_m1 || int(u_f) < 0 || int(u_f) > v.w_m1 || int(u_f_end) < 1 || int(u_f_end) > v.w_m2)
      return false;
    int seg = normal_v > 0 ? 0 : n_seg - 1;
    int dir = normal_v > 0 ? 1 : -1;
    sf[seg] = 1.0f; sb[seg] = 1.0f;
    int segment_idx = 0;
    for (; vv <= v_end; ++vv, u_f += u_step, ++segment_idx) {
      if (segment_idx == v.scale) {
        seg += dir;
        sf[seg] = 1.0f; sb[seg] = 1.0f;
        segment_idx = 0;
      }
      MultiplyPixel(v, hist_f, hist_b, img + size_t(vv) * pitch + 3 * size_t(int(u_f)), &sf[seg], &sb[seg]);
    }
    *normal_component_to_scale = std::fabs(normal_v) / v.fscale;
    *delta_r = (std::round(center_v - v.line_length_minus_1_half) + v.line_length_minus_1_half - center_v) / normal_v;
  }
  // Normalize segment probabilities (:1555-1571)
  if (v.scale > 1) {
    for (int i = 0; i < n_seg; ++i) {
      if (sf[i] || sb[i]) {
        float sum = sf[i];
        sum += sb[i];
        sf[i] /= sum;
        sb[i] /= sum;
      } else {
        sf[i] = 0.5f;
        sb[i] = 0.5f;
      }
    }
  }
  return true;
}

// CalculateDistribution (region_modality.cpp:1600-1637)
void Distribution(const RegionVars& v, int function_length, int distribution_length, const float* sf,
                  const float* sb, float* dist) {
  float area = 0.0f;
  for (int d = 0; d < distribution_length; ++d) {
    float val = 1.0f;
    for (int k = 0; k < function_length; ++k) val *= sf[d + k] * v.lookup_f[k] + sb[d + k] * v.lookup_b[k];
    dist[d] = val;
    area += val;
  }
  for (int d = 0; d < distribution_length; ++d) dist[d] /= area;
}

// CalculateDistributionMoments (region_modality.cpp:1639-1658)
void Moments(const RegionVars& v, int distribution_length, const float* dist, float* mean, float* variance) {
  float mean_from_begin = 0.0f;
  for (int i = 0; i < distribution_length; ++i) mean_from_begin += float(i) * dist[i];
  float var = 0.0f;
  for (int i = 0; i < distribution_length; ++i) {
    float d = float(i) - mean_from_begin;
    var += (d * d) * dist[i];  // powf(x, 2.0f) * dist[i]
  }
  *mean = mean_from_begin - v.dl_minus_1_half;
  *variance = std::max(var, v.min_expected_variance);
}

// ---------------------------------------------------------------------------------------------
// Depth modality precalculated variables (depth_modality.cpp:618-654)
// ---------------------------------------------------------------------------------------------
struct DepthVars {
  float fu, fv, ppu, ppv, depth_scale;
  int w_m1, h_m1;
  float body2camera[12], camera2body[12];
  float considered_distance;
  int max_n_strides;
  float standard_deviation;
};

void DepthPrecalc(const orc_depth_params* p, const orc_depth_frame* f, const float* body2world, int corr_iteration,
                  DepthVars* v) {
  v->fu = f->intrinsics.fu; v->fv = f->intrinsics.fv;
  v->ppu = f->intrinsics.ppu; v->ppv = f->intrinsics.ppv;
  v->depth_scale = f->depth_scale;
  v->w_m1 = f->intrinsics.width - 1; v->h_m1 = f->intrinsics.height - 1;
  PoseMul(f->world2camera, body2world, v->body2camera);  // :642-643
  PoseInverse(v->body2camera, v->camera2body);            // :644
  v->considered_distance = LastValidValue(p->considered_distances, p->n_considered_distances, corr_iteration);
  v->max_n_strides = int(v->considered_distance / p->stride_length + 0.5f);  // :651
  v->standard_deviation = LastValidValue(p->standard_deviations, p->n_standard_deviations, corr_iteration);
}

// DepthModality::FindCorrespondence (depth_modality.cpp:826-884)
bool FindCorrespondence(const orc_depth_params* p, const DepthVars& v, const orc_depth_frame* f,
                        const float* center_f_camera, float center_u, float center_v, float depth_pt,
                        float* correspondence) {
  float considered_distance = v.considered_distance;
  if (p->use_depth_scaling) considered_distance *= depth_pt;
  float meter_to_pixel = v.fu / depth_pt;
  float diameter = 2.0f * considered_distance * meter_to_pixel;
  int stride = int(diameter / float(v.max_n_strides) + 1.0f);
  int n_strides = int(diameter / float(stride) + 0.5f);
  int rounded_diameter = n_strides * stride;
  float rounded_radius = 0.5f * float(rounded_diameter);
  int u_min = int(center_u - rounded_radius + 0.5f);
  int v_min = int(center_v - rounded_radius + 0.5f);
  int u_max = u_min + rounded_diameter;
  int v_max = v_min + rounded_diameter;
  u_min = std::max(u_min, 0);
  v_min = std::max(v_min, 0);
  u_max = std::min(u_max, v.w_m1);
  v_max = std::min(v_max, v.h_m1);
  // NB: the reference really uses std::min(0.0f, ...) here (:851-852), i.e. the lower bound is <= 0.
  float min_depth_value = std::min(0.0f, (depth_pt - considered_distance) / v.depth_scale);
  float max_depth_value = (depth_pt + considered_distance) / v.depth_scale;
  float min_considered_distance_square = considered_distance * considered_distance;
  float min_measured_distance_square = min_considered_distance_square;
  for (int vv = v_min; vv <= v_max; vv += stride) {
    const uint16_t* row = reinterpret_cast<const uint16_t*>(reinterpret_cast<const uint8_t*>(f->depth) + size_t(vv) * f->pitch);
    for (int uu = u_min; uu <= u_max; uu += stride) {
      float depth = float(row[uu]);
      if (depth > min_depth_value && depth < max_depth_value) {
        depth *= v.depth_scale;
        float tx = (float(uu) - v.ppu) * depth / v.fu;
        float ty = (float(vv) - v.ppv) * depth / v.fv;
        float tz = depth;
        float dx = tx - center_f_camera[0], dy = ty - center_f_camera[1], dz = tz - center_f_camera[2];
        float d2 = dx * dx + dy * dy + dz * dz;
        if (d2 < min_measured_distance_square) {
          correspondence[0] = tx; correspondence[1] = ty; correspondence[2] = tz;
          min_measured_distance_square = d2;
        }
      }
    }
  }
  return min_measured_distance_square != min_considered_distance_square;
}

// ---------------------------------------------------------------------------------------------
// Eigen::LDLT<MatrixXf, Lower> restated (Eigen/src/Cholesky/LDLT.h: ldlt_inplace<Lower>::unblocked,
// LDLT::_solve_impl). a: n x n, only the lower triangle is read. Returns false if n is too large.
// ---------------------------------------------------------------------------------------------
constexpr int kMaxN = 128;
bool LdltSolve(int n, const float* a_in, const float* b, float* x) {
  if (n > kMaxN || n < 1) return false;
  std::vector<float> mat(size_t(n) * n, 0.0f);
  auto A = [&](int i, int j) -> float& { return mat[size_t(i) * n + j]; };
  for (int i = 0; i < n; ++i)
    for (int j = 0; j <= i; ++j) A(i, j) = a_in[size_t(i) * n + j];
  std::vector<int> trans(n);
  std::vector<float> temp(n);
  bool zero_matrix = false;
  if (n == 1) {
    trans[0] = 0;
  } else {
    for (int k = 0; k < n; ++k) {
      // Find largest diagonal element (first maximum wins)
      int biggest = k;
      float big = std::fabs(A(k, k));
      for (int i = k + 1; i < n; ++i) {
        float val = std::fabs(A(i, i));
        if (val > big) { big = val; biggest = i; }
      }
      trans[k] = biggest;
      if (k != biggest) {
        int s = n - biggest - 1;
        for (int j = 0; j < k; ++j) std::swap(A(k, j), A(biggest, j));
        for (int i = 0; i < s; ++i) std::swap(A(biggest + 1 + i, k), A(biggest + 1 + i, biggest));
        std::swap(A(k, k), A(biggest, biggest));
        for (int i = k + 1; i < biggest; ++i) {
          float tmp = A(i, k);
          A(i, k) = A(biggest, i);
          A(biggest, i) = tmp;
        }
      }
      int rs = n - k - 1;
      if (k > 0) {
        for (int j = 0; j < k; ++j) temp[j] = A(j, j) * A(k, j);
        float dot = 0.0f;
        for (int j = 0; j < k; ++j) dot += A(k, j) * temp[j];
        A(k, k) -= dot;
        for (int i = k + 1; i < n; ++i) {
          float acc = 0.0f;
          for (int j = 0; j < k; ++j) acc += A(i, j) * temp[j];
          A(i, k) -= acc;
        }
      }
      float akk = A(k, k);
      bool pivot_is_valid = std::fabs(akk) > 0.0f;
      if (k == 0 && !pivot_is_valid) {
        // The entire diagonal is zero, there is nothing more to do except filling the transpositions
        for (int j = 0; j < n; ++j) trans[j] = j;
        zero_matrix = true;
        break;
      }
      if (rs > 0 && pivot_is_valid)
        for (int i = k + 1; i < n; ++i) A(i, k) /= akk;
    }
  }
  (void)zero_matrix;
  // _solve_impl: dst = P b
  std::vector<float> dst(b, b + n);
  for (int k = 0; k < n; ++k) std::swap(dst[k], dst[trans[k]]);
  // dst = L^-1 (P b): unit lower, column oriented
  for (int j = 0; j < n; ++j)
    for (int i = j + 1; i < n; ++i) dst[i] -= A(i, j) * dst[j];
  // dst = D^-1 (L^-1 P b) with Eigen's tolerance 1 / highest()
  const float tolerance = 1.0f / std::numeric_limits<float>::max();
  for (int i = 0; i < n; ++i) {
    if (std::fabs(A(i, i)) > tolerance)
      dst[i] /= A(i, i);
    else
      dst[i] = 0.0f;
  }
  // dst = L^-T (...): unit upper, column oriented backwards
  for (int j = n - 1; j >= 0; --j)
    for (int i = 0; i < j; ++i) dst[i] -= A(j, i) * dst[j];
  // dst = P^T dst
  for (int k = n - 1; k >= 0; --k) std::swap(dst[k], dst[trans[k]]);
  for (int i = 0; i < n; ++i) x[i] = dst[i];
  return true;
}

// ---------------------------------------------------------------------------------------------
// Vector2Skewsymmetric(w).exp()  (common.h:64-70, link.cpp:224; Eigen unsupported MatrixFunctions,
// MatrixExponential.h: matrix_exp_computeUV<_, float> + matrix_exp_compute).
// ---------------------------------------------------------------------------------------------
struct M3 {
  float m[9];
  float& operator()(int i, int j) { return m[3 * i + j]; }
  float operator()(int i, int j) const { return m[3 * i + j]; }
};
M3 Mul(const M3& a, const M3& b) {
  M3 r;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r(i, j) = a(i, 0) * b(0, j) + a(i, 1) * b(1, j) + a(i, 2) * b(2, j);
  return r;
}
M3 Lin(float ca, const M3& a, float cb, const M3& b) {  // ca*a + cb*b
  M3 r;
  for (int k = 0; k < 9; ++k) r.m[k] = ca * a.m[k] + cb * b.m[k];
  return r;
}
M3 Identity3() { return M3{{1, 0, 0, 0, 1, 0, 0, 0, 1}}; }

// denom.partialPivLu().solve(numer) for 3x3
M3 LuSolve(M3 a, M3 b) {
  int perm[3] = {0, 1, 2};
  for (int k = 0; k < 3; ++k) {
    int piv = k;
    float big = std::fabs(a(k, k));
    for (int i = k + 1; i < 3; ++i)
      if (std::fabs(a(i, k)) > big) { big = std::fabs(a(i, k)); piv = i; }
    if (piv != k) {
      for (int j = 0; j < 3; ++j) { std::swap(a(k, j), a(piv, j)); std::swap(b(k, j), b(piv, j)); }
      std::swap(perm[k], perm[piv]);
    }
    for (int i = k + 1; i < 3; ++i) {
      a(i, k) /= a(k, k);
      for (int j = k + 1; j < 3; ++j) a(i, j) -= a(i, k) * a(k, j);
    }
  }
  // forward (unit lower)
  for (int c = 0; c < 3; ++c) {
    for (int i = 1; i < 3; ++i)
      for (int j = 0; j < i; ++j) b(i, c) -= a(i, j) * b(j, c);
    for (int i = 2; i >= 0; --i) {
      for (int j = i + 1; j < 3; ++j) b(i, c) -= a(i, j) * b(j, c);
      b(i, c) /= a(i, i);
    }
  }
  return b;
}

void ExpSkew(const float* w, int exp_mode, float* out) {
  M3 A{{0.0f, -w[2], w[1], w[2], 0.0f, -w[0], -w[1], w[0], 0.0f}};  // common.h:64-70
  if (exp_mode == ORC_EXP_RODRIGUES) {
    // closed form, same expression as the CUDA path (csrc/m3t_b200_math.cuh ExpSkew)
    float t2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    float a, b;
    if (t2 < 0.01f) {
      a = 1.0f + t2 * (-1.0f / 6.0f + t2 * (1.0f / 120.0f + t2 * (-1.0f / 5040.0f)));
      b = 0.5f + t2 * (-1.0f / 24.0f + t2 * (1.0f / 720.0f + t2 * (-1.0f / 40320.0f)));
    } else {
      float t = std::sqrt(t2);
      float sh = std::sin(0.5f * t);
      a = std::sin(t) / t;
      b = 2.0f * sh * sh / t2;
    }
    M3 A2 = Mul(A, A);
    M3 I = Identity3();
    for (int k = 0; k < 9; ++k) out[k] = I.m[k] + a * A.m[k] + b * A2.m[k];
    return;
  }
  float l1norm = 0.0f;
  for (int j = 0; j < 3; ++j) {
    float s = std::fabs(A(0, j)) + std::fabs(A(1, j)) + std::fabs(A(2, j));
    l1norm = std::max(l1norm, s);
  }
  int squarings = 0;
  M3 U, V;
  const M3 I = Identity3();
  if (l1norm < 4.258730016922831e-001f) {
    const float b[] = {120.0f, 60.0f, 12.0f, 1.0f};
    M3 A2 = Mul(A, A);
    M3 tmp = Lin(b[3], A2, b[1], I);
    U = Mul(A, tmp);
    V = Lin(b[2], A2, b[0], I);
  } else if (l1norm < 1.880152677804762e+000f) {
    const float b[] = {30240.0f, 15120.0f, 3360.0f, 420.0f, 30.0f, 1.0f};
    M3 A2 = Mul(A, A);
    M3 A4 = Mul(A2, A2);
    M3 tmp;
    for (int k = 0; k < 9; ++k) tmp.m[k] = b[5] * A4.m[k] + b[3] * A2.m[k] + b[1] * I.m[k];
    U = Mul(A, tmp);
    for (int k = 0; k < 9; ++k) V.m[k] = b[4] * A4.m[k] + b[2] * A2.m[k] + b[0] * I.m[k];
  } else {
    const float maxnorm = 3.925724783138660f;
    std::frexp(l1norm / maxnorm, &squarings);
    if (squarings < 0) squarings = 0;
    M3 As = A;
    for (int k = 0; k < 9; ++k) As.m[k] = std::ldexp(A.m[k], -squarings);
    const float b[] = {17297280.0f, 8648640.0f, 1995840.0f, 277200.0f, 25200.0f, 1512.0f, 56.0f, 1.0f};
    M3 A2 = Mul(As, As);
    M3 A4 = Mul(A2, A2);
    M3 A6 = Mul(A4, A2);
    M3 tmp;
    for (int k = 0; k < 9; ++k) tmp.m[k] = b[7] * A6.m[k] + b[5] * A4.m[k] + b[3] * A2.m[k] + b[1] * I.m[k];
    U = Mul(As, tmp);
    for (int k = 0; k < 9; ++k) V.m[k] = b[6] * A6.m[k] + b[4] * A4.m[k] + b[2] * A2.m[k] + b[0] * I.m[k];
  }
  M3 numer = Lin(1.0f, U, 1.0f, V);
  M3 denom = Lin(-1.0f, U, 1.0f, V);
  M3 result = LuSolve(denom, numer);
  for (int i = 0; i < squarings; ++i) result = Mul(result, result);
  for (int k = 0; k < 9; ++k) out[k] = result.m[k];
}

inline double Now() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

}  // namespace

// =============================================================================================
// extern "C" surface
// =============================================================================================
extern "C" {

void orc_region_params_default(orc_region_params* p) {  // region_modality.h:411-443
  std::memset(p, 0, sizeof(*p));
  p->n_lines_max = 200;
  p->use_adaptive_coverage = 0;
  p->reference_contour_length = 0.0f;
  p->min_continuous_distance = 3.0f;
  p->function_length = 8;
  p->distribution_length = 12;
  p->function_amplitude = 0.43f;
  p->function_slope = 0.5f;
  p->learning_rate = 1.3f;
  p->n_global_iterations = 1;
  p->n_scales = 4;
  const int s[] = {6, 4, 2, 1};
  const float sd[] = {15.0f, 5.0f, 3.5f, 1.5f};
  for (int i = 0; i < 4; ++i) { p->scales[i] = s[i]; p->standard_deviations[i] = sd[i]; }
  p->n_standard_deviations = 4;
  p->n_histogram_bins = 16;
  p->learning_rate_f = 0.2f;
  p->learning_rate_b = 0.2f;
  p->unconsidered_line_length = 0.5f;
  p->max_considered_line_length = 20.0f;
  p->measure_occlusions = 0;
  p->measured_depth_offset_radius = 0.01f;
  p->measured_occlusion_radius = 0.01f;
  p->measured_occlusion_threshold = 0.03f;
  p->n_unoccluded_iterations = 10;
  p->min_n_unoccluded_lines = 0;
  p->modeled_depth_offset_radius = 0.01f;
  p->modeled_occlusion_radius = 0.01f;
  p->modeled_occlusion_threshold = 0.03f;
}

void orc_depth_params_default(orc_depth_params* p) {  // depth_modality.h:302-321
  std::memset(p, 0, sizeof(*p));
  p->n_points_max = 200;
  p->stride_length = 0.005f;
  p->n_considered_distances = 3;
  const float cd[] = {0.05f, 0.02f, 0.01f};
  const float sd[] = {0.05f, 0.03f, 0.02f};
  for (int i = 0; i < 3; ++i) { p->considered_distances[i] = cd[i]; p->standard_deviations[i] = sd[i]; }
  p->n_standard_deviations = 3;
  p->measured_depth_offset_radius = 0.01f;
  p->measured_occlusion_radius = 0.01f;
  p->measured_occlusion_threshold = 0.03f;
  p->n_unoccluded_iterations = 10;
  p->min_n_unoccluded_points = 0;
  p->modeled_depth_offset_radius = 0.01f;
  p->modeled_occlusion_radius = 0.01f;
  p->modeled_occlusion_threshold = 0.03f;
}

void orc_pose_multiply(const float a[12], const float b[12], float out[12]) { PoseMul(a, b, out); }
void orc_pose_inverse(const float a[12], float out[12]) { PoseInverse(a, out); }
void orc_pose_rotation(const float a[12], int rotation_mode, float r[9]) { PoseRotation(a, rotation_mode, r); }
void orc_exp_skew(const float w[3], int exp_mode, float r[9]) { ExpSkew(w, exp_mode, r); }
int orc_ldlt_solve(int n, const float* a, const float* b, float* x) { return LdltSolve(n, a, b, x) ? 1 : 0; }
void orc_function_lookup(const orc_region_params* p, float lookup_f[8], float lookup_b[8], float* mev) {
  FunctionLookup(p, lookup_f, lookup_b, mev);
}

// ---- ColorHistograms ------------------------------------------------------------------------
void orc_hist_clear(int n_bins, float* memory_f, float* memory_b) {  // color_histograms.cpp:49-58
  size_t n = size_t(n_bins) * n_bins * n_bins;
  std::fill(memory_f, memory_f + n, 0.0f);
  std::fill(memory_b, memory_b + n, 0.0f);
}
void orc_hist_add(int n_bins, float* memory, const uint8_t bgr[3]) {  // :60-70
  memory[HistIndex(n_bins, Bitshift(n_bins), bgr)] += 1.0f;
}
void orc_hist_calculate(int n_bins, float learning_rate, const float* memory, float* histogram) {  // :174-214
  int n = n_bins * n_bins * n_bins;
  float sum = 0.0f;
  for (int i = 0; i < n; ++i) sum += memory[i];
  if (!sum) {
    if (learning_rate == 1.0f) {
      float uniform_value = 1.0f / float(n);
      std::fill(histogram, histogram + n, uniform_value);
    }
    return;
  }
  float complement_learning_rate = 1.0f - learning_rate;
  float learning_rate_divide_sum = learning_rate / sum;
  if (complement_learning_rate == 0.0f) {
    for (int i = 0; i < n; ++i) histogram[i] = memory[i] * learning_rate_divide_sum;
  } else {
    for (int i = 0; i < n; ++i) {
      histogram[i] *= complement_learning_rate;
      histogram[i] += memory[i] * learning_rate_divide_sum;
    }
  }
}
void orc_hist_get(int n_bins, const float* hist_f, const float* hist_b, const uint8_t bgr[3], float* pf, float* pb) {
  int idx = HistIndex(n_bins, Bitshift(n_bins), bgr);
  *pf = hist_f[idx];
  *pb = hist_b[idx];
}

int orc_closest_view(const orc_model* model, const float body2camera[12], int rotation_mode) {
  return ClosestView(model, body2camera, rotation_mode);
}

}  // extern "C"
namespace {
constexpr int kMaxNOcclusionStrides = 5;  // region_modality.h:145, depth_modality.h:113

// A NaN diameter or one in (-5, 0) gives the reference's scans a stride of 0 and a loop that never ends. A window whose
// diameter is not finite or is negative (an item behind or level with the camera, a non-finite pose) scans nothing and
// counts as unoccluded, as in the library.
bool ScanDiameterValid(float diameter) { return diameter >= 0.0f && diameter <= 3.40282347e38f; }

// The strided window scan shared by RegionModality::IsLineUnoccludedMeasured (region_modality.cpp:1355-1388) and
// DepthModality::IsPointUnoccludedMeasured (depth_modality.cpp:739-775): false if any valid depth sample inside the
// window lies in front of min_depth. The reference converts the float threshold with ushort(x); that is restated as
// truncation to int followed by reduction modulo 2^16 (what x86 does), so that a negative threshold behaves the same
// on both sides of the parity tests.
bool WindowUnoccluded(const orc_depth_frame* f, float center_u, float center_v, float diameter, float min_depth_value) {
  if (!ScanDiameterValid(diameter)) return true;
  int stride = int(diameter / kMaxNOcclusionStrides + 1.0f);
  int n_strides = int(diameter / stride + 0.5f);
  int rounded_diameter = n_strides * stride;
  float rounded_radius = 0.5f * float(rounded_diameter);
  int u_min = int(center_u - rounded_radius + 0.5f);
  int v_min = int(center_v - rounded_radius + 0.5f);
  int u_max = u_min + rounded_diameter;
  int v_max = v_min + rounded_diameter;
  u_min = std::max(u_min, 0);
  v_min = std::max(v_min, 0);
  u_max = std::min(u_max, f->intrinsics.width - 1);
  v_max = std::min(v_max, f->intrinsics.height - 1);
  const uint16_t min_depth = uint16_t(unsigned(int(min_depth_value)) & 0xffffu);
  for (int v = v_min; v <= v_max; v += stride) {
    const uint16_t* row = reinterpret_cast<const uint16_t*>(reinterpret_cast<const uint8_t*>(f->depth) + size_t(v) * f->pitch);
    for (int u = u_min; u <= u_max; u += stride) {
      uint16_t depth = row[u];
      if (depth > 0 && depth < min_depth) return false;
    }
  }
  return true;
}

// RegionModality::IsLineUnoccludedMeasured (region_modality.cpp:1343-1389)
bool LineUnoccludedMeasured(const orc_region_params* p, const orc_depth_frame* f, const float* body2depth_camera,
                            const float* center_f_body, float depth_offset) {
  float cd[3];
  PoseApply(body2depth_camera, center_f_body, cd);
  float center_u = cd[0] * f->intrinsics.fu / cd[2] + f->intrinsics.ppu;
  float center_v = cd[1] * f->intrinsics.fv / cd[2] + f->intrinsics.ppv;
  float meter_to_pixel = f->intrinsics.fu / cd[2];
  float diameter = 2.0f * p->measured_occlusion_radius * meter_to_pixel;
  return WindowUnoccluded(f, center_u, center_v, diameter,
                          (cd[2] - depth_offset - p->measured_occlusion_threshold) / f->depth_scale);
}

// measured_depth_offset_id_ (region_modality.cpp:965-977); -1 if the radius exceeds the model's table or rounds to an
// id past its 30 entries (max_radius / stride in [29.5, 30) passes the reference's radius test), which the library
// refuses
int RegionOffsetIdOf(float radius, const orc_model* model) {
  if (radius > model->max_radius_depth_offset) return -1;
  const int id = int(radius / model->stride_depth_offset + 0.5f);
  return id < ORC_N_DEPTH_OFFSETS ? id : -1;
}
int RegionOffsetId(const orc_region_params* p, const orc_model* model) {
  return RegionOffsetIdOf(p->measured_depth_offset_radius, model);
}
// modeled_depth_offset_id_ (region_modality.cpp:979-991)
int RegionModeledOffsetId(const orc_region_params* p, const orc_model* model) {
  return RegionOffsetIdOf(p->modeled_depth_offset_radius, model);
}

constexpr int kNRegionStride = 5;      // region_modality.h:146
constexpr float kRegionOffset = 2.0f;  // region_modality.h:147

inline uint8_t SilhouetteAt(const orc_rendering* r, int v, int u) {
  return reinterpret_cast<const uint8_t*>(r->image)[size_t(v) * r->pitch + size_t(u)];
}

// The strided minimum scan shared by RegionModality::IsLineUnoccludedModeled (region_modality.cpp:1391-1431) and
// DepthModality::IsPointUnoccludedModeled (depth_modality.cpp:778-824), in the focused depth rendering.
bool ModeledWindowUnoccluded(const orc_rendering* r, float center_u, float center_v, float diameter, float min_allowed_depth) {
  if (!ScanDiameterValid(diameter)) return true;
  int stride = int(diameter / kMaxNOcclusionStrides + 1.0f);
  int n_strides = int(diameter / stride + 0.5f);
  int rounded_diameter = n_strides * stride;
  float rounded_radius = 0.5f * float(rounded_diameter);
  float focused_center_u = (center_u - r->corner_u) * r->scale;
  float focused_center_v = (center_v - r->corner_v) * r->scale;
  int u_min = int(focused_center_u - rounded_radius + 0.5f);
  int v_min = int(focused_center_v - rounded_radius + 0.5f);
  int u_max = u_min + rounded_diameter;
  int v_max = v_min + rounded_diameter;
  u_min = std::max(u_min, 0);
  v_min = std::max(v_min, 0);
  u_max = std::min(u_max, r->image_size - 1);
  v_max = std::min(v_max, r->image_size - 1);
  uint16_t min_depth_value = 65535;
  for (int v = v_min; v <= v_max; v += stride) {
    const uint16_t* row = reinterpret_cast<const uint16_t*>(reinterpret_cast<const uint8_t*>(r->image) + size_t(v) * r->pitch);
    for (int u = u_min; u <= u_max; u += stride) min_depth_value = std::min(min_depth_value, row[u]);
  }
  float min_depth = r->projection_term_a / (r->projection_term_b - float(min_depth_value));  // FocusedDepthRenderer::Depth
  return min_depth > min_allowed_depth;
}

// RegionModality::IsLineUnoccludedModeled (region_modality.cpp:1391-1431)
bool LineUnoccludedModeled(const orc_region_params* p, const orc_rendering* r, float fu, float center_u, float center_v,
                           float depth, float depth_offset) {
  float meter_to_pixel = (fu / depth) * r->scale;
  float diameter = 2.0f * p->modeled_occlusion_radius * meter_to_pixel;
  return ModeledWindowUnoccluded(r, center_u, center_v, diameter, depth - depth_offset - p->modeled_occlusion_threshold);
}

// RegionModality::IsDynamicLineRegionSufficient (region_modality.cpp:1293-1341)
bool DynamicLineRegionSufficient(const orc_region_params* p, const orc_rendering* r, float fscale, float center_u,
                                 float center_v, float normal_u, float normal_v) {
  const uint8_t region_id = uint8_t(r->id);
  const float fsize = float(r->image_size);
  float focused_min_continuous_distance = p->min_continuous_distance * fscale * r->scale;
  float focused_stride = std::max((focused_min_continuous_distance - kRegionOffset) / float(kNRegionStride), 0.0f);
  float stride_u = focused_stride * normal_u;
  float stride_v = focused_stride * normal_v;
  float offset_u = kRegionOffset * normal_u;
  float offset_v = kRegionOffset * normal_v;
  float focused_center_u = 0.5f + (center_u - r->corner_u) * r->scale;
  float focused_center_v = 0.5f + (center_v - r->corner_v) * r->scale;
  // foreground region. The reference reads silhouette_image.at<uchar>(int(v), int(u)) without a bounds test here; a
  // sample outside the focused image is undefined behaviour there - it is treated as "not this region" on both sides.
  float u = focused_center_u - offset_u;
  float v = focused_center_v - offset_v;
  for (int i = 0; i <= kNRegionStride; ++i) {
    if (u >= fsize || u < 0.0f || v >= fsize || v < 0.0f) return false;
    if (SilhouetteAt(r, int(v), int(u)) != region_id) return false;
    u -= stride_u;
    v -= stride_v;
  }
  // background region
  u = focused_center_u + offset_u;
  v = focused_center_v + offset_v;
  for (int i = 0; i <= kNRegionStride; ++i) {
    if (u >= fsize || u < 0.0f || v >= fsize || v < 0.0f) break;
    if (SilhouetteAt(r, int(v), int(u)) == region_id) return false;
    u += stride_u;
    v += stride_v;
  }
  return true;
}

// RegionModality::DynamicRegionDistance (region_modality.cpp:1157-1223), including its quirk: a background sample of
// the own region at i > i_start overwrites the FOREGROUND distance (:1218)
void DynamicRegionDistance(const orc_region_params* p, const orc_rendering* r, float center_u, float center_v,
                           float normal_u, float normal_v, float* dynamic_foreground_distance,
                           float* dynamic_background_distance) {
  const uint8_t region_id = uint8_t(r->id);
  const float fsize = float(r->image_size);
  float stride = p->max_considered_line_length / float(kNRegionStride);
  float focused_stride = stride * r->scale;
  float focused_stride_u = focused_stride * normal_u;
  float focused_stride_v = focused_stride * normal_v;
  float delta_start = kRegionOffset / r->scale - p->unconsidered_line_length;
  int i_start = std::max(int(delta_start / stride + 1.0f), 0);
  float offset = p->unconsidered_line_length + float(i_start) * stride;
  float focused_offset = offset * r->scale;
  float focused_offset_u = focused_offset * normal_u;
  float focused_offset_v = focused_offset * normal_v;
  float focused_center_u = 0.5f + (center_u - r->corner_u) * r->scale;
  float focused_center_v = 0.5f + (center_v - r->corner_v) * r->scale;
  float u = focused_center_u - focused_offset_u;
  float v = focused_center_v - focused_offset_v;
  for (int i = i_start; i <= kNRegionStride; ++i) {
    if (u >= fsize || u < 0.0f || v >= fsize || v < 0.0f) {
      *dynamic_foreground_distance = stride * float(i);
      break;
    }
    if (SilhouetteAt(r, int(v), int(u)) != region_id) {
      if (i == i_start) *dynamic_foreground_distance = 0.0f;
      else *dynamic_foreground_distance = stride * float(i);
      break;
    }
    u -= focused_stride_u;
    v -= focused_stride_v;
  }
  u = focused_center_u + focused_offset_u;
  v = focused_center_v + focused_offset_v;
  for (int i = i_start; i <= kNRegionStride; ++i) {
    if (u >= fsize || u < 0.0f || v >= fsize || v < 0.0f) {
      *dynamic_background_distance = p->max_considered_line_length;
      break;
    }
    if (SilhouetteAt(r, int(v), int(u)) == region_id) {
      if (i == i_start) *dynamic_background_distance = 0.0f;
      else *dynamic_foreground_distance = stride * float(i);  // sic (:1218)
      break;
    }
    u += focused_stride_u;
    v += focused_stride_v;
  }
}
}  // namespace
extern "C" {

// ---- RegionModality::AddLinePixelColorsToTempHistograms (region_modality.cpp:1025-1155) -------
void orc_region_add_line_pixels(const orc_region_params* p, const orc_model* model, const orc_color_frame* c,
                                const float body2world[12], int rotation_mode, float* memory_f, float* memory_b) {
  orc_region_add_line_pixels_occ(p, model, c, nullptr, 0, body2world, rotation_mode, memory_f, memory_b);
}

void orc_region_add_line_pixels_occ(const orc_region_params* p, const orc_model* model, const orc_color_frame* c,
                                    const orc_depth_frame* occlusion_depth, int handle_occlusions,
                                    const float body2world[12], int rotation_mode, float* memory_f, float* memory_b) {
  const bool occ = handle_occlusions && p->measure_occlusions && occlusion_depth;
  float body2depth_camera[12];
  int offset_id = 0;
  if (occ) {
    PoseMul(occlusion_depth->world2camera, body2world, body2depth_camera);  // region_modality.cpp:1003-1005
    offset_id = std::max(0, RegionOffsetId(p, model));
  }
  // renderer-image checks (:1031-1043): modeled occlusions only with handle_occlusions, region checking always
  const orc_rendering* dr = c->depth_rendering;
  const orc_rendering* sr = c->silhouette_rendering;
  const bool model_occ = handle_occlusions && p->model_occlusions && dr && dr->visible;
  const bool region_checking = p->use_region_checking && sr && sr->visible;
  const int modeled_offset_id = std::max(0, RegionModeledOffsetId(p, model));
  RegionVars v;
  RegionPrecalc(p, c, body2world, 0, rotation_mode, &v);
  int view = ClosestView(model, v.body2camera, rotation_mode);
  int n_lines = AdaptiveCount(p->n_lines_max, p->use_adaptive_coverage, p->reference_contour_length,
                              model->view_scalars ? model->view_scalars[view] : 0.0f, model->max_view_scalar,
                              model->n_points);
  const float* pts = model->points + size_t(view) * model->n_points * ORC_REGION_POINT_FLOATS;
  for (int i = 0; i < n_lines; ++i) {
    const float* dp = pts + size_t(i) * ORC_REGION_POINT_FLOATS;
    const float* center_f_body = dp;
    const float* normal_f_body = dp + 3;
    float foreground_distance = dp[6], background_distance = dp[7];
    float cc[3];
    PoseApply(v.body2camera, center_f_body, cc);
    if (!(cc[2] > 0.0f)) continue;
    float center_u = cc[0] * v.fu / cc[2] + v.ppu;
    float center_v = cc[1] * v.fv / cc[2] + v.ppv;
    int i_center_u = int(center_u + 0.5f);
    int i_center_v = int(center_v + 0.5f);
    if (i_center_u < 0 || i_center_u > v.w_m1 || i_center_v < 0 || i_center_v > v.h_m1) continue;
    if (model_occ && !LineUnoccludedModeled(p, dr, v.fu, center_u, center_v, cc[2], dp[8 + modeled_offset_id]))
      continue;  // :1079-1084
    if (occ && !LineUnoccludedMeasured(p, occlusion_depth, body2depth_camera, center_f_body, dp[8 + offset_id]))
      continue;  // :1086-1089
    float length_f = p->max_considered_line_length;
    float length_b = p->max_considered_line_length;
    if (region_checking) {  // :1092-1099
      float nrm[2] = {v.rot[0] * normal_f_body[0] + v.rot[1] * normal_f_body[1] + v.rot[2] * normal_f_body[2],
                      v.rot[3] * normal_f_body[0] + v.rot[4] * normal_f_body[1] + v.rot[5] * normal_f_body[2]};
      Normalize2(nrm);
      DynamicRegionDistance(p, sr, center_u, center_v, nrm[0], nrm[1], &length_f, &length_b);
    }
    float l_f = foreground_distance * v.fu / cc[2];
    float l_b = background_distance * v.fu / cc[2];
    length_f = std::fmin(length_f, l_f - 2.0f * p->unconsidered_line_length);
    length_b = std::fmin(length_b, l_b - 2.0f * p->unconsidered_line_length);
    float normal[2] = {v.rot[0] * normal_f_body[0] + v.rot[1] * normal_f_body[1] + v.rot[2] * normal_f_body[2],
                       v.rot[3] * normal_f_body[0] + v.rot[4] * normal_f_body[1] + v.rot[5] * normal_f_body[2]};
    Normalize2(normal);
    float u_step, v_step;
    int projected_length_f, projected_length_b;
    float abs_normal_u = std::fabs(normal[0]);
    float abs_normal_v = std::fabs(normal[1]);
    if (abs_normal_u > abs_normal_v) {
      u_step = sgnf(normal[0]);
      v_step = normal[1] / abs_normal_u;
      projected_length_f = int(length_f * abs_normal_u + 0.5f);
      projected_length_b = int(length_b * abs_normal_u + 0.5f);
    } else {
      u_step = normal[0] / abs_normal_v;
      v_step = sgnf(normal[1]);
      projected_length_f = int(length_f * abs_normal_v + 0.5f);
      projected_length_b = int(length_b * abs_normal_v + 0.5f);
    }
    float u = center_u - normal[0] * p->unconsidered_line_length + 0.5f;
    float vv = center_v - normal[1] * p->unconsidered_line_length + 0.5f;
    for (int k = 0; k < projected_length_f; ++k) {
      int i_u = int(u), i_v = int(vv);
      if (i_u < 0 || i_u > v.w_m1 || i_v < 0 || i_v > v.h_m1) break;
      orc_hist_add(p->n_histogram_bins, memory_f, c->bgr + size_t(i_v) * c->pitch + 3 * size_t(i_u));
      u -= u_step;
      vv -= v_step;
    }
    u = center_u + normal[0] * p->unconsidered_line_length + 0.5f;
    vv = center_v + normal[1] * p->unconsidered_line_length + 0.5f;
    for (int k = 0; k < projected_length_b; ++k) {
      int i_u = int(u), i_v = int(vv);
      if (i_u < 0 || i_u > v.w_m1 || i_v < 0 || i_v > v.h_m1) break;
      orc_hist_add(p->n_histogram_bins, memory_b, c->bgr + size_t(i_v) * c->pitch + 3 * size_t(i_u));
      u += u_step;
      vv += v_step;
    }
  }
}

// ---- RegionModality::CalculateCorrespondences (region_modality.cpp:390-465) -------------------
int orc_region_correspondences(const orc_region_params* p, const orc_model* model, const orc_color_frame* c,
                               const orc_depth_frame* occlusion_depth, const float* hist_f, const float* hist_b,
                               const float body2world[12], int iteration, int first_iteration, int corr_iteration,
                               int rotation_mode, orc_region_line* lines, int* view_index) {
  RegionVars v;
  RegionPrecalc(p, c, body2world, corr_iteration, rotation_mode, &v);
  int view = ClosestView(model, v.body2camera, rotation_mode);
  if (view_index) *view_index = view;
  int n_lines = AdaptiveCount(p->n_lines_max, p->use_adaptive_coverage, p->reference_contour_length,
                              model->view_scalars ? model->view_scalars[view] : 0.0f, model->max_view_scalar,
                              model->n_points);
  const float* pts = model->points + size_t(view) * model->n_points * ORC_REGION_POINT_FLOATS;
  float sf[32], sb[32];
  const bool can_measure = p->measure_occlusions && occlusion_depth;
  float body2depth_camera[12];
  int offset_id = 0;
  if (can_measure) {
    PoseMul(occlusion_depth->world2camera, body2world, body2depth_camera);
    offset_id = std::max(0, RegionOffsetId(p, model));
  }
  const orc_rendering* dr = c->depth_rendering;
  const orc_rendering* sr = c->silhouette_rendering;
  const bool can_model = p->model_occlusions && dr && dr->visible;            // :397-401
  const bool region_checking = p->use_region_checking && sr && sr->visible;   // :402-408, both passes
  const int modeled_offset_id = std::max(0, RegionModeledOffsetId(p, model));
  // Two passes (:435-463): the first handles occlusions once the modality has run n_unoccluded_iterations; if too
  // few lines survive, everything is recomputed without occlusion handling. Without an occlusion source the two
  // passes are identical, so one suffices.
  for (int j = 0; j < 2; ++j) {
    const bool handle_occlusions = j == 0 && (iteration - first_iteration) >= p->n_unoccluded_iterations;
    const bool occ = handle_occlusions && can_measure;
    const bool mocc = handle_occlusions && can_model;
    int survivors = 0;
    for (int i = 0; i < n_lines; ++i) {
      const float* dp = pts + size_t(i) * ORC_REGION_POINT_FLOATS;
      orc_region_line& L = lines[i];
      std::memset(&L, 0, sizeof(L));
      L.model_index = i;
      // CalculateBasicLineData (:1231-1250)
      float cc[3];
      PoseApply(v.body2camera, dp, cc);
      float n2[2] = {v.rot[0] * dp[3] + v.rot[1] * dp[4] + v.rot[2] * dp[5],
                     v.rot[3] * dp[3] + v.rot[4] * dp[4] + v.rot[5] * dp[5]};
      Normalize2(n2);
      L.center_f_body[0] = dp[0]; L.center_f_body[1] = dp[1]; L.center_f_body[2] = dp[2];
      L.center_u = cc[0] * v.fu / cc[2] + v.ppu;
      L.center_v = cc[1] * v.fv / cc[2] + v.ppv;
      L.normal_u = n2[0];
      L.normal_v = n2[1];
      float continuous_distance = std::min(dp[7], dp[6]) * v.fu / (cc[2] * v.fscale);
      // IsLineValid (:1252-1291)
      if (continuous_distance < p->min_continuous_distance) continue;
      if (!(cc[2] > 0.0f)) continue;
      int i_center_u = int(L.center_u + 0.5f);
      int i_center_v = int(L.center_v + 0.5f);
      if (i_center_u < 0 || i_center_u > v.w_m1 || i_center_v < 0 || i_center_v > v.h_m1) continue;
      if (region_checking &&
          !DynamicLineRegionSufficient(p, sr, v.fscale, L.center_u, L.center_v, L.normal_u, L.normal_v))
        continue;  // :1269-1274
      if (occ && !LineUnoccludedMeasured(p, occlusion_depth, body2depth_camera, dp, dp[8 + offset_id])) continue;
      if (mocc && !LineUnoccludedModeled(p, dr, v.fu, L.center_u, L.center_v, cc[2], dp[8 + modeled_offset_id]))
        continue;  // :1283-1289
      if (!SegmentProbabilities(v, c, hist_f, hist_b, L.center_u, L.center_v, L.normal_u, L.normal_v, sf, sb,
                                &L.normal_component_to_scale, &L.delta_r))
        continue;
      Distribution(v, p->function_length, p->distribution_length, sf, sb, L.distribution);
      Moments(v, p->distribution_length, L.distribution, &L.mean, &L.measured_variance);
      L.valid = 1;
      survivors++;
    }
    if (!(occ || mocc) || survivors >= p->min_n_unoccluded_lines) break;
  }
  return n_lines;
}

// ---- RegionModality::CalculateGradientAndHessian (region_modality.cpp:485-558) ----------------
void orc_region_gradient_hessian(const orc_region_params* p, const orc_color_frame* c, const float body2world[12],
                                 const orc_region_line* lines, int n_lines, int corr_iteration, int opt_iteration,
                                 int rotation_mode, float g[6], float H[36]) {
  RegionVars v;
  RegionPrecalc(p, c, body2world, corr_iteration, rotation_mode, &v);
  for (int i = 0; i < 6; ++i) g[i] = 0.0f;
  for (int i = 0; i < 36; ++i) H[i] = 0.0f;
  for (int li = 0; li < n_lines; ++li) {
    const orc_region_line& L = lines[li];
    if (!L.valid) continue;
    float cc[3];
    PoseApply(v.body2camera, L.center_f_body, cc);
    float x = cc[0], y = cc[1], z = cc[2];
    float fu_z = v.fu / z;
    float fv_z = v.fv / z;
    float xfu_z = x * fu_z;
    float yfv_z = y * fv_z;
    float delta_cs = (L.normal_u * (xfu_z + v.ppu - L.center_u) + L.normal_v * (yfv_z + v.ppv - L.center_v) - L.delta_r) *
                     L.normal_component_to_scale;
    float dloglikelihood_ddelta_cs;
    if (opt_iteration < p->n_global_iterations) {
      dloglikelihood_ddelta_cs = (L.mean - delta_cs) / L.measured_variance;
    } else {
      int dist_idx_upper = int(delta_cs + v.dl_plus_1_half);
      int dist_idx_lower = dist_idx_upper - 1;
      if (dist_idx_upper <= 0 || dist_idx_upper >= p->distribution_length) continue;
      dloglikelihood_ddelta_cs = (std::log(L.distribution[dist_idx_upper]) - std::log(L.distribution[dist_idx_lower])) *
                                 p->learning_rate / L.measured_variance;
    }
    float ncts = L.normal_component_to_scale;
    float dc[3] = {ncts * L.normal_u * fu_z, ncts * L.normal_v * fv_z,
                   ncts * (-L.normal_u * xfu_z - L.normal_v * yfv_z) / z};
    float dt[3];
    for (int j = 0; j < 3; ++j) dt[j] = dc[0] * v.rot[0 + j] + dc[1] * v.rot[3 + j] + dc[2] * v.rot[6 + j];
    const float* cb = L.center_f_body;
    float J[6] = {cb[1] * dt[2] - cb[2] * dt[1], cb[2] * dt[0] - cb[0] * dt[2], cb[0] * dt[1] - cb[1] * dt[0],
                  dt[0], dt[1], dt[2]};
    float weight = v.min_expected_variance / (ncts * ncts * v.variance);
    float wg = weight * dloglikelihood_ddelta_cs;
    float wh = weight / L.measured_variance;
    for (int i = 0; i < 6; ++i) g[i] += wg * J[i];
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j <= i; ++j) H[6 * i + j] -= (wh * J[i]) * J[j];
  }
  for (int i = 0; i < 6; ++i)
    for (int j = i + 1; j < 6; ++j) H[6 * i + j] = H[6 * j + i];  // selfadjointView<Lower>
}

// ---- DepthModality::CalculateCorrespondences (depth_modality.cpp:252-315) ---------------------
int orc_depth_correspondences(const orc_depth_params* p, const orc_model* model, const orc_depth_frame* f,
                              const float body2world[12], int iteration, int first_iteration, int corr_iteration,
                              int rotation_mode, orc_depth_point* points, int* view_index) {
  DepthVars v;
  DepthPrecalc(p, f, body2world, corr_iteration, &v);
  int view = ClosestView(model, v.body2camera, rotation_mode);
  if (view_index) *view_index = view;
  int n_points = AdaptiveCount(p->n_points_max, p->use_adaptive_coverage, p->reference_surface_area,
                               model->view_scalars ? model->view_scalars[view] : 0.0f, model->max_view_scalar,
                               model->n_points);
  const float* pts = model->points + size_t(view) * model->n_points * ORC_DEPTH_POINT_FLOATS;
  const orc_rendering* dr = f->depth_rendering;
  const orc_rendering* sr = f->silhouette_rendering;
  const bool can_model = p->model_occlusions && dr && dr->visible;              // :259-263
  const bool silhouette_checking = p->use_silhouette_checking && sr && sr->visible;  // :264-270, both passes
  for (int j = 0; j < 2; ++j) {  // :295-313
    const bool handle = j == 0 && (iteration - first_iteration) >= p->n_unoccluded_iterations;
    const bool occ = handle && p->measure_occlusions;
    const bool mocc = handle && can_model;
    int survivors = 0;
    for (int i = 0; i < n_points; ++i) {
      const float* dp = pts + size_t(i) * ORC_DEPTH_POINT_FLOATS;
      orc_depth_point& P = points[i];
      std::memset(&P, 0, sizeof(P));
      P.model_index = i;
      // CalculateBasicPointData (:656-695)
      float cc[3];
      PoseApply(v.body2camera, dp, cc);
      for (int k = 0; k < 3; ++k) { P.center_f_body[k] = dp[k]; P.normal_f_body[k] = dp[3 + k]; }
      float center_u = cc[0] * v.fu / cc[2] + v.ppu;
      float center_v = cc[1] * v.fv / cc[2] + v.ppv;
      float depth = cc[2];
      // IsPointValid (:697-726)
      if (!(depth > 0.0f)) continue;
      int i_center_u = int(center_u + 0.5f);
      int i_center_v = int(center_v + 0.5f);
      if (i_center_u < 0 || i_center_u > v.w_m1 || i_center_v < 0 || i_center_v > v.h_m1) continue;
      if (silhouette_checking) {  // IsPointOnValidSilhouette (:728-734) via FocusedSilhouetteRenderer::SilhouetteValue
        int su = int((float(i_center_u) - sr->corner_u) * sr->scale + 0.5f);
        int sv = int((float(i_center_v) - sr->corner_v) * sr->scale + 0.5f);
        // (outside the focused image the reference reads out of bounds; treated as "another body" on both sides)
        if (su < 0 || su >= sr->image_size || sv < 0 || sv >= sr->image_size) continue;
        if (SilhouetteAt(sr, sv, su) != uint8_t(sr->id)) continue;
      }
      if (occ) {  // IsPointUnoccludedMeasured (:736-776) with the depth offset selected in CalculateBasicPointData
        float radius = p->measured_depth_offset_radius;
        if (p->use_depth_scaling) radius *= depth;
        int id = int(radius / model->stride_depth_offset + 0.5f);
        if (id >= ORC_N_DEPTH_OFFSETS) id = ORC_N_DEPTH_OFFSETS - 1;
        float measured_depth_offset = dp[6 + id];
        float diameter = 2.0f * p->measured_occlusion_radius * v.fu;
        if (!p->use_depth_scaling) diameter /= depth;
        float threshold = p->measured_occlusion_threshold;
        if (p->use_depth_scaling) threshold *= depth;
        if (!WindowUnoccluded(f, center_u, center_v, diameter, (depth - measured_depth_offset - threshold) / v.depth_scale))
          continue;
      }
      if (mocc) {  // IsPointUnoccludedModeled (:778-824), depth offset selected in CalculateBasicPointData (:682-693)
        float radius = p->modeled_depth_offset_radius;
        if (p->use_depth_scaling) radius *= depth;
        int id = int(radius / model->stride_depth_offset + 0.5f);
        if (id >= ORC_N_DEPTH_OFFSETS) id = ORC_N_DEPTH_OFFSETS - 1;
        float modeled_depth_offset = dp[6 + id];
        float meter_to_pixel = v.fu * dr->scale;
        if (!p->use_depth_scaling) meter_to_pixel /= depth;
        float diameter = 2.0f * p->modeled_occlusion_radius * meter_to_pixel;
        float threshold = p->modeled_occlusion_threshold;
        if (p->use_depth_scaling) threshold *= depth;
        if (!ModeledWindowUnoccluded(dr, center_u, center_v, diameter, depth - modeled_depth_offset - threshold)) continue;
      }
      if (!FindCorrespondence(p, v, f, cc, center_u, center_v, depth, P.correspondence_center_f_camera)) continue;
      P.valid = 1;
      survivors++;
    }
    if (!(occ || mocc) || survivors >= p->min_n_unoccluded_points) break;
  }
  return n_points;
}

// ---- DepthModality::CalculateGradientAndHessian (depth_modality.cpp:333-381) ------------------
void orc_depth_gradient_hessian(const orc_depth_params* p, const orc_depth_frame* f, const float body2world[12],
                                const orc_depth_point* points, int n_points, int corr_iteration, float g[6],
                                float H[36]) {
  DepthVars v;
  DepthPrecalc(p, f, body2world, corr_iteration, &v);
  for (int i = 0; i < 6; ++i) g[i] = 0.0f;
  for (int i = 0; i < 36; ++i) H[i] = 0.0f;
  for (int pi = 0; pi < n_points; ++pi) {
    const orc_depth_point& P = points[pi];
    if (!P.valid) continue;
    float yb[3];
    PoseApply(v.camera2body, P.correspondence_center_f_camera, yb);
    const float* n = P.normal_f_body;
    const float* xb = P.center_f_body;
    float epsilon = n[0] * (xb[0] - yb[0]) + n[1] * (xb[1] - yb[1]) + n[2] * (xb[2] - yb[2]);
    float cx[3] = {yb[1] * n[2] - yb[2] * n[1], yb[2] * n[0] - yb[0] * n[2], yb[0] * n[1] - yb[1] * n[0]};
    float correspondence_depth = P.correspondence_center_f_camera[2];
    float weight = 1.0f / (v.standard_deviation * correspondence_depth);
    float squared_weight = weight * weight;
    float wc[3] = {weight * cx[0], weight * cx[1], weight * cx[2]};
    float wn[3] = {weight * n[0], weight * n[1], weight * n[2]};
    float se = squared_weight * epsilon;
    for (int i = 0; i < 3; ++i) {
      g[i] -= se * cx[i];
      g[3 + i] -= se * n[i];
    }
    for (int i = 0; i < 3; ++i)
      for (int j = i; j < 3; ++j) H[6 * i + j] -= wc[i] * wc[j];           // topLeft, Upper
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) H[6 * i + 3 + j] -= wc[i] * wn[j];       // topRight
    for (int i = 0; i < 3; ++i)
      for (int j = i; j < 3; ++j) H[6 * (3 + i) + 3 + j] -= wn[i] * wn[j]; // bottomRight, Upper
  }
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < i; ++j) H[6 * i + j] = H[6 * j + i];  // selfadjointView<Upper>
}

// ---- Optimizer::CalculateOptimization for one rigid body (optimizer.cpp:144-167) --------------
int orc_optimize_rigid(const float g[6], const float H[36], float tikhonov_rotation, float tikhonov_translation,
                       int exp_mode, float body2world[12], float theta_out[6]) {
  float a[36], b[6], theta[6];
  // b += J^T g ; a(lower) -= J^T H J with J = I6 (root link, body2joint = I, all directions free)
  for (int i = 0; i < 6; ++i) {
    b[i] = 0.0f + g[i];
    for (int j = 0; j < 6; ++j) a[6 * i + j] = (j <= i) ? 0.0f - H[6 * i + j] : 0.0f;
  }
  for (int i = 0; i < 6; ++i) a[6 * i + i] += (i < 3) ? tikhonov_rotation : tikhonov_translation;  // :159, :252-271
  LdltSolve(6, a, b, theta);
  if (theta_out) std::memcpy(theta_out, theta, sizeof(theta));
  for (int i = 0; i < 6; ++i)
    if (std::isnan(theta[i])) return 0;  // :165
  // Link::UpdatePoses (link.cpp:205-241), root link: link2world * [exp(skew(theta_r)) | theta_t]
  float e[9];
  ExpSkew(theta, exp_mode, e);
  float var[12] = {e[0], e[1], e[2], theta[3], e[3], e[4], e[5], theta[4], e[6], e[7], e[8], theta[5]};
  float nb[12];
  PoseMul(body2world, var, nb);
  std::memcpy(body2world, nb, sizeof(nb));
  return 1;
}

// ---- batch drivers ---------------------------------------------------------------------------
int orc_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

static void StartOne(orc_body* b, int iteration, int rotation_mode) {
  // RegionModality::StartModality (region_modality.cpp:375-388)
  b->first_iteration = iteration;
  if (!b->region) return;
  int nb = b->region->n_histogram_bins;
  size_t n = size_t(nb) * nb * nb;
  std::vector<float> mf(n, 0.0f), mb(n, 0.0f);
  orc_region_add_line_pixels_occ(b->region, b->region_model, b->color, b->region_occlusion_frame,
                                 b->region->n_unoccluded_iterations == 0, b->body2world, rotation_mode, mf.data(), mb.data());
  orc_hist_calculate(nb, 1.0f, mf.data(), b->histogram_f);  // InitializeHistograms (color_histograms.cpp:72-81)
  orc_hist_calculate(nb, 1.0f, mb.data(), b->histogram_b);
}

// RegionModality::UseSharedColorHistograms (region_modality.cpp:168-179): bodies whose histogram_f pointers are equal use
// ONE ColorHistograms object. Their modalities only add their line pixels (StartModality :382-386, CalculateResults
// :575-582 skip ClearMemory / Initialize / Update); the tracker clears the object before and initialises / updates it
// once after all modalities (tracker.cpp:435-443, 507-515). The object's own learning rates (color_histograms.h) are
// taken from the first body of the group. Returns false if no body shares anything (the per-body path then runs).
static bool SharedHistogramPass(orc_body* bodies, int n_bodies, int iteration, int rotation_mode, bool start) {
  std::vector<int> leader(n_bodies);
  bool any = false;
  for (int i = 0; i < n_bodies; ++i) {
    leader[i] = i;
    if (!bodies[i].region) continue;
    for (int j = 0; j < i; ++j)
      if (bodies[j].region && bodies[j].histogram_f == bodies[i].histogram_f) { leader[i] = j; any = true; break; }
  }
  if (!any) return false;
  for (int l = 0; l < n_bodies; ++l) {
    if (leader[l] != l) continue;
    orc_body* L = &bodies[l];
    if (start) L->first_iteration = iteration;
    if (!L->region) continue;
    int nb = L->region->n_histogram_bins;
    size_t n = size_t(nb) * nb * nb;
    std::vector<float> mf(n, 0.0f), mb(n, 0.0f);  // ClearMemory
    for (int i = l; i < n_bodies; ++i) {
      if (leader[i] != l) continue;
      orc_body* b = &bodies[i];
      if (start) b->first_iteration = iteration;
      const bool handle_occlusions = start ? b->region->n_unoccluded_iterations == 0
                                           : (iteration - b->first_iteration) >= b->region->n_unoccluded_iterations;
      orc_region_add_line_pixels_occ(b->region, b->region_model, b->color, b->region_occlusion_frame, handle_occlusions,
                                     b->body2world, rotation_mode, mf.data(), mb.data());
    }
    orc_hist_calculate(nb, start ? 1.0f : L->region->learning_rate_f, mf.data(), L->histogram_f);
    orc_hist_calculate(nb, start ? 1.0f : L->region->learning_rate_b, mb.data(), L->histogram_b);
  }
  return true;
}

void orc_start_modalities(orc_body* bodies, int n_bodies, int iteration, int rotation_mode, int n_threads) {
  if (SharedHistogramPass(bodies, n_bodies, iteration, rotation_mode, true)) return;
#pragma omp parallel for schedule(dynamic) num_threads(n_threads > 0 ? n_threads : 1)
  for (int i = 0; i < n_bodies; ++i) StartOne(&bodies[i], iteration, rotation_mode);
}

static void ResultsOne(orc_body* b, int iteration, int rotation_mode) {
  // RegionModality::CalculateResults (region_modality.cpp:572-583)
  if (!b->region) return;
  int nb = b->region->n_histogram_bins;
  size_t n = size_t(nb) * nb * nb;
  std::vector<float> mf(n, 0.0f), mb(n, 0.0f);
  orc_region_add_line_pixels_occ(b->region, b->region_model, b->color, b->region_occlusion_frame,
                                 (iteration - b->first_iteration) >= b->region->n_unoccluded_iterations, b->body2world,
                                 rotation_mode, mf.data(), mb.data());
  orc_hist_calculate(nb, b->region->learning_rate_f, mf.data(), b->histogram_f);  // UpdateHistograms (:83-92)
  orc_hist_calculate(nb, b->region->learning_rate_b, mb.data(), b->histogram_b);
}

void orc_calculate_results(orc_body* bodies, int n_bodies, int iteration, int rotation_mode, int n_threads) {
  if (SharedHistogramPass(bodies, n_bodies, iteration, rotation_mode, false)) return;
#pragma omp parallel for schedule(dynamic) num_threads(n_threads > 0 ? n_threads : 1)
  for (int i = 0; i < n_bodies; ++i) ResultsOne(&bodies[i], iteration, rotation_mode);
}

// Tracker::ExecuteTrackingStep (tracker.cpp:344-361) for one body (= one optimizer with a root link).
static void StepOne(orc_body* b, int iteration, int corr_begin, int corr_end, int n_update, int rotation_mode,
                    int exp_mode, double* phase) {
  for (int corr = corr_begin; corr < corr_end; ++corr) {
    double t0 = Now();
    if (b->region)
      b->n_lines = orc_region_correspondences(b->region, b->region_model, b->color, b->region_occlusion_frame,
                                              b->histogram_f, b->histogram_b, b->body2world, iteration,
                                              b->first_iteration, corr, rotation_mode, b->lines, &b->region_view);
    if (b->depth)
      b->n_points = orc_depth_correspondences(b->depth, b->depth_model, b->depth_frame, b->body2world, iteration,
                                              b->first_iteration, corr, rotation_mode, b->points, &b->depth_view);
    double t1 = Now();
    phase[0] += t1 - t0;
    for (int upd = 0; upd < n_update; ++upd) {
      double t2 = Now();
      float g[6] = {0, 0, 0, 0, 0, 0}, H[36], gr[6], Hr[36], gd[6], Hd[36];
      for (int i = 0; i < 36; ++i) H[i] = 0.0f;
      // Link::CalculateGradientAndHessian (link.cpp:184-193): region first, then depth
      if (b->region) {
        orc_region_gradient_hessian(b->region, b->color, b->body2world, b->lines, b->n_lines, corr, upd,
                                    rotation_mode, gr, Hr);
        for (int i = 0; i < 6; ++i) g[i] += gr[i];
        for (int i = 0; i < 36; ++i) H[i] += Hr[i];
      }
      if (b->depth) {
        orc_depth_gradient_hessian(b->depth, b->depth_frame, b->body2world, b->points, b->n_points, corr, gd, Hd);
        for (int i = 0; i < 6; ++i) g[i] += gd[i];
        for (int i = 0; i < 36; ++i) H[i] += Hd[i];
      }
      double t3 = Now();
      phase[1] += t3 - t2;
      orc_optimize_rigid(g, H, b->tikhonov_rotation, b->tikhonov_translation, exp_mode, b->body2world, nullptr);
      phase[2] += Now() - t3;
    }
  }
}

void orc_tracking_step(orc_body* bodies, int n_bodies, int iteration, int corr_begin, int corr_end, int n_update,
                       int rotation_mode, int exp_mode, int n_threads, double* phase_seconds) {
  double p0 = 0, p1 = 0, p2 = 0;
#pragma omp parallel for schedule(dynamic) num_threads(n_threads > 0 ? n_threads : 1) reduction(+ : p0, p1, p2)
  for (int i = 0; i < n_bodies; ++i) {
    double phase[3] = {0, 0, 0};
    StepOne(&bodies[i], iteration, corr_begin, corr_end, n_update, rotation_mode, exp_mode, phase);
    p0 += phase[0]; p1 += phase[1]; p2 += phase[2];
  }
  if (phase_seconds) {
    phase_seconds[0] += p0; phase_seconds[1] += p1; phase_seconds[2] += p2;
  }
}

}  // extern "C"

// =============================================================================================
// Kinematic structures (SURVEY §8 a13-a16): Link tree, Constraint, SoftConstraint, Optimizer over DoF + nc unknowns.
// The reference has no known answers for this part (parity unpinned, see the header); float summation order of the
// small Eigen products is taken as left-to-right.
// =============================================================================================
namespace {

constexpr int kMaxDof = 96;  // 16 links x 6

inline void Skew3(const float* v, float* m /*3x3 row-major*/) {  // Vector2Skewsymmetric (common.h:62-71)
  m[0] = 0.0f; m[1] = -v[2]; m[2] = v[1];
  m[3] = v[2]; m[4] = 0.0f; m[5] = -v[0];
  m[6] = -v[1]; m[7] = v[0]; m[8] = 0.0f;
}
inline void Mul3(const float* a, const float* b, float* o) {
  float r[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r[3 * i + j] = a[3 * i] * b[j] + a[3 * i + 1] * b[3 + j] + a[3 * i + 2] * b[6 + j];
  std::memcpy(o, r, sizeof(r));
}

// Link::Adjoint (link.cpp:341-348): [[R, 0], [skew(t) R, R]], row-major 6x6
void Adjoint(const float* pose, int rotation_mode, float* m) {
  float r[9], s[9], sr[9];
  PoseRotation(pose, rotation_mode, r);
  float t[3] = {T_(pose, 0), T_(pose, 1), T_(pose, 2)};
  Skew3(t, s);
  Mul3(s, r, sr);
  for (int k = 0; k < 36; ++k) m[k] = 0.0f;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      m[6 * i + j] = r[3 * i + j];
      m[6 * (i + 3) + j] = sr[3 * i + j];
      m[6 * (i + 3) + j + 3] = r[3 * i + j];
    }
}

int LinkDof(const orc_link& l) {
  int n = 0;
  for (int d = 0; d < 6; ++d) n += l.free_directions[d] ? 1 : 0;
  return n;
}
int FirstIndex(const orc_structure* s, int link) {
  int n = 0;
  for (int i = 0; i < link; ++i) n += LinkDof(s->links[i]);
  return n;
}
int NRows(const int32_t* directions) {
  int n = 0;
  for (int d = 0; d < 6; ++d) n += directions[d] ? 1 : 0;
  return n;
}

// Eigen::Quaternionf(Matrix3f) (quaternionbase_assign_impl<..,3,3>) followed by AngleAxisf = Quaternionf.
void AngleAxisFromMatrix(const float* m /*row-major 3x3*/, float* angle, float* axis) {
  auto M = [&](int i, int j) { return m[3 * i + j]; };
  float q[4];  // x, y, z, w
  float t = M(0, 0) + M(1, 1) + M(2, 2);
  if (t > 0.0f) {
    t = std::sqrt(t + 1.0f);
    q[3] = 0.5f * t;
    t = 0.5f / t;
    q[0] = (M(2, 1) - M(1, 2)) * t;
    q[1] = (M(0, 2) - M(2, 0)) * t;
    q[2] = (M(1, 0) - M(0, 1)) * t;
  } else {
    int i = 0;
    if (M(1, 1) > M(0, 0)) i = 1;
    if (M(2, 2) > M(i, i)) i = 2;
    int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(M(i, i) - M(j, j) - M(k, k) + 1.0f);
    q[i] = 0.5f * t;
    t = 0.5f / t;
    q[3] = (M(k, j) - M(j, k)) * t;
    q[j] = (M(j, i) + M(i, j)) * t;
    q[k] = (M(k, i) + M(i, k)) * t;
  }
  float n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
  if (n < std::numeric_limits<float>::epsilon()) {  // stableNorm(): scaled to avoid underflow
    double sx = q[0], sy = q[1], sz = q[2];
    n = float(std::sqrt(sx * sx + sy * sy + sz * sz));
  }
  if (n != 0.0f) {
    *angle = 2.0f * std::atan2(n, std::fabs(q[3]));
    if (q[3] < 0.0f) n = -n;
    axis[0] = q[0] / n; axis[1] = q[1] / n; axis[2] = q[2] / n;
  } else {
    *angle = 0.0f;
    axis[0] = 1.0f; axis[1] = 0.0f; axis[2] = 0.0f;
  }
}

float Xcotx(float x) {  // common.h:73-77
  if (std::tan(x) <= std::numeric_limits<float>::min()) return 1.0f;
  if (std::tan(x) >= std::numeric_limits<float>::max()) return 0.0f;
  return float(double(x) / std::tan(double(x)));
}

struct JointGeometry {
  float body22joint1[12], joint22joint1[12];
  float angle, axis[3];
  float rotation_vector[3], translation_vector[3];
};

// the "required poses" block shared by Constraint (constraint.cpp:88-92) and SoftConstraint (soft_constraint.cpp:120-124)
void CalcJointGeometry(const float* body12joint1, const float* body22joint2, const float* link1_2world,
                       const float* link2_2world, int rotation_mode, JointGeometry* jg) {
  float inv1[12], tmp[12], inv22[12], rot[9];
  PoseInverse(link1_2world, inv1);
  PoseMul(body12joint1, inv1, tmp);
  PoseMul(tmp, link2_2world, jg->body22joint1);
  PoseInverse(body22joint2, inv22);
  PoseMul(jg->body22joint1, inv22, jg->joint22joint1);
  PoseRotation(jg->joint22joint1, rotation_mode, rot);
  AngleAxisFromMatrix(rot, &jg->angle, jg->axis);
  for (int i = 0; i < 3; ++i) {
    jg->rotation_vector[i] = jg->angle * jg->axis[i];
    jg->translation_vector[i] = T_(jg->joint22joint1, i);
  }
}

// Constraint::UnprojectedConstraintJacobian (constraint.cpp:205-274) for the selected directions: rows[nr][6]
int UnprojectedJacobian(const JointGeometry& jg, const float* body2joint1, const int32_t* directions, int rotation_mode,
                        bool rotation_rows, bool translation_rows, float* rows) {
  float inv_j[12], body2joint2[12], inv_b[12], r1[9];
  PoseInverse(jg.joint22joint1, inv_j);
  PoseMul(inv_j, body2joint1, body2joint2);
  PoseInverse(body2joint2, inv_b);
  float jt[3] = {T_(inv_b, 0), T_(inv_b, 1), T_(inv_b, 2)};  // joint22body_translation
  PoseRotation(body2joint1, rotation_mode, r1);
  float angle_half = 0.5f * jg.angle;
  float xc = Xcotx(angle_half);
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
      for (int j = 0; j < 3; ++j)
        row[j] = var[3 * d] * r1[j] + var[3 * d + 1] * r1[3 + j] + var[3 * d + 2] * r1[6 + j];
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

void StructureJacobians(const orc_structure* s, int rotation_mode, int dof, float* jac /*[n_links][6][dof]*/) {
  int first = 0;
  for (int l = 0; l < s->n_links; ++l) {
    const orc_link& link = s->links[l];
    float* J = jac + size_t(l) * 6 * dof;
    if (link.parent >= 0) {
      float prod[12], parent2body[12], ad[36];
      PoseMul(link.joint2parent, link.body2joint, prod);
      PoseInverse(prod, parent2body);
      Adjoint(parent2body, rotation_mode, ad);
      const float* Jp = jac + size_t(link.parent) * 6 * dof;
      for (int i = 0; i < 6; ++i)
        for (int c = 0; c < dof; ++c) {
          float acc = 0.0f;
          for (int k = 0; k < 6; ++k) acc += ad[6 * i + k] * Jp[size_t(k) * dof + c];
          J[size_t(i) * dof + c] = acc;
        }
    } else {
      for (int k = 0; k < 6 * dof; ++k) J[k] = 0.0f;
    }
    float joint2body[12], adj[36];
    PoseInverse(link.body2joint, joint2body);
    Adjoint(joint2body, rotation_mode, adj);
    int idx = first;
    for (int d = 0; d < 6; ++d)
      if (link.free_directions[d]) {
        for (int i = 0; i < 6; ++i) J[size_t(i) * dof + idx] = adj[6 * i + d];
        idx++;
      }
    first = idx;
  }
}

// Link::UpdatePoses for every link in pre-order (optimizer.cpp:334-346, link.cpp:205-241)
void StructureUpdatePoses(orc_structure* s, const float* theta, int exp_mode, float* link2world) {
  int idx = 0;
  for (int l = 0; l < s->n_links; ++l) {
    orc_link& link = s->links[l];
    float th[6];
    for (int d = 0; d < 6; ++d) th[d] = link.free_directions[d] ? theta[idx++] : 0.0f;
    float e[9];
    ExpSkew(th, exp_mode, e);
    float var[12] = {e[0], e[1], e[2], th[3], e[3], e[4], e[5], th[4], e[6], e[7], e[8], th[5]};
    float* l2w = link2world + 12 * l;
    float tmp[12], tmp2[12];
    if (link.parent >= 0) {
      if (link.fixed_body2joint_pose) {
        PoseMul(link.joint2parent, var, tmp);
        std::memcpy(link.joint2parent, tmp, sizeof(tmp));
      } else {
        PoseMul(var, link.body2joint, tmp);
        std::memcpy(link.body2joint, tmp, sizeof(tmp));
      }
      PoseMul(link2world + 12 * link.parent, link.joint2parent, tmp);
      PoseMul(tmp, link.body2joint, l2w);
    } else {
      float inv[12];
      PoseInverse(link.body2joint, inv);
      PoseMul(l2w, inv, tmp);
      PoseMul(tmp, var, tmp2);
      PoseMul(tmp2, link.body2joint, l2w);
    }
  }
}

}  // namespace

extern "C" {

int orc_structure_dof(const orc_structure* s) { return FirstIndex(s, s->n_links); }
int orc_structure_n_constraint_rows(const orc_structure* s) {
  int n = 0;
  for (int c = 0; c < s->n_constraints; ++c) n += NRows(s->constraints[c].directions);
  return n;
}
void orc_angle_axis(const float r[9], float* angle, float axis[3]) { AngleAxisFromMatrix(r, angle, axis); }
float orc_xcotx(float x) { return Xcotx(x); }

void orc_structure_jacobians(const orc_structure* s, int rotation_mode, float* jacobians) {
  StructureJacobians(s, rotation_mode, orc_structure_dof(s), jacobians);
}

int orc_constraint_residual_jacobian(const orc_structure* s, int constraint, const float* link2world,
                                     const float* jacobians, int rotation_mode, float* residual, float* jacobian) {
  const orc_constraint& c = s->constraints[constraint];
  const int dof = orc_structure_dof(s);
  JointGeometry jg;
  CalcJointGeometry(c.body12joint1, c.body22joint2, link2world + 12 * c.link1, link2world + 12 * c.link2, rotation_mode, &jg);
  int idx = 0;
  for (int d = 0; d < 6; ++d)  // Constraint::Residual (constraint.cpp:176-203)
    if (c.directions[d]) residual[idx++] = d < 3 ? jg.rotation_vector[d] : jg.translation_vector[d - 3];
  float u2[36], u1[36];
  const int nr = UnprojectedJacobian(jg, jg.body22joint1, c.directions, rotation_mode, true, true, u2);
  UnprojectedJacobian(jg, c.body12joint1, c.directions, rotation_mode, true, true, u1);
  const float* J2 = jacobians + size_t(c.link2) * 6 * dof;
  const float* J1 = jacobians + size_t(c.link1) * 6 * dof;
  for (int r = 0; r < nr; ++r)
    for (int col = 0; col < dof; ++col) {
      float a2 = 0.0f, a1 = 0.0f;
      for (int k = 0; k < 6; ++k) a2 += u2[6 * r + k] * J2[size_t(k) * dof + col];
      for (int k = 0; k < 6; ++k) a1 += u1[6 * r + k] * J1[size_t(k) * dof + col];
      jacobian[size_t(r) * dof + col] = a2 - a1;
    }
  return nr;
}

// SoftConstraint::AddGradientsAndHessiansToLink (soft_constraint.cpp:220-270)
static void SoftAddToLink(const orc_soft_constraint& c, const JointGeometry& jg, const float* body2joint1, float sign,
                          int rotation_mode, float* g, float* H) {
  float grad[6] = {0, 0, 0, 0, 0, 0}, hess[36];
  for (int k = 0; k < 36; ++k) hess[k] = 0.0f;
  for (int part = 0; part < 2; ++part) {
    const int32_t* dirs = c.directions;
    int n = 0;
    float vec[3];
    for (int d = 0; d < 3; ++d)
      if (dirs[d + 3 * part]) vec[n++] = part == 0 ? jg.rotation_vector[d] : jg.translation_vector[d];
    if (!n) continue;
    const float max_d = part == 0 ? c.max_distance_rotation : c.max_distance_translation;
    const float sd = part == 0 ? c.standard_deviation_rotation : c.standard_deviation_translation;
    float sq = 0.0f;
    for (int i = 0; i < n; ++i) sq += vec[i] * vec[i];
    const float dist = std::sqrt(sq);
    if (!(dist > max_d)) continue;
    float rows[18];
    UnprojectedJacobian(jg, body2joint1, dirs, rotation_mode, part == 0, part == 1, rows);
    float unit[3] = {0, 0, 0};
    for (int i = 0; i < n; ++i) unit[i] = vec[i];
    if (sq > 0.0f)
      for (int i = 0; i < n; ++i) unit[i] = vec[i] / dist;
    const float inv_var = 1.0f / (sd * sd);
    // gradient -= (sign / sd^2) * J^T * (vec - unit * max_d)
    float e[3];
    for (int i = 0; i < n; ++i) e[i] = vec[i] - unit[i] * max_d;
    for (int k = 0; k < 6; ++k) {
      float acc = 0.0f;
      for (int i = 0; i < n; ++i) acc += rows[6 * i + k] * e[i];
      grad[k] -= (sign * inv_var) * acc;
    }
    // hessian -= (1 / sd^2) * J^T * (I - (max_d / dist) * (I - unit unit^T)) * J
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
        hess[6 * a + b] -= inv_var * acc;
      }
  }
  for (int k = 0; k < 6; ++k) g[k] += grad[k];      // Link::AddToGradientAndHessian (link.cpp:195-203)
  for (int k = 0; k < 36; ++k) H[k] += hess[k];
}

void orc_soft_constraint_add(const orc_structure* s, int soft_constraint, const float* link2world, int rotation_mode,
                             float* g, float* H) {
  const orc_soft_constraint& c = s->soft_constraints[soft_constraint];
  JointGeometry jg;
  CalcJointGeometry(c.body12joint1, c.body22joint2, link2world + 12 * c.link1, link2world + 12 * c.link2, rotation_mode, &jg);
  SoftAddToLink(c, jg, c.body12joint1, -1.0f, rotation_mode, g + 6 * c.link1, H + 36 * c.link1);
  SoftAddToLink(c, jg, jg.body22joint1, 1.0f, rotation_mode, g + 6 * c.link2, H + 36 * c.link2);
}

int orc_optimize_structure(orc_structure* s, const float* g_in, const float* H_in, int rotation_mode, int exp_mode,
                           float* link2world, float* theta_out) {
  const int dof = orc_structure_dof(s);
  const int nc = orc_structure_n_constraint_rows(s);
  const int n = dof + nc;
  if (dof > kMaxDof || n > kMaxN || n < 1) return -1;
  const int nl = s->n_links;
  std::vector<float> jac(size_t(nl) * 6 * dof), g(g_in, g_in + size_t(nl) * 6), H(H_in, H_in + size_t(nl) * 36);
  // CalculateDataLinks (optimizer.cpp:283-299): Jacobians + modality sums (given), then the soft constraints
  StructureJacobians(s, rotation_mode, dof, jac.data());
  for (int c = 0; c < s->n_soft_constraints; ++c) orc_soft_constraint_add(s, c, link2world, rotation_mode, g.data(), H.data());
  std::vector<float> a(size_t(n) * n, 0.0f), b(n, 0.0f), theta(n, 0.0f);
  // AddProjectedGradientsAndHessians (optimizer.cpp:308-320)
  for (int l = 0; l < nl; ++l) {
    const float* J = jac.data() + size_t(l) * 6 * dof;
    const float* gl = g.data() + 6 * l;
    const float* Hl = H.data() + 36 * l;
    for (int i = 0; i < dof; ++i) {
      float acc = 0.0f;
      for (int k = 0; k < 6; ++k) acc += J[size_t(k) * dof + i] * gl[k];
      b[i] += acc;
      float jh[6];
      for (int q = 0; q < 6; ++q) {
        float t = 0.0f;
        for (int k = 0; k < 6; ++k) t += J[size_t(k) * dof + i] * Hl[6 * k + q];
        jh[q] = t;
      }
      for (int j = 0; j <= i; ++j) {
        float t = 0.0f;
        for (int q = 0; q < 6; ++q) t += jh[q] * J[size_t(q) * dof + j];
        a[size_t(i) * n + j] -= t;
      }
    }
  }
  // AddResidualsAndConstraintJacobians (optimizer.cpp:322-332)
  int idx = dof;
  std::vector<float> res(6), cj(size_t(6) * std::max(dof, 1));
  for (int c = 0; c < s->n_constraints; ++c) {
    const int nr = orc_constraint_residual_jacobian(s, c, link2world, jac.data(), rotation_mode, res.data(), cj.data());
    for (int r = 0; r < nr; ++r) {
      b[idx + r] = res[r];
      for (int col = 0; col < dof; ++col) a[size_t(idx + r) * n + col] = -cj[size_t(r) * dof + col];
    }
    idx += nr;
  }
  // tikhonov_vector_ (optimizer.cpp:236-252)
  int di = 0;
  for (int l = 0; l < nl; ++l)
    for (int d = 0; d < 6; ++d)
      if (s->links[l].free_directions[d]) {
        a[size_t(di) * n + di] += d < 3 ? s->tikhonov_rotation : s->tikhonov_translation;
        di++;
      }
  LdltSolve(n, a.data(), b.data(), theta.data());
  if (theta_out) std::memcpy(theta_out, theta.data(), sizeof(float) * n);
  for (int i = 0; i < n; ++i)
    if (std::isnan(theta[i])) return 0;  // optimizer.cpp:165
  StructureUpdatePoses(s, theta.data(), exp_mode, link2world);
  return 1;
}

void orc_structure_consistent_poses(orc_structure* s, int exp_mode, float* link2world) {
  std::vector<float> theta(size_t(std::max(1, orc_structure_dof(s))), 0.0f);
  StructureUpdatePoses(s, theta.data(), exp_mode, link2world);
}

void orc_tracking_step_structures(orc_body* bodies, orc_structure* structures, int n_structures, int iteration,
                                  int corr_begin, int corr_end, int n_update, int rotation_mode, int exp_mode,
                                  int n_threads, float* bodyless_link2world, int max_links) {
#pragma omp parallel for schedule(dynamic) num_threads(n_threads > 0 ? n_threads : 1)
  for (int si = 0; si < n_structures; ++si) {
    orc_structure* s = &structures[si];
    const int nl = s->n_links;
    std::vector<float> l2w(size_t(nl) * 12), g(size_t(nl) * 6), H(size_t(nl) * 36);
    auto gather = [&]() {
      for (int l = 0; l < nl; ++l) {
        const int bi = s->links[l].body;
        const float* src = bi >= 0 ? bodies[bi].body2world : bodyless_link2world + (size_t(si) * max_links + l) * 12;
        std::memcpy(&l2w[12 * l], src, 12 * sizeof(float));
      }
    };
    auto scatter = [&]() {
      for (int l = 0; l < nl; ++l) {
        const int bi = s->links[l].body;
        float* dst = bi >= 0 ? bodies[bi].body2world : bodyless_link2world + (size_t(si) * max_links + l) * 12;
        std::memcpy(dst, &l2w[12 * l], 12 * sizeof(float));
        for (int x = 0; x < s->links[l].n_extra_bodies; ++x)  // one physical body, several modality sets
          std::memcpy(bodies[s->links[l].extra_bodies[x]].body2world, &l2w[12 * l], 12 * sizeof(float));
      }
    };
    // the modality sets of link l: its body, then the extra bodies (Link::modality_ptrs() order)
    auto n_sets = [&](int l) { return s->links[l].body < 0 ? 0 : 1 + s->links[l].n_extra_bodies; };
    auto set_body = [&](int l, int k) { return k == 0 ? s->links[l].body : s->links[l].extra_bodies[k - 1]; };
    for (int corr = corr_begin; corr < corr_end; ++corr) {
      for (int l = 0; l < nl; ++l)
        for (int k = 0; k < n_sets(l); ++k) {
          orc_body* b = &bodies[set_body(l, k)];
          if (b->region)
            b->n_lines = orc_region_correspondences(b->region, b->region_model, b->color, b->region_occlusion_frame,
                                                    b->histogram_f, b->histogram_b, b->body2world, iteration,
                                                    b->first_iteration, corr, rotation_mode, b->lines, &b->region_view);
          if (b->depth)
            b->n_points = orc_depth_correspondences(b->depth, b->depth_model, b->depth_frame, b->body2world, iteration,
                                                    b->first_iteration, corr, rotation_mode, b->points, &b->depth_view);
        }
      for (int upd = 0; upd < n_update; ++upd) {
        std::fill(g.begin(), g.end(), 0.0f);
        std::fill(H.begin(), H.end(), 0.0f);
        for (int l = 0; l < nl; ++l)
          for (int k = 0; k < n_sets(l); ++k) {
          orc_body* b = &bodies[set_body(l, k)];
          float gm[6], Hm[36];
          if (b->region) {
            orc_region_gradient_hessian(b->region, b->color, b->body2world, b->lines, b->n_lines, corr, upd,
                                        rotation_mode, gm, Hm);
            for (int i = 0; i < 6; ++i) g[6 * l + i] += gm[i];
            for (int i = 0; i < 36; ++i) H[36 * l + i] += Hm[i];
          }
          if (b->depth) {
            orc_depth_gradient_hessian(b->depth, b->depth_frame, b->body2world, b->points, b->n_points, corr, gm, Hm);
            for (int i = 0; i < 6; ++i) g[6 * l + i] += gm[i];
            for (int i = 0; i < 36; ++i) H[36 * l + i] += Hm[i];
          }
        }
        gather();
        orc_optimize_structure(s, g.data(), H.data(), rotation_mode, exp_mode, l2w.data(), nullptr);
        scatter();
      }
    }
  }
}

}  // extern "C"
