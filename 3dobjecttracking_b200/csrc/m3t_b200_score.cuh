// m3t_b200_score.cuh — pose scoring against ground truth: the evaluators' CalculatePoseResults (ycb_evaluator.cpp:803-848,
// rtb_evaluator.cpp:930-989, opt_evaluator.cpp:462-488, rbot_evaluator.cpp:416-433) and OPTEvaluator::CalculateDiameters
// (opt_evaluator.cpp:580-599). DESIGN.md §3 "k_score / k_score_finish / k_diameter" states what is computed.
// The kernels are defined here and compiled in m3t_b200.cu's translation unit: a further .cu file would lengthen the
// cubin name cuobjdump -xelf gives the library's one device image (all unit names joined) past 255 bytes.
// Every float operation is written as one rounding (_rn intrinsics), in the order the reference's Eigen / nanoflann
// expressions evaluate it.
#pragma once

#include <cuda_runtime.h>

#include <cfloat>
#include <cmath>

#include "m3t_b200.h"
#include "m3t_b200_device.cuh"

namespace m3tb {

constexpr int kScoreThreads = 128;
constexpr int kScoreVerts = 4;      // evaluation vertices per thread of k_score / rows per thread of k_diameter
constexpr int kScoreTile = 1024;    // full-set vertices staged in shared memory at a time
constexpr int kScoreBlock = kScoreThreads * kScoreVerts;

// One evaluation model: the full vertex set (the nearest-neighbour search set) and the reduced set
// (GenderateReducedVertices), both as (x, y, z, 0).
struct EvalModelDev {
  const float4* full;
  const float4* reduced;
  int n_full, n_reduced;
};

// Per body: its evaluation model (-1: none) and the OPT evaluator's geometry2body term (kBody2Geometry2BodyPoseMap).
struct EvalBodyDev {
  int model;
  int has_geometry2body;
  float geometry2body[12];
};

struct ScoreArgs {
  const EvalModelDev* models;
  const EvalBodyDev* eval_bodies;
  const float* poses;        // the context's body2world poses [max_bodies][12]
  const int* bodies;         // [n]
  const float* gt;           // [n][12] ground-truth body2world
  int n;
  int n_chunks, chunk;       // the full set is searched in n_chunks slices of `chunk` vertices (a multiple of kScoreTile)
  int max_reduced;           // row length of `partial`
  float* partial;            // [n][n_chunks][max_reduced] squared-distance minimum of each slice
  float threshold_max, curve_scale, auc_scale, translation_threshold, rotation_threshold;
  m3tb_pose_score* out;      // [n]
  float* add_curve;          // [n][M3TB_N_CURVE_VALUES]
  float* adds_curve;
};

struct DiameterArgs {
  const EvalModelDev* models;
  const int* model_ids;      // [n]
  int n_chunks, chunk;
  unsigned* max_sq;          // [n] bits of the largest squared distance, zeroed before the launch
};
namespace score {

// delta_pose of the evaluators: body2world.inverse() * gt (YCB / RTB, whose world2body_pose() is the same inverse), or
// (body2world * geometry2body).inverse() * gt * geometry2body (OPT)
__device__ void DeltaPose(const ScoreArgs& a, int q, float* delta) {
  const int b = a.bodies[q];
  const EvalBodyDev& e = a.eval_bodies[b];
  const float* pose = a.poses + 12 * size_t(b);
  const float* gt = a.gt + 12 * size_t(q);
  float inv[12];
  if (e.has_geometry2body) {
    float p[12], t[12];
    PoseMul(pose, e.geometry2body, p);
    PoseInverse(p, inv);
    PoseMul(inv, gt, t);
    PoseMul(t, e.geometry2body, delta);
  } else {
    PoseInverse(pose, inv);
    PoseMul(inv, gt, delta);
  }
}

// Transform3fA * Vector3f
__device__ __forceinline__ float3 Apply(const float* p, float4 v) {
  return make_float3(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p[0], v.x), __fmul_rn(p[1], v.y)), __fmul_rn(p[2], v.z)), p[3]),
                     __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p[4], v.x), __fmul_rn(p[5], v.y)), __fmul_rn(p[6], v.z)), p[7]),
                     __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p[8], v.x), __fmul_rn(p[9], v.y)), __fmul_rn(p[10], v.z)), p[11]));
}

// ((dx² + dy²) + dz²): Eigen's squaredNorm and nanoflann's L2 adaptor ((0 + dx²) + ..., the 0 + exact) alike
__device__ __forceinline__ float SquaredDistance(float x, float y, float z, float4 w) {
  const float dx = __fsub_rn(x, w.x), dy = __fsub_rn(y, w.y), dz = __fsub_rn(z, w.z);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// Transform3fA::rotation(): the polar factor of the linear block, Newton's iteration X <- (X + X^-T) / 2 in double,
// rounded once to float (the restatement the oracle's PoseRotation uses)
__device__ void PolarRotation(const float* p, float* r) {
  double x[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) x[3 * i + j] = double(p[4 * i + j]);
  for (int it = 0; it < 12; ++it) {
    double c[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        c[3 * i + j] = __dsub_rn(__dmul_rn(x[3 * i1 + j1], x[3 * i2 + j2]), __dmul_rn(x[3 * i1 + j2], x[3 * i2 + j1]));
      }
    const double det = __dadd_rn(__dadd_rn(__dmul_rn(c[0], x[0]), __dmul_rn(c[1], x[1])), __dmul_rn(c[2], x[2]));
    double delta = 0.0;
    for (int k = 0; k < 9; ++k) {
      const double nx = __dmul_rn(0.5, __dadd_rn(x[k], __ddiv_rn(c[k], det)));
      const double d = fabs(__dsub_rn(nx, x[k]));
      delta = delta < d ? d : delta;  // std::max
      x[k] = nx;
    }
    if (delta < 1e-15) break;
  }
  for (int k = 0; k < 9; ++k) r[k] = __double2float_rn(x[k]);
}

}  // namespace score

// grid (n, n_chunks, ceil(max_reduced / kScoreBlock)), kScoreThreads threads: the squared distance from every moved
// evaluation vertex to its nearest full-set vertex within one slice.
__global__ void __launch_bounds__(kScoreThreads) k_score(const __grid_constant__ ScoreArgs a) {
  __shared__ float4 tile[kScoreTile];
  const int q = blockIdx.x;
  const EvalModelDev m = a.models[a.eval_bodies[a.bodies[q]].model];
  const int first = blockIdx.z * kScoreBlock;
  if (first >= m.n_reduced) return;  // uniform over the block
  float delta[12];
  score::DeltaPose(a, q, delta);
  float x[kScoreVerts], y[kScoreVerts], z[kScoreVerts], best[kScoreVerts];
#pragma unroll
  for (int v = 0; v < kScoreVerts; ++v) {
    const int i = first + threadIdx.x + v * kScoreThreads;
    const float3 p = score::Apply(delta, m.reduced[min(i, m.n_reduced - 1)]);
    x[v] = p.x;
    y[v] = p.y;
    z[v] = p.z;
    best[v] = FLT_MAX;  // KNNResultSet::init: the worst distance starts at numeric_limits<float>::max()
  }
  const int j0 = blockIdx.y * a.chunk, j1 = min(j0 + a.chunk, m.n_full);
  for (int t0 = j0; t0 < j1; t0 += kScoreTile) {
    const int nt = min(kScoreTile, j1 - t0);
    __syncthreads();
    for (int k = threadIdx.x; k < nt; k += kScoreThreads) tile[k] = m.full[t0 + k];
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < nt; ++k) {
      const float4 w = tile[k];
#pragma unroll
      for (int v = 0; v < kScoreVerts; ++v) {
        const float d = score::SquaredDistance(x[v], y[v], z[v], w);
        // searchLevel adds a point only when dist < worst_dist: a NaN or infinite distance (a NaN or infinite pose) is
        // never taken, and such a query keeps FLT_MAX
        best[v] = d < best[v] ? d : best[v];
      }
    }
  }
  float* row = a.partial + (size_t(q) * a.n_chunks + blockIdx.y) * a.max_reduced;
#pragma unroll
  for (int v = 0; v < kScoreVerts; ++v) {
    const int i = first + threadIdx.x + v * kScoreThreads;
    if (i < m.n_reduced) row[i] = best[v];
  }
}

// grid n, kScoreThreads threads: the slices merged, both sums in vertex order, curves, AUCs and the RBOT errors.
__global__ void __launch_bounds__(kScoreThreads) k_score_finish(const __grid_constant__ ScoreArgs a) {
  __shared__ float s_add[kScoreThreads], s_adds[kScoreThreads];
  __shared__ float s_error[2];
  const int q = blockIdx.x;
  const EvalModelDev m = a.models[a.eval_bodies[a.bodies[q]].model];
  float delta[12];
  score::DeltaPose(a, q, delta);
  const float* partial = a.partial + size_t(q) * a.n_chunks * a.max_reduced;
  float add = 0.0f, adds = 0.0f;  // thread 0: the two sums, in vertex order
  for (int base = 0; base < m.n_reduced; base += kScoreThreads) {
    const int i = base + threadIdx.x;
    if (i < m.n_reduced) {
      const float4 v = m.reduced[i];
      const float3 p = score::Apply(delta, v);
      const float dx = __fsub_rn(v.x, p.x), dy = __fsub_rn(v.y, p.y), dz = __fsub_rn(v.z, p.z);
      s_add[threadIdx.x] = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
      float d = partial[i];  // every slice holds FLT_MAX or a smaller, non-NaN distance
      for (int c = 1; c < a.n_chunks; ++c) {
        const float e = partial[size_t(c) * a.max_reduced + i];
        d = e < d ? e : d;
      }
      s_adds[threadIdx.x] = __fsqrt_rn(d);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const int nk = min(kScoreThreads, m.n_reduced - base);
      for (int k = 0; k < nk; ++k) {
        add = __fadd_rn(add, s_add[k]);
        adds = __fadd_rn(adds, s_adds[k]);
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float size = float(m.n_reduced);
    add = __fdiv_rn(add, size);
    adds = __fdiv_rn(adds, size);
    s_error[0] = add;
    s_error[1] = adds;
    const float scaled_max = __fmul_rn(a.curve_scale, a.threshold_max);
    m3tb_pose_score s;
    s.add_error = add;
    s.adds_error = adds;
    // 1 - std::min(error / threshold, 1.0f): std::min(NaN, 1.0f) is NaN
    const float ra = __fdiv_rn(add, scaled_max), rs = __fdiv_rn(adds, scaled_max);
    s.add_auc = __fmul_rn(a.auc_scale, __fsub_rn(1.0f, 1.0f < ra ? 1.0f : ra));
    s.adds_auc = __fmul_rn(a.auc_scale, __fsub_rn(1.0f, 1.0f < rs ? 1.0f : rs));
    // RBOTEvaluator::CalculatePoseResults
    const int b = a.bodies[q];
    const float* pose = a.poses + 12 * size_t(b);
    const float* gt = a.gt + 12 * size_t(q);
    const float tx = __fsub_rn(pose[3], gt[3]), ty = __fsub_rn(pose[7], gt[7]), tz = __fsub_rn(pose[11], gt[11]);
    s.translation_error = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(tx, tx), __fmul_rn(ty, ty)), __fmul_rn(tz, tz)));
    float r[9], rg[9];
    score::PolarRotation(pose, r);
    score::PolarRotation(gt, rg);
    float trace = 0.0f;
    for (int i = 0; i < 3; ++i) {
      const float d = __fadd_rn(__fadd_rn(__fmul_rn(r[i], rg[i]), __fmul_rn(r[3 + i], rg[3 + i])), __fmul_rn(r[6 + i], rg[6 + i]));
      trace = i == 0 ? d : __fadd_rn(trace, d);
    }
    s.rotation_error = acosf(__fdiv_rn(__fsub_rn(trace, 1.0f), 2.0f));
    // a NaN error is not above its threshold: the frame counts as a success
    s.tracking_success = (s.translation_error > a.translation_threshold || s.rotation_error > a.rotation_threshold) ? 0.0f : 1.0f;
    a.out[q] = s;
  }
  __syncthreads();
  if (a.add_curve && threadIdx.x < M3TB_N_CURVE_VALUES) {
    // std::fill(1), then zero every value before the first threshold the error falls below
    const float step = __fdiv_rn(a.threshold_max, float(M3TB_N_CURVE_VALUES));
    float c_add = 0.0f, c_adds = 0.0f;
    for (int k = 0; k <= int(threadIdx.x); ++k) {
      const float th = __fmul_rn(a.curve_scale, __fmul_rn(step, __fadd_rn(0.5f, float(k))));
      if (s_error[0] < th) c_add = 1.0f;
      if (s_error[1] < th) c_adds = 1.0f;
    }
    a.add_curve[size_t(q) * M3TB_N_CURVE_VALUES + threadIdx.x] = c_add;
    a.adds_curve[size_t(q) * M3TB_N_CURVE_VALUES + threadIdx.x] = c_adds;
  }
}

// grid (n, n_chunks, ceil(max n_full / kScoreBlock)), kScoreThreads threads
__global__ void __launch_bounds__(kScoreThreads) k_diameter(const __grid_constant__ DiameterArgs a) {
  __shared__ float4 tile[kScoreTile];
  __shared__ float s_max[kScoreThreads];
  const EvalModelDev m = a.models[a.model_ids[blockIdx.x]];
  const int first = blockIdx.z * kScoreBlock;
  // (v_i - v_j).norm() and (v_j - v_i).norm() are equal: slices wholly before this block's rows hold no new pair
  const int j0 = max(blockIdx.y * a.chunk, first), j1 = min((blockIdx.y + 1) * a.chunk, m.n_full);
  if (first >= m.n_full || j0 >= j1) return;  // uniform over the block
  float4 p[kScoreVerts];
#pragma unroll
  for (int v = 0; v < kScoreVerts; ++v) p[v] = m.full[min(first + int(threadIdx.x) + v * kScoreThreads, m.n_full - 1)];
  float best = 0.0f;  // std::max(d_max, d): d_max starts at 0
  for (int t0 = j0; t0 < j1; t0 += kScoreTile) {
    const int nt = min(kScoreTile, j1 - t0);
    __syncthreads();
    for (int k = threadIdx.x; k < nt; k += kScoreThreads) tile[k] = m.full[t0 + k];
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < nt; ++k) {
      const float4 w = tile[k];
#pragma unroll
      for (int v = 0; v < kScoreVerts; ++v) {
        const float d = score::SquaredDistance(p[v].x, p[v].y, p[v].z, w);
        best = best < d ? d : best;
      }
    }
  }
  // the square root is monotone and correctly rounded, so the largest norm is the root of the largest square
  s_max[threadIdx.x] = best;
  __syncthreads();
  for (int s = kScoreThreads / 2; s > 0; s >>= 1) {
    if (int(threadIdx.x) < s) s_max[threadIdx.x] = fmaxf(s_max[threadIdx.x], s_max[threadIdx.x + s]);
    __syncthreads();
  }
  // non-negative floats order as their bit patterns
  if (threadIdx.x == 0) atomicMax(a.max_sq + blockIdx.x, __float_as_uint(s_max[0]));
}

}  // namespace m3tb
