// m3t_b200_views.cuh — exact, pruned RegionModel/DepthModel::GetClosestView (region_model.cpp:105-130,
// depth_model.cpp:81-106).
//
// The reference scans all template views for the largest orientation . R^T normalize(t) (first maximum wins, -1 start
// value). Here the views are grouped once, at model upload, into spatially compact clusters of <= 32 views (recursive
// median bisection of the orientation vectors). Per cluster an upper bound of the dot product with ANY query o follows
// from the decomposition along the cluster axis c (unit):
//     o.v = (o.c)(v.c) + o_perp.v_perp  <=  max((o.c) vc_max, (o.c) vc_min) + |o_perp| vperp_max
// so only clusters whose bound reaches a known lower bound of the maximum (the dot product of the previously selected
// view, any valid view works) can hold the arg-max. Those few clusters (2-4 of ~80 for the 2562-view models) are
// evaluated with the reference's own expression; everything else is provably smaller (a 1e-5 relative slack covers the
// float rounding of bound and dot products). The result is therefore IDENTICAL to the full scan, including the tie rule
// (largest value, smallest view index) - tests/test_view_clusters.py checks that against brute force on the host
// restatement below, tests/test_gpu_views.py on the device.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace m3tb {

constexpr int kViewClusterSize = 32;     // one warp-wide load per cluster
constexpr int kMaxViewClusterSlots = 8;  // clusters per lane in the bound pass: up to 256 clusters (8192 views)

// Device layout: cluster c = two float4:
//   a = (cx, cy, cz, vc_max)    b = (vc_min, vperp_max, slack_scale, bits(first | count << 24))
// sorted views: float4 (x, y, z, bits(original view index)), cluster members contiguous from `first`.
struct ViewClustersHost {
  std::vector<float> info;    // 8 floats per cluster
  std::vector<float> sorted;  // 4 floats per view
  int n_clusters = 0;
};

inline float FloatUp(double v) {
  float f = float(v);
  if (double(f) < v) f = std::nextafterf(f, INFINITY);
  return f;
}
inline float FloatDown(double v) {
  float f = float(v);
  if (double(f) > v) f = std::nextafterf(f, -INFINITY);
  return f;
}

inline void BuildViewClusters(const float* ori, int n, ViewClustersHost& out) {
  out.info.clear();
  out.sorted.assign(size_t(n) * 4, 0.0f);
  out.n_clusters = 0;
  std::vector<int> idx(n);
  for (int i = 0; i < n; ++i) idx[i] = i;
  struct Range { int lo, hi; };
  std::vector<Range> stack, leaves;
  stack.push_back({0, n});
  while (!stack.empty()) {
    const Range r = stack.back();
    stack.pop_back();
    const int cnt = r.hi - r.lo;
    if (cnt <= kViewClusterSize) {
      if (cnt > 0) leaves.push_back(r);
      continue;
    }
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int i = r.lo; i < r.hi; ++i)
      for (int a = 0; a < 3; ++a) {
        const float v = ori[3 * idx[i] + a];
        mn[a] = std::min(mn[a], v);
        mx[a] = std::max(mx[a], v);
      }
    int axis = 0;
    for (int a = 1; a < 3; ++a)
      if (mx[a] - mn[a] > mx[axis] - mn[axis]) axis = a;
    // left part: a multiple of the cluster size next to the median, so that most leaves are full
    int left = ((cnt / 2 + kViewClusterSize - 1) / kViewClusterSize) * kViewClusterSize;
    if (left >= cnt) left = cnt / 2;
    std::sort(idx.begin() + r.lo, idx.begin() + r.hi, [&](int p, int q) {
      const float vp = ori[3 * p + axis], vq = ori[3 * q + axis];
      return vp < vq || (vp == vq && p < q);
    });
    stack.push_back({r.lo + left, r.hi});
    stack.push_back({r.lo, r.lo + left});
  }
  std::sort(leaves.begin(), leaves.end(), [](const Range& p, const Range& q) { return p.lo < q.lo; });
  out.n_clusters = int(leaves.size());
  out.info.assign(size_t(out.n_clusters) * 8, 0.0f);
  for (int c = 0; c < out.n_clusters; ++c) {
    const Range r = leaves[c];
    std::sort(idx.begin() + r.lo, idx.begin() + r.hi);
    double m[3] = {0.0, 0.0, 0.0};
    for (int i = r.lo; i < r.hi; ++i) {
      const float* v = ori + 3 * idx[i];
      const double nv = std::sqrt(double(v[0]) * v[0] + double(v[1]) * v[1] + double(v[2]) * v[2]);
      if (nv > 0.0)
        for (int a = 0; a < 3; ++a) m[a] += v[a] / nv;
    }
    double nm = std::sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2]);
    if (!(nm > 1e-12)) { m[0] = 0.0; m[1] = 0.0; m[2] = 1.0; nm = 1.0; }
    // the axis as the float the device sees; bounds are derived from that float vector, made unit in double
    float cf[3] = {float(m[0] / nm), float(m[1] / nm), float(m[2] / nm)};
    const double cn = std::sqrt(double(cf[0]) * cf[0] + double(cf[1]) * cf[1] + double(cf[2]) * cf[2]);
    double vc_max = -INFINITY, vc_min = INFINITY, vperp_max = 0.0, vnorm_max = 0.0;
    for (int i = r.lo; i < r.hi; ++i) {
      const float* v = ori + 3 * idx[i];
      // decomposition along the (slightly non-unit) float axis cf: o.v = (o.cf)(v.cf)/|cf|^2 + o_perp.v_perp; the
      // device evaluates p = o.cf, so the stored factors absorb 1/|cf|^2 and the perpendicular part uses |cf|
      const double vc = (double(v[0]) * cf[0] + double(v[1]) * cf[1] + double(v[2]) * cf[2]) / (cn * cn);
      double perp2 = 0.0, n2 = 0.0;
      for (int a = 0; a < 3; ++a) {
        const double d = double(v[a]) - vc * cf[a];
        perp2 += d * d;
        n2 += double(v[a]) * v[a];
      }
      vc_max = std::max(vc_max, vc);
      vc_min = std::min(vc_min, vc);
      vperp_max = std::max(vperp_max, std::sqrt(perp2));
      vnorm_max = std::max(vnorm_max, std::sqrt(n2));
      float* s = out.sorted.data() + size_t(i) * 4;
      s[0] = v[0]; s[1] = v[1]; s[2] = v[2];
      const int32_t orig = idx[i];
      std::memcpy(&s[3], &orig, 4);
    }
    float* f = out.info.data() + size_t(c) * 8;
    f[0] = cf[0]; f[1] = cf[1]; f[2] = cf[2];
    f[3] = FloatUp(vc_max);
    f[4] = FloatDown(vc_min);
    // |o_perp| is evaluated on the device as sqrt(|o|^2 - p^2) with p = o.cf; with the non-unit cf the exact value is
    // sqrt(|o|^2 - p^2/|cf|^2) <= sqrt(|o|^2 - p^2) * (1 + 1e-6) for | |cf| - 1 | < 1e-7: covered by the slack
    f[5] = FloatUp(vperp_max * (1.0 + 1e-6));
    f[6] = FloatUp(2e-5 * std::max(vnorm_max, 1e-30));
    const uint32_t packed = uint32_t(r.lo) | (uint32_t(r.hi - r.lo) << 24);
    std::memcpy(&f[7], &packed, 4);
  }
}

// The bound of one cluster for query o (|o| = onorm, |o|^2 = on2). Identical expression on host and device.
__host__ __device__ inline float ViewClusterBound(float cx, float cy, float cz, float vc_max, float vc_min, float vperp_max,
                                                  float slack_scale, float o0, float o1, float o2, float on2, float onorm) {
  const float p = o0 * cx + o1 * cy + o2 * cz;
  const float along = fmaxf(p * vc_max, p * vc_min);
  const float perp = sqrtf(fmaxf(on2 - p * p, 0.0f) + 1e-6f * on2);
  return along + perp * vperp_max + slack_scale * onorm;
}

// Host restatement of the device search (scalar); used by the CPU test and as documentation of the algorithm.
// *n_evaluated receives the number of views whose dot product was computed.
inline int ClosestViewPrunedHost(const ViewClustersHost& vc, const float* ori, int n_views, const float o[3], int prev,
                                 int* n_evaluated) {
  const float on2 = o[0] * o[0] + o[1] * o[1] + o[2] * o[2];
  const float onorm = std::sqrt(on2);
  prev = std::min(std::max(prev, 0), n_views - 1);
  const float lb = o[0] * ori[3 * prev] + o[1] * ori[3 * prev + 1] + o[2] * ori[3 * prev + 2];
  float best = -1.0f;
  int idx = 0x7fffffff, evaluated = 0;
  for (int c = 0; c < vc.n_clusters; ++c) {
    const float* f = vc.info.data() + size_t(c) * 8;
    const float ub = ViewClusterBound(f[0], f[1], f[2], f[3], f[4], f[5], f[6], o[0], o[1], o[2], on2, onorm);
    if (ub < lb) continue;  // NaN-safe: a NaN bound keeps the cluster
    uint32_t packed;
    std::memcpy(&packed, &f[7], 4);
    const int first = int(packed & 0xffffffu), cnt = int(packed >> 24);
    for (int k = 0; k < cnt; ++k) {
      const float* s = vc.sorted.data() + size_t(first + k) * 4;
      const float dot = o[0] * s[0] + o[1] * s[1] + o[2] * s[2];
      int32_t vi;
      std::memcpy(&vi, &s[3], 4);
      if (dot > best || (dot == best && vi < idx)) { best = dot; idx = vi; }
      ++evaluated;
    }
  }
  if (n_evaluated) *n_evaluated = evaluated;
  return idx == 0x7fffffff ? 0 : idx;
}

#ifdef __CUDACC__
// Evaluates the candidate clusters of one warp's bound pass: bit j of `m` (warp-uniform) marks the cluster whose packed
// (first | count << 24) word lane j holds. B clusters at a time, so that their loads are in flight together; lane k
// takes member k (a cluster has <= 32 members) and keeps its running maximum in best / idx (ties: smaller view index).
template <int B>
__device__ __forceinline__ void EvaluateViewCandidates(unsigned m, unsigned packed, const float4* __restrict__ sorted,
                                                       float o0, float o1, float o2, int lane, float& best, int& idx) {
  constexpr unsigned kFull = 0xffffffffu;
  while (m) {  // warp-uniform
    unsigned pk[B];
#pragma unroll
    for (int u = 0; u < B; ++u) {
      const int j = m ? __ffs(m) - 1 : 0;
      const unsigned v = __shfl_sync(kFull, packed, j);
      pk[u] = m ? v : 0u;
      m &= m - 1u;  // 0 stays 0
    }
    float4 q[B];
#pragma unroll
    for (int u = 0; u < B; ++u) {
      const int first = int(pk[u] & 0xffffffu), cnt = int(pk[u] >> 24);
      q[u] = lane < cnt ? __ldg(sorted + first + lane) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
#pragma unroll
    for (int u = 0; u < B; ++u) {
      const int cnt = int(pk[u] >> 24);
      const float dot = o0 * q[u].x + o1 * q[u].y + o2 * q[u].z;
      const int vi = __float_as_int(q[u].w);
      if (lane < cnt && (dot > best || (dot == best && vi < idx))) { best = dot; idx = vi; }
    }
  }
}

// Order-preserving unsigned key of a dot product. -0.0 is folded to +0.0 first: the float comparison of the full scan
// treats the two as equal (the smaller view index wins), and so must the key when the two sit in different lanes.
__device__ __forceinline__ unsigned ViewKey(float v) {
  const unsigned k = __float_as_uint(v == 0.0f ? 0.0f : v);
  return (k & 0x80000000u) ? ~k : (k | 0x80000000u);
}

// Warp arg-max over (key, idx): largest key, then smallest index. Every lane receives both.
__device__ __forceinline__ void WarpViewArgMax(unsigned& key, int& idx) {
  constexpr unsigned kFull = 0xffffffffu;
  const unsigned kmax = __reduce_max_sync(kFull, key);
  idx = int(__reduce_min_sync(kFull, key == kmax ? unsigned(idx) : 0x7fffffffu));
  key = kmax;
}

// The reference's result from the arg-max: views_[0] unless some dot product exceeded its start value -1.
__device__ __forceinline__ int ClosestViewResult(unsigned kmax, int ri) {
  return (ri == 0x7fffffff || kmax <= ViewKey(-1.0f)) ? 0 : ri;
}

// Device search, executed by ONE WARP (all 32 lanes call it with identical arguments; every lane returns the result).
//   info / sorted / n_clusters: the cluster tables of the model; ori4: the model's views in original order (for the
//   lower bound); vo: query (o0, o1, o2, nonzero flag) as the pose-product step leaves it; prev: any view index.
// 32 clusters are bounded per pass (one per lane), two passes per trip to memory; the candidates of a pass are
// evaluated four at a time so that their loads are in flight together. ~5 dependent L1 / L2 trips in total.
//   `info` may point to shared memory (k_track2 stages the tables of <= 96 clusters there) or to global memory.
__device__ __forceinline__ int ClosestViewPrunedWarp(const float4* info, const float4* __restrict__ sorted,
                                                     int n_clusters, const float4* __restrict__ ori4, int n_views,
                                                     const float* vo, int prev) {
  constexpr unsigned kFull = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const float o0 = vo[0], o1 = vo[1], o2 = vo[2];
  if (vo[3] == 0.0f || n_views <= 0) return 0;  // |t| = 0: the reference returns views_[0]
  const float on2 = o0 * o0 + o1 * o1 + o2 * o2;
  const float onorm = sqrtf(on2);
  prev = min(max(prev, 0), n_views - 1);
  const float4 qp = __ldg(ori4 + prev);
  const float lb = o0 * qp.x + o1 * qp.y + o2 * qp.z;
  float best = -1.0f;
  int idx = 0x7fffffff;
  for (int c0 = 0; c0 < n_clusters; c0 += 64) {  // two bound passes per trip: their table loads are in flight together
    float4 ia[2], ib[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = c0 + 32 * h + lane;
      if (c < n_clusters) { ia[h] = info[2 * c]; ib[h] = info[2 * c + 1]; }
      else { ia[h] = make_float4(0.0f, 0.0f, 0.0f, 0.0f); ib[h] = ia[h]; }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = c0 + 32 * h + lane;
      bool cand = false;
      if (c < n_clusters) {
        const float ub = ViewClusterBound(ia[h].x, ia[h].y, ia[h].z, ia[h].w, ib[h].x, ib[h].y, ib[h].z, o0, o1, o2, on2, onorm);
        cand = !(ub < lb);  // NaN-safe: a NaN bound keeps the cluster
      }
      EvaluateViewCandidates<4>(__ballot_sync(kFull, cand), __float_as_uint(ib[h].w), sorted, o0, o1, o2, lane, best, idx);
    }
  }
  unsigned key = ViewKey(best);
  WarpViewArgMax(key, idx);
  return ClosestViewResult(key, idx);
}

// The view that a group search published in `slots`: every thread may call this once the search's barrier has passed,
// until the second search after it starts writing the same slots. `tid` is the calling thread's index (threadIdx.x): the
// caller decides where it is read (k_track2 reads it at the use in its 1024-thread kernel, see NestTid).
template <int G>
__device__ __forceinline__ int ClosestViewOfSlots(const uint2* slots, int tid) {
  const int lane = tid & 31;
  const uint2 s = lane < G / 32 ? slots[lane] : make_uint2(0u, 0x7fffffffu);
  unsigned key = s.x;
  int idx = int(s.y);
  WarpViewArgMax(key, idx);
  return ClosestViewResult(key, idx);
}

// The same search, executed by a warp group of G threads (G / 32 warps; all threads call it with identical arguments
// and every thread returns the result). Shorter dependent chain than the one-warp form: every thread bounds one cluster
// of a round of G (the tables and the lower bound's view in one trip), each warp evaluates its own candidates, and one
// group barrier (`barrier()`) publishes the per-warp maxima. Clusters are dealt to the warps round-robin
// (c = c0 + lane * G/32 + warp): neighbouring clusters, the likely candidates of one query, land in different warps, so
// a warp rarely holds more than one candidate and evaluates them one at a time (a batch of two costs the 1024-thread
// k_track2 more spill traffic than it saves). The result does not depend on how the views are split: largest dot
// product, smallest view index on ties.
//   slots: G / 32 entries of scratch in shared memory, written on every call (also when there is nothing to search).
//   tid: the calling thread's index, threadIdx.x (see ClosestViewOfSlots).
//   Callers alternate two sets between consecutive searches, so that the next search's writes cannot overtake a slow
//   warp's reads of this one, and ClosestViewOfSlots can re-read this result up to the start of the next-but-one search.
template <int G, class Barrier>
__device__ __forceinline__ int ClosestViewPrunedGroup(const float4* info, const float4* __restrict__ sorted,
                                                      int n_clusters, const float4* __restrict__ ori4, int n_views,
                                                      const float* vo, int prev, uint2* slots, int tid, Barrier barrier) {
  constexpr unsigned kFull = 0xffffffffu;
  constexpr int kWarps = G / 32;
  static_assert(kWarps <= 32 && (G & (G - 1)) == 0, "one slot per warp, read by one warp");
  const int lane = tid & 31, warp = (tid & (G - 1)) >> 5;
  const bool search = vo[3] != 0.0f && n_views > 0;  // group-uniform; else (|t| = 0) the reference returns views_[0]
  prev = min(max(prev, 0), n_views - 1);
  // the lower bound's view and the first round's cluster tables are requested together (one trip, not two)
  const float4 qp = search ? __ldg(ori4 + prev) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  int c = lane * kWarps + warp;
  float4 ia = make_float4(0.0f, 0.0f, 0.0f, 0.0f), ib = ia;
  if (search && c < n_clusters) { ia = info[2 * c]; ib = info[2 * c + 1]; }
  const float o0 = vo[0], o1 = vo[1], o2 = vo[2];
  const float on2 = o0 * o0 + o1 * o1 + o2 * o2;
  const float onorm = sqrtf(on2);
  float best = -1.0f;
  int idx = 0x7fffffff;
  for (int c0 = 0; search && c0 < n_clusters; c0 += G, c += G) {
    bool cand = false;
    if (c < n_clusters) {
      const float ub = ViewClusterBound(ia.x, ia.y, ia.z, ia.w, ib.x, ib.y, ib.z, o0, o1, o2, on2, onorm);
      const float lb = o0 * qp.x + o1 * qp.y + o2 * qp.z;
      cand = !(ub < lb);  // NaN-safe: a NaN bound keeps the cluster
    }
    EvaluateViewCandidates<1>(__ballot_sync(kFull, cand), __float_as_uint(ib.w), sorted, o0, o1, o2, lane, best, idx);
    if (c + G < n_clusters) { ia = info[2 * (c + G)]; ib = info[2 * (c + G) + 1]; }  // next round (> G clusters)
  }
  unsigned key = ViewKey(best);
  WarpViewArgMax(key, idx);
  if (lane == 0) slots[warp] = make_uint2(key, unsigned(idx));
  barrier();
  return ClosestViewOfSlots<G>(slots, tid);
}
#endif  // __CUDACC__

}  // namespace m3tb
