// m3t_b200_track2.cuh — k_track2: the fused tracking step for rigid bodies, second generation.
//
// Same arithmetic as k_track (m3t_b200_kernels.cuh: every per-line / per-point expression is evaluated in the
// reference's order, so the stored state is bit-identical to the oracle), different execution shape:
//
//   * 1024 threads per body when a body carries both modalities: warps 16-31 own the correspondence LINES, warps
//     0-15 the depth POINTS, one item per thread, so the two correspondence phases and the two gradient passes of
//     an iteration run concurrently (32 resident warps instead of 16; 64 registers per thread).
//   * 64 registers: the 2 x 19 segment products of a line are never held at once. A line is walked segment by
//     segment; a sliding window of the last 8 segments (16 registers) is all CalculateDistribution
//     (region_modality.cpp:1600-1637) needs to finish one distribution entry per new segment, in the reference's
//     multiplication order, for lines walked in either direction. The 12 entries go to shared memory (24 KB); the
//     local-mode gradient reads its two entries from there by index.
//   * GetClosestView is the exact pruned search of m3t_b200_views.cuh (~200 instead of 2 x 2562 dot products per
//     iteration), split over the 16 warps of each group (ClosestViewPrunedGroup): each warp bounds its share of the
//     clusters and evaluates its candidates (usually one), one group barrier combines the 16 maxima. A single warp
//     needed ~5 dependent trips to memory while the other 15 waited at the barrier.
//   * CalculateOptimization (6 x 6) is k_track's: SolveAndUpdateSerial and PublishPoseProducts of m3t_b200_kernels.cuh,
//     run thread-serially in registers on warp 0 (every lane the same work, no shuffles in the dependent chain).
//
// Serves the fused entry points (m3tb_tracking_step, m3tb_corr_iteration) and the plain correspondence calls for
// bodies with <= 512 lines and <= 512 points, no measured occlusion handling, function lookups identical across the
// batch; everything else stays on k_track.
#pragma once

#include "m3t_b200_kernels.cuh"
#include "m3t_b200_views.cuh"

namespace m3tb {

constexpr int kGroup = 512;                                      // items per modality and threads per warp group
constexpr int kDistBytes = kDistributionLength * kGroup * 4;     // shared-memory home of the line distributions
constexpr int kClusterStage = 96;                                // clusters per model staged in shared memory (3072 views)
constexpr int kClusterBytes = 2 * kClusterStage * 32;            // [region | depth] x kClusterStage x two float4
constexpr int kFixedDynBytes = kDistBytes + kClusterBytes;       // dynamic shared memory before the tiles (after the LUT)

// The camera's histogram bin-index image (valid inside the body's ROI)
struct BinImage {
  const uint16_t* px;  // null: no bin-index image
  unsigned pitch;      // bytes
};

struct Shared2 {
  float pose[12];            // body2world
  float rb2c[12], db2c[12];  // body2camera of the colour / depth camera
  float dc2b[12];            // inverse of db2c
  float cw2c[12], dw2c[12];  // world2camera
  float view_o[2][4];        // GetClosestView queries, [3] = 1 if |t| > 0
  Tile ctile, dtile;
  unsigned long long depth_bar, lut_bar, ctile_bar;
  float red[32][32];         // per-warp partial sums g[6] + H lower[21] (+5 pad)
  float a[36], b[6], x[6];   // normal equations
  uint2 view_slots[2][2][kGroup / 32];  // [corr parity][region | depth] per-warp maxima of the closest-view searches
  FrameView cframe, dframe;  // how the body sees its colour / depth frame (read on the rare out-of-tile paths)
  int stamp_n[2];            // profiling aid: slots filled so far by the solver warp / the point group's leader warp
  int view0[2];              // the region / depth view the first closest-view searches start from (the body's record)
  int n_items[2];            // lines / points of the last correspondence iteration (written by item 0 of the group)
  // Per-body parameters, cameras and model headers are read all over the iteration loops. With 225 KB of the SM's
  // 228 KB configured as shared memory the L1 cache is ~3 KB, so from global memory each of those reads is an L2 round
  // trip (long-scoreboard stalls); one copy here instead.
  BodyDev body;
  CameraDev cams[2];         // colour, depth
  ModelDev models[2];        // region, depth
  const float4* info[2];     // cluster tables of the pruned closest-view searches (region, depth)
  BinImage bins;             // the colour camera's bin-index image, when the TMA path maintains it
};

// barrier of one warp group (512 threads) when the CTA has two; id 1 = lines, id 2 = points
template <int T>
__device__ __forceinline__ void GroupBarrier(int group) {
  if (T == kGroup) __syncthreads();
  else asm volatile("bar.sync %0, %1;" ::"r"(group + 1), "r"(kGroup) : "memory");
}

// Thread and block index, read where they are used. The asm is volatile so that the value is not hoisted out of the loop
// nest, where it would occupy a register, or a stack slot, all the way through.
__device__ __forceinline__ int TidX() {
  unsigned v;
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(v));
  return int(v);
}
__device__ __forceinline__ int CtaX() {
  unsigned v;
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(v));
  return int(v);
}
// The indices as the loop nest of k_track2<T> reads them. The 1024-thread kernel (64 registers) re-reads them at every
// use: hoisted, the lane / warp index of the view search and the solve and the block index sat in stack slots. The
// 512-thread kernel has the registers to keep them, and keeping them is cheaper than an S2R on the dependent chains of
// the view search and the solve.
template <int T>
__device__ __forceinline__ int NestTid() {
  return T > kGroup ? TidX() : int(threadIdx.x);
}
template <int T>
__device__ __forceinline__ int NestCta() {
  return T > kGroup ? CtaX() : int(blockIdx.x);
}

struct LineRegs {  // RegionModality::DataLine without the distribution (shared memory)
  float cbx, cby, cbz, cu, cv, nu, nv, dr, ncts, mean, var;
  bool valid;
};

// profiling aid (M3TB_TIMING=1): the solver warp (last warp) stamps slots [0, 128), the point group's leader warp slots
// [128, 256). Which warp stamps where follows from threadIdx and the kernel parameters, and the slot counters live in
// shared memory (each one written by lane 0 of one warp), so the instrumentation holds no registers across the loop nest.
template <int T>
__device__ __forceinline__ void Stamp2(const TrackArgs& args, Shared2& sh) {
  if (!args.phase_clock) return;
  const int tid = NestTid<T>(), warp = tid >> 5;
  if ((tid & 31) != 0) return;
  if (warp != T / 32 - 1 && !(T > kGroup && warp == kGroup / 32 - 1)) return;
  const int half = (T > kGroup && tid < kGroup) ? 1 : 0;
  const int i = sh.stamp_n[half];
  if (i < kPhaseSlots / 2) {
    args.phase_clock[size_t(NestCta<T>()) * kPhaseSlots + half * (kPhaseSlots / 2) + i] = clock64();
    sh.stamp_n[half] = i + 1;
  }
}

// prologue detail (profiling aid): fixed slots past the ones Stamp2 fills
#define M3TB_STAMP_AT(slot, cond)                                                                  \
  do {                                                                                             \
    if (args.phase_clock && (cond)) args.phase_clock[size_t(body_id) * kPhaseSlots + (slot)] = clock64(); \
  } while (0)

// dynamic shared memory: [LUT when staged] [line distributions] [cluster tables] [tiles]
__device__ __forceinline__ unsigned char* DynSmem() {
  extern __shared__ __align__(128) unsigned char dyn[];
  return dyn;
}
template <bool LUT_SMEM>
constexpr unsigned kLutBytes = LUT_SMEM ? unsigned(16 * 16 * 16 * sizeof(float2)) : 0u;  // the LUT opens dynamic smem
// This thread's column of the line distributions, its address formed from the thread index where it is needed (TidX)
template <bool LUT_SMEM>
__device__ __forceinline__ float* DistCol() {
  return reinterpret_cast<float*>(DynSmem() + kLutBytes<LUT_SMEM>) + (TidX() & (kGroup - 1));
}
// ---------------------------------------------------------------------------------------------
// One correspondence line, streaming form. Walks the 19 segments of the line in pixel order; after segment w >= 7 the
// distribution entry that has just become computable is finished from the 8-segment window:
//   line walked front to back (n_major > 0): entry d = w - 7 uses the segments walked at w-7 .. w, in that order;
//   line walked back to front: segment index = 18 - walk index (region_modality.cpp:1470-1484), so entry d = 18 - w
//   uses the segments walked at w, w-1, .. w-7, in that order.
// Either way the factors are multiplied for k = 0..7 exactly as CalculateDistribution does.
// The loop over the segments is rolled: unrolled 19 times for each compile-time scale, the walk was almost half of the
// kernel's code, far more than the SM's instruction caches hold, and the 16 line warps streamed it in again every
// correspondence iteration. The S samples of a segment stay unrolled. The window is a register shift (slot 7 = the
// segment just walked, slot 0 = the one 7 steps earlier), so every index into it is a compile-time constant and it
// stays in registers; the entry's address is formed from the thread index at the store, so the walk carries no pointer
// to this thread's distribution column.
// ---------------------------------------------------------------------------------------------
template <bool LUT_SMEM, int S>
__device__ __forceinline__ void WalkFast(int scale, int base, float minor_f, float step, int stride_major, int stride_minor,
                                         const uint16_t* tile_px, const float2* __restrict__ lut_g, const float2* lut_s,
                                         const float* __restrict__ lf, const float* __restrict__ lb, bool rev) {
  float wf[8], wb[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) wf[k] = wb[k] = 0.0f;
  // two segments per trip: with one, the loop's bookkeeping made the 512-thread kernel slower than the unrolled walk
#pragma unroll 2
  for (int w = 0; w < kLineSegments; ++w) {
    float pf = 1.0f, pb = 1.0f;
    if (S > 0) {
      int idx[S > 0 ? S : 1];
#pragma unroll
      for (int k = 0; k < S; ++k) {
        idx[k] = tile_px[base + int(minor_f) * stride_minor];
        base += stride_major;
        minor_f += step;
      }
      float2 l[S > 0 ? S : 1];
#pragma unroll
      for (int k = 0; k < S; ++k) l[k] = LutFetch<LUT_SMEM>(lut_g, lut_s, idx[k]);
#pragma unroll
      for (int k = 0; k < S; ++k) { pf *= l[k].x; pb *= l[k].y; }
    } else {
#pragma unroll 1
      for (int k = 0; k < scale; ++k) {
        const int idx = tile_px[base + int(minor_f) * stride_minor];
        const float2 l = LutFetch<LUT_SMEM>(lut_g, lut_s, idx);
        pf *= l.x;
        pb *= l.y;
        base += stride_major;
        minor_f += step;
      }
    }
    if (S > 1 || (S == 0 && scale > 1)) {  // region_modality.cpp:1555-1571
      if (pf != 0.0f || pb != 0.0f) {
        float sum = pf;
        sum += pb;
        pf /= sum;
        pb /= sum;
      } else {
        pf = 0.5f;
        pb = 0.5f;
      }
    }
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      wf[k] = wf[k + 1];
      wb[k] = wb[k + 1];
    }
    wf[7] = pf;
    wb[7] = pb;
    if (w >= 7) {
      float val = 1.0f;
#pragma unroll
      for (int k = 0; k < kFunctionLength; ++k) {
        const float f = rev ? wf[7 - k] : wf[k];
        const float b = rev ? wb[7 - k] : wb[k];
        val *= f * lf[k] + b * lb[k];
      }
      DistCol<LUT_SMEM>()[(rev ? kLineSegments - 1 - w : w - 7) * kGroup] = val;
    }
  }
}

// Rare path: a sample may lie outside the tile. All 19 segments go to local memory first (as in k_track). Samples
// outside the tile come from the camera's bin-index image where it is valid (inside the body's ROI), else from the frame.
template <bool LUT_SMEM>
__device__ __noinline__ void WalkSlow(int scale, int bs, int nb, bool horizontal, int major, float minor_f, float step,
                                      const FrameView& frame, const Tile& tile, const uint16_t* tile_px, const BinImage& bins,
                                      const float2* __restrict__ lut_g, const float2* lut_s, const float* lf,
                                      const float* lb, bool rev, float* dist_col) {
  float sf[kLineSegments], sb[kLineSegments];
#pragma unroll 1
  for (int s = 0; s < kLineSegments; ++s) {
    float pf = 1.0f, pb = 1.0f;
#pragma unroll 1
    for (int k = 0; k < scale; ++k) {
      const int minor = int(minor_f);
      const int x = horizontal ? major : minor, y = horizontal ? minor : major;
      const unsigned tx = unsigned(x - tile.x0), ty = unsigned(y - tile.y0);
      int idx;
      if (tx < unsigned(tile.w) && ty < unsigned(tile.h)) {
        idx = tile_px[ty * unsigned(tile.pitch) + tx];
      } else if (bins.px && x >= frame.x0 && x < frame.x1 && y >= frame.y0 && y < frame.y1) {
        idx = __ldg(reinterpret_cast<const uint16_t*>(reinterpret_cast<const uint8_t*>(bins.px) + size_t(unsigned(y)) * bins.pitch) + x);
      } else {
        const uint8_t* p = FramePtr(frame, x, y, 3u);
        idx = int(LutSlot(unsigned((int(__ldg(p)) >> bs) * nb * nb + (int(__ldg(p + 1)) >> bs) * nb + (int(__ldg(p + 2)) >> bs))));
      }
      const float2 l = LutFetch<LUT_SMEM>(lut_g, lut_s, idx);
      pf *= l.x;
      pb *= l.y;
      ++major;
      minor_f += step;
    }
    sf[s] = pf;
    sb[s] = pb;
  }
  if (scale > 1) {
#pragma unroll 1
    for (int s = 0; s < kLineSegments; ++s) {
      if (sf[s] != 0.0f || sb[s] != 0.0f) {
        float sum = sf[s];
        sum += sb[s];
        sf[s] /= sum;
        sb[s] /= sum;
      } else {
        sf[s] = 0.5f;
        sb[s] = 0.5f;
      }
    }
  }
#pragma unroll 1
  for (int d = 0; d < kDistributionLength; ++d) {
    float val = 1.0f;
#pragma unroll 1
    for (int k = 0; k < kFunctionLength; ++k) {
      const int s = rev ? kLineSegments - 1 - (d + k) : d + k;
      val *= sf[s] * lf[k] + sb[s] * lb[k];
    }
    dist_col[d * kGroup] = val;
  }
}

template <bool LUT_SMEM>
__device__ __forceinline__ void RegionLine2(const RegionIter& it, const RegionParamsDev& rp, const float4 p0, const float4 p1,
                                            const FrameView& frame, const Tile& tile, const uint16_t* tile_px,
                                            const BinImage& bins, const float2* __restrict__ lut_g, const float2* lut_s,
                                            const float* __restrict__ lf, const float* __restrict__ lb, LineRegs& L) {
  L.valid = false;
  // CalculateBasicLineData (:1231-1250)
  float x, y, z;
  PoseApply(it.b2c, p0.x, p0.y, p0.z, x, y, z);
  float nu = it.b2c[0] * p0.w + it.b2c[1] * p1.x + it.b2c[2] * p1.y;
  float nv = it.b2c[4] * p0.w + it.b2c[5] * p1.x + it.b2c[6] * p1.y;
  {
    float zz = nu * nu + nv * nv;
    if (zz > 0.0f) { float n = sqrtf(zz); nu /= n; nv /= n; }
  }
  float center_u = x * it.fu / z + it.ppu;
  float center_v = y * it.fv / z + it.ppv;
  L.cbx = p0.x; L.cby = p0.y; L.cbz = p0.z;
  L.cu = center_u; L.cv = center_v; L.nu = nu; L.nv = nv;
  float continuous_distance = fminf(p1.w, p1.z) * it.fu / (z * it.fscale);
  // IsLineValid (:1252-1291)
  if (continuous_distance < rp.min_continuous_distance) return;
  if (z <= 0.0f) return;
  int icu = int(center_u + 0.5f), icv = int(center_v + 0.5f);
  if (icu < 0 || icu > it.w_m1 || icv < 0 || icv > it.h_m1) return;
  // CalculateSegmentProbabilities (:1433-1573); horizontal / vertical cases folded into major / minor axes
  const bool horizontal = fabsf(nv) < fabsf(nu);
  const float c_major = horizontal ? center_u : center_v;
  const float c_minor = horizontal ? center_v : center_u;
  const float n_major = horizontal ? nu : nv;
  const float n_minor = horizontal ? nv : nu;
  const int major_m1 = horizontal ? it.w_m1 : it.h_m1;
  const int minor_m1 = horizontal ? it.h_m1 : it.w_m1;
  const int minor_m2 = horizontal ? it.h_m2 : it.w_m2;
  const float step = n_minor / n_major;
  int major = int(c_major - it.ll_half_m1);
  const int major_end = major + it.ll_m1;
  float minor_f = c_minor + step * (float(major) - c_major) + 0.5f;
  const float minor_f_end = minor_f + step * float(it.ll_m1);
  if (major < 0 || major_end > major_m1 || int(minor_f) < 0 || int(minor_f) > minor_m1 || int(minor_f_end) < 1 ||
      int(minor_f_end) > minor_m2)
    return;
  const bool rev = !(n_major > 0.0f);  // segments are filled back to front (:1470-1484)
  {
    const int mi0 = int(minor_f), mi1 = int(minor_f_end);
    const int minor_lo = min(mi0, mi1) - 1, minor_hi = max(mi0, mi1) + 1;
    const int x_lo = horizontal ? major : minor_lo, x_hi = horizontal ? major_end : minor_hi;
    const int y_lo = horizontal ? minor_lo : major, y_hi = horizontal ? minor_hi : major_end;
    const bool inside = x_lo >= tile.x0 && x_hi < tile.x0 + tile.w && y_lo >= tile.y0 && y_hi < tile.y0 + tile.h;
    if (inside) {
      const int stride_major = horizontal ? 1 : tile.pitch;
      const int stride_minor = horizontal ? tile.pitch : 1;
      const int base = horizontal ? (major - tile.x0) - tile.y0 * tile.pitch : (major - tile.y0) * tile.pitch - tile.x0;
      switch (it.scale) {
        case 1: WalkFast<LUT_SMEM, 1>(1, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, lf, lb, rev); break;
        case 2: WalkFast<LUT_SMEM, 2>(2, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, lf, lb, rev); break;
        case 4: WalkFast<LUT_SMEM, 4>(4, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, lf, lb, rev); break;
        case 6: WalkFast<LUT_SMEM, 6>(6, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, lf, lb, rev); break;
        default: WalkFast<LUT_SMEM, 0>(it.scale, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, lf, lb, rev); break;
      }
    } else {
      // the lookups from the body's parameters in shared memory (the host checked them equal to the kernel parameters):
      // the generic address of a kernel parameter was held in registers through the loop nest
      WalkSlow<LUT_SMEM>(it.scale, rp.bitshift, rp.n_bins, horizontal, major, minor_f, step, frame, tile, tile_px, bins,
                         lut_g, lut_s, rp.lookup_f, rp.lookup_b, rev, DistCol<LUT_SMEM>());
    }
  }
  L.ncts = fabsf(n_major) / it.fscale;
  L.dr = (roundf(c_major - it.ll_m1_half) + it.ll_m1_half - c_major) / n_major;
  // CalculateDistribution, normalisation (:1630-1636) and CalculateDistributionMoments (:1639-1658)
  float* dist_col = DistCol<LUT_SMEM>();
  float dist[kDistributionLength];
  float area = 0.0f;
#pragma unroll
  for (int d = 0; d < kDistributionLength; ++d) {
    dist[d] = dist_col[d * kGroup];
    area += dist[d];
  }
#pragma unroll
  for (int d = 0; d < kDistributionLength; ++d) {
    dist[d] /= area;
    dist_col[d * kGroup] = dist[d];
  }
  float mean_from_begin = 0.0f;
#pragma unroll
  for (int d = 0; d < kDistributionLength; ++d) mean_from_begin += float(d) * dist[d];
  float var = 0.0f;
#pragma unroll
  for (int d = 0; d < kDistributionLength; ++d) {
    float dd = float(d) - mean_from_begin;
    var += (dd * dd) * dist[d];
  }
  L.mean = mean_from_begin - (float(kDistributionLength) - 1.0f) / 2.0f;
  L.var = fmaxf(var, rp.min_expected_variance);
  L.valid = true;
}

// K2 region (region_modality.cpp:485-558), in two steps: the line's Jacobian J and weights (wg, wh), then the 27 sums
// (AddRegionSums). The pose (b2c), the camera and the body's parameters are read from shared memory where they are
// used, the two distribution entries of the local mode too: nothing of the iteration state is carried into the update
// loop besides the line itself. Returns false, leaving J, wg and wh as they are, when the line adds nothing.
__device__ __forceinline__ bool RegionJacobian2(const float* b2c, const CameraDev& cam, const RegionParamsDev& rp,
                                                const LineRegs& L, const float* dist_col, int corr, int opt_iteration,
                                                float (&J)[6], float& wg, float& wh) {
  if (!L.valid) return false;
  float x, y, z;
  PoseApply(b2c, L.cbx, L.cby, L.cbz, x, y, z);
  float fu_z = cam.fu / z, fv_z = cam.fv / z;
  float xfu_z = x * fu_z, yfv_z = y * fv_z;
  float delta_cs = (L.nu * (xfu_z + cam.ppu - L.cu) + L.nv * (yfv_z + cam.ppv - L.cv) - L.dr) * L.ncts;
  float dll;
  if (opt_iteration < rp.n_global_iterations) {
    dll = (L.mean - delta_cs) / L.var;
  } else {
    int upper = int(delta_cs + (float(kDistributionLength) + 1.0f) / 2.0f);
    int lower = upper - 1;
    if (upper <= 0 || upper >= kDistributionLength) return false;
    dll = (logf(dist_col[upper * kGroup]) - logf(dist_col[lower * kGroup])) * rp.learning_rate / L.var;
  }
  float dc0 = L.ncts * L.nu * fu_z;
  float dc1 = L.ncts * L.nv * fv_z;
  float dc2 = L.ncts * (-L.nu * xfu_z - L.nv * yfv_z) / z;
  J[3] = dc0 * b2c[0] + dc1 * b2c[4] + dc2 * b2c[8];
  J[4] = dc0 * b2c[1] + dc1 * b2c[5] + dc2 * b2c[9];
  J[5] = dc0 * b2c[2] + dc1 * b2c[6] + dc2 * b2c[10];
  J[0] = L.cby * J[5] - L.cbz * J[4];
  J[1] = L.cbz * J[3] - L.cbx * J[5];
  J[2] = L.cbx * J[4] - L.cby * J[3];
  const float sd = LastValid(rp.standard_deviations, rp.n_standard_deviations, corr);  // as MakeRegionIter
  float weight = rp.min_expected_variance / (L.ncts * L.ncts * (sd * sd));
  wg = weight * dll;
  wh = weight / L.var;
  return true;
}
__device__ __forceinline__ void AddRegionSums(const float (&J)[6], float wg, float wh, float (&acc)[27]) {
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    acc[r] += wg * J[r];
#pragma unroll
    for (int c = 0; c <= r; ++c) acc[6 + Tri(r, c)] -= (wh * J[r]) * J[c];
  }
}

// ---------------------------------------------------------------------------------------------
// TMA tensor tiles
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void TensorCopyG2S(void* dst_smem, const CUtensorMap* map, int x, int y, int z,
                                              unsigned long long* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
          SmemAddr(dst_smem)),
      "l"(reinterpret_cast<unsigned long long>(map)), "r"(x), "r"(y), "r"(z), "r"(SmemAddr(bar))
      : "memory");
}

// Fits the wanted rectangle `t` to what a stack of TMA boxes can deliver: a width from {64, 96, .. 256}, a height that
// is a multiple of kTileBoxRows, inside the region where the device copy of the frame is valid (`f`), at most `budget`
// bytes. Wider / taller than wanted is fine (more samples take the fast path); smaller is clipped symmetrically, the
// samples outside go through the frame in global memory. No tile (w = h = 0) if even the smallest box does not fit.
__device__ __forceinline__ void SnapTile(Tile& t, const FrameView& f, int budget, int max_w = 256) {
  const int vx0 = f.x0, vx1 = f.x1, vy0 = f.y0, vy1 = f.y1;
  if (t.w <= 0 || t.h <= 0 || vx1 - vx0 < 64 || vy1 - vy0 < kTileBoxRows || budget < 64 * kTileBoxRows * 2) {
    t.w = t.h = t.pitch = 0;
    return;
  }
  int w = min(max_w, (max(t.w, 64) + 31) / 32 * 32);         // smallest box width that covers the rectangle
  w = min(w, (vx1 - vx0) / 32 * 32);                         // ... that fits the valid columns
  w = max(w, 64);
  if (w > vx1 - vx0) { t.w = t.h = t.pitch = 0; return; }
  int h = (t.h + kTileBoxRows - 1) / kTileBoxRows * kTileBoxRows;
  h = min(h, (vy1 - vy0) / kTileBoxRows * kTileBoxRows);
  while (w * h * 2 > budget) {                               // over budget: shrink the longer side first
    if (h >= w && h > kTileBoxRows) h -= kTileBoxRows;
    else if (w > 64) w -= 32;
    else if (h > kTileBoxRows) h -= kTileBoxRows;
    else { t.w = t.h = t.pitch = 0; return; }
  }
  // centre on the wanted rectangle, then push back inside the valid region. The first column is a multiple of 8 pixels:
  // TMA needs the global address of a box (base + 2 * x0) 16-byte aligned (an unaligned x0 traps as "illegal
  // instruction", measured with scripts/probes/tma_probe.cu).
  int x0 = (t.x0 + (t.w - w) / 2) & ~7, y0 = t.y0 + (t.h - h) / 2;
  x0 = max((vx0 + 7) & ~7, min(x0, (vx1 - w) & ~7));
  y0 = max(vy0, min(y0, vy1 - h));
  if (x0 < vx0 || x0 + w > vx1) { t.w = t.h = t.pitch = 0; return; }
  t.x0 = x0; t.y0 = y0; t.w = w; t.h = h; t.pitch = w;
}

// ---------------------------------------------------------------------------------------------
// The correspondence / update loop nest, by role. A thread of the 1024-thread kernel owns either a line or a depth point,
// so the kernel runs the nest once per role (ItemLoop<.., LINES, POINTS>) and a thread carries the state of its own role
// only; at 64 registers per thread that keeps the line walk and the gradient reduction out of local memory. The
// 512-thread kernel, where one group owns both, runs the nest with both roles, phase after phase as before. Every
// instantiation meets the same CTA barriers in the same order: two __syncthreads per update iteration.
// ---------------------------------------------------------------------------------------------
// The loop nest reaches what the prologue settled (per-body copies, tiles, lookups) through `sh`, the kernel parameters and
// threadIdx where it uses it, so that no pointer or flag is carried in registers through the loop nest.
__device__ __forceinline__ bool DoPhase(const Shared2& sh, const TrackArgs& args, bool region, unsigned phase) {
  return (region ? sh.body.has_region : sh.body.has_depth) && (args.phases & phase);
}

// The readers of the prologue's bulk copies wait for them in the first correspondence iteration (the loop nest's first
// use) and before the kernel exits. Whether a copy was issued follows from the kernel parameters and the tiles in `sh`,
// and a wait on the completed phase of an mbarrier returns at once, so no "copy has landed" flag is carried through the
// loop nest.
template <bool LUT_SMEM>
__device__ __forceinline__ void WaitColourCopies(const TrackArgs& args, Shared2& sh) {
  if (LUT_SMEM) MbarWait(&sh.lut_bar, 0);
  if (args.tma_mode != 0 && sh.ctile.w > 0) MbarWait(&sh.ctile_bar, 0);
}
__device__ __forceinline__ void WaitDepthCopies(Shared2& sh) {
  if (sh.dtile.w > 0) MbarWait(&sh.depth_bar, 0);
}

// Closest view of model m (0: region, searched by the line group; 1: depth, by the point group, or by the only group of
// the 512-thread kernel), by all threads of the group. The lower bound starts from the previous iteration's answer,
// re-read from that search's slots in shared memory: a register copy kept across the loop nest sits in local memory in
// the 1024-thread kernel, one more L2 round trip ahead of the search. The first iteration starts from the view of the
// body's record (Shared2::view0).
template <int T>
__device__ __forceinline__ int GroupClosestView(const TrackArgs& args, Shared2& sh, int corr, int m) {
  const ModelDev& model = sh.models[m];
  const int prev =
      corr > args.corr_begin ? ClosestViewOfSlots<kGroup>(sh.view_slots[(corr - 1) & 1][m], NestTid<T>()) : sh.view0[m];
  return ClosestViewPrunedGroup<kGroup>(sh.info[m], model.sorted_views, model.n_clusters, model.orientations4,
                                        model.n_views, sh.view_o[m], prev, sh.view_slots[corr & 1][m], NestTid<T>(),
                                        [m] { GroupBarrier<T>(m); });
}

// The view of model m that the body's record keeps: the last search's answer, or the record's own view when the
// correspondence phase of the model did not run (by all threads of the group, like the search)
template <int T>
__device__ __forceinline__ int RecordView(const TrackArgs& args, const Shared2& sh, bool searched, int m) {
  return (searched && args.corr_end > args.corr_begin)
             ? ClosestViewOfSlots<kGroup>(sh.view_slots[(args.corr_end - 1) & 1][m], NestTid<T>()) : sh.view0[m];
}

// Line role, one correspondence iteration: closest view of the region model (the whole group), then RegionLine2. With
// one warp group (POINTS: T = 512) the group searches the depth model right after. L arrives empty (ItemLoop).
template <int T, bool LUT_SMEM, bool POINTS>
__device__ __forceinline__ void LineCorrespondence(const TrackArgs& args, Shared2& sh, int corr, LineRegs& L) {
  const BodyDev& body = sh.body;
  const ModelDev* rmodel = &sh.models[0];
  const int view_r = GroupClosestView<T>(args, sh, corr, 0);
  if (POINTS && DoPhase(sh, args, false, PH_DEPTH_CORR)) GroupClosestView<T>(args, sh, corr, 1);
  Stamp2<T>(args, sh);  // closest view (region)
  RegionIter rit;
  MakeRegionIter(body.rp, sh.cams[0], sh.rb2c, corr, rit);
  // the model record does not depend on the line count: load it first, the count (one more trip to memory when the
  // coverage is adaptive) meanwhile
  const int item = NestTid<T>() & (kGroup - 1);
  const float4* pts = rmodel->points + size_t(view_r) * rmodel->n_points * 2;
  float4 p0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), p1 = p0;
  if (item < min(rmodel->n_points, min(args.line_cap, kGroup))) { p0 = __ldg(pts + 2 * item); p1 = __ldg(pts + 2 * item + 1); }
  int n_lines = AdaptiveCount(body.rp.n_lines_max, body.rp.use_adaptive_coverage, body.rp.reference_contour_length,
                              body.rp.use_adaptive_coverage ? __ldg(rmodel->view_scalars + view_r) : 0.0f,
                              rmodel->max_view_scalar, rmodel->n_points);
  n_lines = min(n_lines, min(args.line_cap, kGroup));
  if (item == 0) sh.n_items[0] = n_lines;
  const int body_id = NestCta<T>();
  if (corr == args.corr_begin) {
    const bool tile_wait = args.tma_mode != 0 && sh.ctile.w > 0;
    M3TB_STAMP_AT(118, tile_wait && NestTid<T>() == T - 32);
    WaitColourCopies<LUT_SMEM>(args, sh);
    M3TB_STAMP_AT(119, tile_wait && NestTid<T>() == T - 32);
  }
  if (item < n_lines) {
    const uint16_t* tile_px = reinterpret_cast<const uint16_t*>(DynSmem() + sh.ctile.offset);
    const float2* lut_g = args.lut + size_t(NestCta<T>()) * args.lut_stride;
    const float2* lut_s = reinterpret_cast<const float2*>(DynSmem());
    // function lookups (identical for every body of the launch, checked by the host): kernel-parameter constants
    RegionLine2<LUT_SMEM>(rit, body.rp, p0, p1, sh.cframe, sh.ctile, tile_px, sh.bins, lut_g, lut_s, args.lookup_f,
                          args.lookup_b, L);
  }
  Stamp2<T>(args, sh);  // region lines
}

// Point role, one correspondence iteration: closest view of the depth model (the whole group; with one warp group and
// lines it was searched in LineCorrespondence, and its answer is re-read from the search's slots), then DepthPoint. P
// arrives empty (ItemLoop).
template <int T, bool LINES>
__device__ __forceinline__ void PointCorrespondence(const TrackArgs& args, Shared2& sh, int corr, PointState& P) {
  const BodyDev& body = sh.body;
  const ModelDev* dmodel = &sh.models[1];
  const int view_d = (!LINES || !DoPhase(sh, args, true, PH_REGION_CORR))
                         ? GroupClosestView<T>(args, sh, corr, 1)
                         : ClosestViewOfSlots<kGroup>(sh.view_slots[corr & 1][1], NestTid<T>());
  Stamp2<T>(args, sh);  // closest view (depth)
  DepthIter dit;
  MakeDepthIter(body.dp, sh.cams[1], sh.db2c, sh.dc2b, corr, dit);
  const int item = NestTid<T>() & (kGroup - 1);
  const float4* pts = dmodel->points + size_t(view_d) * dmodel->n_points * 2;
  float4 p0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), p1 = p0;
  if (item < min(dmodel->n_points, min(args.point_cap, kGroup))) { p0 = __ldg(pts + 2 * item); p1 = __ldg(pts + 2 * item + 1); }
  int n_points = AdaptiveCount(body.dp.n_points_max, body.dp.use_adaptive_coverage, body.dp.reference_surface_area,
                               body.dp.use_adaptive_coverage ? __ldg(dmodel->view_scalars + view_d) : 0.0f,
                               dmodel->max_view_scalar, dmodel->n_points);
  n_points = min(n_points, min(args.point_cap, kGroup));
  if (item == 0) sh.n_items[1] = n_points;
  if (corr == args.corr_begin) WaitDepthCopies(sh);
  if (item < n_points) {
    const uint16_t* tile_px = reinterpret_cast<const uint16_t*>(DynSmem() + sh.dtile.offset);
    DepthPoint<false>(dit, body.dp, p0, p1, sh.dframe, sh.dtile, tile_px, P);
  }
  Stamp2<T>(args, sh);  // depth points
}

// Warp sum of the 27 accumulators by recursive halving (see k_track); lane k < 27 returns entry k. One function per
// level, so that every loop has a constant trip count: a loop over the levels is not always unrolled, and then v[] is
// indexed at run time and lives in local memory.
template <int HALF>
__device__ __forceinline__ void HalvingLevel(float (&v)[32], int lane) {
  const bool upper = (lane & HALF) != 0;
#pragma unroll
  for (int k = 0; k < HALF; ++k) {
    const float send = upper ? v[k] : v[k + HALF];
    const float keep = upper ? v[k + HALF] : v[k];
    v[k] = keep + __shfl_xor_sync(0xffffffffu, send, HALF);
  }
}
__device__ __forceinline__ float WarpReduce27(const float (&acc)[27]) {
  const int lane = threadIdx.x & 31;
  float v[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) v[k] = k < 27 ? acc[k] : 0.0f;
  HalvingLevel<16>(v, lane);
  HalvingLevel<8>(v, lane);
  HalvingLevel<4>(v, lane);
  HalvingLevel<2>(v, lane);
  HalvingLevel<1>(v, lane);
  return v[0];
}

// Last warp: cross-warp sum of the per-warp partials, normal equations, solve and pose update. Without the point role
// in the calling group the depth camera's pose products are left to the point group's leader (see ItemLoop).
template <int T, bool POINTS>
__device__ __forceinline__ void SumAndSolve(const TrackArgs& args, Shared2& sh) {
  constexpr int kW = T / 32;
  const int lane = NestTid<T>() & 31;
  const int l = lane < 27 ? lane : 26;
  // cross-warp sum, four interleaved partial sums (fixed order: deterministic)
  float s4[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
  for (int w = 0; w < kW; ++w) s4[w & 3] += sh.red[w][l];
  const float v = (s4[0] + s4[1]) + (s4[2] + s4[3]);
  // Optimizer: b = J^T g, a(lower) = -J^T H J with J = I6, a.diagonal() += tikhonov (optimizer.cpp:144-159)
  int i, j;
  TriInv(l >= 6 ? l - 6 : 0, i, j);
  float aval = 0.0f - v;
  if (i == j) aval += (i < 3) ? sh.body.tikhonov_rotation : sh.body.tikhonov_translation;
  const bool is_b = l < 6;
  float* p1 = is_b ? &sh.b[l] : &sh.a[i * 6 + j];
  float* p2 = is_b ? &sh.b[l] : &sh.a[j * 6 + i];
  const float val = is_b ? 0.0f + v : aval;
  *p1 = val;
  *p2 = val;
  __syncwarp();
  Stamp2<T>(args, sh);  // cross-warp sum + normal equations
  SolveAndUpdateSerial(sh, sh.body.has_region != 0, POINTS && sh.body.has_depth);
  Stamp2<T>(args, sh);  // solve + pose update + pose products
}

// The loop nest of one role (T = 1024: LINES on warps 16-31, POINTS on warps 0-15) or of both (T = 512), followed by
// the role's per-line / per-point records. Across the nest a thread carries its line or point, the accumulators and the
// two loop counters; everything else (counts, views, which copies have landed, and in the 1024-thread kernel the thread
// and block index) is re-derived from shared memory, the kernel parameters or the special registers where it is used. At 64 registers anything more
// went to local memory, an L2 round trip per access with ~3 KB of L1 left next to 225 KB of shared memory.
template <int T, bool LUT_SMEM, bool LINES, bool POINTS>
__device__ __forceinline__ void ItemLoop(const TrackArgs& args, Shared2& sh) {
  constexpr int kW = T / 32;
  LineRegs L = LineRegs{};
  PointState P = PointState{};

  for (int corr = args.corr_begin; corr < args.corr_end; ++corr) {
    // ---------------- CalculateCorrespondences -------------------------------------------------
    // Each iteration starts from an empty line / point: one without an item this iteration keeps nothing of an earlier
    // one (the gradient skips it, its record is not written), and nothing of the previous iteration is live across the
    // closest-view search and the walk. Without the correspondence phase the state stays empty, as it starts.
    L = LineRegs{};
    P = PointState{};
    if (LINES && DoPhase(sh, args, true, PH_REGION_CORR)) LineCorrespondence<T, LUT_SMEM, POINTS>(args, sh, corr, L);
    if (POINTS && DoPhase(sh, args, false, PH_DEPTH_CORR)) PointCorrespondence<T, LINES>(args, sh, corr, P);

    // ---------------- n_update x (CalculateGradientAndHessian + CalculateOptimization) ---------
    for (int upd = 0; upd < args.n_update; ++upd) {
      float acc[27];
#pragma unroll
      for (int k = 0; k < 27; ++k) acc[k] = 0.0f;
      if (LINES) {
        // A line that adds nothing contributes J = 0, wg = wh = 0: its sums, 0 + 0 * 0 and 0 - (0 * 0) * 0, are the +0
        // of untouched accumulators, so the sums are formed on every path. With the zeros written before a conditional
        // gradient instead, all 27 accumulators held a register through it, and at 64 registers the line spilled.
        float J[6], wg, wh;
        if (!(DoPhase(sh, args, true, PH_REGION_GH) &&
              RegionJacobian2(sh.rb2c, sh.cams[0], sh.body.rp, L, DistCol<LUT_SMEM>(), corr, args.opt_base + upd, J, wg,
                              wh))) {
#pragma unroll
          for (int k = 0; k < 6; ++k) J[k] = 0.0f;
          wg = wh = 0.0f;
        }
        AddRegionSums(J, wg, wh, acc);
      }
      if (POINTS && DoPhase(sh, args, false, PH_DEPTH_GH)) {
        DepthIter dit;  // registers: DepthGradient reads the pose products (dc2b) and the deviation only
        MakeDepthIter(sh.body.dp, sh.cams[1], sh.db2c, sh.dc2b, corr, dit);
        DepthGradient(dit, P, acc);
      }
      const float red = WarpReduce27(acc);
      sh.red[NestTid<T>() >> 5][NestTid<T>() & 31] = red;
      Stamp2<T>(args, sh);  // accumulate + warp reduce
      __syncthreads();
      Stamp2<T>(args, sh);  // all warps arrived
      if (LINES && (NestTid<T>() >> 5) == kW - 1) SumAndSolve<T, POINTS>(args, sh);
      __syncthreads();
      if (!LINES && sh.body.has_depth) {
        // the depth camera's pose products: off the critical path here, so the serial section every warp waits for
        // gets shorter
        if ((NestTid<T>() & (kGroup - 1)) >= kGroup - 32) {
          float pose[12];
#pragma unroll
          for (int i = 0; i < 12; ++i) pose[i] = sh.pose[i];
          PublishPoseProducts(pose, false, true, false, sh);
        }
        GroupBarrier<T>(1);
      }
      Stamp2<T>(args, sh);  // released
    }
  }

  // ---------------- the role's records ------------------------------------------------------------
  // The counts in sh.n_items come from item 0 of the group: one group barrier before they are read (the update loop's
  // barriers order them too, but it may have had no iteration).
  const BodyDev& body = sh.body;
  const int body_id = NestCta<T>(), item = NestTid<T>() & (kGroup - 1);
  int* counts = args.counts + 4 * body_id;
  if (LINES && (args.phases & PH_STORE_REGION) && body.has_region) {
    GroupBarrier<T>(0);
    const int n_lines = sh.n_items[0];
    const int lcap = args.line_cap;
    float* g_rst = args.region_state + size_t(body_id) * RF_COUNT * lcap;
    if (item < n_lines) {
      const int i = item;
      g_rst[RF_CBX * lcap + i] = L.cbx; g_rst[RF_CBY * lcap + i] = L.cby; g_rst[RF_CBZ * lcap + i] = L.cbz;
      g_rst[RF_CU * lcap + i] = L.cu; g_rst[RF_CV * lcap + i] = L.cv;
      g_rst[RF_NU * lcap + i] = L.nu; g_rst[RF_NV * lcap + i] = L.nv;
      g_rst[RF_VALID * lcap + i] = L.valid ? 1.0f : 0.0f;
      if (L.valid) {
        g_rst[RF_DR * lcap + i] = L.dr; g_rst[RF_NCTS * lcap + i] = L.ncts;
        g_rst[RF_MEAN * lcap + i] = L.mean; g_rst[RF_VAR * lcap + i] = L.var;
#pragma unroll
        for (int d = 0; d < kDistributionLength; ++d) g_rst[(RF_DIST0 + d) * lcap + i] = DistCol<LUT_SMEM>()[d * kGroup];
      }
    }
    const int view_r = RecordView<T>(args, sh, DoPhase(sh, args, true, PH_REGION_CORR), 0);
    if (item == 0) { counts[0] = n_lines; counts[2] = view_r; }
  }
  if (POINTS && (args.phases & PH_STORE_DEPTH) && body.has_depth) {
    GroupBarrier<T>(1);
    const int n_points = sh.n_items[1];
    const int pcap = args.point_cap;
    float* g_dst = args.depth_state + size_t(body_id) * DF_COUNT * pcap;
    if (item < n_points) {
      const int i = item;
      g_dst[DF_CBX * pcap + i] = P.cbx; g_dst[DF_CBY * pcap + i] = P.cby; g_dst[DF_CBZ * pcap + i] = P.cbz;
      g_dst[DF_NX * pcap + i] = P.nx; g_dst[DF_NY * pcap + i] = P.ny; g_dst[DF_NZ * pcap + i] = P.nz;
      g_dst[DF_VALID * pcap + i] = P.valid ? 1.0f : 0.0f;
      if (P.valid) {
        g_dst[DF_YX * pcap + i] = P.yx; g_dst[DF_YY * pcap + i] = P.yy; g_dst[DF_YZ * pcap + i] = P.yz;
      }
    }
    const int view_d = RecordView<T>(args, sh, DoPhase(sh, args, false, PH_DEPTH_CORR), 1);
    if (item == 0) { counts[1] = n_points; counts[3] = view_d; }
  }
}

// ---------------------------------------------------------------------------------------------
// The kernel. T = 1024: points on warps 0-15, lines on warps 16-31. T = 512: one group does both in turn
// (batches in which no body has both modalities).
// ---------------------------------------------------------------------------------------------
template <int T, bool LUT_SMEM>
__global__ void __launch_bounds__(T, 1) k_track2(const __grid_constant__ TrackArgs args) {
  extern __shared__ __align__(128) unsigned char dyn[];
  __shared__ Shared2 sh;
  constexpr int kW = T / 32;
  const int body_id = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const BodyDev& gbody = args.bodies[body_id];
  if (!gbody.set) return;
  {  // per-body copies (Shared2::body, cams, models)
    const int* src = reinterpret_cast<const int*>(&gbody);
    int* dst = reinterpret_cast<int*>(&sh.body);
    for (int k = tid; k < int(sizeof(BodyDev) / 4); k += T) dst[k] = __ldg(src + k);
    if (gbody.has_region) {
      const int* c = reinterpret_cast<const int*>(&args.color_cams[gbody.color_camera]);
      const int* m = reinterpret_cast<const int*>(&args.region_models[gbody.region_model]);
      for (int k = tid; k < int(sizeof(CameraDev) / 4); k += T) reinterpret_cast<int*>(&sh.cams[0])[k] = __ldg(c + k);
      for (int k = tid; k < int(sizeof(ModelDev) / 4); k += T) reinterpret_cast<int*>(&sh.models[0])[k] = __ldg(m + k);
    }
    if (gbody.has_depth) {
      const int* c = reinterpret_cast<const int*>(&args.depth_cams[gbody.depth_camera]);
      const int* m = reinterpret_cast<const int*>(&args.depth_models[gbody.depth_model]);
      for (int k = tid; k < int(sizeof(CameraDev) / 4); k += T) reinterpret_cast<int*>(&sh.cams[1])[k] = __ldg(c + k);
      for (int k = tid; k < int(sizeof(ModelDev) / 4); k += T) reinterpret_cast<int*>(&sh.models[1])[k] = __ldg(m + k);
    }
    if (tid < 2) {
      sh.stamp_n[tid] = 0;
      sh.view0[tid] = args.counts[4 * body_id + 2 + tid];  // any valid view index: the first search's lower bound
      sh.n_items[tid] = 0;
    }
  }
  __syncthreads();
  M3TB_STAMP_AT(120, tid == T - 32);
  const BodyDev& body = sh.body;
  const bool has_region = body.has_region, has_depth = body.has_depth;
  const float2* lut_g = args.lut + size_t(body_id) * args.lut_stride;
  constexpr unsigned lut_bytes = kLutBytes<LUT_SMEM>;
  Stamp2<T>(args, sh);

  // ---- prologue: pose, LUT bulk copy, ROI tiles (as in k_track) -----------------------------------------
  const CameraDev* ccam = has_region ? &sh.cams[0] : nullptr;
  const CameraDev* dcam = has_depth ? &sh.cams[1] : nullptr;
  const ModelDev* rmodel = has_region ? &sh.models[0] : nullptr;
  const ModelDev* dmodel = has_depth ? &sh.models[1] : nullptr;
  const bool do_rcorr = has_region && (args.phases & PH_REGION_CORR);
  const bool do_dcorr = has_depth && (args.phases & PH_DEPTH_CORR);
  FrameView cframe, dframe;
  cframe.dev = cframe.host = dframe.dev = dframe.host = nullptr;
  cframe.dev_pitch = cframe.host_pitch = dframe.dev_pitch = dframe.host_pitch = 0u;
  cframe.x0 = cframe.y0 = cframe.x1 = cframe.y1 = dframe.x0 = dframe.y0 = dframe.x1 = dframe.y1 = 0;
  if (ccam) cframe = MakeFrameView(*ccam, args.roi[2 * body_id + 0]);
  if (dcam) dframe = MakeFrameView(*dcam, args.roi[2 * body_id + 1]);
  if (tid < 12) sh.pose[tid] = args.poses[12 * body_id + tid];
  if (tid >= 32 && tid < 44 && ccam) sh.cw2c[tid - 32] = ccam->w2c[tid - 32];
  if (tid >= 64 && tid < 76 && dcam) sh.dw2c[tid - 64] = dcam->w2c[tid - 64];
  // cluster tables of the pruned closest-view search: shared memory when they fit (they are read every iteration)
  float4* cl_smem = reinterpret_cast<float4*>(dyn + lut_bytes + kDistBytes);
  const bool stage_r = do_rcorr && rmodel->n_clusters <= kClusterStage;
  const bool stage_d = do_dcorr && dmodel->n_clusters <= kClusterStage;
  if (stage_r)
    for (int k = tid; k < 2 * rmodel->n_clusters; k += T) cl_smem[k] = __ldg(rmodel->cluster_info + k);
  if (stage_d)
    for (int k = tid; k < 2 * dmodel->n_clusters; k += T) cl_smem[2 * kClusterStage + k] = __ldg(dmodel->cluster_info + k);
  const bool need_lut = LUT_SMEM && do_rcorr;
  const bool tma = args.tma_mode != 0;
  if (tid == 0) {
    if (LUT_SMEM) MbarInit(&sh.lut_bar, 1);
    MbarInit(&sh.depth_bar, 1);
    MbarInit(&sh.ctile_bar, 1);
    sh.cframe = cframe;
    sh.dframe = dframe;
    sh.info[0] = stage_r ? cl_smem : (rmodel ? rmodel->cluster_info : nullptr);
    sh.info[1] = stage_d ? cl_smem + 2 * kClusterStage : (dmodel ? dmodel->cluster_info : nullptr);
    // the bin-index image is valid wherever the device copy of the colour frame is (the body's ROI), when the TMA path
    // maintains it
    sh.bins.px = (tma && ccam) ? ccam->bins : nullptr;
    sh.bins.pitch = ccam ? ccam->bin_pitch : 0u;
  }
  __syncthreads();
  M3TB_STAMP_AT(121, tid == T - 32);
  if (warp == kW - 1) {
    float pose[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) pose[i] = sh.pose[i];
    PublishPoseProducts(pose, ccam != nullptr, dcam != nullptr, false, sh);
    M3TB_STAMP_AT(122, lane == 0);
  }
  if (need_lut && tid == 0) {
    const unsigned bytes = unsigned(body.rp.n_bins * body.rp.n_bins * body.rp.n_bins) * sizeof(float2);
    MbarExpectTx(&sh.lut_bar, bytes);
    BulkCopyG2S(dyn, lut_g, bytes, &sh.lut_bar);
  }
  if (tma) {
    // ROI tiles: one thread sizes them and issues the TMA tensor copies (cp.async.bulk.tensor.3d, SASS UTMALDG): the
    // colour tile comes from the camera's BIN-INDEX image (u16 per pixel, written once per frame by k_bin / k_ingest),
    // the depth tile from the raw U16 frame; boxes of kTileBoxRows rows x the tile width, stacked -> row-major tile.
    if (tid == 32 % T) {
      M3TB_STAMP_AT(124, true);
      Tile ct, dt;
      ct.x0 = ct.y0 = ct.w = ct.h = ct.pitch = 0; ct.offset = lut_bytes + kFixedDynBytes;
      dt = ct;
      if (args.tile_bytes > 0) {
        float b2c[12];
        if (do_rcorr) {
          int s_max = 1;
          for (int c = args.corr_begin; c < args.corr_end; ++c) s_max = max(s_max, LastValid(body.rp.scales, body.rp.n_scales, c));
          PoseMul(ccam->w2c, sh.pose, b2c);
          RoiRect(b2c, ccam->fu, ccam->fv, ccam->ppu, ccam->ppv, ccam->width, ccam->height, rmodel->radius,
                  0.5f * float(kLineSegments * s_max) + 2.0f + 12.0f, 1, ct);
        }
        if (do_dcorr) {
          float d_max = 0.0f;
          for (int c = args.corr_begin; c < args.corr_end; ++c)
            d_max = fmaxf(d_max, LastValid(body.dp.considered_distances, body.dp.n_considered_distances, c));
          PoseMul(dcam->w2c, sh.pose, b2c);
          const float z = b2c[11];
          const float reach = (z > 2.0f * dmodel->radius) ? d_max * dcam->fu / (z - dmodel->radius) + 2.0f + 8.0f : 0.0f;
          RoiRect(b2c, dcam->fu, dcam->fv, dcam->ppu, dcam->ppv, dcam->width, dcam->height, dmodel->radius, reach, 1, dt);
        }
        // split the budget: the depth tile is the smaller one, give it what it asks for up to 40 %
        const int budget = args.tile_bytes - 256;
        SnapTile(dt, dframe, budget * 2 / 5, args.tma_max_w);
        const int dbytes = dt.w * dt.h * 2;
        SnapTile(ct, cframe, budget - dbytes, args.tma_max_w);
        dt.offset = lut_bytes + kFixedDynBytes + unsigned(ct.w * ct.h * 2);
      }
      sh.ctile = ct;
      sh.dtile = dt;
      M3TB_STAMP_AT(125, true);
      if (ct.w > 0) {
        const CUtensorMap* map = (args.tma_mode == 2 ? args.tmaps_global : args.bin_maps) + ((ct.w - 64) >> 5);
        MbarExpectTx(&sh.ctile_bar, unsigned(ct.w * ct.h * 2));
#pragma unroll 1
        for (int r = 0; r < ct.h; r += kTileBoxRows)
          TensorCopyG2S(dyn + ct.offset + size_t(r) * ct.w * 2, map, ct.x0, ct.y0 + r, body.color_camera, &sh.ctile_bar);
      }
      if (dt.w > 0) {
        const CUtensorMap* map = (args.tma_mode == 2 ? args.tmaps_global + kTileWidths : args.depth_maps) + ((dt.w - 64) >> 5);
        MbarExpectTx(&sh.depth_bar, unsigned(dt.w * dt.h * 2));
#pragma unroll 1
        for (int r = 0; r < dt.h; r += kTileBoxRows)
          TensorCopyG2S(dyn + dt.offset + size_t(r) * dt.w * 2, map, dt.x0, dt.y0 + r, body.depth_camera, &sh.depth_bar);
      }
      M3TB_STAMP_AT(126, true);
    }
  } else {  // legacy staging (tma_mode 0): depth rows by 1-D bulk copies, colour bins converted from the BGR frame
    if (tid == 32 % T) {
      Tile ct, dt;
      ct.x0 = ct.y0 = ct.w = ct.h = ct.pitch = 0; ct.offset = lut_bytes + kFixedDynBytes;
      dt = ct;
      if (args.tile_bytes > 0) {
        float b2c[12];
        if (do_rcorr) {
          int s_max = 1;
          for (int c = args.corr_begin; c < args.corr_end; ++c) s_max = max(s_max, LastValid(body.rp.scales, body.rp.n_scales, c));
          PoseMul(ccam->w2c, sh.pose, b2c);
          RoiRect(b2c, ccam->fu, ccam->fv, ccam->ppu, ccam->ppv, ccam->width, ccam->height, rmodel->radius,
                  0.5f * float(kLineSegments * s_max) + 2.0f + 12.0f, 4, ct);
        }
        if (do_dcorr) {
          float d_max = 0.0f;
          for (int c = args.corr_begin; c < args.corr_end; ++c)
            d_max = fmaxf(d_max, LastValid(body.dp.considered_distances, body.dp.n_considered_distances, c));
          PoseMul(dcam->w2c, sh.pose, b2c);
          const float z = b2c[11];
          const float reach = (z > 2.0f * dmodel->radius) ? d_max * dcam->fu / (z - dmodel->radius) + 2.0f + 8.0f : 0.0f;
          RoiRect(b2c, dcam->fu, dcam->fv, dcam->ppu, dcam->ppv, dcam->width, dcam->height, dmodel->radius, reach, 8, dt);
        }
        ClipTile(ct, cframe, 4);
        ClipTile(dt, dframe, 8);
        int budget = args.tile_bytes - 256;
        FitTile(dt, budget * 2 / 5, 8);
        const int dbytes = (dt.w * dt.h * 2 + 127) / 128 * 128;
        FitTile(ct, budget - dbytes, 4);
        const int cbytes = (ct.w * ct.h * 2 + 127) / 128 * 128;
        dt.offset = lut_bytes + kFixedDynBytes + unsigned(cbytes);
      }
      sh.ctile = ct;
      sh.dtile = dt;
    }
  }
  __syncthreads();  // tiles sized (TMA copies in flight); also orders the initial pose products before their first readers
  const Tile ctile = sh.ctile, dtile = sh.dtile;
  if (!tma) {
    if (dtile.w > 0) {
      if (warp == 0) {  // a point warp issues the depth rows while the others convert the colour tile
        const unsigned row_bytes = unsigned(dtile.w) * 2u;
        if (lane == 0) MbarExpectTx(&sh.depth_bar, row_bytes * unsigned(dtile.h));
        __syncwarp();
        for (int r = lane; r < dtile.h; r += 32)
          BulkCopyG2S(dyn + dtile.offset + size_t(r) * row_bytes,
                      dcam->image + size_t(dtile.y0 + r) * dcam->pitch + size_t(dtile.x0) * 2u, row_bytes, &sh.depth_bar);
      }
    }
    if (ctile.w > 0) {
      const int groups_per_row = ctile.w >> 2;
      const int n_groups = groups_per_row * ctile.h;
      const int bs = body.rp.bitshift, nb = body.rp.n_bins;
      uint2* out = reinterpret_cast<uint2*>(dyn + ctile.offset);
      auto bin = [&](unsigned b, unsigned gch, unsigned rch) {
        return LutSlot(((b >> bs) * unsigned(nb) + (gch >> bs)) * unsigned(nb) + (rch >> bs));
      };
      for (int g0 = tid; g0 < n_groups; g0 += 4 * T) {
        unsigned w[4][3];
  #pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int g = g0 + u * T;
          if (g < n_groups) {
            const int r = g / groups_per_row, c = g - r * groups_per_row;
            const unsigned* src = reinterpret_cast<const unsigned*>(ccam->image + size_t(ctile.y0 + r) * ccam->pitch +
                                                                    size_t(ctile.x0 + 4 * c) * 3u);
            w[u][0] = __ldg(src); w[u][1] = __ldg(src + 1); w[u][2] = __ldg(src + 2);
          }
        }
  #pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int g = g0 + u * T;
          if (g < n_groups) {
            const unsigned w0 = w[u][0], w1 = w[u][1], w2 = w[u][2];
            const unsigned i0 = bin(w0 & 0xffu, (w0 >> 8) & 0xffu, (w0 >> 16) & 0xffu);
            const unsigned i1 = bin(w0 >> 24, w1 & 0xffu, (w1 >> 8) & 0xffu);
            const unsigned i2 = bin((w1 >> 16) & 0xffu, w1 >> 24, w2 & 0xffu);
            const unsigned i3 = bin((w2 >> 8) & 0xffu, (w2 >> 16) & 0xffu, w2 >> 24);
            out[g] = make_uint2(i0 | (i1 << 16), i2 | (i3 << 16));
          }
        }
      }
    }
    __syncthreads();  // colour tile complete
  }

  Stamp2<T>(args, sh);  // prologue done

  // Warp priority: an SM sub-partition issues from its highest-numbered eligible warp first. The lines are the critical
  // path of every iteration (the points finish earlier and wait), so they get the HIGH warps, and the single-warp
  // sections (view search, solve) run on the last warp of their group.
  if (T == kGroup) ItemLoop<T, LUT_SMEM, true, true>(args, sh);
  else if (tid >= kGroup) ItemLoop<T, LUT_SMEM, true, false>(args, sh);
  else ItemLoop<T, LUT_SMEM, false, true>(args, sh);

  // ---------------- epilogue ----------------------------------------------------------------------
  if (args.phases & PH_SOLVE)
    if (NestTid<T>() < 12) args.poses[12 * NestCta<T>() + NestTid<T>()] = sh.pose[NestTid<T>()];
  // never leave with a bulk copy in flight
  if (DoPhase(sh, args, true, PH_REGION_CORR)) WaitColourCopies<LUT_SMEM>(args, sh);
  WaitDepthCopies(sh);
}

}  // namespace m3tb
