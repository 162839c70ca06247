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
//     iteration), done by the last warp of each group while the other warps wait at the group's named barrier
//     (every warp searching redundantly would spend the issue slots of the whole group on the same search).
//   * CalculateOptimization (6 x 6) runs thread-serially in registers on warp 0 (every lane the same work, no
//     shuffles in the dependent chain): pivot order from the original diagonal, gather of the permuted matrix,
//     unrolled left-looking LDL^T, substitutions, Rodrigues, pose products; shorter than the lane-parallel form.
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
  int views[2][2];           // [corr parity][region | depth] closest views, published by the group leaders
};

// barrier of one warp group (512 threads) when the CTA has two; id 1 = lines, id 2 = points
template <int T>
__device__ __forceinline__ void GroupBarrier(int group) {
  if (T == kGroup) __syncthreads();
  else asm volatile("bar.sync %0, %1;" ::"r"(group + 1), "r"(kGroup) : "memory");
}

struct LineRegs {  // RegionModality::DataLine without the distribution (shared memory)
  float cbx, cby, cbz, cu, cv, nu, nv, dr, ncts, mean, var;
  bool valid;
};

#define M3TB_STAMP2(base)                                                                                   \
  do {                                                                                                      \
    if (stamp_ptr && lane == 0 && stamp_i < kPhaseSlots / 2) stamp_ptr[(base) + stamp_i++] = clock64();     \
  } while (0)

// prologue detail (profiling aid): fixed slots past the ones M3TB_STAMP2 fills
#define M3TB_STAMP_AT(slot, cond)                                                                  \
  do {                                                                                             \
    if (args.phase_clock && (cond)) args.phase_clock[size_t(body_id) * kPhaseSlots + (slot)] = clock64(); \
  } while (0)

// ---------------------------------------------------------------------------------------------
// One correspondence line, streaming form. Walks the 19 segments of the line in pixel order; after segment w >= 7 the
// distribution entry that has just become computable is finished from the 8-segment window:
//   line walked front to back (n_major > 0): entry d = w - 7 uses the segments walked at w-7 .. w, in that order;
//   line walked back to front: segment index = 18 - walk index (region_modality.cpp:1470-1484), so entry d = 18 - w
//   uses the segments walked at w, w-1, .. w-7, in that order.
// Either way the factors are multiplied for k = 0..7 exactly as CalculateDistribution does.
// ---------------------------------------------------------------------------------------------
template <bool LUT_SMEM, int S>
__device__ __forceinline__ void WalkFast(int scale, int base, float minor_f, float step, int stride_major, int stride_minor,
                                         const uint16_t* tile_px, const float2* __restrict__ lut_g, const float2* lut_s,
                                         const float* __restrict__ lf, const float* __restrict__ lb, bool rev,
                                         float* dist_col) {
  float wf[8], wb[8];
#pragma unroll
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
    wf[w & 7] = pf;
    wb[w & 7] = pb;
    if (w >= 7) {
      float val = 1.0f;
#pragma unroll
      for (int k = 0; k < kFunctionLength; ++k) {
        const float f = rev ? wf[(w - k) & 7] : wf[(w + 1 + k) & 7];
        const float b = rev ? wb[(w - k) & 7] : wb[(w + 1 + k) & 7];
        val *= f * lf[k] + b * lb[k];
      }
      dist_col[(rev ? kLineSegments - 1 - w : w - 7) * kGroup] = val;
    }
  }
}

// Rare path: a sample may lie outside the tile. All 19 segments go to local memory first (as in k_track). Samples
// outside the tile come from the camera's bin-index image where it is valid (inside the body's ROI), else from the frame.
struct BinImage {
  const uint16_t* px;  // null: no bin-index image
  unsigned pitch;      // bytes
};
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
                                            const float* __restrict__ lf, const float* __restrict__ lb,
                                            float* dist_col, LineRegs& L) {
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
        case 1: WalkFast<LUT_SMEM, 1>(1, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, lf, lb, rev, dist_col); break;
        case 2: WalkFast<LUT_SMEM, 2>(2, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, lf, lb, rev, dist_col); break;
        case 4: WalkFast<LUT_SMEM, 4>(4, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, lf, lb, rev, dist_col); break;
        case 6: WalkFast<LUT_SMEM, 6>(6, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, lf, lb, rev, dist_col); break;
        default: WalkFast<LUT_SMEM, 0>(it.scale, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, lf, lb, rev, dist_col); break;
      }
    } else {
      WalkSlow<LUT_SMEM>(it.scale, rp.bitshift, rp.n_bins, horizontal, major, minor_f, step, frame, tile, tile_px, bins,
                         lut_g, lut_s, lf, lb, rev, dist_col);
    }
  }
  L.ncts = fabsf(n_major) / it.fscale;
  L.dr = (roundf(c_major - it.ll_m1_half) + it.ll_m1_half - c_major) / n_major;
  // CalculateDistribution, normalisation (:1630-1636) and CalculateDistributionMoments (:1639-1658)
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

// K2 region (region_modality.cpp:485-558); the two distribution entries of the local mode come from shared memory
__device__ __forceinline__ void RegionGradient2(const RegionIter& it, const RegionParamsDev& rp, const LineRegs& L,
                                                const float* dist_col, int opt_iteration, float (&acc)[27]) {
  if (!L.valid) return;
  float x, y, z;
  PoseApply(it.b2c, L.cbx, L.cby, L.cbz, x, y, z);
  float fu_z = it.fu / z, fv_z = it.fv / z;
  float xfu_z = x * fu_z, yfv_z = y * fv_z;
  float delta_cs = (L.nu * (xfu_z + it.ppu - L.cu) + L.nv * (yfv_z + it.ppv - L.cv) - L.dr) * L.ncts;
  float dll;
  if (opt_iteration < rp.n_global_iterations) {
    dll = (L.mean - delta_cs) / L.var;
  } else {
    int upper = int(delta_cs + (float(kDistributionLength) + 1.0f) / 2.0f);
    int lower = upper - 1;
    if (upper <= 0 || upper >= kDistributionLength) return;
    dll = (logf(dist_col[upper * kGroup]) - logf(dist_col[lower * kGroup])) * rp.learning_rate / L.var;
  }
  float dc0 = L.ncts * L.nu * fu_z;
  float dc1 = L.ncts * L.nv * fv_z;
  float dc2 = L.ncts * (-L.nu * xfu_z - L.nv * yfv_z) / z;
  float J[6];
  J[3] = dc0 * it.b2c[0] + dc1 * it.b2c[4] + dc2 * it.b2c[8];
  J[4] = dc0 * it.b2c[1] + dc1 * it.b2c[5] + dc2 * it.b2c[9];
  J[5] = dc0 * it.b2c[2] + dc1 * it.b2c[6] + dc2 * it.b2c[10];
  J[0] = L.cby * J[5] - L.cbz * J[4];
  J[1] = L.cbz * J[3] - L.cbx * J[5];
  J[2] = L.cbx * J[4] - L.cby * J[3];
  float weight = rp.min_expected_variance / (L.ncts * L.ncts * it.variance);
  float wg = weight * dll;
  float wh = weight / L.var;
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
// Pose products, thread-serial (every calling lane computes everything; lane 0 publishes). Expressions are those of
// PoseMul / PoseInverse / ViewOrientation, i.e. of PoseProductsWarp in k_track.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void PublishPoseProducts(const float (&pose)[12], bool has_color, bool has_depth, bool store_pose,
                                                    Shared2& sh) {
  const bool writer = (threadIdx.x & 31) == 0;
  if (store_pose && writer) {
#pragma unroll
    for (int i = 0; i < 12; ++i) sh.pose[i] = pose[i];
  }
  if (has_color) {
    float w[12], o[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) w[i] = sh.cw2c[i];
    PoseMul(w, pose, o);
    float v0 = 0.0f, v1 = 0.0f, v2 = 0.0f;
    const bool nz = ViewOrientation(o, v0, v1, v2);
    if (writer) {
#pragma unroll
      for (int i = 0; i < 12; ++i) sh.rb2c[i] = o[i];
      sh.view_o[0][0] = v0; sh.view_o[0][1] = v1; sh.view_o[0][2] = v2; sh.view_o[0][3] = nz ? 1.0f : 0.0f;
    }
  }
  if (has_depth) {
    float w[12], o[12], inv[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) w[i] = sh.dw2c[i];
    PoseMul(w, pose, o);
    PoseInverse(o, inv);
    float v0 = 0.0f, v1 = 0.0f, v2 = 0.0f;
    const bool nz = ViewOrientation(o, v0, v1, v2);
    if (writer) {
#pragma unroll
      for (int i = 0; i < 12; ++i) { sh.db2c[i] = o[i]; sh.dc2b[i] = inv[i]; }
      sh.view_o[1][0] = v0; sh.view_o[1][1] = v1; sh.view_o[1][2] = v2; sh.view_o[1][3] = nz ? 1.0f : 0.0f;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// K4, thread-serial: Optimizer::CalculateOptimization for a rigid body (optimizer.cpp:144-167) = Eigen LDLT<Lower>
// (pivot = largest remaining diagonal entry, first maximum wins; left-looking update) restated for n = 6, then
// Link::UpdatePoses (link.cpp:205-241). Same arithmetic, element by element, as SolveAndUpdateWarp of k_track; the
// difference is that one thread holds the whole permuted matrix in registers, so the dependent chain contains no
// shuffles or shared-memory round trips. sh.a (full symmetric 6x6) and sh.b must be visible to the calling warp.
// Returns true if the pose was updated (sh.pose and the pose products are then refreshed).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool SolveAndUpdateSerial(Shared2& sh, bool has_color, bool has_depth) {
  constexpr int n = 6;
  // 1. transposition sequence from the ORIGINAL diagonal (see SolveAndUpdateWarp)
  unsigned key[n];
  int pm[n];
#pragma unroll
  for (int i = 0; i < n; ++i) { key[i] = __float_as_uint(fabsf(sh.a[i * (n + 1)])); pm[i] = i; }
#pragma unroll
  for (int k = 0; k < n - 1; ++k) {
    int p = k;
    unsigned big = key[k];
#pragma unroll
    for (int q = k + 1; q < n; ++q)
      if (key[q] > big) { big = key[q]; p = q; }
#pragma unroll
    for (int q = k + 1; q < n; ++q)
      if (p == q) {
        const unsigned tk = key[k]; key[k] = key[q]; key[q] = tk;
        const int tp = pm[k]; pm[k] = pm[q]; pm[q] = tp;
      }
  }
  // 2. lower triangle of P A P^T and P b
  float A[n][n];
  float dst[n];
#pragma unroll
  for (int i = 0; i < n; ++i) {
#pragma unroll
    for (int j = 0; j <= i; ++j) A[i][j] = sh.a[pm[i] * n + pm[j]];
    dst[i] = sh.b[pm[i]];
  }
  // 3. ldlt_inplace<Lower>::unblocked
  float D[n];
  bool zero_matrix = false;
#pragma unroll
  for (int k = 0; k < n; ++k) {
    if (k > 0) {
      float temp[n];
#pragma unroll
      for (int j = 0; j < k; ++j) temp[j] = D[j] * A[k][j];
#pragma unroll
      for (int i = k; i < n; ++i) {
        float acc = 0.0f;
#pragma unroll
        for (int j = 0; j < k; ++j) acc += A[i][j] * temp[j];
        if (!zero_matrix) A[i][k] -= acc;
      }
    }
    const float akk = A[k][k];
    const bool pivot_is_valid = fabsf(akk) > 0.0f;
    if (k == 0 && !pivot_is_valid) zero_matrix = true;
    D[k] = akk;
    if (!zero_matrix && pivot_is_valid) {
#pragma unroll
      for (int i = k + 1; i < n; ++i) A[i][k] /= akk;
    }
  }
  // 4. LDLT::_solve_impl: L^-1, D^-1 (tolerance 1/highest), L^-T, P^T
#pragma unroll
  for (int j = 0; j < n; ++j) {
#pragma unroll
    for (int r = j + 1; r < n; ++r) dst[r] -= A[r][j] * dst[j];
  }
  {
    const float tolerance = 1.0f / 3.402823466e+38f;
#pragma unroll
    for (int r = 0; r < n; ++r) {
      if (fabsf(D[r]) > tolerance) dst[r] /= D[r];
      else dst[r] = 0.0f;
    }
  }
#pragma unroll
  for (int j = n - 1; j >= 1; --j) {
#pragma unroll
    for (int r = 0; r < j; ++r) dst[r] -= A[j][r] * dst[j];
  }
  __syncwarp();
#pragma unroll
  for (int r = 0; r < n; ++r) sh.x[pm[r]] = dst[r];  // every lane stores the same value to the same address
  __syncwarp();
  float theta[n];
  bool nan = false;
#pragma unroll
  for (int i = 0; i < n; ++i) { theta[i] = sh.x[i]; nan = nan || isnan(theta[i]); }
  if (nan) return false;  // optimizer.cpp:165
  float e[9];
  ExpSkew(theta, e);
  float var[12] = {e[0], e[1], e[2], theta[3], e[3], e[4], e[5], theta[4], e[6], e[7], e[8], theta[5]};
  float cur[12], np[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) cur[i] = sh.pose[i];
  PoseMul(cur, var, np);  // link2world * [exp | t] (link.cpp:222-238, body2joint = I)
  __syncwarp();
  PublishPoseProducts(np, has_color, has_depth, true, sh);
  return true;
}

// ---------------------------------------------------------------------------------------------
// The kernel. T = 1024: lines on warps 0-15, points on warps 16-31. T = 512: one group does both in turn
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
  // Per-body parameters, cameras and model headers are read all over the iteration loops. With 225 KB of the SM's
  // 228 KB configured as shared memory the L1 cache is ~3 KB, so from global memory each of those reads is an L2 round
  // trip (long-scoreboard stalls); one copy into shared memory instead.
  __shared__ BodyDev s_body;
  __shared__ CameraDev s_cams[2];
  __shared__ ModelDev s_models[2];
  {
    const int* src = reinterpret_cast<const int*>(&gbody);
    int* dst = reinterpret_cast<int*>(&s_body);
    for (int k = tid; k < int(sizeof(BodyDev) / 4); k += T) dst[k] = __ldg(src + k);
    if (gbody.has_region) {
      const int* c = reinterpret_cast<const int*>(&args.color_cams[gbody.color_camera]);
      const int* m = reinterpret_cast<const int*>(&args.region_models[gbody.region_model]);
      for (int k = tid; k < int(sizeof(CameraDev) / 4); k += T) reinterpret_cast<int*>(&s_cams[0])[k] = __ldg(c + k);
      for (int k = tid; k < int(sizeof(ModelDev) / 4); k += T) reinterpret_cast<int*>(&s_models[0])[k] = __ldg(m + k);
    }
    if (gbody.has_depth) {
      const int* c = reinterpret_cast<const int*>(&args.depth_cams[gbody.depth_camera]);
      const int* m = reinterpret_cast<const int*>(&args.depth_models[gbody.depth_model]);
      for (int k = tid; k < int(sizeof(CameraDev) / 4); k += T) reinterpret_cast<int*>(&s_cams[1])[k] = __ldg(c + k);
      for (int k = tid; k < int(sizeof(ModelDev) / 4); k += T) reinterpret_cast<int*>(&s_models[1])[k] = __ldg(m + k);
    }
  }
  __syncthreads();
  M3TB_STAMP_AT(120, tid == T - 32);
  const BodyDev& body = s_body;
  const bool has_region = body.has_region, has_depth = body.has_depth;
  const int item = tid & (kGroup - 1);
  // Warp priority: an SM sub-partition issues from its highest-numbered eligible warp first. The lines are the critical
  // path of every iteration (the points finish earlier and wait), so they get the HIGH warps, and the single-warp
  // sections (view search, solve) run on the last warp of their group.
  const bool line_group = T == kGroup || tid >= kGroup;
  const bool point_group = T == kGroup || tid < kGroup;
  const bool group_leader = (tid & (kGroup - 1)) >= kGroup - 32;
  const int lcap = args.line_cap, pcap = args.point_cap;
  float* g_rst = args.region_state + size_t(body_id) * RF_COUNT * lcap;
  float* g_dst = args.depth_state + size_t(body_id) * DF_COUNT * pcap;
  int* counts = args.counts + 4 * body_id;
  const float2* lut_g = args.lut + size_t(body_id) * args.lut_stride;
  const float2* lut_s = reinterpret_cast<const float2*>(dyn);
  constexpr unsigned lut_bytes = LUT_SMEM ? unsigned(16 * 16 * 16 * sizeof(float2)) : 0u;
  float* dist_col = reinterpret_cast<float*>(dyn + lut_bytes) + item;

  // profiling aid: the solver warp (last warp) stamps slots [0, 128), the point group's leader warp slots [128, 256)
  long long* stamp_ptr = nullptr;
  int stamp_i = 0;
  const int stamp_base = (T > kGroup && tid < kGroup) ? kPhaseSlots / 2 : 0;
  if (args.phase_clock && (warp == kW - 1 || (T > kGroup && warp == kGroup / 32 - 1)))
    stamp_ptr = args.phase_clock + size_t(body_id) * kPhaseSlots;
  M3TB_STAMP2(stamp_base);

  // ---- prologue: pose, LUT bulk copy, ROI tiles (as in k_track) -----------------------------------------
  const CameraDev* ccam = has_region ? &s_cams[0] : nullptr;
  const CameraDev* dcam = has_depth ? &s_cams[1] : nullptr;
  const ModelDev* rmodel = has_region ? &s_models[0] : nullptr;
  const ModelDev* dmodel = has_depth ? &s_models[1] : nullptr;
  const bool do_rcorr = has_region && (args.phases & PH_REGION_CORR);
  const bool do_dcorr = has_depth && (args.phases & PH_DEPTH_CORR);
  const bool do_rgh = has_region && (args.phases & PH_REGION_GH);
  const bool do_dgh = has_depth && (args.phases & PH_DEPTH_GH);
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
  const float4* info_r = stage_r ? cl_smem : (rmodel ? rmodel->cluster_info : nullptr);
  const float4* info_d = stage_d ? cl_smem + 2 * kClusterStage : (dmodel ? dmodel->cluster_info : nullptr);
  const bool need_lut = LUT_SMEM && do_rcorr;
  if (tid == 0) {
    if (LUT_SMEM) MbarInit(&sh.lut_bar, 1);
    MbarInit(&sh.depth_bar, 1);
    MbarInit(&sh.ctile_bar, 1);
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
  const bool tma = args.tma_mode != 0;
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
  const uint16_t* ctile_px = reinterpret_cast<const uint16_t*>(dyn + ctile.offset);
  const uint16_t* dtile_px = reinterpret_cast<const uint16_t*>(dyn + dtile.offset);
  bool depth_ready = dtile.w <= 0;
  bool ctile_ready = ctile.w <= 0 || !tma;
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

  LineRegs L;
  PointState P;
  L.valid = false;
  P.valid = false;
  L.cbx = L.cby = L.cbz = L.cu = L.cv = L.nu = L.nv = L.dr = L.ncts = L.mean = L.var = 0.0f;
  P.cbx = P.cby = P.cbz = P.nx = P.ny = P.nz = P.yx = P.yy = P.yz = 0.0f;
  int n_lines = 0, n_points = 0;
  int view_r = counts[2], view_d = counts[3];  // any valid view index: the lower bound of the pruned search
  bool lut_ready = !need_lut;
  BinImage bin_image;  // valid wherever the device copy of the colour frame is (the body's ROI), when the TMA path maintains it
  bin_image.px = (tma && ccam) ? ccam->bins : nullptr;
  bin_image.pitch = ccam ? ccam->bin_pitch : 0u;
  // function lookups (identical for every body of the launch, checked by the host): kernel-parameter constants
  const float* lf = args.lookup_f;
  const float* lb = args.lookup_b;
  M3TB_STAMP2(stamp_base);  // prologue done

  for (int corr = args.corr_begin; corr < args.corr_end; ++corr) {
    // ---------------- CalculateCorrespondences -------------------------------------------------
    if (do_rcorr && line_group) {
      if (group_leader) {
        const int v = ClosestViewPrunedWarp(info_r, rmodel->sorted_views, rmodel->n_clusters,
                                            rmodel->orientations4, rmodel->n_views, sh.view_o[0], view_r);
        if (lane == 0) sh.views[corr & 1][0] = v;
      }
      if (T == kGroup && do_dcorr && warp == kW - 2) {  // single group: another warp searches the depth model meanwhile
        const int v = ClosestViewPrunedWarp(info_d, dmodel->sorted_views, dmodel->n_clusters,
                                            dmodel->orientations4, dmodel->n_views, sh.view_o[1], view_d);
        if (lane == 0) sh.views[corr & 1][1] = v;
      }
      GroupBarrier<T>(0);
      view_r = sh.views[corr & 1][0];
      M3TB_STAMP2(stamp_base);  // closest view (region)
      RegionIter rit;
      MakeRegionIter(body.rp, *ccam, sh.rb2c, corr, rit);
      // the model record does not depend on the line count: load it first, the count (one more trip to memory when the
      // coverage is adaptive) meanwhile
      const float4* pts = rmodel->points + size_t(view_r) * rmodel->n_points * 2;
      float4 p0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), p1 = p0;
      if (item < min(rmodel->n_points, min(lcap, kGroup))) { p0 = __ldg(pts + 2 * item); p1 = __ldg(pts + 2 * item + 1); }
      n_lines = AdaptiveCount(body.rp.n_lines_max, body.rp.use_adaptive_coverage, body.rp.reference_contour_length,
                              body.rp.use_adaptive_coverage ? __ldg(rmodel->view_scalars + view_r) : 0.0f,
                              rmodel->max_view_scalar, rmodel->n_points);
      n_lines = min(n_lines, min(lcap, kGroup));
      M3TB_STAMP_AT(118, tid == T - 32 && !ctile_ready);
      if (!lut_ready) { MbarWait(&sh.lut_bar, 0); lut_ready = true; }
      if (!ctile_ready) { MbarWait(&sh.ctile_bar, 0); ctile_ready = true; M3TB_STAMP_AT(119, tid == T - 32); }
      L.valid = false;
      if (item < n_lines) {
        RegionLine2<LUT_SMEM>(rit, body.rp, p0, p1, cframe, ctile, ctile_px, bin_image, lut_g, lut_s, lf, lb, dist_col, L);
      }
      M3TB_STAMP2(stamp_base);  // region lines
    }
    if (do_dcorr && point_group) {
      if (T > kGroup || !do_rcorr) {  // (single group with lines: searched above, behind the same barrier)
        if (group_leader) {
          const int v = ClosestViewPrunedWarp(info_d, dmodel->sorted_views, dmodel->n_clusters,
                                              dmodel->orientations4, dmodel->n_views, sh.view_o[1], view_d);
          if (lane == 0) sh.views[corr & 1][1] = v;
        }
        GroupBarrier<T>(1);
      }
      view_d = sh.views[corr & 1][1];
      M3TB_STAMP2(stamp_base);  // closest view (depth)
      DepthIter dit;
      MakeDepthIter(body.dp, *dcam, sh.db2c, sh.dc2b, corr, dit);
      const float4* pts = dmodel->points + size_t(view_d) * dmodel->n_points * 2;
      float4 p0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), p1 = p0;
      if (item < min(dmodel->n_points, min(pcap, kGroup))) { p0 = __ldg(pts + 2 * item); p1 = __ldg(pts + 2 * item + 1); }
      n_points = AdaptiveCount(body.dp.n_points_max, body.dp.use_adaptive_coverage, body.dp.reference_surface_area,
                               body.dp.use_adaptive_coverage ? __ldg(dmodel->view_scalars + view_d) : 0.0f,
                               dmodel->max_view_scalar, dmodel->n_points);
      n_points = min(n_points, min(pcap, kGroup));
      if (!depth_ready) { MbarWait(&sh.depth_bar, 0); depth_ready = true; }
      P.valid = false;
      if (item < n_points) {
        DepthPoint<false>(dit, body.dp, p0, p1, dframe, dtile, dtile_px, P);
      }
      M3TB_STAMP2(stamp_base);  // depth points
    }

    // ---------------- n_update x (CalculateGradientAndHessian + CalculateOptimization) ---------
    for (int upd = 0; upd < args.n_update; ++upd) {
      const int opt_iteration = args.opt_base + upd;
      float acc[27];
#pragma unroll
      for (int k = 0; k < 27; ++k) acc[k] = 0.0f;
      if (do_rgh && line_group) {
        RegionIter rit;
        MakeRegionIter(body.rp, *ccam, sh.rb2c, corr, rit);
        RegionGradient2(rit, body.rp, L, dist_col, opt_iteration, acc);
      }
      if (do_dgh && point_group) {
        DepthIter dit;
        MakeDepthIter(body.dp, *dcam, sh.db2c, sh.dc2b, corr, dit);
        DepthGradient(dit, P, acc);
      }
      {  // warp reduction by recursive halving (see k_track)
        float v[32];
#pragma unroll
        for (int k = 0; k < 32; ++k) v[k] = k < 27 ? acc[k] : 0.0f;
#pragma unroll
        for (int half = 16; half >= 1; half >>= 1) {
          const bool upper = (lane & half) != 0;
#pragma unroll
          for (int k = 0; k < half; ++k) {
            const float send = upper ? v[k] : v[k + half];
            const float keep = upper ? v[k + half] : v[k];
            v[k] = keep + __shfl_xor_sync(0xffffffffu, send, half);
          }
        }
        sh.red[warp][lane] = v[0];
      }
      M3TB_STAMP2(stamp_base);  // accumulate + warp reduce
      __syncthreads();
      M3TB_STAMP2(stamp_base);  // all warps arrived
      if (warp == kW - 1) {
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
        if (i == j) aval += (i < 3) ? body.tikhonov_rotation : body.tikhonov_translation;
        const bool is_b = l < 6;
        float* p1 = is_b ? &sh.b[l] : &sh.a[i * 6 + j];
        float* p2 = is_b ? &sh.b[l] : &sh.a[j * 6 + i];
        const float val = is_b ? 0.0f + v : aval;
        *p1 = val;
        *p2 = val;
        __syncwarp();
        M3TB_STAMP2(stamp_base);  // cross-warp sum + normal equations
        // with two warp groups the depth camera's pose products are left to the point group's leader (below): they are
        // off the critical path there, and the serial section every warp waits for gets shorter
        SolveAndUpdateSerial(sh, ccam != nullptr, dcam != nullptr && T == kGroup);
        M3TB_STAMP2(stamp_base);  // solve + pose update + pose products
      }
      __syncthreads();
      if (T > kGroup && dcam != nullptr && point_group) {
        if (group_leader) {
          float pose[12];
#pragma unroll
          for (int i = 0; i < 12; ++i) pose[i] = sh.pose[i];
          PublishPoseProducts(pose, false, true, false, sh);
        }
        GroupBarrier<T>(1);
      }
      M3TB_STAMP2(stamp_base);  // released
    }
  }

  // ---------------- epilogue ----------------------------------------------------------------------
  if (args.phases & PH_SOLVE)
    if (tid < 12) args.poses[12 * body_id + tid] = sh.pose[tid];
  if ((args.phases & PH_STORE_REGION) && has_region && line_group) {
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
        for (int d = 0; d < kDistributionLength; ++d) g_rst[(RF_DIST0 + d) * lcap + i] = dist_col[d * kGroup];
      }
    }
    if (item == 0) { counts[0] = n_lines; counts[2] = view_r; }
  }
  if ((args.phases & PH_STORE_DEPTH) && has_depth && point_group) {
    if (item < n_points) {
      const int i = item;
      g_dst[DF_CBX * pcap + i] = P.cbx; g_dst[DF_CBY * pcap + i] = P.cby; g_dst[DF_CBZ * pcap + i] = P.cbz;
      g_dst[DF_NX * pcap + i] = P.nx; g_dst[DF_NY * pcap + i] = P.ny; g_dst[DF_NZ * pcap + i] = P.nz;
      g_dst[DF_VALID * pcap + i] = P.valid ? 1.0f : 0.0f;
      if (P.valid) {
        g_dst[DF_YX * pcap + i] = P.yx; g_dst[DF_YY * pcap + i] = P.yy; g_dst[DF_YZ * pcap + i] = P.yz;
      }
    }
    if (item == 0) { counts[1] = n_points; counts[3] = view_d; }
  }
  if (need_lut && !lut_ready) MbarWait(&sh.lut_bar, 0);  // never leave with a bulk copy in flight
  if (!depth_ready) MbarWait(&sh.depth_bar, 0);
  if (!ctile_ready) MbarWait(&sh.ctile_bar, 0);
}

}  // namespace m3tb
