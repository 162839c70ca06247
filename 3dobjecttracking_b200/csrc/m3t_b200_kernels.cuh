// m3t_b200_kernels.cuh — the kernels of the pose-optimisation path.
//
//   k_track<T,K,LUT_SMEM>
//       one CTA of T threads per body for a whole tracking step; thread t owns correspondence lines /
//       surface points t, t+T, ... (K of each) and keeps their state (RegionModality::DataLine,
//       DepthModality::DataPoint) in REGISTERS between CalculateCorrespondences and the n_update
//       gradient passes. Per correspondence iteration:
//         K5 closest view (block arg-max)  ->  K1 region lines (project, validate, DDA gather,
//         normalised-LUT lookup, segment products, distribution, moments)  +  K3 depth search
//         ->  n_update x ( K2 gradient/Hessian (27 accumulators/thread, warp-shuffle + one smem hop)
//                          ->  K4 6x6 pivoted LDL^T + SE(3) update, thread-serial on warp 0 ).
//       The normalised histogram LUT (32 KB at 16 bins) is staged into shared memory once per launch
//       by a TMA bulk copy (cp.async.bulk + mbarrier). The same kernel serves the fine-grained C-ABI
//       calls via `phases`.
//   k_histogram  RegionModality::StartModality / CalculateResults histogram side (SURVEY §8 f1).
//   k_lut        per-bin normalisation of (hist_f, hist_b) -> float2 LUT.
#pragma once

#include "m3t_b200_device.cuh"
#include "m3t_b200_structures.cuh"
#include "m3t_b200_texture.cuh"
#include "m3t_b200_views.cuh"

namespace m3tb {

constexpr int kMaxWarps = 16;
constexpr int kDynSmemBytes = 220 * 1024;  // dynamic shared memory per CTA when ROI tiles are on (1 CTA / SM)

// ROI tile staged in shared memory: pixels [x0, x0+w) x [y0, y0+h) of one camera frame, `pitch` elements per row.
// Colour tiles hold the histogram BIN INDEX of every pixel (u16, computed once per launch instead of once per
// line sample); depth tiles hold the raw U16 depth, copied row by row with TMA bulk copies.
struct Tile {
  int x0, y0, w, h, pitch;
  unsigned offset;  // byte offset in dynamic shared memory
};

struct Shared {
  // pose products shared by all threads; recomputed by warp 0 after every pose update
  float rb2c[12];                // colour-camera body2camera  (region_modality.cpp:1001-1002)
  float db2c[12];                // depth-camera body2camera   (depth_modality.cpp:642-643)
  float dc2b[12];                // its inverse                (depth_modality.cpp:644)
  float cw2c[12], dw2c[12];      // world2camera of the two cameras (copied once per launch)
  float view_o[2][4];            // R^T normalize(t) of rb2c / db2c, [3] = 1 if |t| > 0 (GetClosestView query)
  Tile ctile, dtile;
  unsigned long long depth_bar;  // mbarrier of the depth-tile bulk copies
  float pose[12];                // body2world (Body::body2world_pose)
  float red[kMaxWarps][32];      // per-warp partial sums: g[6] + H lower[21] (+5 pad)
  float a[36];                   // normal matrix, full symmetric
  float b[6];
  float x[6];
  unsigned best_key[2][2][kMaxWarps];  // [call parity][model][warp]
  int best_idx[2][2][kMaxWarps];
  unsigned long long lut_bar;    // mbarrier of the LUT bulk copy
};


// ---------------------------------------------------------------------------------------------
// TMA bulk copy + mbarrier (sm_90+ PTX; SASS: UBLKCP / SYNCS)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned SmemAddr(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void MbarInit(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(SmemAddr(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void MbarExpectTx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(SmemAddr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void BulkCopyG2S(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   SmemAddr(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(SmemAddr(bar))
               : "memory");
}
__device__ __forceinline__ bool MbarTryWait(unsigned long long* bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(SmemAddr(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void MbarWait(unsigned long long* bar, unsigned parity) {
  while (!MbarTryWait(bar, parity)) {
  }
}

// ---------------------------------------------------------------------------------------------
// K5: RegionModel/DepthModel::GetClosestView (region_model.cpp:105-130, depth_model.cpp:81-106)
// orientation = R^T * normalize(t) (linear block of body2camera, see DESIGN.md "Numerics");
// arg-max of the dot product, first maximum wins. Two models (region + depth) share one block pass.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool ViewOrientation(const float* b2c, float& o0, float& o1, float& o2) {
  float tx = b2c[3], ty = b2c[7], tz = b2c[11];
  float z = tx * tx + ty * ty + tz * tz;
  float norm = sqrtf(z);
  if (norm == 0.0f) return false;  // reference returns views_[0]
  if (z > 0.0f) { tx /= norm; ty /= norm; tz /= norm; }
  o0 = b2c[0] * tx + b2c[4] * ty + b2c[8] * tz;
  o1 = b2c[1] * tx + b2c[5] * ty + b2c[9] * tz;
  o2 = b2c[2] * tx + b2c[6] * ty + b2c[10] * tz;
  return true;
}

__device__ __forceinline__ void ArgmaxMerge(float& best, int& idx, float ob, int oi) {
  if (ob > best || (ob == best && oi < idx)) { best = ob; idx = oi; }
}

// float -> unsigned key with the same ordering (finite values)
__device__ __forceinline__ unsigned SortableKey(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// warp arg-max with "first maximum wins": REDUX.MAX on the key, then REDUX.MIN of the index among the lanes holding it
__device__ __forceinline__ void WarpArgmax(unsigned& key, int& idx) {
  const unsigned kmax = __reduce_max_sync(0xffffffffu, key);
  const unsigned cand = key == kmax ? unsigned(idx) : 0x7fffffffu;
  idx = int(__reduce_min_sync(0xffffffffu, cand));
  key = kmax;
}

template <int T>
__device__ void ClosestViews(const ModelDev* m0, const ModelDev* m1, Shared& sh, int parity, int& view0, int& view1) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int kW = T / 32;
  float best[2] = {-1.0f, -1.0f};
  int idx[2] = {0x7fffffff, 0x7fffffff};
  float o[2][3];
  bool nonzero[2];
  int nv[2] = {0, 0};
  const float4* ori[2] = {nullptr, nullptr};
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    o[s][0] = sh.view_o[s][0]; o[s][1] = sh.view_o[s][1]; o[s][2] = sh.view_o[s][2];
    nonzero[s] = sh.view_o[s][3] != 0.0f;
  }
  if (m0) { nv[0] = nonzero[0] ? m0->n_views : 0; ori[0] = m0->orientations4; }
  if (m1) { nv[1] = nonzero[1] ? m1->n_views : 0; ori[1] = m1->orientations4; }
  const int nv_max = max(nv[0], nv[1]);
  // both models share one pass: eight independent 16-byte loads in flight per thread
  for (int v0 = tid; v0 < nv_max; v0 += 4 * T) {
    float4 q[2][4];
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int v = v0 + u * T;
        q[s][u] = v < nv[s] ? __ldg(ori[s] + v) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      }
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int v = v0 + u * T;
        const float dot = o[s][0] * q[s][u].x + o[s][1] * q[s][u].y + o[s][2] * q[s][u].z;
        if (v < nv[s] && dot > best[s]) { best[s] = dot; idx[s] = v; }
      }
  }
  // warp arg-max (REDUX), one shared-memory hop, the same arg-max over the per-warp results inside every warp:
  // one __syncthreads per call; the buffers alternate with the call parity so that the next call cannot overwrite
  // values a slow warp is still reading.
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    unsigned key = SortableKey(best[s]);
    WarpArgmax(key, idx[s]);
    if (lane == 0) { sh.best_key[parity][s][warp] = key; sh.best_idx[parity][s][warp] = idx[s]; }
  }
  __syncthreads();
  int out[2] = {0, 0};
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    unsigned key = lane < kW ? sh.best_key[parity][s][lane] : 0u;
    int ri = lane < kW ? sh.best_idx[parity][s][lane] : 0x7fffffff;
    WarpArgmax(key, ri);
    // nothing beat the initial -1 (or |t| = 0): the reference leaves / returns views_[0]
    out[s] = (ri == 0x7fffffff || !nonzero[s] || key <= SortableKey(-1.0f)) ? 0 : ri;
  }
  view0 = out[0];
  view1 = out[1];
}

// ---------------------------------------------------------------------------------------------
// K1: one correspondence line (region_modality.cpp:1231-1291, 1433-1658)
// ---------------------------------------------------------------------------------------------
struct RegionIter {  // PrecalculateCameraVariables / PoseVariables / IterationDependentVariables
  float b2c[12];
  float fu, fv, ppu, ppv;
  int w_m1, h_m1, w_m2, h_m2;
  int scale;
  float fscale;
  int ll_m1;
  float ll_m1_half, ll_half_m1;
  float variance;
};

__device__ __forceinline__ void MakeRegionIter(const RegionParamsDev& rp, const CameraDev& cam, const float* b2c,
                                               int corr_iteration, RegionIter& it) {
#pragma unroll
  for (int i = 0; i < 12; ++i) it.b2c[i] = b2c[i];
  it.fu = cam.fu; it.fv = cam.fv; it.ppu = cam.ppu; it.ppv = cam.ppv;
  it.w_m1 = cam.width - 1; it.h_m1 = cam.height - 1; it.w_m2 = cam.width - 2; it.h_m2 = cam.height - 2;
  it.scale = LastValid(rp.scales, rp.n_scales, corr_iteration);  // :1011-1023
  it.fscale = float(it.scale);
  int line_length = kLineSegments * it.scale;
  it.ll_m1 = line_length - 1;
  it.ll_m1_half = float(line_length - 1) * 0.5f;
  it.ll_half_m1 = float(line_length) * 0.5f - 1.0f;
  float sd = LastValid(rp.standard_deviations, rp.n_standard_deviations, corr_iteration);
  it.variance = sd * sd;
}

__device__ __forceinline__ FrameView MakeFrameView(const CameraDev& cam, const RoiRecord& r) {
  FrameView f;
  f.dev = cam.image; f.dev_pitch = cam.pitch;
  f.host = cam.host_src; f.host_pitch = cam.host_pitch;
  if (cam.host_src) { f.x0 = r.x0; f.y0 = r.y0; f.x1 = r.x1; f.y1 = r.y1; }
  else { f.x0 = 0; f.y0 = 0; f.x1 = cam.width; f.y1 = cam.height; }
  return f;
}
__device__ __forceinline__ const uint8_t* FramePtr(const FrameView& f, int x, int y, unsigned bytes_per_pixel) {
  const bool in_roi = x >= f.x0 && x < f.x1 && y >= f.y0 && y < f.y1;
  return in_roi ? f.dev + size_t(unsigned(y)) * f.dev_pitch + bytes_per_pixel * unsigned(x)
                : f.host + size_t(unsigned(y)) * f.host_pitch + bytes_per_pixel * unsigned(x);
}

// Histogram bin index of pixel (x, y): from the shared-memory tile when inside it, else from the frame
// (same integer result either way, so tiling never changes a line).
__device__ __forceinline__ int PixelBin(const Tile& t, const uint16_t* tile, const FrameView& f, int bs, int nb, int x,
                                        int y) {
  const unsigned tx = unsigned(x - t.x0), ty = unsigned(y - t.y0);
  if (tx < unsigned(t.w) && ty < unsigned(t.h)) return tile[ty * unsigned(t.pitch) + tx];
  const uint8_t* px = FramePtr(f, x, y, 3u);
  // ColorHistograms::GetProbabilities index (color_histograms.cpp:97-99), BGR memory order
  return int(LutSlot(unsigned((int(__ldg(px)) >> bs) * nb * nb + (int(__ldg(px + 1)) >> bs) * nb + (int(__ldg(px + 2)) >> bs))));
}

__device__ __forceinline__ unsigned DepthAt(const Tile& t, const uint16_t* tile, const FrameView& f, int x, int y) {
  const unsigned tx = unsigned(x - t.x0), ty = unsigned(y - t.y0);
  if (tx < unsigned(t.w) && ty < unsigned(t.h)) return tile[ty * unsigned(t.pitch) + tx];
  return __ldg(reinterpret_cast<const uint16_t*>(FramePtr(f, x, y, 2u)));
}

struct LineState {  // RegionModality::DataLine (region_modality.h:150-165), the fields the math uses
  float cbx, cby, cbz, cu, cv, nu, nv, dr, ncts, mean, var;
  float dist[kDistributionLength];
  bool valid;
};

// The strided window scan shared by RegionModality::IsLineUnoccludedMeasured (region_modality.cpp:1355-1388) and
// DepthModality::IsPointUnoccludedMeasured (depth_modality.cpp:739-775). ushort(x) of the reference is restated as
// truncation to int and reduction modulo 2^16 (identical to the oracle).
static __device__ __noinline__ bool WindowUnoccluded(const Tile& t, const uint16_t* tile, const FrameView& f, int w_m1, int h_m1,
                                              float center_u, float center_v, float diameter, float min_depth_value) {
  if (!ScanDiameterValid(diameter)) return true;
  const int stride = int(diameter / float(kMaxNOcclusionStrides) + 1.0f);
  const int n_strides = int(diameter / float(stride) + 0.5f);
  const int rounded_diameter = n_strides * stride;
  const float rounded_radius = 0.5f * float(rounded_diameter);
  int u_min = int(center_u - rounded_radius + 0.5f);
  int v_min = int(center_v - rounded_radius + 0.5f);
  int u_max = u_min + rounded_diameter;
  int v_max = v_min + rounded_diameter;
  u_min = max(u_min, 0);
  v_min = max(v_min, 0);
  u_max = min(u_max, w_m1);
  v_max = min(v_max, h_m1);
  const unsigned min_depth = unsigned(int(min_depth_value)) & 0xffffu;
  for (int v = v_min; v <= v_max; v += stride)
    for (int u = u_min; u <= u_max; u += stride) {
      const unsigned depth = DepthAt(t, tile, f, u, v);
      if (depth > 0u && depth < min_depth) return false;
    }
  return true;
}

// What RegionModality needs of its depth camera to measure occlusions (region_modality.cpp:944-962,1003-1005)
struct RegionOcclusion {
  const float* b2d;          // body2depth_camera_pose_
  const float* offsets;      // depth_offsets of the closest view: [n_points][30]
  int offset_id;             // measured_depth_offset_id_
  float fu, fv, ppu, ppv, depth_scale;
  int w_m1, h_m1;
  float radius, threshold;
  const FrameView* frame;
  const Tile* tile;
  const uint16_t* tile_px;
};

// RegionModality::IsLineUnoccludedMeasured (region_modality.cpp:1343-1389)
__device__ __forceinline__ bool LineUnoccludedMeasured(const RegionOcclusion& o, float cbx, float cby, float cbz, int point) {
  float x, y, z;
  PoseApply(o.b2d, cbx, cby, cbz, x, y, z);
  const float center_u = x * o.fu / z + o.ppu;
  const float center_v = y * o.fv / z + o.ppv;
  const float meter_to_pixel = o.fu / z;
  const float diameter = 2.0f * o.radius * meter_to_pixel;
  const float depth_offset = __ldg(o.offsets + size_t(point) * kDepthOffsets + o.offset_id);
  return WindowUnoccluded(*o.tile, o.tile_px, *o.frame, o.w_m1, o.h_m1, center_u, center_v, diameter,
                          (z - depth_offset - o.threshold) / o.depth_scale);
}

// ---- checks on renderer images (SURVEY f4: modeled occlusion handling, region checking, silhouette checking) ----------
// The strided minimum scan of RegionModality::IsLineUnoccludedModeled (region_modality.cpp:1391-1431) and
// DepthModality::IsPointUnoccludedModeled (depth_modality.cpp:778-824) in the focused depth rendering.
static __device__ __noinline__ bool ModeledWindowUnoccluded(const RenderingDev& r, float center_u, float center_v, float diameter,
                                                            float min_allowed_depth) {
  if (!ScanDiameterValid(diameter)) return true;
  const int stride = int(diameter / float(kMaxNOcclusionStrides) + 1.0f);
  const int n_strides = int(diameter / float(stride) + 0.5f);
  const int rounded_diameter = n_strides * stride;
  const float rounded_radius = 0.5f * float(rounded_diameter);
  const float focused_center_u = (center_u - r.corner_u) * r.scale;
  const float focused_center_v = (center_v - r.corner_v) * r.scale;
  int u_min = int(focused_center_u - rounded_radius + 0.5f);
  int v_min = int(focused_center_v - rounded_radius + 0.5f);
  int u_max = u_min + rounded_diameter;
  int v_max = v_min + rounded_diameter;
  u_min = max(u_min, 0);
  v_min = max(v_min, 0);
  u_max = min(u_max, r.image_size - 1);
  v_max = min(v_max, r.image_size - 1);
  unsigned min_depth_value = 65535u;
  for (int v = v_min; v <= v_max; v += stride) {
    const uint16_t* row = reinterpret_cast<const uint16_t*>(r.image + size_t(v) * r.pitch);
    for (int u = u_min; u <= u_max; u += stride) min_depth_value = min(min_depth_value, unsigned(__ldg(row + u)));
  }
  const float min_depth = r.projection_term_a / (r.projection_term_b - float(min_depth_value));  // FocusedDepthRenderer::Depth
  return min_depth > min_allowed_depth;
}

__device__ __forceinline__ unsigned SilhouetteAt(const RenderingDev& r, int v, int u) {
  return __ldg(r.image + size_t(v) * r.pitch + size_t(u));
}

// RegionModality::IsDynamicLineRegionSufficient (region_modality.cpp:1293-1341); a foreground sample outside the focused
// image (undefined behaviour in the reference) counts as "not this region", as in the oracle
static __device__ __noinline__ bool DynamicLineRegionSufficient(const RenderingDev& r, float min_continuous_distance, float fscale,
                                                                float center_u, float center_v, float normal_u, float normal_v) {
  const unsigned region_id = unsigned(r.id) & 0xffu;
  const float fsize = float(r.image_size);
  const float focused_min_continuous_distance = min_continuous_distance * fscale * r.scale;
  const float focused_stride = fmaxf((focused_min_continuous_distance - kRegionOffset) / float(kNRegionStride), 0.0f);
  const float stride_u = focused_stride * normal_u;
  const float stride_v = focused_stride * normal_v;
  const float offset_u = kRegionOffset * normal_u;
  const float offset_v = kRegionOffset * normal_v;
  const float focused_center_u = 0.5f + (center_u - r.corner_u) * r.scale;
  const float focused_center_v = 0.5f + (center_v - r.corner_v) * r.scale;
  float u = focused_center_u - offset_u;
  float v = focused_center_v - offset_v;
  for (int i = 0; i <= kNRegionStride; ++i) {
    if (u >= fsize || u < 0.0f || v >= fsize || v < 0.0f) return false;
    if (SilhouetteAt(r, int(v), int(u)) != region_id) return false;
    u -= stride_u;
    v -= stride_v;
  }
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

// RegionModality::DynamicRegionDistance (region_modality.cpp:1157-1223), quirk of :1218 included
static __device__ __noinline__ void DynamicRegionDistance(const RenderingDev& r, float max_considered_line_length,
                                                          float unconsidered_line_length, float center_u, float center_v,
                                                          float normal_u, float normal_v, float& dynamic_foreground_distance,
                                                          float& dynamic_background_distance) {
  const unsigned region_id = unsigned(r.id) & 0xffu;
  const float fsize = float(r.image_size);
  const float stride = max_considered_line_length / float(kNRegionStride);
  const float focused_stride = stride * r.scale;
  const float focused_stride_u = focused_stride * normal_u;
  const float focused_stride_v = focused_stride * normal_v;
  const float delta_start = kRegionOffset / r.scale - unconsidered_line_length;
  const int i_start = max(int(delta_start / stride + 1.0f), 0);
  const float offset = unconsidered_line_length + float(i_start) * stride;
  const float focused_offset = offset * r.scale;
  const float focused_offset_u = focused_offset * normal_u;
  const float focused_offset_v = focused_offset * normal_v;
  const float focused_center_u = 0.5f + (center_u - r.corner_u) * r.scale;
  const float focused_center_v = 0.5f + (center_v - r.corner_v) * r.scale;
  float u = focused_center_u - focused_offset_u;
  float v = focused_center_v - focused_offset_v;
  for (int i = i_start; i <= kNRegionStride; ++i) {
    if (u >= fsize || u < 0.0f || v >= fsize || v < 0.0f) {
      dynamic_foreground_distance = stride * float(i);
      break;
    }
    if (SilhouetteAt(r, int(v), int(u)) != region_id) {
      dynamic_foreground_distance = i == i_start ? 0.0f : stride * float(i);
      break;
    }
    u -= focused_stride_u;
    v -= focused_stride_v;
  }
  u = focused_center_u + focused_offset_u;
  v = focused_center_v + focused_offset_v;
  for (int i = i_start; i <= kNRegionStride; ++i) {
    if (u >= fsize || u < 0.0f || v >= fsize || v < 0.0f) {
      dynamic_background_distance = max_considered_line_length;
      break;
    }
    if (SilhouetteAt(r, int(v), int(u)) == region_id) {
      if (i == i_start) dynamic_background_distance = 0.0f;
      else dynamic_foreground_distance = stride * float(i);  // sic (:1218)
      break;
    }
    u += focused_stride_u;
    v += focused_stride_v;
  }
}

// What RegionLine / DepthPoint need for the renderer-image checks of one pass
struct RenderChecks {
  const RenderingDev* silhouette;  // region checking / silhouette checking (both passes), or null
  const RenderingDev* depth;       // modeled occlusion handling (first pass only), or null
  const float* offsets;            // depth offsets of the closest view: [n_points][30]
  int modeled_offset_id;           // region: modeled_depth_offset_id_
  float radius, threshold, offset_radius;
};

template <bool LUT_SMEM>
__device__ __forceinline__ float2 LutFetch(const float2* __restrict__ lut_g, const float2* lut_s, int idx) {
  if (LUT_SMEM) return lut_s[idx];
  return __ldg(lut_g + idx);
}

// Hot gather: every sample of the line is inside the shared-memory tile. S > 0: compile-time scale, the S pixels
// of a segment are unrolled (loads batched, multiplications still in pixel order); S == 0: run-time scale.
template <bool LUT_SMEM, int S>
__device__ __forceinline__ void GatherFast(int scale, int base, float minor_f, float step, int stride_major,
                                           int stride_minor, const uint16_t* tile_px, const float2* __restrict__ lut_g,
                                           const float2* lut_s, float (&sf)[kLineSegments], float (&sb)[kLineSegments]) {
#pragma unroll
  for (int s = 0; s < kLineSegments; ++s) {
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
      for (int k = 0; k < S; ++k) l[k] = LutFetch<LUT_SMEM>(lut_g, lut_s, idx[k]);  // normalised per bin (:1575-1598)
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
    sf[s] = pf;
    sb[s] = pb;
  }
}

// Generic (rare) gather: any sample may lie outside the tile. Kept out of line so that the hot loop stays small.
template <bool LUT_SMEM>
__device__ __noinline__ void GatherSlow(int scale, int bs, int nb, bool horizontal, int major, float minor_f, float step,
                                        const FrameView& frame, const Tile& tile,
                                        const uint16_t* tile_px, const float2* __restrict__ lut_g, const float2* lut_s,
                                        float* sf, float* sb) {
#pragma unroll 1
  for (int s = 0; s < kLineSegments; ++s) {
    float pf = 1.0f, pb = 1.0f;
#pragma unroll 1
    for (int k = 0; k < scale; ++k) {
      const int minor = int(minor_f);
      const int idx = PixelBin(tile, tile_px, frame, bs, nb, horizontal ? major : minor, horizontal ? minor : major);
      const float2 l = LutFetch<LUT_SMEM>(lut_g, lut_s, idx);
      pf *= l.x;
      pb *= l.y;
      ++major;
      minor_f += step;
    }
    sf[s] = pf;
    sb[s] = pb;
  }
}

template <bool LUT_SMEM, bool OCC = false>
__device__ __forceinline__ void RegionLine(const RegionIter& it, const RegionParamsDev& rp, const float4 p0,
                                           const float4 p1, const FrameView& frame,
                                           const Tile& tile, const uint16_t* tile_px,
                                           const float2* __restrict__ lut_g, const float2* lut_s, LineState& L,
                                           const RegionOcclusion* occ = nullptr, int point = 0,
                                           const RenderChecks* rc = nullptr) {
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
  if (!(z > 0.0f)) return;
  int icu = int(center_u + 0.5f), icv = int(center_v + 0.5f);
  if (icu < 0 || icu > it.w_m1 || icv < 0 || icv > it.h_m1) return;
  if (OCC) {  // region checking (:1269-1274), measured occlusions (:1274-1281), modeled occlusions (:1283-1289)
    if (rc && rc->silhouette &&
        !DynamicLineRegionSufficient(*rc->silhouette, rp.min_continuous_distance, it.fscale, center_u, center_v, nu, nv))
      return;
    if (occ && !LineUnoccludedMeasured(*occ, p0.x, p0.y, p0.z, point)) return;
    if (rc && rc->depth) {
      const float meter_to_pixel = (it.fu / z) * rc->depth->scale;
      const float diameter = 2.0f * rc->radius * meter_to_pixel;
      const float depth_offset = __ldg(rc->offsets + size_t(point) * kDepthOffsets + rc->modeled_offset_id);
      if (!ModeledWindowUnoccluded(*rc->depth, center_u, center_v, diameter, z - depth_offset - rc->threshold)) return;
    }
  }

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
  float sf[kLineSegments], sb[kLineSegments];
  {
    // Is the whole line inside the shared-memory tile? (+-1 on the minor axis for the rounding of the running sum)
    const int mi0 = int(minor_f), mi1 = int(minor_f_end);
    const int minor_lo = min(mi0, mi1) - 1, minor_hi = max(mi0, mi1) + 1;
    const int x_lo = horizontal ? major : minor_lo, x_hi = horizontal ? major_end : minor_hi;
    const int y_lo = horizontal ? minor_lo : major, y_hi = horizontal ? minor_hi : major_end;
    const bool inside = x_lo >= tile.x0 && x_hi < tile.x0 + tile.w && y_lo >= tile.y0 && y_hi < tile.y0 + tile.h;
    if (inside) {
      // fast path: no per-sample bounds checks; tile element index = base + int(minor_f) * stride_minor.
      // For the usual scales the pixels of a segment are unrolled so that their loads are issued together.
      const int stride_major = horizontal ? 1 : tile.pitch;
      const int stride_minor = horizontal ? tile.pitch : 1;
      int base = horizontal ? (major - tile.x0) - tile.y0 * tile.pitch : (major - tile.y0) * tile.pitch - tile.x0;
      switch (it.scale) {
        case 1: GatherFast<LUT_SMEM, 1>(1, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, sf, sb); break;
        case 2: GatherFast<LUT_SMEM, 2>(2, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, sf, sb); break;
        case 4: GatherFast<LUT_SMEM, 4>(4, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, sf, sb); break;
        case 6: GatherFast<LUT_SMEM, 6>(6, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, sf, sb); break;
        default: GatherFast<LUT_SMEM, 0>(it.scale, base, minor_f, step, stride_major, stride_minor, tile_px, lut_g, lut_s, sf, sb); break;
      }
    } else {
      float tf[kLineSegments], tb[kLineSegments];
      GatherSlow<LUT_SMEM>(it.scale, rp.bitshift, rp.n_bins, horizontal, major, minor_f, step, frame, tile, tile_px,
                           lut_g, lut_s, tf, tb);
#pragma unroll
      for (int s = 0; s < kLineSegments; ++s) { sf[s] = tf[s]; sb[s] = tb[s]; }
    }
  }
  if (!(n_major > 0.0f)) {  // segments are filled back to front (:1470-1484)
#pragma unroll
    for (int s = 0; s < kLineSegments / 2; ++s) {
      float t = sf[s]; sf[s] = sf[kLineSegments - 1 - s]; sf[kLineSegments - 1 - s] = t;
      t = sb[s]; sb[s] = sb[kLineSegments - 1 - s]; sb[kLineSegments - 1 - s] = t;
    }
  }
  if (it.scale > 1) {  // :1555-1571
#pragma unroll
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
  L.ncts = fabsf(n_major) / it.fscale;
  L.dr = (roundf(c_major - it.ll_m1_half) + it.ll_m1_half - c_major) / n_major;

  // CalculateDistribution (:1600-1637)
  float area = 0.0f;
#pragma unroll
  for (int d = 0; d < kDistributionLength; ++d) {
    float val = 1.0f;
#pragma unroll
    for (int k = 0; k < kFunctionLength; ++k) val *= sf[d + k] * rp.lookup_f[k] + sb[d + k] * rp.lookup_b[k];
    L.dist[d] = val;
    area += val;
  }
#pragma unroll
  for (int d = 0; d < kDistributionLength; ++d) L.dist[d] /= area;
  // CalculateDistributionMoments (:1639-1658)
  float mean_from_begin = 0.0f;
#pragma unroll
  for (int d = 0; d < kDistributionLength; ++d) mean_from_begin += float(d) * L.dist[d];
  float var = 0.0f;
#pragma unroll
  for (int d = 0; d < kDistributionLength; ++d) {
    float dd = float(d) - mean_from_begin;
    var += (dd * dd) * L.dist[d];
  }
  L.mean = mean_from_begin - (float(kDistributionLength) - 1.0f) / 2.0f;
  L.var = var < rp.min_expected_variance ? rp.min_expected_variance : var;  // std::max: a NaN variance stays NaN
  L.valid = true;
}

__device__ __forceinline__ float Select12(const float (&d)[kDistributionLength], int i) {
  float r = d[0];
#pragma unroll
  for (int k = 1; k < kDistributionLength; ++k) r = (i == k) ? d[k] : r;
  return r;
}

// K2 region: one line's contribution to g / H (region_modality.cpp:485-558)
__device__ __forceinline__ void RegionGradient(const RegionIter& it, const RegionParamsDev& rp, const LineState& L,
                                               int opt_iteration, float (&acc)[27]) {
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
    dll = (logf(Select12(L.dist, upper)) - logf(Select12(L.dist, lower))) * rp.learning_rate / L.var;
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
// K3: depth correspondence search (depth_modality.cpp:656-726, 826-884)
// ---------------------------------------------------------------------------------------------
struct DepthIter {
  float b2c[12], c2b[12];
  float fu, fv, ppu, ppv, depth_scale;
  int w_m1, h_m1;
  float considered_distance, standard_deviation;
  int max_n_strides;
};

__device__ __forceinline__ void MakeDepthIter(const DepthParamsDev& dp, const CameraDev& cam, const float* b2c,
                                              const float* c2b, int corr_iteration, DepthIter& it) {
#pragma unroll
  for (int i = 0; i < 12; ++i) { it.b2c[i] = b2c[i]; it.c2b[i] = c2b[i]; }
  it.fu = cam.fu; it.fv = cam.fv; it.ppu = cam.ppu; it.ppv = cam.ppv;
  it.depth_scale = cam.depth_scale;
  it.w_m1 = cam.width - 1; it.h_m1 = cam.height - 1;
  it.considered_distance = LastValid(dp.considered_distances, dp.n_considered_distances, corr_iteration);
  it.max_n_strides = int(it.considered_distance / dp.stride_length + 0.5f);  // :651
  it.standard_deviation = LastValid(dp.standard_deviations, dp.n_standard_deviations, corr_iteration);
}

struct PointState {  // DepthModality::DataPoint (depth_modality.h:139-150)
  float cbx, cby, cbz, nx, ny, nz, yx, yy, yz;
  bool valid;
};

// Rare path of FindCorrespondence: the search window leaves the tile. Takes the camera scalars by value and returns
// (best, x, y, z) by value, so that neither the caller's DepthIter nor its result has its address taken: an
// address-taken struct lives in local memory, and k_track2 rebuilt its DepthIter there every update iteration.
static __device__ __noinline__ float4 DepthSearchSlow(float ppu, float ppv, float fu, float fv, float depth_scale, int u_min,
                                                      int u_max, int v_min, int v_max, int stride, float min_depth_value,
                                                      float max_depth_value, float x, float y, float z,
                                                      const FrameView& frame, const Tile& tile, const uint16_t* tile_px,
                                                      float best) {
  float bx = 0.0f, by = 0.0f, bz = 0.0f;
  for (int v = v_min; v <= v_max; v += stride) {
    for (int u = u_min; u <= u_max; u += stride) {
      float depth = float(DepthAt(tile, tile_px, frame, u, v));
      if (depth > min_depth_value && depth < max_depth_value) {
        depth *= depth_scale;
        float tx = (float(u) - ppu) * depth / fu;
        float ty = (float(v) - ppv) * depth / fv;
        float dx = tx - x, dy = ty - y, dz = depth - z;
        float d2 = dx * dx + dy * dy + dz * dz;
        if (d2 < best) { bx = tx; by = ty; bz = depth; best = d2; }
      }
    }
  }
  return make_float4(best, bx, by, bz);
}

template <bool OCC = false>
__device__ __forceinline__ void DepthPoint(const DepthIter& it, const DepthParamsDev& dp, const float4 p0, const float4 p1,
                                           const FrameView& frame, const Tile& tile, const uint16_t* tile_px,
                                           PointState& P, const float* offsets = nullptr, float stride_depth_offset = 1.0f,
                                           const RenderChecks* rc = nullptr) {
  P.valid = false;
  float x, y, z;
  PoseApply(it.b2c, p0.x, p0.y, p0.z, x, y, z);
  P.cbx = p0.x; P.cby = p0.y; P.cbz = p0.z;
  P.nx = p0.w; P.ny = p1.x; P.nz = p1.y;
  float center_u = x * it.fu / z + it.ppu;
  float center_v = y * it.fv / z + it.ppv;
  // IsPointValid (:697-726)
  if (!(z > 0.0f)) return;
  int icu = int(center_u + 0.5f), icv = int(center_v + 0.5f);
  if (icu < 0 || icu > it.w_m1 || icv < 0 || icv > it.h_m1) return;
  if (OCC) {  // IsPointOnValidSilhouette (:728-734) via FocusedSilhouetteRenderer::SilhouetteValue
    if (rc && rc->silhouette) {
      const RenderingDev& sr = *rc->silhouette;
      const int su = int((float(icu) - sr.corner_u) * sr.scale + 0.5f);
      const int sv = int((float(icv) - sr.corner_v) * sr.scale + 0.5f);
      if (su < 0 || su >= sr.image_size || sv < 0 || sv >= sr.image_size) return;
      if (SilhouetteAt(sr, sv, su) != (unsigned(sr.id) & 0xffu)) return;
    }
  }
  if (OCC) {  // IsPointUnoccludedMeasured (:736-776), depth offset selected as in CalculateBasicPointData (:669-681)
    if (offsets) {
      float radius = dp.measured_depth_offset_radius;
      if (dp.use_depth_scaling) radius *= z;
      int id = int(radius / stride_depth_offset + 0.5f);
      if (id >= kDepthOffsets) id = kDepthOffsets - 1;
      const float measured_depth_offset = __ldg(offsets + id);
      float diameter = 2.0f * dp.measured_occlusion_radius * it.fu;
      if (!dp.use_depth_scaling) diameter /= z;
      float threshold = dp.measured_occlusion_threshold;
      if (dp.use_depth_scaling) threshold *= z;
      if (!WindowUnoccluded(tile, tile_px, frame, it.w_m1, it.h_m1, center_u, center_v, diameter,
                            (z - measured_depth_offset - threshold) / it.depth_scale))
        return;
    }
  }
  if (OCC) {  // IsPointUnoccludedModeled (:778-824), depth offset as in CalculateBasicPointData (:682-693)
    if (rc && rc->depth) {
      float radius = rc->offset_radius;
      if (dp.use_depth_scaling) radius *= z;
      int id = int(radius / stride_depth_offset + 0.5f);
      if (id >= kDepthOffsets) id = kDepthOffsets - 1;
      const float modeled_depth_offset = __ldg(rc->offsets + id);
      float meter_to_pixel = it.fu * rc->depth->scale;
      if (!dp.use_depth_scaling) meter_to_pixel /= z;
      const float diameter = 2.0f * rc->radius * meter_to_pixel;
      float threshold = rc->threshold;
      if (dp.use_depth_scaling) threshold *= z;
      if (!ModeledWindowUnoccluded(*rc->depth, center_u, center_v, diameter, z - modeled_depth_offset - threshold)) return;
    }
  }
  // FindCorrespondence (:826-884)
  float considered_distance = it.considered_distance;
  if (dp.use_depth_scaling) considered_distance *= z;
  float meter_to_pixel = it.fu / z;
  float diameter = 2.0f * considered_distance * meter_to_pixel;
  int stride = int(diameter / float(it.max_n_strides) + 1.0f);
  int n_strides = int(diameter / float(stride) + 0.5f);
  int rounded_diameter = n_strides * stride;
  float rounded_radius = 0.5f * float(rounded_diameter);
  int u_min = int(center_u - rounded_radius + 0.5f);
  int v_min = int(center_v - rounded_radius + 0.5f);
  int u_max = u_min + rounded_diameter;
  int v_max = v_min + rounded_diameter;
  u_min = max(u_min, 0);
  v_min = max(v_min, 0);
  u_max = min(u_max, it.w_m1);
  v_max = min(v_max, it.h_m1);
  float min_depth_value = fminf(0.0f, (z - considered_distance) / it.depth_scale);  // sic, :851-852
  float max_depth_value = (z + considered_distance) / it.depth_scale;
  float min_considered_distance_square = considered_distance * considered_distance;
  float best = min_considered_distance_square;
  float bx = 0.0f, by = 0.0f, bz = 0.0f;
  const bool inside = u_min >= tile.x0 && u_max < tile.x0 + tile.w && v_min >= tile.y0 && v_max < tile.y0 + tile.h;
  if (inside) {
    const uint16_t* trow = tile_px + (v_min - tile.y0) * tile.pitch - tile.x0;
    const int row_step = stride * tile.pitch;
    // The reference's tests, restated so that most samples cost a handful of instructions (results unchanged):
    //  * depth > min && depth < max on the raw integer sample (a u16 is exact in float: raw > m <=> raw >= floor(m) + 1);
    //  * dz * dz >= best: the exact early-out (d2 >= dz * dz under round-to-nearest);
    //  * a SCREEN with reciprocal multiplies instead of the two divisions: whenever d2 < best, its squared distance s
    //    satisfies s <= best * (1 + 2^-9) + 2^-34 * (|x| + |y|)^2 (DESIGN.md section 3), so a sample with
    //    s > best * (1 + 2^-8) + 2^-33 * (|x| + |y|)^2 + 2^-126 cannot pass the strict test d2 < best, at any depth,
    //    depth scale or considered distance. Everything else is evaluated with the reference's expression, and only
    //    those values are ever stored.
    const int raw_lo = int(floorf(fmaxf(min_depth_value, -2.0f))) + 1;
    const int raw_hi = int(ceilf(fminf(max_depth_value, 70000.0f))) - 1;
    const float rfu = 1.0f / it.fu, rfv = 1.0f / it.fv;
    const float q = fabsf(x) + fabsf(y);
    const float k = 0x1p-33f * (q * q) + 0x1p-126f;  // 2^-126: the roundings of k where q * q is subnormal
    float screen = best * (1.0f + 0x1p-8f) + k;
    for (int v = v_min; v <= v_max; v += stride, trow += row_step) {
      const float vy = float(v) - it.ppv;
#pragma unroll 4
      for (int u = u_min; u <= u_max; u += stride) {
        const int raw = trow[u];
        if (raw >= raw_lo && raw <= raw_hi) {
          const float depth = float(raw) * it.depth_scale;
          const float dz0 = depth - z;
          const float dz2 = dz0 * dz0;
          if (dz2 >= best) continue;
          const float ux = float(u) - it.ppu;
          const float ax = ux * depth * rfu - x, ay = vy * depth * rfv - y;
          if (ax * ax + ay * ay + dz2 > screen) continue;
          float tx = ux * depth / it.fu;
          float ty = vy * depth / it.fv;
          float dx = tx - x, dy = ty - y, dz = depth - z;
          float d2 = dx * dx + dy * dy + dz * dz;
          if (d2 < best) { bx = tx; by = ty; bz = depth; best = d2; screen = best * (1.0f + 0x1p-8f) + k; }
        }
      }
    }
  } else {
    const float4 r = DepthSearchSlow(it.ppu, it.ppv, it.fu, it.fv, it.depth_scale, u_min, u_max, v_min, v_max, stride,
                                     min_depth_value, max_depth_value, x, y, z, frame, tile, tile_px, best);
    best = r.x; bx = r.y; by = r.z; bz = r.w;
  }
  if (best == min_considered_distance_square) return;
  P.yx = bx; P.yy = by; P.yz = bz;
  P.valid = true;
}

// K2 depth: one point's contribution (depth_modality.cpp:333-381)
__device__ __forceinline__ void DepthGradient(const DepthIter& it, const PointState& P, float (&acc)[27]) {
  if (!P.valid) return;
  float yb0, yb1, yb2;
  PoseApply(it.c2b, P.yx, P.yy, P.yz, yb0, yb1, yb2);
  float epsilon = P.nx * (P.cbx - yb0) + P.ny * (P.cby - yb1) + P.nz * (P.cbz - yb2);
  float cx[3] = {yb1 * P.nz - yb2 * P.ny, yb2 * P.nx - yb0 * P.nz, yb0 * P.ny - yb1 * P.nx};
  float weight = 1.0f / (it.standard_deviation * P.yz);
  float squared_weight = weight * weight;
  float v[6] = {weight * cx[0], weight * cx[1], weight * cx[2], weight * P.nx, weight * P.ny, weight * P.nz};
  float se = squared_weight * epsilon;
  float nn[3] = {P.nx, P.ny, P.nz};
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    acc[r] -= se * cx[r];
    acc[3 + r] -= se * nn[r];
  }
  // upper-triangle products v[r] * v[c], r <= c, stored at the mirrored lower index
#pragma unroll
  for (int c = 0; c < 6; ++c)
#pragma unroll
    for (int r = 0; r <= c; ++r) acc[6 + Tri(c, r)] -= v[r] * v[c];
}

// All 32 lanes of warp 0 take the stamp and store it to the same shared-memory slot: warp-uniform control flow,
// so the instrumentation cannot split the warp in front of its full-mask collectives.
#define M3TB_STAMP()                                                              \
  do {                                                                            \
    if (stamp_ptr && (tid >> 5) == 0 && stamp_i < kPhaseSlots) g_stamps[stamp_i++] = clock64(); \
  } while (0)

// ---------------------------------------------------------------------------------------------
// Pose products every thread needs (one evaluation per pose instead of one per thread), thread-serial: every calling
// lane computes everything, lane 0 publishes. body2camera of the colour / depth camera (region_modality.cpp:1001-1002,
// depth_modality.cpp:642-643), the inverse of the depth one (depth_modality.cpp:644) and the GetClosestView queries
// (region_model.cpp:112-120). Expressions are those of PoseMul / PoseInverse / ViewOrientation. sh.cw2c / sh.dw2c must
// be visible. Sh is the shared-memory layout of k_track (Shared) or of k_track2 (Shared2).
// ---------------------------------------------------------------------------------------------
template <class Sh>
__device__ __forceinline__ void PublishPoseProducts(const float (&pose)[12], bool has_color, bool has_depth, bool store_pose,
                                                    Sh& sh) {
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

constexpr unsigned kFloatInfBits = 0x7f800000u;  // bits of +inf: the bits of |x| are greater exactly when x is NaN

// ---------------------------------------------------------------------------------------------
// K4: Optimizer::CalculateOptimization for a rigid body (optimizer.cpp:144-167) = Eigen LDLT<Lower> (pivot = largest
// remaining diagonal entry, first maximum wins; left-looking update) restated for n = 6, then Link::UpdatePoses
// (link.cpp:205-241). The one rigid-body solve of k_track and k_track2 (Sh = Shared / Shared2). Executed redundantly
// by every lane of warp 0: one thread holds the whole permuted matrix in registers, so the dependent chain contains no
// shuffles or shared-memory round trips. sh.a (full symmetric 6x6), sh.b, sh.pose and sh.cw2c / sh.dw2c must be
// visible to the calling warp. Returns true if the pose was updated (sh.pose and the pose products are then refreshed).
// ---------------------------------------------------------------------------------------------
template <class Sh>
__device__ __forceinline__ bool SolveAndUpdateSerial(Sh& sh, bool has_color, bool has_depth) {
  constexpr int n = 6;
  // 1. transposition sequence from the ORIGINAL diagonal: the left-looking factorisation never touches a diagonal
  //    entry before it is chosen as pivot (Eigen LDLT.h, "Find largest diagonal element"). |d| >= 0, so the float bit
  //    patterns order like the values.
  unsigned key[n];
  int pm[n];
  // A NaN is pivoted only when it heads the tail and never wins below it, so it never moves: the NaN positions are
  // those of the original diagonal, their keys are 0 and no step that a NaN heads swaps. A NaN first pivot is the
  // zero-matrix exit (identity transpositions); with a zero first pivot every key is 0 and no step swaps either.
  unsigned nan_steps = 0u;
#pragma unroll
  for (int i = 0; i < n; ++i) {
    const unsigned bits = __float_as_uint(fabsf(sh.a[i * (n + 1)]));
    nan_steps |= unsigned(bits > kFloatInfBits) << i;
    key[i] = bits > kFloatInfBits ? 0u : bits;
    pm[i] = i;
  }
  if (nan_steps & 1u) nan_steps = (1u << n) - 1u;
#pragma unroll
  for (int k = 0; k < n - 1; ++k) {
    int p = k;
    unsigned big = key[k];
#pragma unroll
    for (int q = k + 1; q < n; ++q)
      if (key[q] > big) { big = key[q]; p = q; }
    if (nan_steps & (1u << k)) p = k;
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

// (i, j) of packed lower-triangle index e
__device__ __forceinline__ void TriInv(int e, int& i, int& j) {
  i = (e >= 15) ? 5 : (e >= 10) ? 4 : (e >= 6) ? 3 : (e >= 3) ? 2 : (e >= 1) ? 1 : 0;
  j = e - i * (i + 1) / 2;
}

// ---------------------------------------------------------------------------------------------
// ROI tiles. The rectangle every line sample / depth window of this launch can touch is bounded by the
// projected bounding sphere of the model plus the longest line (or the widest search window) plus a
// motion margin; it is computed once from the pose at launch. Samples that still fall outside (large pose
// updates, clipped tiles) are read from the frame in global memory, so tiling never changes a result.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void RoiRect(const float* b2c, float fu, float fv, float ppu, float ppv, int width, int height,
                                        float radius, float reach_px, int align_x, Tile& t) {
  const float z = b2c[11];
  t.x0 = t.y0 = t.w = t.h = t.pitch = 0;
  if (!(z > 2.0f * radius)) return;  // too close / behind: no tile, global path only
  const float cu = b2c[3] * fu / z + ppu, cv = b2c[7] * fv / z + ppv;
  const float ru = radius * fu / (z - radius) + reach_px, rv = radius * fv / (z - radius) + reach_px;
  int x0 = int(floorf(cu - ru)), x1 = int(ceilf(cu + ru)) + 1;
  int y0 = int(floorf(cv - rv)), y1 = int(ceilf(cv + rv)) + 1;
  x0 = max(x0, 0) / align_x * align_x;
  x1 = min((min(x1, width) + align_x - 1) / align_x * align_x, width / align_x * align_x);
  y0 = max(y0, 0);
  y1 = min(y1, height);
  if (x1 <= x0 || y1 <= y0) return;
  t.x0 = x0; t.y0 = y0; t.w = x1 - x0; t.h = y1 - y0; t.pitch = t.w;
}

__device__ __forceinline__ void ClipTile(Tile& t, const FrameView& f, int align_x) {
  if (t.w <= 0) return;
  int x0 = max(t.x0, (f.x0 + align_x - 1) / align_x * align_x), x1 = min(t.x0 + t.w, f.x1 / align_x * align_x);
  int y0 = max(t.y0, f.y0), y1 = min(t.y0 + t.h, f.y1);
  if (x1 <= x0 || y1 <= y0) { t.w = t.h = t.pitch = 0; return; }
  t.x0 = x0; t.y0 = y0; t.w = x1 - x0; t.h = y1 - y0; t.pitch = t.w;
}

// shrink symmetric about the centre until the tile fits `budget` bytes (2 bytes per pixel)
__device__ __forceinline__ void FitTile(Tile& t, int budget, int align_x) {
  while (t.w > 0 && t.h > 0 && t.w * t.h * 2 > budget) {
    if (t.h >= t.w && t.h > 16) { t.y0 += 4; t.h -= 8; }
    else if (t.w > 2 * align_x) { t.x0 += align_x; t.w -= 2 * align_x; }
    else { t.w = t.h = 0; }
  }
  t.pitch = t.w;
}

// ---------------------------------------------------------------------------------------------
// The fused kernel
// ---------------------------------------------------------------------------------------------

template <int T, int K, bool LUT_SMEM, bool OCC>
__global__ void __launch_bounds__(T, 512 / T) k_track(const __grid_constant__ TrackArgs args) {
  extern __shared__ __align__(128) unsigned char dyn[];
  __shared__ Shared sh;
  constexpr int kW = T / 32;
  const int body_id = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const BodyDev& body = args.bodies[body_id];
  if (!body.set) return;
  const bool has_region = body.has_region, has_depth = body.has_depth;
  const int lcap = args.line_cap, pcap = args.point_cap;
  float* g_rst = args.region_state + size_t(body_id) * RF_COUNT * lcap;
  float* g_dst = args.depth_state + size_t(body_id) * DF_COUNT * pcap;
  int* counts = args.counts + 4 * body_id;
  const float2* lut_g = args.lut + size_t(body_id) * args.lut_stride;
  const float2* lut_s = reinterpret_cast<const float2*>(dyn);

  // profiling aid: stamps go to shared memory (cheap) and are flushed at the end of the kernel
  __shared__ long long g_stamps_storage[kPhaseSlots];
  long long* g_stamps = g_stamps_storage;
  long long* stamp_ptr = args.phase_clock ? args.phase_clock + size_t(body_id) * kPhaseSlots : nullptr;
  int stamp_i = 0;
  M3TB_STAMP();
  // ---- prologue: pose, LUT bulk copy, ROI tiles ----------------------------------------------------
  const CameraDev* ccam = has_region ? &args.color_cams[body.color_camera] : nullptr;
  // the depth camera serves the depth modality and, with measured occlusion handling, the region modality
  const bool region_occ = OCC && has_region && body.rp.measure_occlusions;
  const CameraDev* dcam = (has_depth || region_occ) ? &args.depth_cams[body.depth_camera] : nullptr;
  const ModelDev* rmodel = has_region ? &args.region_models[body.region_model] : nullptr;
  const ModelDev* dmodel = has_depth ? &args.depth_models[body.depth_model] : nullptr;
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
  const bool need_lut = LUT_SMEM && do_rcorr;
  const unsigned lut_bytes = LUT_SMEM ? unsigned(16 * 16 * 16 * sizeof(float2)) : 0u;
  if (tid == 0) {
    if (LUT_SMEM) MbarInit(&sh.lut_bar, 1);
    MbarInit(&sh.depth_bar, 1);
  }
  __syncthreads();
  if (warp == 0) {
    float pose[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) pose[i] = sh.pose[i];
    PublishPoseProducts(pose, ccam != nullptr, dcam != nullptr, /*store_pose=*/false, sh);
  }
  if (need_lut && tid == 0) {
    const unsigned bytes = unsigned(body.rp.n_bins * body.rp.n_bins * body.rp.n_bins) * sizeof(float2);
    MbarExpectTx(&sh.lut_bar, bytes);
    BulkCopyG2S(dyn, lut_g, bytes, &sh.lut_bar);
  }
  if (tid == 0) {
    Tile ct, dt;
    ct.x0 = ct.y0 = ct.w = ct.h = ct.pitch = 0; ct.offset = lut_bytes;
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
      // tiles are built from the device copy: keep them inside the rectangle where that copy is valid
      ClipTile(ct, cframe, 4);
      ClipTile(dt, dframe, 8);
      // split the budget: the depth tile is the smaller one, give it what it asks for up to 40 %
      int budget = args.tile_bytes - 256;
      FitTile(dt, budget * 2 / 5, 8);
      const int dbytes = (dt.w * dt.h * 2 + 127) / 128 * 128;
      FitTile(ct, budget - dbytes, 4);
      const int cbytes = (ct.w * ct.h * 2 + 127) / 128 * 128;
      dt.offset = lut_bytes + unsigned(cbytes);
    }
    sh.ctile = ct;
    sh.dtile = dt;
  }
  __syncthreads();
  const Tile ctile = sh.ctile, dtile = sh.dtile;
  const uint16_t* ctile_px = reinterpret_cast<const uint16_t*>(dyn + ctile.offset);
  const uint16_t* dtile_px = reinterpret_cast<const uint16_t*>(dyn + dtile.offset);
  // depth tile: one TMA bulk copy per row (16 B aligned: x0 and w are multiples of 8 pixels), all rows complete
  // on one mbarrier; issued by warp 1 so that it overlaps the colour conversion below.
  bool depth_ready = true;
  if (dtile.w > 0) {
    depth_ready = false;
    if (warp == 1 % kW) {
      const unsigned row_bytes = unsigned(dtile.w) * 2u;
      if (lane == 0) MbarExpectTx(&sh.depth_bar, row_bytes * unsigned(dtile.h));
      __syncwarp();
      for (int r = lane; r < dtile.h; r += 32)
        BulkCopyG2S(dyn + dtile.offset + size_t(r) * row_bytes,
                    dcam->image + size_t(dtile.y0 + r) * dcam->pitch + size_t(dtile.x0) * 2u, row_bytes, &sh.depth_bar);
    }
  }
  // colour tile: 4 pixels (12 bytes, three aligned words) -> 4 bin indices (one 8-byte store) per work item
  if (ctile.w > 0) {
    const int groups_per_row = ctile.w >> 2;
    const int n_groups = groups_per_row * ctile.h;
    const int bs = body.rp.bitshift, nb = body.rp.n_bins;
    uint2* out = reinterpret_cast<uint2*>(dyn + ctile.offset);
    auto bin = [&](unsigned b, unsigned gch, unsigned rch) {
      return LutSlot(((b >> bs) * unsigned(nb) + (gch >> bs)) * unsigned(nb) + (rch >> bs));
    };
    for (int g0 = tid; g0 < n_groups; g0 += 4 * T) {  // 12 independent word loads in flight per thread
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
    __syncthreads();
  }

  LineState L[K];
  PointState P[K];
  int n_lines = 0, n_points = 0, view_r = 0, view_d = 0;
#pragma unroll
  for (int k = 0; k < K; ++k) { L[k].valid = false; P[k].valid = false; }
  if (args.phases & PH_LOAD_REGION) {
    n_lines = counts[0];
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int i = tid + k * T;
      if (i < n_lines) {
        L[k].cbx = g_rst[RF_CBX * lcap + i]; L[k].cby = g_rst[RF_CBY * lcap + i]; L[k].cbz = g_rst[RF_CBZ * lcap + i];
        L[k].cu = g_rst[RF_CU * lcap + i]; L[k].cv = g_rst[RF_CV * lcap + i];
        L[k].nu = g_rst[RF_NU * lcap + i]; L[k].nv = g_rst[RF_NV * lcap + i];
        L[k].dr = g_rst[RF_DR * lcap + i]; L[k].ncts = g_rst[RF_NCTS * lcap + i];
        L[k].mean = g_rst[RF_MEAN * lcap + i]; L[k].var = g_rst[RF_VAR * lcap + i];
#pragma unroll
        for (int d = 0; d < kDistributionLength; ++d) L[k].dist[d] = g_rst[(RF_DIST0 + d) * lcap + i];
        L[k].valid = g_rst[RF_VALID * lcap + i] != 0.0f;
      }
    }
  }
  if (args.phases & PH_LOAD_DEPTH) {
    n_points = counts[1];
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int i = tid + k * T;
      if (i < n_points) {
        P[k].cbx = g_dst[DF_CBX * pcap + i]; P[k].cby = g_dst[DF_CBY * pcap + i]; P[k].cbz = g_dst[DF_CBZ * pcap + i];
        P[k].nx = g_dst[DF_NX * pcap + i]; P[k].ny = g_dst[DF_NY * pcap + i]; P[k].nz = g_dst[DF_NZ * pcap + i];
        P[k].yx = g_dst[DF_YX * pcap + i]; P[k].yy = g_dst[DF_YY * pcap + i]; P[k].yz = g_dst[DF_YZ * pcap + i];
        P[k].valid = g_dst[DF_VALID * pcap + i] != 0.0f;
      }
    }
  }

  bool lut_ready = !need_lut;
  M3TB_STAMP();  // prologue done

  for (int corr = args.corr_begin; corr < args.corr_end; ++corr) {
    // ---------------- CalculateCorrespondences -------------------------------------------------
    if (do_rcorr || do_dcorr) {
      int v0, v1;
      ClosestViews<T>(do_rcorr ? rmodel : nullptr, do_dcorr ? dmodel : nullptr, sh, corr & 1, v0, v1);
      M3TB_STAMP();  // closest views
      if (do_rcorr) {
        RegionIter rit;
        MakeRegionIter(body.rp, *ccam, sh.rb2c, corr, rit);
        view_r = v0;
        n_lines = AdaptiveCount(body.rp.n_lines_max, body.rp.use_adaptive_coverage, body.rp.reference_contour_length,
                                __ldg(rmodel->view_scalars + view_r), rmodel->max_view_scalar, rmodel->n_points);
        n_lines = min(n_lines, min(lcap, K * T));
        if (!lut_ready) { MbarWait(&sh.lut_bar, 0); lut_ready = true; }
        const float4* pts = rmodel->points + size_t(view_r) * rmodel->n_points * 2;
        // measured occlusion handling: two passes (region_modality.cpp:435-463)
        RegionOcclusion rocc;
        bool handle = false;
        if (OCC) {
          handle = region_occ && rmodel->depth_offsets != nullptr &&
                   (args.iteration - body.first_iteration) >= body.rp.n_unoccluded_iterations;
          if (handle) {
            if (!depth_ready) { MbarWait(&sh.depth_bar, 0); depth_ready = true; }
            rocc.b2d = sh.db2c;
            rocc.offsets = rmodel->depth_offsets + size_t(view_r) * rmodel->n_points * kDepthOffsets;
            rocc.offset_id = int(body.rp.measured_depth_offset_radius / rmodel->stride_depth_offset + 0.5f);
            rocc.fu = dcam->fu; rocc.fv = dcam->fv; rocc.ppu = dcam->ppu; rocc.ppv = dcam->ppv;
            rocc.depth_scale = dcam->depth_scale;
            rocc.w_m1 = dcam->width - 1; rocc.h_m1 = dcam->height - 1;
            rocc.radius = body.rp.measured_occlusion_radius; rocc.threshold = body.rp.measured_occlusion_threshold;
            rocc.frame = &dframe; rocc.tile = &dtile; rocc.tile_px = dtile_px;
          }
        }
        // checks on renderer images: region checking in both passes (:402-408), modeled occlusions in the first (:447)
        RenderChecks rchk;
        bool use_rchk = false, handle_modeled = false;
        if (OCC) {
          const RenderingDev& sr = body.rend[RS_REGION_SILHOUETTE];
          const RenderingDev& dr = body.rend[RS_REGION_DEPTH];
          rchk.silhouette = (body.rp.use_region_checking && sr.image && sr.visible) ? &sr : nullptr;
          handle_modeled = body.rp.model_occlusions && dr.image && dr.visible && rmodel->depth_offsets != nullptr &&
                           (args.iteration - body.first_iteration) >= body.rp.n_unoccluded_iterations;
          rchk.depth = handle_modeled ? &dr : nullptr;
          rchk.offsets = rmodel->depth_offsets ? rmodel->depth_offsets + size_t(view_r) * rmodel->n_points * kDepthOffsets : nullptr;
          rchk.modeled_offset_id = int(body.rp.modeled_depth_offset_radius / rmodel->stride_depth_offset + 0.5f);
          rchk.radius = body.rp.modeled_occlusion_radius;
          rchk.threshold = body.rp.modeled_occlusion_threshold;
          rchk.offset_radius = body.rp.modeled_depth_offset_radius;
          use_rchk = rchk.silhouette != nullptr || rchk.depth != nullptr;
        }
        for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
          for (int k = 0; k < K; ++k) {
            const int i = tid + k * T;
            L[k].valid = false;
            if (i < n_lines) {
              float4 p0 = __ldg(pts + 2 * i), p1 = __ldg(pts + 2 * i + 1);
              RegionLine<LUT_SMEM, OCC>(rit, body.rp, p0, p1, cframe, ctile, ctile_px, lut_g, lut_s, L[k],
                                        handle ? &rocc : nullptr, i, use_rchk ? &rchk : nullptr);
            }
          }
          if (!OCC || !(handle || handle_modeled)) break;
          int survivors = 0;
#pragma unroll
          for (int k = 0; k < K; ++k) survivors += __syncthreads_count(L[k].valid);
          if (survivors >= body.rp.min_n_unoccluded_lines) break;
          handle = false;
          handle_modeled = false;
          rchk.depth = nullptr;
          use_rchk = rchk.silhouette != nullptr;
        }
      }
      M3TB_STAMP();  // region lines (thread 0's own line)
      if (do_dcorr) {
        DepthIter dit;
        MakeDepthIter(body.dp, *dcam, sh.db2c, sh.dc2b, corr, dit);
        view_d = v1;
        n_points = AdaptiveCount(body.dp.n_points_max, body.dp.use_adaptive_coverage, body.dp.reference_surface_area,
                                 __ldg(dmodel->view_scalars + view_d), dmodel->max_view_scalar, dmodel->n_points);
        n_points = min(n_points, min(pcap, K * T));
        if (!depth_ready) { MbarWait(&sh.depth_bar, 0); depth_ready = true; }
        const float4* pts = dmodel->points + size_t(view_d) * dmodel->n_points * 2;
        bool handle = false;
        const float* offs = nullptr;
        if (OCC) {  // depth_modality.cpp:295-313
          handle = body.dp.measure_occlusions && dmodel->depth_offsets != nullptr &&
                   (args.iteration - body.first_iteration) >= body.dp.n_unoccluded_iterations;
          if (handle) offs = dmodel->depth_offsets + size_t(view_d) * dmodel->n_points * kDepthOffsets;
        }
        RenderChecks dchk;  // silhouette checking in both passes (:264-270), modeled occlusions in the first
        bool use_dchk = false, handle_modeled = false;
        if (OCC) {
          const RenderingDev& sr = body.rend[RS_DEPTH_SILHOUETTE];
          const RenderingDev& dr = body.rend[RS_DEPTH_DEPTH];
          dchk.silhouette = (body.dp.use_silhouette_checking && sr.image && sr.visible) ? &sr : nullptr;
          handle_modeled = body.dp.model_occlusions && dr.image && dr.visible && dmodel->depth_offsets != nullptr &&
                           (args.iteration - body.first_iteration) >= body.dp.n_unoccluded_iterations;
          dchk.depth = handle_modeled ? &dr : nullptr;
          dchk.offsets = nullptr;
          dchk.modeled_offset_id = 0;
          dchk.radius = body.dp.modeled_occlusion_radius;
          dchk.threshold = body.dp.modeled_occlusion_threshold;
          dchk.offset_radius = body.dp.modeled_depth_offset_radius;
          use_dchk = dchk.silhouette != nullptr || dchk.depth != nullptr;
        }
        for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
          for (int k = 0; k < K; ++k) {
            const int i = tid + k * T;
            P[k].valid = false;
            if (i < n_points) {
              float4 p0 = __ldg(pts + 2 * i), p1 = __ldg(pts + 2 * i + 1);
              RenderChecks mine = dchk;  // per-point depth offsets
              if (OCC && dmodel->depth_offsets)
                mine.offsets = dmodel->depth_offsets + (size_t(view_d) * dmodel->n_points + i) * kDepthOffsets;
              DepthPoint<OCC>(dit, body.dp, p0, p1, dframe, dtile, dtile_px, P[k],
                              handle ? offs + size_t(i) * kDepthOffsets : nullptr, dmodel->stride_depth_offset,
                              use_dchk ? &mine : nullptr);
            }
          }
          if (!OCC || !(handle || handle_modeled)) break;
          int survivors = 0;
#pragma unroll
          for (int k = 0; k < K; ++k) survivors += __syncthreads_count(P[k].valid);
          if (survivors >= body.dp.min_n_unoccluded_points) break;
          handle = false;
          handle_modeled = false;
          dchk.depth = nullptr;
          use_dchk = dchk.silhouette != nullptr;
        }
      }
    }

    M3TB_STAMP();  // depth points (thread 0's own point)
    // ---------------- n_update x (CalculateGradientAndHessian + CalculateOptimization) ---------
    for (int upd = 0; upd < args.n_update; ++upd) {
      const int opt_iteration = args.opt_base + upd;
      float acc[27];
#pragma unroll
      for (int k = 0; k < 27; ++k) acc[k] = 0.0f;
      if (has_region && (args.phases & PH_REGION_GH)) {
        RegionIter rit;
        MakeRegionIter(body.rp, *ccam, sh.rb2c, corr, rit);
#pragma unroll
        for (int k = 0; k < K; ++k) RegionGradient(rit, body.rp, L[k], opt_iteration, acc);
      }
      if (has_depth && (args.phases & PH_DEPTH_GH)) {
        DepthIter dit;
        MakeDepthIter(body.dp, *dcam, sh.db2c, sh.dc2b, corr, dit);
#pragma unroll
        for (int k = 0; k < K; ++k) DepthGradient(dit, P[k], acc);
      }
      const bool tex_gh = body.has_texture && (args.phases & PH_TEXTURE_GH);
      if (tex_gh) {  // the texture term after region and depth (the evaluators' AddModality order)
        TextureGradient(args.color_cams[body.texture_camera], sh.pose, body.tp, corr,
                        args.tex_points + size_t(body_id) * TF_COUNT * args.tex_point_cap, args.tex_point_cap,
                        args.tex_counts[body_id], tid, T, acc);
        // PrecalculatePoseVariables of this pass: CalculateResults reconstructs keyframes with it (sh.pose changes
        // only in the solve, behind the barrier below)
        if (tid < 12) args.tex_pose[12 * body_id + tid] = sh.pose[tid];
      }
      // Warp reduction by recursive halving: the 27 sums are padded to 32; at each of the 5 butterfly steps a
      // lane keeps one half of its values and hands the other half to its partner, so 31 shuffle+add pairs per
      // lane replace the 135 of a value-by-value tree, and lane l ends up with the warp total of value kSlot(l).
      {
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
        // value index held by this lane: bit b of the index is set iff lane bit b is set (same bit, same weight)
        sh.red[warp][lane] = v[0];
      }
      M3TB_STAMP();  // accumulate + warp reduce
      __syncthreads();
      M3TB_STAMP();  // all warps arrived
      if (warp == 0) {
        // Branch-free on purpose: a divergent branch here would leave the warp split when it reaches the
        // full-mask shuffles of the solve (the compiler then runs their slow divergent path). Lanes >= 27
        // shadow lane 26 and redundantly store the same values to the same addresses.
        const int l = lane < 27 ? lane : 26;
        float v = sh.red[0][l];
#pragma unroll
        for (int w = 1; w < kW; ++w) v += sh.red[w][l];
        if (args.phases & PH_STORE_GH) {
          if (args.phases & PH_REGION_GH) args.gh_region[27 * body_id + l] = v;
          if (args.phases & PH_DEPTH_GH) args.gh_depth[27 * body_id + l] = v;
          if (args.phases & PH_TEXTURE_GH) args.gh_texture[27 * body_id + l] = v;
        }
        if (args.phases & PH_STORE_LINK_GH) args.gh_link[27 * body_id + l] = v;
        if (args.phases & PH_LOAD_GH) {  // Link::CalculateGradientAndHessian (link.cpp:184-193): region, depth, texture
          v = 0.0f + args.gh_region[27 * body_id + l] + args.gh_depth[27 * body_id + l];
          if (body.has_texture) v = v + args.gh_texture[27 * body_id + l];
        }
        if (args.phases & PH_SOLVE) {
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
          M3TB_STAMP();  // cross-warp sum + normal equations
          SolveAndUpdateSerial(sh, ccam != nullptr, dcam != nullptr);
        }
      }
      if (args.phases & PH_SOLVE) M3TB_STAMP();  // solve + pose products (warp 0)
      __syncthreads();
      M3TB_STAMP();  // solve + pose update
    }
  }

  // ---------------- epilogue ----------------------------------------------------------------------
  if (args.phases & PH_SOLVE)
    if (tid < 12) args.poses[12 * body_id + tid] = sh.pose[tid];
  if (args.phases & PH_STORE_REGION) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int i = tid + k * T;
      if (i < n_lines) {
        g_rst[RF_CBX * lcap + i] = L[k].cbx; g_rst[RF_CBY * lcap + i] = L[k].cby; g_rst[RF_CBZ * lcap + i] = L[k].cbz;
        g_rst[RF_CU * lcap + i] = L[k].cu; g_rst[RF_CV * lcap + i] = L[k].cv;
        g_rst[RF_NU * lcap + i] = L[k].nu; g_rst[RF_NV * lcap + i] = L[k].nv;
        g_rst[RF_VALID * lcap + i] = L[k].valid ? 1.0f : 0.0f;
        if (L[k].valid) {
          g_rst[RF_DR * lcap + i] = L[k].dr; g_rst[RF_NCTS * lcap + i] = L[k].ncts;
          g_rst[RF_MEAN * lcap + i] = L[k].mean; g_rst[RF_VAR * lcap + i] = L[k].var;
#pragma unroll
          for (int d = 0; d < kDistributionLength; ++d) g_rst[(RF_DIST0 + d) * lcap + i] = L[k].dist[d];
        }
      }
    }
    if (tid == 0) { counts[0] = n_lines; counts[2] = view_r; }
  }
  if (args.phases & PH_STORE_DEPTH) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int i = tid + k * T;
      if (i < n_points) {
        g_dst[DF_CBX * pcap + i] = P[k].cbx; g_dst[DF_CBY * pcap + i] = P[k].cby; g_dst[DF_CBZ * pcap + i] = P[k].cbz;
        g_dst[DF_NX * pcap + i] = P[k].nx; g_dst[DF_NY * pcap + i] = P[k].ny; g_dst[DF_NZ * pcap + i] = P[k].nz;
        g_dst[DF_VALID * pcap + i] = P[k].valid ? 1.0f : 0.0f;
        if (P[k].valid) {
          g_dst[DF_YX * pcap + i] = P[k].yx; g_dst[DF_YY * pcap + i] = P[k].yy; g_dst[DF_YZ * pcap + i] = P[k].yz;
        }
      }
    }
    if (tid == 0) { counts[1] = n_points; counts[3] = view_d; }
  }
  if (stamp_ptr && tid == 0)
    for (int k = 0; k < kPhaseSlots; ++k) stamp_ptr[k] = k < stamp_i ? g_stamps[k] : 0;
  if (need_lut && !lut_ready) MbarWait(&sh.lut_bar, 0);  // never leave with a bulk copy in flight
  if (!depth_ready) MbarWait(&sh.depth_bar, 0);
}

// ---------------------------------------------------------------------------------------------
// k_lut: per-bin normalisation (pf, pb) -> (pf/(pf+pb), pb/(pf+pb)) or (0.5, 0.5) if both are zero.
// This is MultiplyPixelColorProbability's per-pixel normalisation (region_modality.cpp:1585-1593)
// hoisted to once per bin; same IEEE divisions, hence bit-identical per-pixel values.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 NormaliseBin(float pf, float pb) {
  if (pf != 0.0f || pb != 0.0f) {
    float sum = pf;
    sum += pb;
    return make_float2(pf / sum, pb / sum);
  }
  return make_float2(0.5f, 0.5f);
}

#ifndef M3TB_TRACK_TU  // the auxiliary kernels are compiled once, in m3t_b200.cu
__global__ void k_lut(const float* hist_f, const float* hist_b, float2* lut, int n, size_t stride, int first_body) {
  const int body = first_body + blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) lut[size_t(body) * stride + LutSlot(unsigned(i))] = NormaliseBin(hist_f[size_t(body) * stride + i], hist_b[size_t(body) * stride + i]);
}

// ---------------------------------------------------------------------------------------------
// k_histogram: RegionModality::AddLinePixelColorsToTempHistograms (region_modality.cpp:1025-1155)
// + ColorHistograms::InitializeHistograms / UpdateHistograms (color_histograms.cpp:72-92,174-214).
// One CTA per body. Counts are integer-valued floats (< 2^24), so atomic accumulation order and the
// tree-shaped sum are exact; the blend h = h*(1-lr) + mem*(lr/sum) rounds as the reference does.
// mode 0: StartModality (learning rate 1), 1: CalculateResults.
// ---------------------------------------------------------------------------------------------
struct HistArgs {
  const BodyDev* bodies;
  const float* poses;
  const CameraDev* color_cams;
  const ModelDev* region_models;
  float* hist_f;
  float* hist_b;
  float* mem_f;
  float* mem_b;
  float2* lut;
  size_t stride;
  int mode;
  const RoiRecord* roi;
  const CameraDev* depth_cams;  // measured occlusion handling
  int iteration;
  const int* shared_owner;      // per body: -1 = its own ColorHistograms, else the owner of the shared one (or null: none shared)
  const int* body_list;         // optional: CTA i handles body body_list[i] (m3tb_refine_poses), null: body i
};

// RegionModality::UseSharedColorHistograms (region_modality.cpp:168-179): the members of a group only ADD their line
// pixels (k_histogram, into their own count arrays); the tracker then runs InitializeHistograms / UpdateHistograms once on
// the shared object (tracker.cpp:435-443, 507-515) - k_histogram_shared, one CTA per group.
struct SharedHistArgs {
  const BodyDev* bodies;
  float* hist_f;
  float* hist_b;
  float* mem_f;
  float* mem_b;
  float2* lut;
  size_t stride;
  int mode;
  const int* group_owner;   // [n_groups]
  const int* group_first;   // [n_groups + 1] into members
  const int* members;       // body indices, owner first
  const int* group_summed;  // optional [n_groups]: only members [first, first + summed) add their counts (the refined
                            //   ones, m3tb_refine_poses); the result still goes to every member. null: all of them
};

// ---------------------------------------------------------------------------------------------
// k_ingest: frame ingest for pinned host frames (SURVEY §8 f3). One CTA per body: the rectangle of the colour /
// depth frame this body can touch during a whole tracking cycle (projected bounding sphere + longest
// correspondence line or widest depth window + a motion margin) is fetched straight from the caller's pinned
// frame over PCIe into the device copy - ~1/7 of the frame at 0.6 m - and recorded as the body's RoiRecord.
// Pixels outside it are still reachable (FrameView falls back to the pinned frame), so this never changes a result.
// ---------------------------------------------------------------------------------------------
// pixels of pose motion (since the ROI was fetched) that stay inside the device copy; beyond it samples are served
// from the pinned frame directly (correct, slower)
constexpr float kIngestMotionMarginPx = 8.0f;

struct IngestArgs {
  const BodyDev* bodies;
  const float* poses;
  const CameraDev* color_cams;
  const CameraDev* depth_cams;
  const ModelDev* region_models;
  const ModelDev* depth_models;
  RoiRecord* roi;
  unsigned long long* bytes;  // total bytes fetched by this launch
  int n_bodies;               // the grid may be smaller: CTAs loop over the bodies (see m3tb_prefetch_frames)
  const int* body_list;       // optional: the n_bodies bodies to fetch for (m3tb_refine_poses), null: bodies 0..n_bodies
};

__device__ __forceinline__ void IngestRect(const CameraDev& cam, const Tile& t, unsigned bpp, unsigned long long* bytes) {
  if (t.w <= 0 || t.h <= 0) return;
  const unsigned row_bytes = unsigned(t.w) * bpp;
  const uint8_t* src0 = cam.host_src + size_t(t.y0) * cam.host_pitch + size_t(t.x0) * bpp;
  uint8_t* dst0 = const_cast<uint8_t*>(cam.image) + size_t(t.y0) * cam.pitch + size_t(t.x0) * bpp;
  const bool vec16 = ((reinterpret_cast<size_t>(src0) | cam.host_pitch | row_bytes) & 15u) == 0;  // dst is 16 B aligned by construction
  if (vec16) {
    const int per_row = int(row_bytes >> 4);
    const int total = per_row * t.h;
    for (int c0 = threadIdx.x; c0 < total; c0 += 4 * blockDim.x) {  // four 16-byte PCIe reads in flight per thread
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int c = c0 + u * blockDim.x;
        if (c < total) {
          const int r = c / per_row, k = c - r * per_row;
          v[u] = __ldg(reinterpret_cast<const uint4*>(src0 + size_t(r) * cam.host_pitch) + k);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int c = c0 + u * blockDim.x;
        if (c < total) {
          const int r = c / per_row, k = c - r * per_row;
          reinterpret_cast<uint4*>(dst0 + size_t(r) * cam.pitch)[k] = v[u];
        }
      }
    }
  } else {
    const int total = int(row_bytes) * t.h;
    for (int c = threadIdx.x; c < total; c += blockDim.x) {
      const int r = c / int(row_bytes), k = c - r * int(row_bytes);
      dst0[size_t(r) * cam.pitch + k] = __ldg(src0 + size_t(r) * cam.host_pitch + k);
    }
  }
  if (threadIdx.x == 0) atomicAdd(bytes, static_cast<unsigned long long>(row_bytes) * t.h);
}

__device__ __forceinline__ unsigned BinOf(unsigned b, unsigned g, unsigned r, int bs, unsigned nb) {  // -> lookup-table slot
  return LutSlot(((b >> bs) * nb + (g >> bs)) * nb + (r >> bs));  // color_histograms.cpp:97-99, BGR memory order
}
// 16 pixels = 48 bytes (three 16-byte words) -> 16 bin indices (two 16-byte words)
__device__ __forceinline__ void Bins16(const uint4 (&w)[3], int bs, unsigned nb, uint4& lo, uint4& hi) {
  unsigned char px[48];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const unsigned v[4] = {w[k].x, w[k].y, w[k].z, w[k].w};
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int b = 0; b < 4; ++b) px[16 * k + 4 * q + b] = (unsigned char)((v[q] >> (8 * b)) & 0xffu);
  }
  unsigned o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const unsigned a = BinOf(px[6 * i], px[6 * i + 1], px[6 * i + 2], bs, nb);
    const unsigned c = BinOf(px[6 * i + 3], px[6 * i + 4], px[6 * i + 5], bs, nb);
    o[i] = a | (c << 16);
  }
  lo = make_uint4(o[0], o[1], o[2], o[3]);
  hi = make_uint4(o[4], o[5], o[6], o[7]);
}

// Colour ROI ingest that also writes the bin-index image (source of k_track2's TMA colour tiles): x0 and w are
// multiples of 16 pixels, so a work item is 48 bytes in, 48 + 32 bytes out.
__device__ __forceinline__ void IngestColorRect(const CameraDev& cam, const Tile& t, int bs, unsigned nb, unsigned long long* bytes) {
  if (t.w <= 0 || t.h <= 0) return;
  const unsigned row_bytes = unsigned(t.w) * 3u;
  const uint8_t* src0 = cam.host_src + size_t(t.y0) * cam.host_pitch + size_t(t.x0) * 3u;
  uint8_t* dst0 = const_cast<uint8_t*>(cam.image) + size_t(t.y0) * cam.pitch + size_t(t.x0) * 3u;
  uint8_t* bin0 = reinterpret_cast<uint8_t*>(cam.bins) + size_t(t.y0) * cam.bin_pitch + size_t(t.x0) * 2u;
  const bool vec16 = ((reinterpret_cast<size_t>(src0) | cam.host_pitch) & 15u) == 0 && (t.w & 15) == 0 && (t.x0 & 15) == 0;
  if (vec16) {
    const int per_row = t.w >> 4;
    const int total = per_row * t.h;
    for (int c0 = threadIdx.x; c0 < total; c0 += 2 * blockDim.x) {  // six 16-byte PCIe reads in flight per thread
      uint4 v[2][3];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int c = c0 + u * blockDim.x;
        if (c < total) {
          const int r = c / per_row, k = c - r * per_row;
          const uint4* s = reinterpret_cast<const uint4*>(src0 + size_t(r) * cam.host_pitch) + 3 * k;
          v[u][0] = __ldg(s); v[u][1] = __ldg(s + 1); v[u][2] = __ldg(s + 2);
        }
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int c = c0 + u * blockDim.x;
        if (c < total) {
          const int r = c / per_row, k = c - r * per_row;
          uint4* d = reinterpret_cast<uint4*>(dst0 + size_t(r) * cam.pitch) + 3 * k;
          d[0] = v[u][0]; d[1] = v[u][1]; d[2] = v[u][2];
          uint4 lo, hi;
          Bins16(v[u], bs, nb, lo, hi);
          uint4* b = reinterpret_cast<uint4*>(bin0 + size_t(r) * cam.bin_pitch) + 2 * k;
          b[0] = lo; b[1] = hi;
        }
      }
    }
  } else {
    const int total = t.w * t.h;
    for (int c = threadIdx.x; c < total; c += blockDim.x) {
      const int r = c / t.w, k = c - r * t.w;
      const uint8_t* s = src0 + size_t(r) * cam.host_pitch + 3 * k;
      uint8_t* d = dst0 + size_t(r) * cam.pitch + 3 * k;
      const unsigned b0 = __ldg(s), b1 = __ldg(s + 1), b2 = __ldg(s + 2);
      d[0] = (uint8_t)b0; d[1] = (uint8_t)b1; d[2] = (uint8_t)b2;
      reinterpret_cast<uint16_t*>(bin0 + size_t(r) * cam.bin_pitch)[k] = (uint16_t)BinOf(b0, b1, b2, bs, nb);
    }
  }
  if (threadIdx.x == 0) atomicAdd(bytes, static_cast<unsigned long long>(row_bytes) * t.h);
}

// k_bin: bin-index image of whole colour frames (frames that were copied in full; grid = (rows, cameras)).
struct BinArgs {
  const CameraDev* cams;
  const int* cam_ids;   // cameras to convert
  int bitshift, n_bins;
};
__global__ void __launch_bounds__(kBlockThreads) k_bin(BinArgs args) {
  const CameraDev& cam = args.cams[args.cam_ids[blockIdx.y]];
  if (!cam.bins || !cam.image) return;
  const int groups = (cam.width + 3) >> 2;  // 4 pixels = 12 bytes = three aligned words (pitch is a multiple of 16)
  for (int y = blockIdx.x; y < cam.height; y += gridDim.x) {
    const unsigned* src = reinterpret_cast<const unsigned*>(cam.image + size_t(y) * cam.pitch);
    uint2* dst = reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(cam.bins) + size_t(y) * cam.bin_pitch);
    for (int g = threadIdx.x; g < groups; g += blockDim.x) {
      const unsigned w0 = __ldg(src + 3 * g), w1 = __ldg(src + 3 * g + 1), w2 = __ldg(src + 3 * g + 2);
      const unsigned nb = unsigned(args.n_bins);
      const int bs = args.bitshift;
      const unsigned i0 = BinOf(w0 & 0xffu, (w0 >> 8) & 0xffu, (w0 >> 16) & 0xffu, bs, nb);
      const unsigned i1 = BinOf(w0 >> 24, w1 & 0xffu, (w1 >> 8) & 0xffu, bs, nb);
      const unsigned i2 = BinOf((w1 >> 16) & 0xffu, w1 >> 24, w2 & 0xffu, bs, nb);
      const unsigned i3 = BinOf((w2 >> 8) & 0xffu, (w2 >> 16) & 0xffu, w2 >> 24, bs, nb);
      dst[g] = make_uint2(i0 | (i1 << 16), i2 | (i3 << 16));
    }
  }
}

// The rectangle is the bounding box of the closest template view's points projected with the current pose (a tight
// fit: for the triangle prism at 0.6 m ~200 x 200 instead of the ~240 x 240 pixels of the projected bounding sphere),
// grown by the reach of the correspondence lines / search windows and a motion margin. Whatever it misses is served from
// the pinned frame directly (FrameView), so this only decides how many bytes cross PCIe.
__device__ __forceinline__ bool ProjectedViewBox(const ModelDev& m, const CameraDev& cam, const float* b2c, float* s_red,
                                                 int* s_view, float (&box)[4]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (!m.cluster_info || m.n_views <= 0) return false;
  if (warp == 0) {
    float vo[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    vo[3] = ViewOrientation(b2c, vo[0], vo[1], vo[2]) ? 1.0f : 0.0f;
    const int v = ClosestViewPrunedWarp(m.cluster_info, m.sorted_views, m.n_clusters, m.orientations4, m.n_views, vo, 0);
    if (lane == 0) *s_view = v;
  }
  __syncthreads();
  const float4* pts = m.points + size_t(*s_view) * m.n_points * 2;
  float umin = 3.0e38f, umax = -3.0e38f, vmin = 3.0e38f, vmax = -3.0e38f, bad = 0.0f;
  for (int i = tid; i < m.n_points; i += blockDim.x) {
    const float4 p = __ldg(pts + 2 * i);
    float x, y, z;
    PoseApply(b2c, p.x, p.y, p.z, x, y, z);
    if (!(z > 0.0f)) { bad = 1.0f; continue; }
    const float u = x * cam.fu / z + cam.ppu, v = y * cam.fv / z + cam.ppv;
    umin = fminf(umin, u); umax = fmaxf(umax, u); vmin = fminf(vmin, v); vmax = fmaxf(vmax, v);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    umin = fminf(umin, __shfl_xor_sync(0xffffffffu, umin, off));
    umax = fmaxf(umax, __shfl_xor_sync(0xffffffffu, umax, off));
    vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, off));
    vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, off));
    bad = fmaxf(bad, __shfl_xor_sync(0xffffffffu, bad, off));
  }
  if (lane == 0) { s_red[5 * warp + 0] = umin; s_red[5 * warp + 1] = umax; s_red[5 * warp + 2] = vmin; s_red[5 * warp + 3] = vmax; s_red[5 * warp + 4] = bad; }
  __syncthreads();
  const int nw = blockDim.x >> 5;
  umin = s_red[0]; umax = s_red[1]; vmin = s_red[2]; vmax = s_red[3]; bad = s_red[4];
  for (int w = 1; w < nw; ++w) {
    umin = fminf(umin, s_red[5 * w + 0]); umax = fmaxf(umax, s_red[5 * w + 1]);
    vmin = fminf(vmin, s_red[5 * w + 2]); vmax = fmaxf(vmax, s_red[5 * w + 3]); bad = fmaxf(bad, s_red[5 * w + 4]);
  }
  __syncthreads();  // s_red / s_view are reused by the next call
  box[0] = umin; box[1] = umax; box[2] = vmin; box[3] = vmax;
  return bad == 0.0f && umax >= umin && vmax >= vmin;
}

__device__ __forceinline__ void BoxRect(const float (&box)[4], float reach_px, int width, int height, int align_x, Tile& t) {
  int x0 = int(floorf(box[0] - reach_px)), x1 = int(ceilf(box[1] + reach_px)) + 1;
  int y0 = int(floorf(box[2] - reach_px)), y1 = int(ceilf(box[3] + reach_px)) + 1;
  x0 = max(x0, 0) / align_x * align_x;
  x1 = min((min(x1, width) + align_x - 1) / align_x * align_x, width / align_x * align_x);
  y0 = max(y0, 0);
  y1 = min(y1, height);
  t.x0 = t.y0 = t.w = t.h = t.pitch = 0;
  if (x1 <= x0 || y1 <= y0) return;
  t.x0 = x0; t.y0 = y0; t.w = x1 - x0; t.h = y1 - y0; t.pitch = t.w;
}

__device__ __forceinline__ void IngestBody(const IngestArgs& args, int body_id, Tile (&rect)[2], int (&todo)[2], float* s_red,
                                           int& s_view) {
  const BodyDev& body = args.bodies[body_id];
  if (!body.set) return;  // block-uniform
  float pose[12];
  for (int i = 0; i < 12; ++i) pose[i] = args.poses[12 * body_id + i];
  const bool region_occ = body.has_region && body.rp.measure_occlusions;
  if (threadIdx.x == 0) {  // which cameras have a frame this body's ROI record does not cover yet (decided once, by one thread)
    for (int which = 0; which < 2; ++which) {
      const bool present = which == 0 ? body.has_region : (body.has_depth || region_occ);
      int need = 0;
      if (present) {
        const CameraDev& cam = which == 0 ? args.color_cams[body.color_camera] : args.depth_cams[body.depth_camera];
        need = cam.host_src && args.roi[2 * body_id + which].generation != cam.generation;
      }
      todo[which] = need;
    }
  }
  __syncthreads();
  for (int which = 0; which < 2; ++which) {  // block-uniform control flow
    if (!todo[which]) continue;
    const CameraDev& cam = which == 0 ? args.color_cams[body.color_camera] : args.depth_cams[body.depth_camera];
    RoiRecord& rec = args.roi[2 * body_id + which];
    float b2c[12];
    PoseMul(cam.w2c, pose, b2c);
    Tile t;
    float box[4];
    if (which == 0) {
      const ModelDev& m = args.region_models[body.region_model];
      int s_max = 1;
      for (int c = 0; c < body.rp.n_scales; ++c) s_max = max(s_max, body.rp.scales[c]);
      const float reach = fmaxf(0.5f * float(kLineSegments * s_max) + 2.0f, body.rp.max_considered_line_length + 2.0f) + kIngestMotionMarginPx;
      if (ProjectedViewBox(m, cam, b2c, s_red, &s_view, box)) BoxRect(box, reach, cam.width, cam.height, 16, t);
      else RoiRect(b2c, cam.fu, cam.fv, cam.ppu, cam.ppv, cam.width, cam.height, m.radius, reach, 16, t);
    } else {
      // depth search windows and, with measured occlusion handling, the occlusion windows around the region points
      const ModelDev& m = body.has_depth ? args.depth_models[body.depth_model] : args.region_models[body.region_model];
      float d_max = 0.0f;
      if (body.has_depth) {
        for (int c = 0; c < body.dp.n_considered_distances; ++c) d_max = fmaxf(d_max, body.dp.considered_distances[c]);
        if (body.dp.measure_occlusions) d_max = fmaxf(d_max, body.dp.measured_occlusion_radius);
      }
      float radius = m.radius;
      if (region_occ) {
        d_max = fmaxf(d_max, body.rp.measured_occlusion_radius);
        radius = fmaxf(radius, args.region_models[body.region_model].radius);
      }
      const float z = b2c[11];
      const float reach = (z > 2.0f * radius) ? d_max * cam.fu / (z - radius) + 2.0f + kIngestMotionMarginPx : 0.0f;
      // (with region occlusion handling the windows sit around the REGION points: keep the bounding sphere there)
      if (!region_occ && z > 2.0f * radius && ProjectedViewBox(m, cam, b2c, s_red, &s_view, box))
        BoxRect(box, reach, cam.width, cam.height, 8, t);
      else
        RoiRect(b2c, cam.fu, cam.fv, cam.ppu, cam.ppv, cam.width, cam.height, radius, reach, 8, t);
    }
    if (threadIdx.x == 0) {
      rect[which] = t;
      rec.x0 = t.x0; rec.y0 = t.y0; rec.x1 = t.x0 + t.w; rec.y1 = t.y0 + t.h;
      rec.generation = cam.generation;
    }
  }
  __syncthreads();
  if (todo[0]) {
    const CameraDev& cc = args.color_cams[body.color_camera];
    if (cc.bins && body.rp.n_bins <= 32) IngestColorRect(cc, rect[0], body.rp.bitshift, unsigned(body.rp.n_bins), args.bytes);
    else IngestRect(cc, rect[0], 3u, args.bytes);
  }
  if (todo[1]) IngestRect(args.depth_cams[body.depth_camera], rect[1], 2u, args.bytes);
}

__global__ void __launch_bounds__(kBlockThreads) k_ingest(IngestArgs args) {
  __shared__ Tile rect[2];
  __shared__ int todo[2];
  __shared__ float s_red[5 * (kBlockThreads / 32)];
  __shared__ int s_view;
  for (int i = blockIdx.x; i < args.n_bodies; i += gridDim.x) {
    IngestBody(args, args.body_list ? args.body_list[i] : i, rect, todo, s_red, s_view);
    __syncthreads();  // rect / todo belong to the next body now
  }
}

__device__ __forceinline__ float sgnf_dev(float v) { return v < 0.0f ? -1.0f : (v > 0.0f ? 1.0f : 0.0f); }

__global__ void __launch_bounds__(kBlockThreads) k_histogram(HistArgs args) {
  __shared__ Shared sh;
  __shared__ float s_sum[2][kWarps];
  const int body_id = args.body_list ? args.body_list[blockIdx.x] : int(blockIdx.x);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const BodyDev& body = args.bodies[body_id];
  if (!body.set || !body.has_region) return;
  const RegionParamsDev& rp = body.rp;
  const int nbins3 = rp.n_bins * rp.n_bins * rp.n_bins;
  float* mem_f = args.mem_f + size_t(body_id) * args.stride;
  float* mem_b = args.mem_b + size_t(body_id) * args.stride;
  float* hist_f = args.hist_f + size_t(body_id) * args.stride;
  float* hist_b = args.hist_b + size_t(body_id) * args.stride;
  float2* lut = args.lut + size_t(body_id) * args.stride;
  for (int k = tid; k < nbins3; k += kBlockThreads) { mem_f[k] = 0.0f; mem_b[k] = 0.0f; }  // ClearMemory
  const CameraDev& cam = args.color_cams[body.color_camera];
  if (tid < 12) sh.pose[tid] = args.poses[12 * body_id + tid];
  if (tid >= 32 && tid < 44) sh.cw2c[tid - 32] = cam.w2c[tid - 32];
  __syncthreads();
  const ModelDev& model = args.region_models[body.region_model];
  if (warp == 0) {
    float pose[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) pose[i] = sh.pose[i];
    PublishPoseProducts(pose, true, false, /*store_pose=*/false, sh);
  }
  __syncthreads();
  RegionIter it;
  MakeRegionIter(rp, cam, sh.rb2c, 0, it);
  int view, unused;
  ClosestViews<kBlockThreads>(&model, nullptr, sh, 0, view, unused);
  int n_lines = AdaptiveCount(rp.n_lines_max, rp.use_adaptive_coverage, rp.reference_contour_length,
                              __ldg(model.view_scalars + view), model.max_view_scalar, model.n_points);
  const float4* pts = model.points + size_t(view) * model.n_points * 2;
  const FrameView frame = MakeFrameView(cam, args.roi[2 * body_id + 0]);
  const int bs = rp.bitshift, nb = rp.n_bins;
  // handle_occlusions: StartModality (:382) n_unoccluded_iterations == 0, CalculateResults (:578-579)
  const bool handle_occlusions = args.mode == 0 ? rp.n_unoccluded_iterations == 0
                                                : (args.iteration - body.first_iteration) >= rp.n_unoccluded_iterations;
  const bool occ_on = handle_occlusions && rp.measure_occlusions && model.depth_offsets != nullptr;
  RegionOcclusion occ;
  FrameView dframe;
  Tile no_tile;
  float b2d[12];
  no_tile.x0 = no_tile.y0 = no_tile.w = no_tile.h = no_tile.pitch = 0; no_tile.offset = 0u;
  if (occ_on) {
    const CameraDev& dcam = args.depth_cams[body.depth_camera];
    PoseMul(dcam.w2c, sh.pose, b2d);
    dframe = MakeFrameView(dcam, args.roi[2 * body_id + 1]);
    occ.b2d = b2d;
    occ.offsets = model.depth_offsets + size_t(view) * model.n_points * kDepthOffsets;
    occ.offset_id = int(rp.measured_depth_offset_radius / model.stride_depth_offset + 0.5f);
    occ.fu = dcam.fu; occ.fv = dcam.fv; occ.ppu = dcam.ppu; occ.ppv = dcam.ppv; occ.depth_scale = dcam.depth_scale;
    occ.w_m1 = dcam.width - 1; occ.h_m1 = dcam.height - 1;
    occ.radius = rp.measured_occlusion_radius; occ.threshold = rp.measured_occlusion_threshold;
    occ.frame = &dframe; occ.tile = &no_tile; occ.tile_px = nullptr;
  }
  // renderer-image checks (:1031-1043): modeled occlusions with handle_occlusions, region checking always
  const RenderingDev& rdep = body.rend[RS_REGION_DEPTH];
  const RenderingDev& rsil = body.rend[RS_REGION_SILHOUETTE];
  const bool model_on = handle_occlusions && rp.model_occlusions && rdep.image && rdep.visible && model.depth_offsets != nullptr;
  const bool region_checking = rp.use_region_checking && rsil.image && rsil.visible;
  const int modeled_offset_id = int(rp.modeled_depth_offset_radius / model.stride_depth_offset + 0.5f);
  for (int i = tid; i < n_lines; i += kBlockThreads) {
    float4 p0 = __ldg(pts + 2 * i), p1 = __ldg(pts + 2 * i + 1);
    float x, y, z;
    PoseApply(it.b2c, p0.x, p0.y, p0.z, x, y, z);
    if (!(z > 0.0f)) continue;
    float center_u = x * it.fu / z + it.ppu;
    float center_v = y * it.fv / z + it.ppv;
    int icu = int(center_u + 0.5f), icv = int(center_v + 0.5f);
    if (icu < 0 || icu > it.w_m1 || icv < 0 || icv > it.h_m1) continue;
    if (model_on) {  // :1079-1084
      const float meter_to_pixel = (it.fu / z) * rdep.scale;
      const float diameter = 2.0f * rp.modeled_occlusion_radius * meter_to_pixel;
      const float depth_offset = __ldg(model.depth_offsets + (size_t(view) * model.n_points + i) * kDepthOffsets + modeled_offset_id);
      if (!ModeledWindowUnoccluded(rdep, center_u, center_v, diameter, z - depth_offset - rp.modeled_occlusion_threshold)) continue;
    }
    if (occ_on && !LineUnoccludedMeasured(occ, p0.x, p0.y, p0.z, i)) continue;  // :1086-1089
    float length_f = rp.max_considered_line_length, length_b = rp.max_considered_line_length;
    if (region_checking) {  // :1092-1099
      float rnu = it.b2c[0] * p0.w + it.b2c[1] * p1.x + it.b2c[2] * p1.y;
      float rnv = it.b2c[4] * p0.w + it.b2c[5] * p1.x + it.b2c[6] * p1.y;
      const float zz = rnu * rnu + rnv * rnv;
      if (zz > 0.0f) { const float n = sqrtf(zz); rnu /= n; rnv /= n; }
      DynamicRegionDistance(rsil, rp.max_considered_line_length, rp.unconsidered_line_length, center_u, center_v, rnu, rnv,
                            length_f, length_b);
    }
    float l_f = p1.z * it.fu / z;
    float l_b = p1.w * it.fu / z;
    length_f = fminf(length_f, l_f - 2.0f * rp.unconsidered_line_length);
    length_b = fminf(length_b, l_b - 2.0f * rp.unconsidered_line_length);
    float nu = it.b2c[0] * p0.w + it.b2c[1] * p1.x + it.b2c[2] * p1.y;
    float nv = it.b2c[4] * p0.w + it.b2c[5] * p1.x + it.b2c[6] * p1.y;
    {
      float zz = nu * nu + nv * nv;
      if (zz > 0.0f) { float n = sqrtf(zz); nu /= n; nv /= n; }
    }
    float u_step, v_step;
    int plf, plb;
    float anu = fabsf(nu), anv = fabsf(nv);
    if (anu > anv) {
      u_step = sgnf_dev(nu);
      v_step = nv / anu;
      plf = int(length_f * anu + 0.5f);
      plb = int(length_b * anu + 0.5f);
    } else {
      u_step = nu / anv;
      v_step = sgnf_dev(nv);
      plf = int(length_f * anv + 0.5f);
      plb = int(length_b * anv + 0.5f);
    }
    float u = center_u - nu * rp.unconsidered_line_length + 0.5f;
    float v = center_v - nv * rp.unconsidered_line_length + 0.5f;
    for (int k = 0; k < plf; ++k) {
      int iu = int(u), iv = int(v);
      if (iu < 0 || iu > it.w_m1 || iv < 0 || iv > it.h_m1) break;
      const uint8_t* px = FramePtr(frame, iu, iv, 3u);
      int idx = (int(__ldg(px)) >> bs) * nb * nb + (int(__ldg(px + 1)) >> bs) * nb + (int(__ldg(px + 2)) >> bs);
      atomicAdd(mem_f + idx, 1.0f);
      u -= u_step;
      v -= v_step;
    }
    u = center_u + nu * rp.unconsidered_line_length + 0.5f;
    v = center_v + nv * rp.unconsidered_line_length + 0.5f;
    for (int k = 0; k < plb; ++k) {
      int iu = int(u), iv = int(v);
      if (iu < 0 || iu > it.w_m1 || iv < 0 || iv > it.h_m1) break;
      const uint8_t* px = FramePtr(frame, iu, iv, 3u);
      int idx = (int(__ldg(px)) >> bs) * nb * nb + (int(__ldg(px + 1)) >> bs) * nb + (int(__ldg(px + 2)) >> bs);
      atomicAdd(mem_b + idx, 1.0f);
      u += u_step;
      v += v_step;
    }
  }
  __threadfence();
  __syncthreads();
  if (args.shared_owner && args.shared_owner[body_id] >= 0) return;  // shared ColorHistograms: k_histogram_shared finishes
  // CalculateHistogram (color_histograms.cpp:174-214)
  float sf = 0.0f, sb = 0.0f;
  for (int k = tid; k < nbins3; k += kBlockThreads) { sf += mem_f[k]; sb += mem_b[k]; }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    sf += __shfl_down_sync(0xffffffffu, sf, off);
    sb += __shfl_down_sync(0xffffffffu, sb, off);
  }
  if (lane == 0) { s_sum[0][warp] = sf; s_sum[1][warp] = sb; }
  __syncthreads();
  float sum_f = 0.0f, sum_b = 0.0f;
  for (int w = 0; w < kWarps; ++w) { sum_f += s_sum[0][w]; sum_b += s_sum[1][w]; }
  const float lr_f = args.mode == 0 ? 1.0f : rp.learning_rate_f;
  const float lr_b = args.mode == 0 ? 1.0f : rp.learning_rate_b;
  const float uniform = 1.0f / float(nbins3);
  const float cf = 1.0f - lr_f, cb = 1.0f - lr_b;
  const float rf = lr_f / sum_f, rb = lr_b / sum_b;
  for (int k = tid; k < nbins3; k += kBlockThreads) {
    float hf = hist_f[k], hb = hist_b[k];
    if (sum_f == 0.0f) {
      if (lr_f == 1.0f) hf = uniform;
    } else if (cf == 0.0f) {
      hf = mem_f[k] * rf;
    } else {
      hf *= cf;
      hf += mem_f[k] * rf;
    }
    if (sum_b == 0.0f) {
      if (lr_b == 1.0f) hb = uniform;
    } else if (cb == 0.0f) {
      hb = mem_b[k] * rb;
    } else {
      hb *= cb;
      hb += mem_b[k] * rb;
    }
    hist_f[k] = hf;
    hist_b[k] = hb;
    lut[LutSlot(unsigned(k))] = NormaliseBin(hf, hb);
  }
}

// One CTA per shared ColorHistograms object. The members' counts are whole numbers, so their sum (and the sum over the
// bins) is exact in any order as long as it stays below 2^24 - the same value the reference gets by adding pixel after
// pixel into one array. Then CalculateHistogram with the OWNER's learning rates, and the result goes to every member's
// copy of the histograms and of the lookup table (the tracking kernels keep reading per-body tables).
__global__ void __launch_bounds__(kBlockThreads) k_histogram_shared(SharedHistArgs args) {
  __shared__ float s_sum[2][kWarps];
  const int g = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int owner = args.group_owner[g];
  const int first = args.group_first[g], last = args.group_first[g + 1];
  const int summed = args.group_summed ? first + args.group_summed[g] : last;
  const RegionParamsDev& rp = args.bodies[owner].rp;
  const int nbins3 = rp.n_bins * rp.n_bins * rp.n_bins;
  float* mem_f = args.mem_f + size_t(owner) * args.stride;
  float* mem_b = args.mem_b + size_t(owner) * args.stride;
  float* hist_f = args.hist_f + size_t(owner) * args.stride;
  float* hist_b = args.hist_b + size_t(owner) * args.stride;
  float sf = 0.0f, sb = 0.0f;
  for (int k = tid; k < nbins3; k += kBlockThreads) {
    float mf = 0.0f, mb = 0.0f;
    for (int q = first; q < summed; ++q) {
      const size_t off = size_t(args.members[q]) * args.stride + k;
      mf += args.mem_f[off];
      mb += args.mem_b[off];
    }
    mem_f[k] = mf;  // the owner's own counts, if summed, were read above, by this thread
    mem_b[k] = mb;
    sf += mf;
    sb += mb;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    sf += __shfl_down_sync(0xffffffffu, sf, off);
    sb += __shfl_down_sync(0xffffffffu, sb, off);
  }
  if (lane == 0) { s_sum[0][warp] = sf; s_sum[1][warp] = sb; }
  __syncthreads();
  float sum_f = 0.0f, sum_b = 0.0f;
  for (int w = 0; w < kWarps; ++w) { sum_f += s_sum[0][w]; sum_b += s_sum[1][w]; }
  const float lr_f = args.mode == 0 ? 1.0f : rp.learning_rate_f;
  const float lr_b = args.mode == 0 ? 1.0f : rp.learning_rate_b;
  const float uniform = 1.0f / float(nbins3);
  const float cf = 1.0f - lr_f, cb = 1.0f - lr_b;
  const float rf = lr_f / sum_f, rb = lr_b / sum_b;
  for (int k = tid; k < nbins3; k += kBlockThreads) {  // each thread revisits the bins it summed
    float hf = hist_f[k], hb = hist_b[k];
    if (sum_f == 0.0f) {
      if (lr_f == 1.0f) hf = uniform;
    } else if (cf == 0.0f) {
      hf = mem_f[k] * rf;
    } else {
      hf *= cf;
      hf += mem_f[k] * rf;
    }
    if (sum_b == 0.0f) {
      if (lr_b == 1.0f) hb = uniform;
    } else if (cb == 0.0f) {
      hb = mem_b[k] * rb;
    } else {
      hb *= cb;
      hb += mem_b[k] * rb;
    }
    const float2 l = NormaliseBin(hf, hb);
    for (int q = first; q < last; ++q) {
      const size_t base = size_t(args.members[q]) * args.stride;
      args.hist_f[base + k] = hf;
      args.hist_b[base + k] = hb;
      args.lut[base + LutSlot(unsigned(k))] = l;
    }
  }
}

#endif  // M3TB_TRACK_TU

}  // namespace m3tb
