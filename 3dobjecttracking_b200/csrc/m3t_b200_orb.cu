// m3t_b200_orb.cu — k_texture_orb: cv::ORB (OpenCV 4) detect, then compute, on each body's focused crop, at M3T's
// settings (texture_modality.cpp:858-888; only n_features, scale_factor and n_levels vary). One CTA per body walks
// the levels in turn; every image and candidate list lives in the body's slice of the context's scratch (global
// memory, so crops of any size fit). tests/texture_orb_reference.py restates each stage and DESIGN.md §3
// "k_texture_orb" lists the arithmetic; the build's -fmad=false keeps every float expression unfused, and the blur's
// fused multiply-adds are written as fmaf.
#include "m3t_b200_texture.cuh"
#include "m3t_b200_orb_pattern.h"

namespace m3tb {

namespace {

constexpr int kOrbWarps = kOrbThreads / 32;
constexpr int kEdge = 31;         // edgeThreshold
constexpr int kHalfPatch = 15;    // patchSize / 2
constexpr int kFastThreshold = 20;

// fast.cpp's offsets16: the radius-3 circle as (dx, dy)
__constant__ signed char kFastDx[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
__constant__ signed char kFastDy[16] = {3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1, 0, 1, 2, 3};
// ICAngles' u_max for the radius-15 patch (orb.cpp, made symmetric)
__constant__ signed char kUmax[16] = {15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3};
// getGaussianKernel(7, 2, CV_32F)
__constant__ float kGauss[7] = {0.0701593235f, 0.131074876f, 0.190712824f, 0.216105938f,
                                0.190712824f, 0.131074876f, 0.0701593235f};
__constant__ signed char kPattern[M3TB_ORB_PATTERN_VALUES] = M3TB_ORB_BIT_PATTERN_31;

// resize_bitExact's interpolationLinear for output position d of n_dst from n_src: the source offset and weight c1 in
// 1/256; pin -1 before the first source pixel, +1 at the last (both take that pixel whole)
__device__ __forceinline__ void ExactTap(int d, int n_src, int n_dst, int& offset, int& c1, int& pin) {
  const double scale = 1.0 / (double(n_dst) / double(n_src));
  const double f = scale * (double(d) + 0.5) - 0.5;
  const double i = floor(f);
  offset = 0; c1 = 0; pin = -1;
  if (i >= 0.0 && n_src > 1) {
    if (i < double(n_src - 1)) {
      offset = int(i);
      c1 = int(rint((f - i) * 256.0));
      pin = 0;
    } else {
      offset = n_src - 1;
      pin = 1;
    }
  }
}

// one source row resized horizontally at output column x, in 1/256
__device__ __forceinline__ int ExactRow(const uint8_t* row, int ox, int c1, int pin) {
  if (pin < 0) return int(row[0]) * 256;
  if (pin > 0) return int(row[ox]) * 256;
  return int(row[ox]) * (256 - c1) + int(row[ox + 1]) * c1;
}

// cv::resize(src, dst, Size(dw, dh), 0, 0, INTER_LINEAR_EXACT), both `pitch` bytes per row
__device__ void ResizeExact(const uint8_t* src, int sw, int sh, uint8_t* dst, int dw, int dh, int pitch) {
  for (int p = threadIdx.x; p < dw * dh; p += kOrbThreads) {
    const int y = p / dw, x = p - y * dw;
    int ox, cx, px, oy, cy, py;
    ExactTap(x, sw, dw, ox, cx, px);
    ExactTap(y, sh, dh, oy, cy, py);
    int v;
    if (py < 0) v = (ExactRow(src, ox, cx, px) + 128) >> 8;
    else if (py > 0) v = (ExactRow(src + size_t(sh - 1) * pitch, ox, cx, px) + 128) >> 8;
    else v = (ExactRow(src + size_t(oy) * pitch, ox, cx, px) * (256 - cy) +
              ExactRow(src + size_t(oy + 1) * pitch, ox, cx, px) * cy + 32768) >> 16;
    dst[size_t(y) * pitch + x] = uint8_t(min(max(v, 0), 255));
  }
}

// cornerScore<16> where FAST-9 finds a corner (an arc of 9 all darker or all brighter than the centre by more than
// the threshold), 0 elsewhere
__device__ __forceinline__ int FastScore(const uint8_t* img, int pitch, int x, int y) {
  const uint8_t* c = img + size_t(y) * pitch + x;
  const int v = c[0];
  // darker (v - p) and brighter (p - v) margins of the 16 circle pixels, each arc of 9 a plain minimum of one of
  // them: cornerScore's max(min over the arc, -(max over the arc)) without a negation
  int dark[16], bright[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int p = c[kFastDy[k] * pitch + kFastDx[k]];
    dark[k] = v - p;
    bright[k] = p - v;
  }
  int best = 0;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    int a = dark[k], b = bright[k];
#pragma unroll
    for (int j = 1; j < 9; ++j) {
      a = min(a, dark[(k + j) & 15]);
      b = min(b, bright[(k + j) & 15]);
    }
    best = max(best, max(a, b));
  }
  return best > kFastThreshold ? best - 1 : 0;
}

// order-preserving key of a float (-0 and +0 equal, as the cuts compare them)
__device__ __forceinline__ uint32_t FloatKey(float f) {
  const uint32_t u = f == 0.0f ? 0u : __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// The k-th largest of keys[0 .. n) (1 <= k <= n), by radix select over bits [0, bits) in 8-bit digits from the top.
__device__ uint32_t KthLargest(const uint32_t* keys, int n, int k, int bits, int* hist, int* shared) {
  uint32_t prefix = 0, mask = 0;
  for (int shift = bits - 8; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += kOrbThreads) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kOrbThreads) {
      const uint32_t key = keys[i];
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int above = 0, bin = 255;
      for (; bin > 0 && above + hist[bin] < k; --bin) above += hist[bin];
      shared[0] = bin;
      shared[1] = k - above;
    }
    __syncthreads();
    prefix |= uint32_t(shared[0]) << shift;
    mask |= 255u << shift;
    k = shared[1];
    __syncthreads();
  }
  return prefix;
}

// Stable block-wide compaction: thread t of the current chunk keeps its element when `keep`; returns its slot in the
// output (or -1) and adds the chunk's count to *total (shared) after a barrier. All threads must call it.
__device__ __forceinline__ int CompactSlot(bool keep, int* warp_counts, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ballot = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) warp_counts[warp] = __popc(ballot);
  __syncthreads();
  int before = *total;
  for (int w = 0; w < warp; ++w) before += warp_counts[w];
  const int slot = keep ? before + __popc(ballot & ((1u << lane) - 1u)) : -1;
  __syncthreads();
  if (threadIdx.x == 0) {
    int sum = 0;
    for (int w = 0; w < kOrbWarps; ++w) sum += warp_counts[w];
    *total += sum;
  }
  __syncthreads();
  return slot;
}

// Keeps the elements of pos / keys / resp (resp may be null) whose key is at least `cut`, in order; returns the count
__device__ int KeepAtLeast(uint32_t* pos, uint32_t* keys, float* resp, int n, uint32_t cut, int* warp_counts,
                           int* total) {
  if (threadIdx.x == 0) *total = 0;
  __syncthreads();
  for (int base = 0; base < n; base += kOrbThreads) {
    const int i = base + threadIdx.x;
    const bool in = i < n;
    const uint32_t p = in ? pos[i] : 0u, key = in ? keys[i] : 0u;
    const float r = in && resp ? resp[i] : 0.0f;
    const int slot = CompactSlot(in && key >= cut, warp_counts, total);  // barriers: every read precedes every write
    if (slot >= 0) {
      pos[slot] = p;
      keys[slot] = key;
      if (resp) resp[slot] = r;
    }
  }
  __syncthreads();
  return *total;
}

// HarrisResponses (block 7, k 0.04): integer Sobel sums, then the float formula in OpenCV's order
__device__ __forceinline__ float Harris(const uint8_t* img, int pitch, int x0, int y0) {
  int a = 0, b = 0, c = 0;
  for (int by = -3; by <= 3; ++by)
    for (int bx = -3; bx <= 3; ++bx) {
      const uint8_t* p = img + size_t(y0 + by) * pitch + (x0 + bx);
      const int ix = (int(p[1]) - int(p[-1])) * 2 + (int(p[-pitch + 1]) - int(p[-pitch - 1])) +
                     (int(p[pitch + 1]) - int(p[pitch - 1]));
      const int iy = (int(p[pitch]) - int(p[-pitch])) * 2 + (int(p[pitch - 1]) - int(p[-pitch - 1])) +
                     (int(p[pitch + 1]) - int(p[-pitch + 1]));
      a += ix * ix;
      b += iy * iy;
      c += ix * iy;
    }
  const float scale = 1.0f / (float(4 * 7) * 255.0f);
  const float sss = scale * scale * scale * scale;
  const float fa = float(a), fb = float(b), fc = float(c);
  return (fa * fb - fc * fc - 0.04f * (fa + fb) * (fa + fb)) * sss;
}

// cv::fastAtan2, degrees
__device__ __forceinline__ float FastAtan2(float y, float x) {
  const float deg = float(180.0 / 3.141592653589793);
  const float p1 = 0.9997878412794807f * deg, p3 = -0.3258083974640975f * deg;
  const float p5 = 0.1555786518463281f * deg, p7 = -0.04432655554792128f * deg;
  const float eps = float(2.220446049250313e-16);
  const float ax = fabsf(x), ay = fabsf(y);
  float a;
  if (ax >= ay) {
    const float c = ay / (ax + eps), c2 = c * c;
    a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  } else {
    const float c = ax / (ay + eps), c2 = c * c;
    a = 90.0f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
  }
  if (x < 0.0f) a = 180.0f - a;
  if (y < 0.0f) a = 360.0f - a;
  return a;
}

// GaussianBlur(7 x 7, sigma 2) at (x, y), 3 <= x < w - 3, 3 <= y < h - 3: OpenCV's separable float path as ORB's
// in-place blur of a pyramid view takes it (rows sequential, columns symmetric about the centre, both fused)
__device__ __forceinline__ uint8_t Blur(const uint8_t* img, int pitch, int x, int y) {
  float rows[7];
#pragma unroll
  for (int r = 0; r < 7; ++r) {
    const uint8_t* p = img + size_t(y + r - 3) * pitch + (x - 3);
    float s = float(p[0]) * kGauss[0];
#pragma unroll
    for (int t = 1; t < 7; ++t) s = fmaf(float(p[t]), kGauss[t], s);
    rows[r] = s;
  }
  float s = kGauss[3] * rows[3];
#pragma unroll
  for (int t = 1; t <= 3; ++t) s = fmaf(rows[3 + t] + rows[3 - t], kGauss[3 + t], s);
  return uint8_t(min(max(__float2int_rn(s), 0), 255));
}

}  // namespace

__global__ void __launch_bounds__(kOrbThreads) k_texture_orb(const __grid_constant__ TexOrbArgs a) {
  const TexOrbJob& j = a.jobs[blockIdx.x];
  __shared__ int hist[256];
  __shared__ int warp_counts[kOrbWarps];
  __shared__ int sh[4];  // [0] compaction total, [2..3] KthLargest
  const int tid = threadIdx.x, b = j.body, pitch = a.pitch;
  const size_t area = size_t(pitch) * size_t(a.height);
  uint8_t* base = a.scratch + a.job_bytes * blockIdx.x;
  // levels alternate between base and base + area; level 0 is the crop k_texture_crop wrote at base
  uint8_t* blur = base + 2 * area;
  uint8_t* score = base + 3 * area;
  uint32_t* pos = reinterpret_cast<uint32_t*>(base + 4 * area);
  uint32_t* keys = pos + area;
  float* resp = reinterpret_cast<float*>(keys + area);
  const size_t cap = size_t(a.cap);
  float2* out_xy = a.feat_xy + size_t(b) * cap;
  uint32_t* out_desc = a.feat_desc + size_t(b) * cap * kTexDescWords;
  const size_t orb_cap = size_t(a.orb_cap);
  float2* orb_xy = a.orb_xy + size_t(b) * orb_cap;
  float* orb_angle = a.orb_angle + size_t(b) * orb_cap;
  float* orb_resp = a.orb_response + size_t(b) * orb_cap;
  int* orb_octave = a.orb_octave + size_t(b) * orb_cap;
  uint32_t* orb_desc = a.orb_desc + size_t(b) * orb_cap * kTexDescWords;

  int total = 0;
  // w[0] = 0: no focus, or a pyramid with a level of size 0 (cv::ORB detects nothing then); otherwise every level
  // has at least one pixel
  for (int level = 0; level < j.n_levels && j.w[0] > 0; ++level) {
    const int w = j.w[level], h = j.h[level];
    uint8_t* im = base + (level & 1) * area;
    if (level > 0) ResizeExact(base + ((level - 1) & 1) * area, j.w[level - 1], j.h[level - 1], im, w, h, pitch);
    __syncthreads();
    if (h <= 2 * kEdge || w <= 2 * kEdge) continue;  // runByImageBorder(31) empties the level
    // FAST-9/16 scores over the rows and columns fast.cpp tests; 0 elsewhere (non-max suppression reads them)
    for (int p = tid; p < w * h; p += kOrbThreads) {
      const int y = p / w, x = p - y * w;
      score[size_t(y) * pitch + x] = uint8_t(x >= 3 && x < w - 3 && y >= 3 && y < h - 3 ? FastScore(im, pitch, x, y) : 0);
    }
    __syncthreads();
    // corners that beat their 8 neighbours, inside the 31-pixel border, in row-major order
    const int iw = w - 2 * kEdge, ih = h - 2 * kEdge;
    if (tid == 0) sh[0] = 0;
    __syncthreads();
    for (int p0 = 0; p0 < iw * ih; p0 += kOrbThreads) {
      const int p = p0 + tid;
      bool keep = false;
      uint32_t s = 0;
      int x = 0, y = 0;
      if (p < iw * ih) {
        y = kEdge + p / iw;
        x = kEdge + p % iw;
        const uint8_t* c = score + size_t(y) * pitch + x;
        s = c[0];
        keep = s > 0 && s > c[-1] && s > c[1] && s > c[-pitch - 1] && s > c[-pitch] && s > c[-pitch + 1] &&
               s > c[pitch - 1] && s > c[pitch] && s > c[pitch + 1];
      }
      const int slot = CompactSlot(keep, warp_counts, &sh[0]);
      if (slot >= 0) {
        pos[slot] = (uint32_t(y) << 16) | uint32_t(x);
        keys[slot] = s;
      }
    }
    __syncthreads();
    int n = sh[0];
    // retainBest(2 n_level) by FAST score, then Harris, then retainBest(n_level) by Harris, keeping ties at both cuts
    const int want = j.per_level[level];
    if (n > 2 * want) n = want == 0 ? 0 : KeepAtLeast(pos, keys, nullptr, n, KthLargest(keys, n, 2 * want, 8, hist, &sh[2]), warp_counts, &sh[0]);
    for (int i = tid; i < n; i += kOrbThreads) {
      const int x = int(pos[i] & 0xffffu), y = int(pos[i] >> 16);
      const float r = Harris(im, pitch, x, y);
      resp[i] = r;
      keys[i] = FloatKey(r);
    }
    __syncthreads();
    if (n > want) n = want == 0 ? 0 : KeepAtLeast(pos, keys, resp, n, KthLargest(keys, n, want, 32, hist, &sh[2]), warp_counts, &sh[0]);
    if (n == 0) continue;
    // the blurred level (only interior pixels: descriptors read at least 12 pixels inside)
    for (int p = tid; p < w * h; p += kOrbThreads) {
      const int y = p / w, x = p - y * w;
      if (x >= 3 && x < w - 3 && y >= 3 && y < h - 3) blur[size_t(y) * pitch + x] = Blur(im, pitch, x, y);
    }
    __syncthreads();
    // one warp per keypoint: intensity-centroid angle, then one descriptor byte per lane
    const float layer_scale = j.layer_scale[level];
    for (int i = tid >> 5; i < n; i += kOrbWarps) {
      const int lane = tid & 31;
      const int x = int(pos[i] & 0xffffu), y = int(pos[i] >> 16);
      int m01 = 0, m10 = 0;
      if (lane <= 2 * kHalfPatch) {
        const int u = lane - kHalfPatch;
        for (int v = -kHalfPatch; v <= kHalfPatch; ++v)
          if (abs(u) <= kUmax[abs(v)]) {
            const int val = im[size_t(y + v) * pitch + (x + u)];
            m10 += u * val;
            m01 += v * val;
          }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        m01 += __shfl_xor_sync(0xffffffffu, m01, o);
        m10 += __shfl_xor_sync(0xffffffffu, m10, o);
      }
      const float angle = FastAtan2(float(m01), float(m10));
      const float rad = angle * float(3.141592653589793 / 180.0);
      // OpenCV takes (float)cos / sin of double(rad). sincospi(double(rad) / pi) is a documented approximation of
      // that: the quotient rounds and pi is rounded, so the argument differs by about an ulp of a double, which the
      // cast to float hides but for a vanishing share of angles (CUDA's double cos / sin are not correctly rounded
      // either). It keeps the kernel free of sincos's slow-path reduction buffer, which lives in local memory.
      double sd, cd;
      sincospi(double(rad) / 3.141592653589793, &sd, &cd);
      const float ca = float(cd), sa = float(sd);
      uint32_t byte = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        int t[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int q = 2 * (16 * lane + 2 * k + e);
          const float px = float(kPattern[q]), py = float(kPattern[q + 1]);
          const int ix = __float2int_rn(px * ca - py * sa), iy = __float2int_rn(px * sa + py * ca);
          t[e] = blur[size_t(y + iy) * pitch + (x + ix)];
        }
        byte |= uint32_t(t[0] < t[1]) << k;
      }
      const int o = total + i;
      if (o < j.n_features_max) {
        // the crop-coordinate keypoint (KeyPoint::pt *= layer scale), the image one as the upload converts it
        const float cx = float(x) * layer_scale, cy = float(y) * layer_scale;
        reinterpret_cast<uint8_t*>(out_desc + size_t(o) * kTexDescWords)[lane] = uint8_t(byte);
        reinterpret_cast<uint8_t*>(orb_desc + size_t(o) * kTexDescWords)[lane] = uint8_t(byte);
        if (lane == 0) {
          out_xy[o] = make_float2(float(j.roi_x) + cx / j.scale, float(j.roi_y) + cy / j.scale);
          orb_xy[o] = make_float2(cx, cy);
          orb_angle[o] = angle;
          orb_resp[o] = resp[i];
          orb_octave[o] = level;
        }
      }
    }
    total += n;
    __syncthreads();
  }
  if (tid == 0) {
    a.found[b] = total;
    a.feat_n[b] = total <= j.n_features_max ? total : 0;
  }
}

}  // namespace m3tb
