// m3t_b200_model.cu — sparse-viewpoint-model generation. k_model_raster draws the geodesic views of a batch into
// global-memory z-buffers, one per renderer of the table. Depth models: k_model_points samples and describes the
// surface points of each view, k_model_images reads one view back as the reference's normal / depth / silhouette
// images. Region models: k_region_contours traces the contours of the main silhouette, k_region_points samples and
// describes the contour points, k_region_images reads one view's silhouettes back. Float32, one rounding per operation
// in the order written (-fmad=false); DESIGN.md §3 "k_model_raster / k_model_points" and "k_region_contours /
// k_region_points" state the contract, tests/model_generation_reference.py and
// tests/region_model_generation_reference.py restate it.
#include "m3t_b200_model.cuh"
#include "m3t_b200_raster.cuh"

#include <cfloat>
#include <climits>

namespace m3tb {

namespace {

constexpr int kMtN = 624, kMtM = 397;

// std::mt19937 (Matsumoto & Nishimura 1998): seeding and one tempered output
__device__ void MtSeed(uint32_t* mt, uint32_t seed) {
  mt[0] = seed;
  for (int i = 1; i < kMtN; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + uint32_t(i);
}

__device__ uint32_t MtNext(uint32_t* mt, int& index) {
  if (index >= kMtN) {
    for (int i = 0; i < kMtN; ++i) {
      const uint32_t y = (mt[i] & 0x80000000u) | (mt[i + 1 < kMtN ? i + 1 : 0] & 0x7fffffffu);
      const int k = i + kMtM < kMtN ? i + kMtM : i + kMtM - kMtN;
      mt[i] = mt[k] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    index = 0;
  }
  uint32_t y = mt[index++];
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

// occlusion silhouette (depth_model.cpp:171-178): the body is kMainBodyID (255), occlusion bodies kBackgroundID (0).
// Without occlusion bodies the silhouette renderer draws what the main renderer draws, so its coverage is used.
__device__ __forceinline__ bool Silhouette(uint64_t key, int n_renderers) {
  if (key == kModelClear) return false;
  return n_renderers == 1 || ((key >> 32) & 0xffffu) == 0u;
}

// the normal image at one pixel (normal_renderer.cpp:11-31): EncodeNormal of the winning triangle; background 0
__device__ __forceinline__ void NormalBytes(const ModelPointArgs& a, int view, uint64_t key, unsigned b[4]) {
  if (key == kModelClear) {
    b[0] = b[1] = b[2] = b[3] = 0u;
    return;
  }
  EncodeNormal(a.rot + 9 * size_t(view), a.face_normals + 3 * size_t(key & 0xffffffffu), b);
}

// Model::CalculateDepthOffsets (model.cpp:338-384) around pixel (x, y) of a main depth image held as z-buffer z0 [S][S],
// shared by both generators. One warp; s_min holds the warp's kModelMaxOffsets slots. The distance is the double
// std::sqrt of the integer squared distance, stored as a float. Lane 0 writes the 30 offsets to o.
__device__ void DepthOffsets(const uint64_t* z0, int S, int x, int y, unsigned d16c, float depth, float pixel_to_meter,
                             float stride_depth_offset, int n_values, float projection_term_a, float projection_term_b,
                             unsigned* s_min, float* o, int lane) {
  const float stride = stride_depth_offset / pixel_to_meter;
  const float max_diameter = 2.0f * float(n_values) * stride;
  const int image_stride = int(stride + 1.0f);
  const int n_image_strides = int(max_diameter / float(image_stride) + 1.0f);
  const int image_diameter = n_image_strides * image_stride;
  const int radius_minus = image_diameter / 2;
  const int radius_plus = image_diameter - radius_minus;
  const int v_min = max(y - radius_minus, 0), v_max = min(y + radius_plus, S - 1);
  const int u_min = max(x - radius_minus, 0), u_max = min(x + radius_plus, S - 1);
  if (lane < kModelMaxOffsets) s_min[lane] = lane == 0 ? d16c : 0xffffu;
  __syncwarp();
  const int nu = u_max >= u_min ? (u_max - u_min) / image_stride + 1 : 0;
  const int nv = v_max >= v_min ? (v_max - v_min) / image_stride + 1 : 0;
  for (int k = lane; k < nu * nv; k += 32) {
    const int u = u_min + (k % nu) * image_stride, v = v_min + (k / nu) * image_stride;
    const int du = u - x, dv = v - y;
    const float distance = float(sqrt(double(du * du + dv * dv)));  // std::sqrt(int) is a double
    const int i = int(distance / stride);
    if (i < n_values) atomicMin(&s_min[i], unsigned(z0[size_t(v) * S + u] >> 48));
  }
  __syncwarp();
  if (lane == 0) {
    unsigned m = s_min[0];
    o[0] = depth - projection_term_a / (projection_term_b - float(m));
    for (int i = 1; i < kModelMaxOffsets; ++i) {
      m = min(s_min[i], m);
      o[i] = depth - projection_term_a / (projection_term_b - float(m));
    }
  }
  __syncwarp();  // s_min is reset for the next point
}

}  // namespace

__global__ void __launch_bounds__(kModelThreads) k_model_raster(const __grid_constant__ ModelRasterArgs a) {
  const int view = blockIdx.y, r = blockIdx.z;
  const int S = a.image_size;
  const size_t n_pix = size_t(S) * S;
  unsigned long long* zb = reinterpret_cast<unsigned long long*>(a.zbuf + (size_t(view) * a.R.n_renderers + r) * n_pix);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const float half = 0.5f * float(S);
  const int d0 = a.R.first[r], d1 = a.R.first[r + 1];
  for (int d = d0; d < d1; ++d) {
    const ModelBodyDev B = a.R.draws[d];
    const float* Mg = a.M + (size_t(view) * a.n_draws + d) * 16;
    float M[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) M[k] = Mg[k];
    for (int t0 = blockIdx.x * kModelTrianglesPerCta; t0 < B.n_triangles; t0 += gridDim.x * kModelTrianglesPerCta) {
      const int t_end = min(t0 + kModelTrianglesPerCta, B.n_triangles);
      for (int t = t0 + warp; t < t_end; t += n_warps) {
        const unsigned long long tag = ModelKey(0u, unsigned(d - d0), unsigned(t));
        auto frag = [&](int i, int j, unsigned d16) {
          atomicMin(zb + size_t(j) * S + i, (static_cast<unsigned long long>(d16) << 48) | tag);
        };
        DrawTriangle(M, B.triangles + 9 * size_t(t), B.enable_culling, S, S, half, half, frag, lane);
      }
    }
  }
}

__global__ void __launch_bounds__(kModelThreads) k_model_points(const __grid_constant__ ModelPointArgs a) {
  __shared__ uint32_t mt[kMtN];
  __shared__ uint32_t cand[32];
  __shared__ unsigned s_count;
  __shared__ unsigned s_min[kModelThreads / 32][kModelMaxOffsets];
  const int view = blockIdx.x;
  const int S = a.image_size;
  const int n_pix = S * S;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
  const uint64_t* z0 = a.zbuf + size_t(view) * a.n_renderers * n_pix;  // main renderer
  const uint64_t* zs = a.n_renderers == 2 ? z0 + n_pix : z0;              // silhouette renderer
  float* out = a.points + size_t(view) * a.n_points * 36;

  // surface area: countNonZero(silhouette) * square(sphere_radius / fu)
  if (tid == 0) s_count = 0;
  __syncthreads();
  unsigned c = 0;
  for (int p = tid; p < n_pix; p += blockDim.x) c += Silhouette(zs[p], a.n_renderers) ? 1u : 0u;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) atomicAdd(&s_count, c);
  __syncthreads();
  const float px = a.sphere_radius / a.fu;
  const float area = float(s_count) * (px * px);
  if (tid == 0) a.surface_area[view] = area;
  if (area == 0.0f) {  // the reference leaves the points of such a view uninitialised
    for (int k = tid; k < a.n_points * 36; k += blockDim.x) out[k] = 0.0f;
    return;
  }

  // SampleSurfacePointCoordinate: a fresh std::mt19937 per view; lane 0 draws 32 values at a time and the warp tests
  // them, keeping the accepted ones in stream order, so the result is that of the reference's serial loop
  int* coords = a.coords + size_t(view) * a.n_points;
  if (warp == 0) {
    int mt_index = kMtN;
    if (lane == 0) MtSeed(mt, a.seed);
    int taken = 0;
    while (taken < a.n_points) {
      if (lane == 0)
        for (int k = 0; k < 32; ++k) cand[k] = MtNext(mt, mt_index);
      __syncwarp();
      const int idx = int(cand[lane] % unsigned(n_pix));
      const int x = idx / S, y = idx % S;  // cv::Point2i{idx / rows, idx % cols}
      const bool ok = Silhouette(zs[size_t(y) * S + x], a.n_renderers);
      const unsigned m = __ballot_sync(0xffffffffu, ok);
      const int rank = __popc(m & ((1u << lane) - 1u));
      if (ok && taken + rank < a.n_points) coords[taken + rank] = y * S + x;
      taken += __popc(m);
      __syncwarp();  // cand is refilled
    }
  }
  __syncthreads();

  // GeneratePointData + CalculateDepthOffsets, one warp per point
  const float* T = a.camera2body + 12 * size_t(view);
  for (int p = warp; p < a.n_points; p += n_warps) {
    const int pix = coords[p];
    const int y = pix / S, x = pix % S;
    const uint64_t key = z0[pix];
    const unsigned d16c = unsigned(key >> 48);
    const float depth = a.projection_term_a / (a.projection_term_b - float(d16c));  // FullDepthRenderer::PointVector
    const float cx = depth * (float(x) - a.ppu) / a.fu;
    const float cy = depth * (float(y) - a.ppv) / a.fv;
    const float cz = depth;
    const float pixel_to_meter = cz / a.fu;
    float* o = out + size_t(p) * 36;
    DepthOffsets(z0, S, x, y, d16c, depth, pixel_to_meter, a.stride_depth_offset, a.n_values, a.projection_term_a,
                 a.projection_term_b, s_min[warp], o + 6, lane);
    if (lane == 0) {
      unsigned nb[4];
      NormalBytes(a, view, key, nb);
      const float nx = 1.0f - float(nb[0]) / 127.5f;  // FullNormalRenderer::NormalVector
      const float ny = 1.0f - float(nb[1]) / 127.5f;
      const float nz = 1.0f - float(nb[2]) / 127.5f;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        o[r] = T[4 * r] * cx + T[4 * r + 1] * cy + T[4 * r + 2] * cz + T[4 * r + 3];
        o[3 + r] = T[4 * r] * nx + T[4 * r + 1] * ny + T[4 * r + 2] * nz;
      }
    }
  }
}

__global__ void k_model_images(const __grid_constant__ ModelPointArgs a, int view, uint8_t* normal, uint16_t* depth,
                               uint8_t* silhouette) {
  const int n_pix = a.image_size * a.image_size;
  const uint64_t* z0 = a.zbuf + size_t(view) * a.n_renderers * n_pix;
  const uint64_t* zs = a.n_renderers == 2 ? z0 + n_pix : z0;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n_pix; p += gridDim.x * blockDim.x) {
    unsigned nb[4];
    NormalBytes(a, view, z0[p], nb);
#pragma unroll
    for (int k = 0; k < 4; ++k) normal[4 * size_t(p) + k] = uint8_t(nb[k]);
    depth[p] = uint16_t(z0[p] >> 48);
    silhouette[p] = Silhouette(zs[p], a.n_renderers) ? 255 : 0;
  }
}

// ---- region-model generation ---------------------------------------------------------------------------------------

namespace {

__device__ __forceinline__ uint32_t PackXY(int x, int y) { return uint32_t(x) | (uint32_t(y) << 16); }
__device__ __forceinline__ int PX(uint32_t q) { return int(q & 0xffffu); }
__device__ __forceinline__ int PY(uint32_t q) { return int(q >> 16); }

// chain code s (0 = +x, counter-clockwise with y down) as a step in x, in y, and in a row-major image of width W
__device__ __forceinline__ int ChainDx(int s) { return (s == 0 || s == 1 || s == 7) ? 1 : (s >= 3 && s <= 5) ? -1 : 0; }
__device__ __forceinline__ int ChainDy(int s) { return (s >= 1 && s <= 3) ? -1 : (s >= 5) ? 1 : 0; }
__device__ __forceinline__ int ChainDelta(int s, int W) { return ChainDx(s) + ChainDy(s) * W; }

// One border of the zero-padded label image from (x0, y0), as OpenCV's icvFetchContour follows it with nbd 2 and
// CHAIN_APPROX_NONE: visited pixels become 2, pixels whose right neighbour was examined -126. Appends the points, in
// unpadded coordinates, to out[n..] (those at or beyond cap are counted but not written); returns the new count.
__device__ int TraceBorder(int8_t* lab, int W, int x0, int y0, bool hole, uint32_t* out, int n, int cap) {
  const int i0 = y0 * W + x0;
  int s = hole ? 0 : 4, s_end = s, i1;
  do {
    s = (s - 1) & 7;
    i1 = i0 + ChainDelta(s, W);
  } while (lab[i1] == 0 && s != s_end);
  if (s == s_end) {  // a single pixel
    lab[i0] = -126;
    if (n < cap) out[n] = PackXY(x0 - 1, y0 - 1);
    return n + 1;
  }
  int i3 = i0, x = x0, y = y0;
  for (;;) {
    s_end = s;
    int i4;
    do {
      ++s;
      i4 = i3 + ChainDelta(s & 7, W);
    } while (lab[i4] == 0 && s < 15);
    s &= 7;
    if (unsigned(s - 1) < unsigned(s_end)) lab[i3] = -126;
    else if (lab[i3] == 1) lab[i3] = 2;
    if (n < cap) out[n] = PackXY(x - 1, y - 1);
    ++n;
    x += ChainDx(s);
    y += ChainDy(s);
    if (i4 == i0 && i3 == i1) break;
    i3 = i4;
    s = (s + 4) & 7;
  }
  return n;
}

// glibc's hypotf: the double squares of two floats are exact, their sum and the square root are rounded once each in
// double, the result once to float. CUDA's hypotf differs in the last bit, which decides argmin ties.
__device__ __forceinline__ float HypotF(float a, float b) {
  const double da = a, db = b;
  return float(sqrt(da * da + db * db));
}

// FindClosestContourPoint (region_model.cpp:768-782) over all n contour points: a warp argmin that keeps the first
// index among equal distances, as the serial loop with its strict < does
__device__ uint32_t ClosestContourPoint(const uint32_t* C, int n, float u, float v, int lane) {
  float best = FLT_MAX;
  int bi = INT_MAX;
  for (int f = lane; f < n; f += 32) {
    const uint32_t q = C[f];
    const float d = HypotF(float(PX(q)) - u, float(PY(q)) - v);
    if (d < best) {
      best = d;
      bi = f;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob < best || (ob == best && oi < bi)) {
      best = ob;
      bi = oi;
    }
  }
  return C[bi];
}

__device__ __forceinline__ int RegionStartStride(int cap) { return cap / kRegionMinContourLength + 2; }

}  // namespace

// cv::findContours(main silhouette == 255, RETR_LIST, CHAIN_APPROX_NONE) + the length filter of
// GenerateValidContours. Per row of the padded image the CTA marks the 0 <-> nonzero steps in shared memory (ballots);
// thread 0 then visits them in raster order and follows each border that starts there (Suzuki & Abe: an outer border
// at 0 -> 1, a hole border from a pixel marked 1 or 2 to 0). Finally the kept contours are copied in reverse order of
// discovery, which is the order cv::findContours lists them in.
__global__ void __launch_bounds__(kModelThreads) k_region_contours(const __grid_constant__ RegionContourArgs a) {
  __shared__ uint32_t s_steps[(8192 + 31) / 32];
  __shared__ int s_n, s_nc, s_overflow;
  const int view = blockIdx.x, S = a.image_size, W = S + 2;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
  const uint64_t* z0 = a.zbuf + size_t(view) * a.R.n_renderers * S * S;
  int8_t* lab = a.label + size_t(view) * W * W;
  uint32_t* raw = a.raw + size_t(view) * a.cap;
  int* raw_start = a.raw_start + size_t(view) * RegionStartStride(a.cap);
  const int max_contours = RegionStartStride(a.cap) - 1;
  for (int k = tid; k < W * W; k += blockDim.x) {
    const int y = k / W - 1, x = k % W - 1;
    lab[k] = (x >= 0 && x < S && y >= 0 && y < S && SilhouetteId(a.R, 0, z0[size_t(y) * S + x]) == 255u) ? 1 : 0;
  }
  __syncthreads();
  const int n_words = (S + 31) / 32;
  int n = 0, nc = 0, overflow = 0;  // thread 0's
  for (int y = 1; y <= S; ++y) {
    const int8_t* row = lab + size_t(y) * W;
    for (int w = warp; w < n_words; w += n_warps) {
      const int x = 1 + 32 * w + lane;
      const bool step = x <= S && ((row[x] != 0) != (row[x - 1] != 0));
      const unsigned m = __ballot_sync(0xffffffffu, step);
      if (lane == 0) s_steps[w] = m;
    }
    __syncthreads();
    if (tid == 0) {
      for (int w = 0; w < n_words; ++w) {
        for (unsigned m = s_steps[w]; m; m &= m - 1) {
          const int x = 1 + 32 * w + __ffs(m) - 1;
          const int8_t p = row[x], prev = row[x - 1];
          bool hole;
          if (prev == 0 && p == 1) hole = false;
          else if (p == 0 && prev >= 1) hole = true;
          else continue;
          const int begin = n;
          n = TraceBorder(lab, W, hole ? x - 1 : x, y, hole, raw, n, a.cap);
          if (n - begin < kRegionMinContourLength) {
            n = begin;  // too short: dropped
          } else if (n > a.cap || nc >= max_contours) {
            overflow = 1;
          } else {
            raw_start[nc++] = begin;
          }
        }
      }
    }
    __syncthreads();
  }
  if (tid == 0) {
    raw_start[nc] = n;
    s_n = n;
    s_nc = nc;
    s_overflow = overflow;
    if (overflow) atomicExch(a.overflow, 1);
  }
  __syncthreads();
  n = s_n;
  nc = s_nc;
  int* counts = a.counts + 2 * view;
  if (s_overflow) {
    if (tid == 0) counts[0] = counts[1] = 0;
    return;
  }
  uint32_t* C = a.contour + size_t(view) * a.cap;
  int* CS = a.contour_start + size_t(view) * RegionStartStride(a.cap);
  for (int j = 0; j < nc; ++j) {  // discovery contour j is contour nc - 1 - j of the list, starting at n - end_j
    const int b = raw_start[j], len = raw_start[j + 1] - b, f = n - raw_start[j + 1];
    for (int i = tid; i < len; i += blockDim.x) C[f + i] = raw[b + i];
  }
  for (int k = tid; k <= nc; k += blockDim.x) CS[k] = n - raw_start[nc - k];
  if (tid == 0) {
    counts[0] = nc;
    counts[1] = n;
  }
}

// RegionModel::GeneratePointData (region_model.cpp:479-554) with IsContourPointValid, SampleContourPointCoordinate,
// CalculateContourSegment, ApproximateNormalVector and CalculateLineDistances. The CTA compacts the valid contour
// points in contour order, then replays the serial sampling loop (thread 0 draws, the CTA finds the first occurrence of
// the centre), then one warp per accepted point computes its DataPoint.
__global__ void __launch_bounds__(kModelThreads) k_region_points(const __grid_constant__ RegionPointArgs a) {
  __shared__ uint32_t mt[kMtN];
  __shared__ unsigned s_min[kModelThreads / 32][kModelMaxOffsets];
  __shared__ int s_warp[kModelThreads / 32];
  __shared__ int s_first, s_ok;
  __shared__ uint32_t s_center;
  const int view = blockIdx.x, S = a.image_size;
  const size_t n_pix = size_t(S) * S;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
  const uint64_t* z = a.zbuf + size_t(view) * a.R.n_renderers * n_pix;
  const int total = a.counts[2 * view + 1];
  const uint32_t* C = a.contour + size_t(view) * a.cap;
  const int* CS = a.contour_start + size_t(view) * RegionStartStride(a.cap);
  uint32_t* V = a.valid + size_t(view) * a.cap;
  float* out = a.points + size_t(view) * a.n_points * kRegionPointFloats;
  // silhouette of renderer r, 0 off the image; depth of the main renderer (FullDepthRenderer::Depth)
  auto sil = [&](int r, int x, int y) -> unsigned {
    if (x < 0 || x >= S || y < 0 || y >= S) return 0u;
    return SilhouetteId(a.R, r, z[size_t(r) * n_pix + size_t(y) * S + x]);
  };
  auto depth_at = [&](int x, int y) {
    return a.projection_term_a / (a.projection_term_b - float(unsigned(z[size_t(y) * S + x] >> 48)));
  };
  const float pixel_to_meter0 = a.sphere_radius / a.fu;
  const float max_depth_difference = pixel_to_meter0 * kRegionMaxSurfaceGradient;

  // IsContourPointValid over the contour list, compacted in order
  int n_valid = 0;
  for (int base = 0; base < total; base += blockDim.x) {
    const int f = base + tid;
    bool ok = false;
    uint32_t q = 0;
    if (f < total) {
      q = C[f];
      const int x = PX(q), y = PY(q);
      const int nx[4] = {x, x, x + 1, x - 1}, ny[4] = {y + 1, y - 1, y, y};
      ok = true;
      if (a.r_same >= 0)
        for (int k = 0; k < 4; ++k) ok = ok && sil(a.r_same, nx[k], ny[k]) == 0u;
      if (ok && a.r_occ >= 0) ok = sil(a.r_occ, x, y) == 0u;
      if (ok) {
        float sum = 0.0f;
        int cnt = 0;
        for (int k = 0; k < 4; ++k)
          if (sil(0, nx[k], ny[k]) == 120u) {
            sum = sum + depth_at(nx[k], ny[k]);
            ++cnt;
          }
        if (cnt > 0 && sum / float(cnt) < depth_at(x, y) - max_depth_difference) ok = false;
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int off = n_valid, sum = 0;
    for (int w = 0; w < n_warps; ++w) {
      if (w < warp) off += s_warp[w];
      sum += s_warp[w];
    }
    if (ok) V[off + __popc(m & ((1u << lane) - 1u))] = q;
    n_valid += sum;
    __syncthreads();
  }
  if (n_valid == 0) {  // no contour, or no valid point: contour_length 0 and zero-filled points
    if (tid == 0) a.contour_length[view] = 0.0f;
    for (int k = tid; k < a.n_points * kRegionPointFloats; k += blockDim.x) out[k] = 0.0f;
    return;
  }

  // sampling: a fresh std::mt19937 per view, idx = gen() % n_valid, at most kRegionMaxSamplingTries + 1 consecutive
  // rejections
  int* coords = a.coords + size_t(view) * a.n_points;
  float* nrm = a.normals + size_t(view) * a.n_points * 2;
  int mt_index = kMtN;
  if (tid == 0) MtSeed(mt, a.seed);
  int produced = 0, tries = 0;
  bool exhausted = false;
  while (produced < a.n_points) {
    if (tries++ > kRegionMaxSamplingTries) {
      exhausted = true;
      break;
    }
    if (tid == 0) {
      s_center = V[MtNext(mt, mt_index) % unsigned(n_valid)];
      s_first = INT_MAX;
    }
    __syncthreads();
    const uint32_t c = s_center;
    for (int base = 0; base < total; base += blockDim.x) {  // the first contour and index that hold the centre
      const bool hit = base + tid < total && C[base + tid] == c;
      if (hit) atomicMin(&s_first, base + tid);
      if (__syncthreads_or(hit)) break;
    }
    if (tid == 0) {
      s_ok = 0;
      const int f = s_first;
      if (f != INT_MAX) {
        int k = 0;
        while (CS[k + 1] <= f) ++k;
        const int b = CS[k], len = CS[k + 1] - b, i = f - b;
        const uint32_t front = C[b + (i - kRegionNormalApproxRadius + len) % len];
        const uint32_t back = C[b + (i + kRegionNormalApproxRadius) % len];
        const int dx = PX(back) - PX(front), dy = PY(back) - PY(front);
        if (HypotF(float(dx), float(dy)) > float(kRegionNormalApproxRadius)) {
          const float vx = -float(dy), vy = float(dx);  // Eigen normalized(): v / sqrt(squaredNorm)
          const float sn = sqrtf(vx * vx + vy * vy);
          coords[produced] = PY(c) * S + PX(c);
          nrm[2 * produced] = vx / sn;
          nrm[2 * produced + 1] = vy / sn;
          s_ok = 1;
        }
      }
    }
    __syncthreads();
    if (s_ok) {
      ++produced;
      tries = 0;
    }
    __syncthreads();  // s_ok and s_center are rewritten by the next attempt
  }
  if (tid == 0) a.contour_length[view] = exhausted ? 0.0f : float(n_valid) * pixel_to_meter0;
  for (int k = produced * kRegionPointFloats + tid; k < a.n_points * kRegionPointFloats; k += blockDim.x) out[k] = 0.0f;

  // the DataPoints, one warp per point
  const float* T = a.camera2body + 12 * size_t(view);
  const int r_fg = a.r_fg >= 0 ? a.r_fg : 0, r_bg = a.r_bg >= 0 ? a.r_bg : 0;
  for (int p = warp; p < produced; p += n_warps) {
    const int pix = coords[p];
    const int y = pix / S, x = pix % S;
    const float nx = nrm[2 * p], ny = nrm[2 * p + 1];
    const unsigned d16c = unsigned(z[pix] >> 48);
    const float depth = a.projection_term_a / (a.projection_term_b - float(d16c));  // FullDepthRenderer::PointVector
    const float cx = depth * (float(x) - a.ppu) / a.fu;
    const float cy = depth * (float(y) - a.ppv) / a.fv;
    const float cz = depth;
    const float pixel_to_meter = cz / a.fu;
    float* o = out + size_t(p) * kRegionPointFloats;
    DepthOffsets(z, S, x, y, d16c, depth, pixel_to_meter, a.stride_depth_offset, a.n_values, a.projection_term_a,
                 a.projection_term_b, s_min[warp], o + 8, lane);
    // CalculateLineDistances: every lane walks the same line, the warp finds the closest contour point
    float u_step, v_step;
    if (fabsf(ny) < fabsf(nx)) {
      u_step = float((0.0f < nx) - (nx < 0.0f));
      v_step = ny / fabsf(nx);
    } else {
      u_step = nx / fabsf(ny);
      v_step = float((0.0f < ny) - (ny < 0.0f));
    }
    float u = float(x) + 0.5f, v = float(y) + 0.5f;
    do {  // inwards on the foreground image; off the image counts as leaving the body
      u = u - u_step;
      v = v - v_step;
    } while (sil(r_fg, int(u), int(v)) == 255u);
    const uint32_t e_in = ClosestContourPoint(C, total, u + u_step - 0.5f, v + v_step - 0.5f, lane);
    const float foreground_distance = pixel_to_meter * HypotF(float(PX(e_in) - x), float(PY(e_in) - y));
    float background_distance = FLT_MAX;
    u = float(x) + 0.5f;
    v = float(y) + 0.5f;
    for (;;) {  // outwards on the background image
      u = u + u_step;
      v = v + v_step;
      if (int(u) < 0 || int(u) >= S || int(v) < 0 || int(v) >= S) break;
      if (sil(r_bg, int(u), int(v)) == 255u) {
        const uint32_t e = ClosestContourPoint(C, total, u - 0.5f, v - 0.5f, lane);
        background_distance = pixel_to_meter * HypotF(float(PX(e) - x), float(PY(e) - y));
        break;
      }
    }
    if (lane == 0) {
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        o[r] = T[4 * r] * cx + T[4 * r + 1] * cy + T[4 * r + 2] * cz + T[4 * r + 3];
        o[3 + r] = T[4 * r] * nx + T[4 * r + 1] * ny + T[4 * r + 2] * 0.0f;  // linear block times (nx, ny, 0)
      }
      o[6] = foreground_distance;
      o[7] = background_distance;
    }
  }
}

__global__ void k_region_images(const uint64_t* zbuf, ModelRenderers R, int image_size, uint8_t* silhouettes,
                                uint16_t* depth) {
  const size_t n_pix = size_t(image_size) * image_size;
  for (size_t p = blockIdx.x * size_t(blockDim.x) + threadIdx.x; p < n_pix; p += size_t(gridDim.x) * blockDim.x) {
    for (int r = 0; r < R.n_renderers; ++r) silhouettes[r * n_pix + p] = uint8_t(SilhouetteId(R, r, zbuf[r * n_pix + p]));
    depth[p] = uint16_t(zbuf[p] >> 48);
  }
}

}  // namespace m3tb
