// m3t_b200_model.cu — depth-model generation: k_model_raster draws the geodesic views of a batch into global-memory
// z-buffers, k_model_points samples and describes the surface points of each view, k_model_images reads one view back
// as the reference's normal / depth / silhouette images. Float32, one rounding per operation in the order written
// (-fmad=false); DESIGN.md §3 "k_model_raster / k_model_points" states the contract and
// tests/model_generation_reference.py restates it.
#include "m3t_b200_model.cuh"
#include "m3t_b200_raster.cuh"

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

// float -> unorm8 of the GL colour attachment: clamp to [0, 1], scale by 255, round to nearest even
__device__ __forceinline__ unsigned Unorm8(float c) { return unsigned(rintf(fminf(fmaxf(c, 0.0f), 1.0f) * 255.0f)); }

// the normal image at one pixel (normal_renderer.cpp:11-31): 0.5 - 0.5 * Rot * n of the winning triangle, bytes in
// GL_BGRA read-back order (byte 0 encodes x); background 0
__device__ __forceinline__ void NormalBytes(const ModelPointArgs& a, int view, uint64_t key, unsigned b[4]) {
  if (key == kModelClear) {
    b[0] = b[1] = b[2] = b[3] = 0u;
    return;
  }
  const float* n = a.face_normals + 3 * size_t(key & 0xffffffffu);
  const float* R = a.rot + 9 * size_t(view);
#pragma unroll
  for (int r = 0; r < 3; ++r) b[r] = Unorm8(0.5f - 0.5f * (R[3 * r] * n[0] + R[3 * r + 1] * n[1] + R[3 * r + 2] * n[2]));
  b[3] = 255u;
}

}  // namespace

__global__ void __launch_bounds__(kModelThreads) k_model_raster(const __grid_constant__ ModelRasterArgs a) {
  const int view = blockIdx.y, r = blockIdx.z;
  const int S = a.image_size;
  const size_t n_pix = size_t(S) * S;
  unsigned long long* zb = reinterpret_cast<unsigned long long*>(a.zbuf + (size_t(view) * a.n_renderers + r) * n_pix);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const int n_bodies = r == 0 ? 1 : 1 + a.n_occlusion;
  const int n_slots = 2 + a.n_occlusion;
  const float half = 0.5f * float(S);
  for (int g = 0; g < n_bodies; ++g) {
    const ModelBodyDev B = a.bodies[g];
    const float* Mg = a.M + (size_t(view) * n_slots + (r == 0 ? 0 : 1 + g)) * 16;
    float M[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) M[k] = Mg[k];
    for (int t0 = blockIdx.x * kModelTrianglesPerCta; t0 < B.n_triangles; t0 += gridDim.x * kModelTrianglesPerCta) {
      const int t_end = min(t0 + kModelTrianglesPerCta, B.n_triangles);
      for (int t = t0 + warp; t < t_end; t += n_warps) {
        const unsigned long long tag = ModelKey(0u, unsigned(g), unsigned(t));
        auto frag = [&](int i, int j, unsigned d16) {
          atomicMin(zb + size_t(j) * S + i, (static_cast<unsigned long long>(d16) << 48) | tag);
        };
        DrawTriangle(M, B.triangles + 9 * size_t(t), B.enable_culling, S, half, frag, lane);
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
    const float stride = a.stride_depth_offset / pixel_to_meter;
    const float max_diameter = 2.0f * float(a.n_values) * stride;
    const int image_stride = int(stride + 1.0f);
    const int n_image_strides = int(max_diameter / float(image_stride) + 1.0f);
    const int image_diameter = n_image_strides * image_stride;
    const int radius_minus = image_diameter / 2;
    const int radius_plus = image_diameter - radius_minus;
    const int v_min = max(y - radius_minus, 0), v_max = min(y + radius_plus, S - 1);
    const int u_min = max(x - radius_minus, 0), u_max = min(x + radius_plus, S - 1);
    if (lane < kModelMaxOffsets) s_min[warp][lane] = lane == 0 ? d16c : 0xffffu;
    __syncwarp();
    const int nu = u_max >= u_min ? (u_max - u_min) / image_stride + 1 : 0;
    const int nv = v_max >= v_min ? (v_max - v_min) / image_stride + 1 : 0;
    for (int k = lane; k < nu * nv; k += 32) {
      const int u = u_min + (k % nu) * image_stride, v = v_min + (k / nu) * image_stride;
      const int du = u - x, dv = v - y;
      const float distance = float(sqrt(double(du * du + dv * dv)));  // std::sqrt(int) is a double
      const int i = int(distance / stride);
      if (i < a.n_values) atomicMin(&s_min[warp][i], unsigned(z0[size_t(v) * S + u] >> 48));
    }
    __syncwarp();
    if (lane == 0) {
      unsigned nb[4];
      NormalBytes(a, view, key, nb);
      const float nx = 1.0f - float(nb[0]) / 127.5f;  // FullNormalRenderer::NormalVector
      const float ny = 1.0f - float(nb[1]) / 127.5f;
      const float nz = 1.0f - float(nb[2]) / 127.5f;
      float* o = out + size_t(p) * 36;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        o[r] = T[4 * r] * cx + T[4 * r + 1] * cy + T[4 * r + 2] * cz + T[4 * r + 3];
        o[3 + r] = T[4 * r] * nx + T[4 * r + 1] * ny + T[4 * r + 2] * nz;
      }
      unsigned m = s_min[warp][0];
      o[6] = depth - a.projection_term_a / (a.projection_term_b - float(m));
      for (int i = 1; i < kModelMaxOffsets; ++i) {
        m = min(s_min[warp][i], m);
        o[6 + i] = depth - a.projection_term_a / (a.projection_term_b - float(m));
      }
    }
    __syncwarp();  // s_min is reset for the next point
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

}  // namespace m3tb
