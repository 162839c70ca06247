// m3t_b200_view.cu — the viewers' full normal renderers and the overlay they are blended into (NormalColorViewer /
// NormalDepthViewer::UpdateViewer, normal_viewer.cpp; FullNormalRenderer, normal_renderer.cpp), and the full renderers
// (FullBasicDepthRenderer / FullSilhouetteRenderer / FullNormalRenderer, m3tb_render_full). Three launches for all
// viewers (or all full renderers) of a context: k_view_setup clips and sets up every triangle, k_view_raster walks
// (triangle, screen tile) pairs so that a large triangle is shared by many warps, k_view_resolve writes the normal and
// viewer images (the depth, silhouette and normal images of a full renderer). Focused normal renderers
// (FocusedNormalRenderer, m3tb_render_focused_normals) take a fourth launch first, k_view_focus, which focuses each on
// its referenced bodies from the current poses. k_normalized_depth writes NormalizedDepthImage. Float32,
// one rounding per operation in the order written (-fmad=false); DESIGN.md §3 "k_view_setup / k_view_raster /
// k_view_resolve" states the contract, tests/viewer_reference.py restates it.
#include "m3t_b200_view.cuh"
#include "m3t_b200_device.cuh"
#include "m3t_b200_raster.cuh"

namespace m3tb {

namespace {

__device__ void EmitFan(const ViewArgs& a, WinVertex v0, WinVertex v1, WinVertex v2, int culling, const ViewerDev& V,
                        int viewer, uint64_t tag) {
  float A;
  if (!OrientTriangle(v0, v1, v2, culling, A)) return;
  int i0, j0, nx, ny;
  if (!PixelBox(v0, v1, v2, V.width, V.height, i0, j0, nx, ny)) return;
  const int ntx = (i0 + nx - 1) / kViewTile - i0 / kViewTile + 1;
  const int nty = (j0 + ny - 1) / kViewTile - j0 / kViewTile + 1;
  // one atomic takes the slot and the work items together, so that slots and first work items grow together
  const unsigned long long old = atomicAdd(a.counter, (1ull << kViewFanShift) | (unsigned long long)(ntx * nty));
  const int slot = int(old >> kViewFanShift);
  if (slot >= a.fan_cap) return;  // cannot happen: two fan triangles per triangle at most
  ViewFanDev f;
  f.v[0] = v0.x; f.v[1] = v0.y; f.v[2] = v0.z;
  f.v[3] = v1.x; f.v[4] = v1.y; f.v[5] = v1.z;
  f.v[6] = v2.x; f.v[7] = v2.y; f.v[8] = v2.z;
  f.A = A;
  f.i0 = i0; f.j0 = j0; f.nx = nx; f.ny = ny;
  f.viewer = viewer;
  f.tag = tag;
  a.fans[slot] = f;
  a.fan_tile[slot] = old & kViewTileMask;
}

// (p2 - p1).cross(p0 - p1).normalized() (RendererGeometry::AssembleVertexData, renderer_geometry.cpp:199-204); Eigen's
// normalized() leaves a zero vector unchanged
__device__ __forceinline__ void FaceNormal(const float* v, float n[3]) {
  const float ax = v[6] - v[3], ay = v[7] - v[4], az = v[8] - v[5];
  const float bx = v[0] - v[3], by = v[1] - v[4], bz = v[2] - v[5];
  n[0] = ay * bz - az * by;
  n[1] = az * bx - ax * bz;
  n[2] = ax * by - ay * bx;
  const float q = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
  if (!(q > 0.0f)) return;
  const float s = sqrtf(q);
  n[0] = n[0] / s;
  n[1] = n[1] / s;
  n[2] = n[2] / s;
}

// char(x) of the blend on x86-64: the low byte of the 32-bit truncation (cvttss2si), whose out-of-range and NaN
// result is 0x80000000
__device__ __forceinline__ unsigned CharOf(float x) {
  if (!(x >= -2147483648.0f && x < 2147483648.0f)) return 0u;
  return unsigned(int(x)) & 0xffu;
}

// saturate_cast<uchar>(src * alpha + beta) of cv::Mat::convertTo as OpenCV 4.13 computes it on x86-64 (AVX2 / FMA3
// path): one fused multiply-add, cvRound (half to even; out of the int range the result is INT_MIN), saturation
__device__ __forceinline__ unsigned DepthGray(unsigned d, float alpha, float beta) {
  const float r = rintf(__fmaf_rn(float(d), alpha, beta));
  if (!(r >= -2147483648.0f && r < 2147483648.0f)) return 0u;
  return unsigned(fminf(fmaxf(r, 0.0f), 255.0f));
}

}  // namespace

__global__ void __launch_bounds__(kViewThreads) k_view_focus(const __grid_constant__ FocusArgs a) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= a.n_focus) return;
  const FocusDev& F = a.focus[f];
  auto body = [&](int k, float& rr, const float*& p) {
    rr = a.radius[F.first_referenced + k];
    p = a.poses + 12 * a.referenced[F.first_referenced + k];
  };
  float P[6];
  RenderOutDev o;
  const bool any =
      FocusProjection(F.cam, F.image_size, F.z_min, F.z_max, F.n_referenced, body, a.visible + F.first_referenced, o, P);
  a.out[f] = o;
  ViewerDev& V = a.viewers[F.viewer];
  V.P00 = P[0];
  V.P02 = P[1];
  V.P11 = P[2];
  V.P12 = P[3];
  V.P22 = P[4];
  V.P23 = P[5];
  if (!any)  // as k_render: nothing is drawn, the images stay cleared
    for (int g = 0; g < V.n_draws; ++g) a.draws[V.first_draw + g].n_triangles = 0;
}

__global__ void __launch_bounds__(kViewThreads) k_view_setup(const __grid_constant__ ViewArgs a) {
  const int d = blockIdx.y;
  if (d >= a.n_draws) return;  // no draw at all: the launch is one idle block
  const ViewDrawDev& D = a.draws[d];
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= D.n_triangles) return;
  const ViewerDev& V = a.viewers[D.viewer];
  float g2w[12], T[12], M[16];
  PoseMul(a.poses + 12 * D.body, D.geometry2body, g2w);  // Body::geometry2world_pose (body.cpp:88)
  PoseMul(V.w2c, g2w, T);                                // world2camera * geometry2world
  // P * [T; 0 0 0 1]; the products with P's zero entries are left out, as in k_render
  for (int c = 0; c < 4; ++c) {
    M[c] = V.P00 * T[c] + V.P02 * T[8 + c];
    M[4 + c] = V.P11 * T[4 + c] + V.P12 * T[8 + c];
    M[8 + c] = V.P22 * T[8 + c];
    M[12 + c] = T[8 + c];
  }
  M[11] = M[11] + V.P23;
  if (t == 0)
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) a.rot[9 * size_t(d) + 3 * i + j] = T[4 * i + j];
  ClipVertex poly[4];
  const int n = ClipTriangle(M, D.triangles + 9 * size_t(t), poly);
  if (n < 3) return;
  const float half_x = 0.5f * float(V.width), half_y = 0.5f * float(V.height);
  const WinVertex w0 = Window(poly[0], half_x, half_y), w1 = Window(poly[1], half_x, half_y),
                  w2 = Window(poly[2], half_x, half_y);
  const uint64_t tag = (uint64_t(unsigned(D.draw)) << 32) | uint64_t(unsigned(t));
  EmitFan(a, w0, w1, w2, D.enable_culling, V, D.viewer, tag);
  if (n == 4) EmitFan(a, w0, w2, Window(poly[3], half_x, half_y), D.enable_culling, V, D.viewer, tag);
}

__global__ void __launch_bounds__(kViewThreads) k_view_raster(const __grid_constant__ ViewArgs a) {
  const unsigned long long c = *a.counter;
  const int n_fans = int(c >> kViewFanShift);
  const uint64_t n_items = c & kViewTileMask;
  const int lane = threadIdx.x & 31;
  const uint64_t n_warps = uint64_t(gridDim.x) * (blockDim.x >> 5);
  for (uint64_t w = uint64_t(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); w < n_items; w += n_warps) {
    int lo = 0, hi = n_fans - 1;  // the last fan whose first work item is at or before w
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (a.fan_tile[mid] <= w) lo = mid;
      else hi = mid - 1;
    }
    const ViewFanDev& F = a.fans[lo];
    const WinVertex v0 = {F.v[0], F.v[1], F.v[2]}, v1 = {F.v[3], F.v[4], F.v[5]}, v2 = {F.v[6], F.v[7], F.v[8]};
    const int k = int(w - a.fan_tile[lo]);
    const int tx0 = F.i0 / kViewTile, ntx = (F.i0 + F.nx - 1) / kViewTile - tx0 + 1;
    const int tx = tx0 + k % ntx, ty = F.j0 / kViewTile + k / ntx;
    const int x0 = max(F.i0, tx * kViewTile), x1 = min(F.i0 + F.nx, (tx + 1) * kViewTile);
    const int y0 = max(F.j0, ty * kViewTile), y1 = min(F.j0 + F.ny, (ty + 1) * kViewTile);
    const int wx = x1 - x0, n = wx * (y1 - y0);
    const ViewerDev& V = a.viewers[F.viewer];
    unsigned long long* zb = reinterpret_cast<unsigned long long*>(V.zbuf);
    for (int p = lane; p < n; p += 32) {
      const int i = x0 + p % wx, j = y0 + p / wx;
      unsigned d16;
      if (PixelDepth(v0, v1, v2, F.A, i, j, d16))
        atomicMin(zb + size_t(j) * V.width + i, (static_cast<unsigned long long>(d16) << 48) | F.tag);
    }
  }
}

__global__ void __launch_bounds__(kViewThreads) k_view_resolve(const __grid_constant__ ViewArgs a) {
  const ViewerDev& V = a.viewers[blockIdx.y];
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *a.counter = 0ull;  // k_view_raster has run
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= V.width * V.height) return;
  const int i = p % V.width, j = p / V.width;
  const uint64_t key = V.zbuf[p];
  V.zbuf[p] = kViewClear;  // glClear of the next update
  unsigned nb[4] = {0u, 0u, 0u, 0u};  // glClearColor(0, 0, 0, 0)
  const int d = V.first_draw + int((key >> 32) & 0xffffu);
  if (key != kViewClear) {
    float n[3];
    FaceNormal(a.draws[d].triangles + 9 * size_t(key & 0xffffffffu), n);
    EncodeNormal(a.rot + 9 * size_t(d), n, nb);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) V.normal[4 * size_t(p) + k] = uint8_t(nb[k]);
  if (V.kind >= VK_FULL) {
    // glReadPixels of GL_DEPTH_COMPONENT16 (the cleared key reads 65535) and of the silhouette id attachment
    V.depth[p] = uint16_t(key >> 48);
    if (V.kind == VK_FULL) V.silhouette[p] = key != kViewClear ? uint8_t(a.draws[d].silhouette_id) : uint8_t(0);
    return;
  }
  unsigned cam[3];
  const uint8_t* row = V.frame + size_t(j) * V.frame_pitch;
  if (V.kind == VK_COLOR) {
    cam[0] = row[3 * i];
    cam[1] = row[3 * i + 1];
    cam[2] = row[3 * i + 2];
  } else {  // NormalizedDepthImage, then COLOR_GRAY2BGR
    cam[0] = cam[1] = cam[2] = DepthGray(reinterpret_cast<const uint16_t*>(row)[i], V.depth_alpha, V.depth_beta);
  }
  // CalculateAlphaBlend (normal_viewer.cpp:8-44)
  const float alpha_scale = V.opacity / 255.0f;
  const float alpha = float(nb[3]) * alpha_scale;
  const float alpha_inv = 1.0f - alpha;
#pragma unroll
  for (int k = 0; k < 3; ++k)
    V.image[3 * size_t(p) + k] = uint8_t(CharOf(float(cam[k]) * alpha_inv + float(nb[k]) * alpha));
}

__global__ void __launch_bounds__(kViewThreads) k_normalized_depth(const __grid_constant__ NormalizedDepthArgs a) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.width * a.height) return;
  const int i = p % a.width, j = p / a.width;
  const unsigned v = reinterpret_cast<const uint16_t*>(a.src + size_t(j) * a.src_pitch)[i];
  unsigned g;
  if (!a.renderer) {
    g = DepthGray(v, a.alpha, a.beta);  // DepthCamera::NormalizedDepthImage, as NormalDepthViewer reads its frame
  } else {  // FullDepthRenderer::NormalizedDepthImage (renderer.cpp:407-427)
    float depth = a.a / (a.b - float(v));
    depth = depth - a.min_depth;
    depth = depth < 0.0f ? 0.0f : depth;        // std::max(depth - min_depth, 0.0f)
    depth = a.delta < depth ? a.delta : depth;  // std::min(..., delta_depth)
    g = CharOf(depth * a.scale);                // uchar(depth * scale)
  }
  a.dst[size_t(j) * a.dst_pitch + i] = uint8_t(g);
}

}  // namespace m3tb
