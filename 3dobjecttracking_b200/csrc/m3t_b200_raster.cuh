// m3t_b200_raster.cuh — the triangle walk shared by k_render (focused renderers, shared-memory z-buffer),
// k_model_raster (full-frame model-generation renderers, global-memory z-buffer) and k_view_setup / k_view_raster
// (full-camera-image viewer renderers, W x H, triangles split into screen tiles): transform to clip space, near-plane
// clipping, window mapping, watertight edge functions with a top-left tie rule, GL-style culling and DEPTH_COMPONENT16
// quantisation. The caller supplies the fragment write. DESIGN.md §3 "k_render" states the contract and
// tests/render_reference.py restates it.
#pragma once

#include <cuda_runtime.h>

namespace m3tb {

struct ClipVertex {
  float x, y, z, w;
};
struct WinVertex {
  float x, y, z;
};

// E(a -> b, p) with the endpoints taken in a fixed (x, then y) order, so that the two triangles sharing an edge
// evaluate it with the same operations and get values of opposite sign (negation is exact)
__device__ __forceinline__ float EdgeValue(const WinVertex& a, const WinVertex& b, float px, float py) {
  const bool fwd = a.x < b.x || (a.x == b.x && a.y < b.y);
  const WinVertex& s = fwd ? a : b;
  const WinVertex& t = fwd ? b : a;
  const float e = (t.x - s.x) * (py - s.y) - (t.y - s.y) * (px - s.x);
  return fwd ? e : -e;
}

// inside test of one edge of a positively oriented triangle, top-left style tie rule for centres on the edge
__device__ __forceinline__ bool EdgeCovers(float e, const WinVertex& a, const WinVertex& b) {
  if (e > 0.0f) return true;
  if (e < 0.0f) return false;
  const float dy = b.y - a.y, dx = b.x - a.x;
  return dy > 0.0f || (dy == 0.0f && dx < 0.0f);
}

__device__ __forceinline__ ClipVertex Intersect(const ClipVertex& in, float d_in, const ClipVertex& out, float d_out) {
  const float t = d_in / (d_in - d_out);
  return {in.x + t * (out.x - in.x), in.y + t * (out.y - in.y), in.z + t * (out.z - in.z), in.w + t * (out.w - in.w)};
}

__device__ __forceinline__ WinVertex Window(const ClipVertex& c, float half_x, float half_y) {
  return {(c.x / c.w + 1.0f) * half_x, (c.y / c.w + 1.0f) * half_y, (c.z / c.w + 1.0f) * 0.5f};
}

// the pixel centre (i, j) of a positively oriented triangle of twice the area A: true and its DEPTH_COMPONENT16 value
// when it is covered and in front of the far plane
__device__ __forceinline__ bool PixelDepth(const WinVertex& v0, const WinVertex& v1, const WinVertex& v2, float A, int i,
                                           int j, unsigned& d16) {
  const float px = float(i) + 0.5f, py = float(j) + 0.5f;
  const float e0 = EdgeValue(v1, v2, px, py);
  const float e1 = EdgeValue(v2, v0, px, py);
  const float e2 = EdgeValue(v0, v1, px, py);
  if (!EdgeCovers(e0, v1, v2) || !EdgeCovers(e1, v2, v0) || !EdgeCovers(e2, v0, v1)) return false;
  const float z = (e0 * v0.z + e1 * v1.z + e2 * v2.z) / A;
  const float q = rintf(z * 65535.0f);   // DEPTH_COMPONENT16
  if (!(q < 65535.0f)) return false;     // GL_LESS against the cleared 1.0 (and beyond the far plane)
  d16 = unsigned(fmaxf(q, 0.0f));
  return true;
}

// twice the signed area, GL-style culling and orientation: false when the triangle has no fragments, else v1 and v2
// are swapped and A made positive for a negatively oriented triangle
__device__ __forceinline__ bool OrientTriangle(const WinVertex& v0, WinVertex& v1, WinVertex& v2, int culling, float& A) {
  A = (v1.x - v0.x) * (v2.y - v0.y) - (v2.x - v0.x) * (v1.y - v0.y);
  if (!(A != 0.0f)) return false;         // zero area (or NaN): no fragments
  if (culling && A > 0.0f) return false;  // glFrontFace(GL_CCW) + glCullFace(GL_FRONT)
  if (A < 0.0f) {
    const WinVertex t = v1; v1 = v2; v2 = t;
    A = -A;
  }
  return true;
}

// the pixel bounding box [i0, i0 + nx) x [j0, j0 + ny) of a triangle, clipped to the W x H image; false when empty
__device__ __forceinline__ bool PixelBox(const WinVertex& v0, const WinVertex& v1, const WinVertex& v2, int W, int H,
                                         int& i0, int& j0, int& nx, int& ny) {
  const float fW = float(W), fH = float(H);
  const float lo_x = fminf(fmaxf(ceilf(fminf(fminf(v0.x, v1.x), v2.x) - 0.5f), 0.0f), fW);
  const float hi_x = fminf(fmaxf(floorf(fmaxf(fmaxf(v0.x, v1.x), v2.x) - 0.5f), -1.0f), fW - 1.0f);
  const float lo_y = fminf(fmaxf(ceilf(fminf(fminf(v0.y, v1.y), v2.y) - 0.5f), 0.0f), fH);
  const float hi_y = fminf(fmaxf(floorf(fmaxf(fmaxf(v0.y, v1.y), v2.y) - 0.5f), -1.0f), fH - 1.0f);
  i0 = int(lo_x);
  j0 = int(lo_y);
  nx = int(hi_x) - i0 + 1;
  ny = int(hi_y) - j0 + 1;
  return nx > 0 && ny > 0;
}

// one (clipped) triangle, the 32 lanes of a warp stride over its pixel bounding box; frag(i, j, depth16) is called for
// every covered pixel centre in front of the far plane
template <class Frag>
__device__ void RasterTriangle(WinVertex v0, WinVertex v1, WinVertex v2, int culling, int W, int H, Frag& frag,
                               int lane) {
  float A;
  if (!OrientTriangle(v0, v1, v2, culling, A)) return;
  int i0, j0, nx, ny;
  if (!PixelBox(v0, v1, v2, W, H, i0, j0, nx, ny)) return;
  const int n = nx * ny;
  for (int k = lane; k < n; k += 32) {
    const int i = i0 + k % nx, j = j0 + k / nx;
    unsigned d16;
    if (PixelDepth(v0, v1, v2, A, i, j, d16)) frag(i, j, d16);
  }
}

// one geometry-frame triangle tv[9] through M = P * world2camera * geometry2world (row-major 4x4) to clip space and
// Sutherland-Hodgman against the near plane: returns the polygon's vertex count (0, 3 or 4; drawn as a fan from the
// first vertex)
__device__ __forceinline__ int ClipTriangle(const float (&M)[16], const float* tv, ClipVertex (&poly)[4]) {
  ClipVertex c[3];
  float dist[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float vx = tv[3 * k], vy = tv[3 * k + 1], vz = tv[3 * k + 2];
    c[k].x = M[0] * vx + M[1] * vy + M[2] * vz + M[3];
    c[k].y = M[4] * vx + M[5] * vy + M[6] * vz + M[7];
    c[k].z = M[8] * vx + M[9] * vy + M[10] * vz + M[11];
    c[k].w = M[12] * vx + M[13] * vy + M[14] * vz + M[15];
    dist[k] = c[k].z + c[k].w;  // near plane: z_clip >= -w_clip
  }
  int n = 0;
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    const int e1 = e == 2 ? 0 : e + 1;
    const bool in0 = dist[e] >= 0.0f, in1 = dist[e1] >= 0.0f;
    if (in0) poly[n++] = c[e];
    if (in0 != in1)  // computed from the inside vertex, so that both triangles of the edge get the same point
      poly[n++] = in0 ? Intersect(c[e], dist[e], c[e1], dist[e1]) : Intersect(c[e1], dist[e1], c[e], dist[e]);
  }
  return n;
}

// one geometry-frame triangle: ClipTriangle, window mapping onto a W x H image (half_x = W / 2, half_y = H / 2),
// rasterisation. One warp per triangle.
template <class Frag>
__device__ void DrawTriangle(const float (&M)[16], const float* tv, int culling, int W, int H, float half_x,
                             float half_y, Frag& frag, int lane) {
  ClipVertex poly[4];
  const int n = ClipTriangle(M, tv, poly);
  if (n < 3) return;
  const WinVertex w0 = Window(poly[0], half_x, half_y), w1 = Window(poly[1], half_x, half_y),
                  w2 = Window(poly[2], half_x, half_y);
  RasterTriangle(w0, w1, w2, culling, W, H, frag, lane);
  if (n == 4) RasterTriangle(w0, w2, Window(poly[3], half_x, half_y), culling, W, H, frag, lane);
}

// float -> unorm8 of the GL colour attachment: clamp to [0, 1], scale by 255, round to nearest even
__device__ __forceinline__ unsigned Unorm8(float c) { return unsigned(rintf(fminf(fmaxf(c, 0.0f), 1.0f) * 255.0f)); }

// NormalRendererCore's fragment colour (normal_renderer.cpp:11-31): vec4(0.5 - 0.5 * Rot * n, 1).zyxw for the face
// normal n and the rotation block R (row-major 3x3) of world2camera * geometry2world, as bytes in GL_BGRA read-back
// order (byte 0 encodes x)
__device__ __forceinline__ void EncodeNormal(const float* R, const float* n, unsigned b[4]) {
#pragma unroll
  for (int r = 0; r < 3; ++r) b[r] = Unorm8(0.5f - 0.5f * (R[3 * r] * n[0] + R[3 * r + 1] * n[1] + R[3 * r + 2] * n[2]));
  b[3] = 255u;
}

}  // namespace m3tb
