// m3t_b200_raster.cuh — the triangle walk shared by k_render (focused renderers, shared-memory z-buffer) and
// k_model_raster (full-frame model-generation renderers, global-memory z-buffer): transform to clip space, near-plane
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

__device__ __forceinline__ WinVertex Window(const ClipVertex& c, float half) {
  return {(c.x / c.w + 1.0f) * half, (c.y / c.w + 1.0f) * half, (c.z / c.w + 1.0f) * 0.5f};
}

// one (clipped) triangle, the 32 lanes of a warp stride over its pixel bounding box; frag(i, j, depth16) is called for
// every covered pixel centre in front of the far plane
template <class Frag>
__device__ void RasterTriangle(WinVertex v0, WinVertex v1, WinVertex v2, int culling, int S, Frag& frag, int lane) {
  float A = (v1.x - v0.x) * (v2.y - v0.y) - (v2.x - v0.x) * (v1.y - v0.y);
  if (!(A != 0.0f)) return;             // zero area (or NaN): no fragments
  if (culling && A > 0.0f) return;      // glFrontFace(GL_CCW) + glCullFace(GL_FRONT)
  if (A < 0.0f) {
    const WinVertex t = v1; v1 = v2; v2 = t;
    A = -A;
  }
  const float fS = float(S);
  const float lo_x = fminf(fmaxf(ceilf(fminf(fminf(v0.x, v1.x), v2.x) - 0.5f), 0.0f), fS);
  const float hi_x = fminf(fmaxf(floorf(fmaxf(fmaxf(v0.x, v1.x), v2.x) - 0.5f), -1.0f), fS - 1.0f);
  const float lo_y = fminf(fmaxf(ceilf(fminf(fminf(v0.y, v1.y), v2.y) - 0.5f), 0.0f), fS);
  const float hi_y = fminf(fmaxf(floorf(fmaxf(fmaxf(v0.y, v1.y), v2.y) - 0.5f), -1.0f), fS - 1.0f);
  const int i0 = int(lo_x), j0 = int(lo_y);
  const int nx = int(hi_x) - i0 + 1, ny = int(hi_y) - j0 + 1;
  if (nx <= 0 || ny <= 0) return;
  const int n = nx * ny;
  for (int k = lane; k < n; k += 32) {
    const int i = i0 + k % nx, j = j0 + k / nx;
    const float px = float(i) + 0.5f, py = float(j) + 0.5f;
    const float e0 = EdgeValue(v1, v2, px, py);
    const float e1 = EdgeValue(v2, v0, px, py);
    const float e2 = EdgeValue(v0, v1, px, py);
    if (!EdgeCovers(e0, v1, v2) || !EdgeCovers(e1, v2, v0) || !EdgeCovers(e2, v0, v1)) continue;
    const float z = (e0 * v0.z + e1 * v1.z + e2 * v2.z) / A;
    const float q = rintf(z * 65535.0f);   // DEPTH_COMPONENT16
    if (!(q < 65535.0f)) continue;         // GL_LESS against the cleared 1.0 (and beyond the far plane)
    frag(i, j, unsigned(fmaxf(q, 0.0f)));
  }
}

// one geometry-frame triangle tv[9] through M = P * world2camera * geometry2world (row-major 4x4): clip-space
// transform, Sutherland-Hodgman against the near plane (0, 3 or 4 vertices, fanned from the first), window mapping,
// rasterisation. One warp per triangle.
template <class Frag>
__device__ void DrawTriangle(const float (&M)[16], const float* tv, int culling, int S, float half, Frag& frag, int lane) {
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
  ClipVertex poly[4];
  int n = 0;
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    const int e1 = e == 2 ? 0 : e + 1;
    const bool in0 = dist[e] >= 0.0f, in1 = dist[e1] >= 0.0f;
    if (in0) poly[n++] = c[e];
    if (in0 != in1)  // computed from the inside vertex, so that both triangles of the edge get the same point
      poly[n++] = in0 ? Intersect(c[e], dist[e], c[e1], dist[e1]) : Intersect(c[e1], dist[e1], c[e], dist[e]);
  }
  if (n < 3) return;
  const WinVertex w0 = Window(poly[0], half), w1 = Window(poly[1], half), w2 = Window(poly[2], half);
  RasterTriangle(w0, w1, w2, culling, S, frag, lane);
  if (n == 4) RasterTriangle(w0, w2, Window(poly[3], half), culling, S, frag, lane);
}

}  // namespace m3tb
