// m3t_b200_render.cuh — focused depth / silhouette rendering on the device (FocusedRenderer::CalculateProjectionMatrix,
// FocusedBasicDepthRenderer / FocusedSilhouetteRenderer::StartRendering). The rasterisation contract is DESIGN.md §3
// "k_render"; tests/render_reference.py restates it operation for operation.
#pragma once

#include <cfloat>

#include "m3t_b200_device.cuh"

namespace m3tb {

constexpr int kRenderThreads = 512;
// the z-buffer (u32 per pixel) lives in shared memory: 240 x 240 x 4 B = 225 KB of the 227 KB a CTA may use
constexpr int kRenderMaxImageSize = 240;

// Body geometry as RendererGeometry::AddBody uploads it (body.cpp:201-249 already applied by the caller)
struct GeometryDev {
  const float* triangles;  // [n_triangles][3][3], metres, geometry frame
  int n_triangles;
  float geometry2body[12];
  float radius;            // 0.5f * Body::maximum_body_diameter()
  int enable_culling;
  int body_id, region_id;  // Body::body_id() / region_id() (uint8)
  int set;
};

enum RenderIdType { RID_BODY = 0, RID_REGION = 1 };

// One focused renderer (FocusedRenderer, renderer.h:156-230): draws geometry_bodies, focuses on referenced_bodies
struct RendererDev {
  int camera_kind;         // 0 colour, 1 depth
  int camera;
  int image_size;
  int id_type;             // RenderIdType
  float z_min, z_max;
  int first_geometry, n_geometry;      // range of RenderArgs::geometry_bodies
  int first_referenced, n_referenced;  // range of RenderArgs::referenced_bodies / visible
  uint16_t* depth;         // focused depth image, u16
  uint8_t* silhouette;     // focused silhouette image, u8 id (0 = background)
  unsigned depth_pitch, silhouette_pitch;  // bytes
  int set;
};

// What StartRendering leaves besides the images (renderer.h:195-197, FocusedDepthRenderer::projection_term_a/b)
struct RenderOutDev {
  float corner_u, corner_v, scale;
  float projection_term_a, projection_term_b;
};

// A body's renderer slot fed by a device renderer (RegionModality / DepthModality::ModelOcclusions, UseRegionChecking,
// UseSilhouetteChecking)
struct RenderAttachDev {
  int body, slot, renderer, referenced_index;
};

// FocusedRenderer::CalculateProjectionMatrix (renderer.cpp:348-405) and CalculateProjectionTerms (:567-570) of an
// S x S renderer of camera `cam` with z range [z_min, z_max]: body(k, r, pose) gives the radius and body2world pose of
// referenced body k. Writes one FocusedRenderer::IsBodyVisible flag per referenced body, the focus `o` and the
// projection P = (P00, P02, P11, P12, P22, P23). False when no referenced body is visible: the matrix is then not
// finite, nothing is drawn and the images stay cleared. Used by k_render and k_view_focus.
template <class Body>
__device__ __forceinline__ bool FocusProjection(const CameraDev& cam, int S, float z_min, float z_max, int n_referenced,
                                                Body body, int* visible, RenderOutDev& o, float* P) {
  const float* w = cam.w2c;
  float u_min = FLT_MAX, u_max = FLT_MIN, v_min = FLT_MAX, v_max = FLT_MIN;  // numeric_limits<float>::min() as written
  bool any = false;
  for (int k = 0; k < n_referenced; ++k) {
    int vis = 0;
    float rr;
    const float* p;
    body(k, rr, p);
    const float x = w[0] * p[3] + w[1] * p[7] + w[2] * p[11] + w[3];
    const float y = w[4] * p[3] + w[5] * p[7] + w[6] * p[11] + w[7];
    const float z = w[8] * p[3] + w[9] * p[7] + w[10] * p[11] + w[11];
    if (!(z < rr * 1.5f || z - rr < z_min || z + rr > z_max)) {
      const float abs_x = fabsf(x), abs_y = fabsf(y);
      const float x2 = x * x, y2 = y * y, z2 = z * z, r2 = rr * rr, rz = rr * z;
      const float z2_r2 = z2 - r2;
      const float z3_zr2 = z2_r2 * z;
      const float r_u = cam.fu * (abs_x * r2 + rz * sqrtf(z2_r2 + x2)) / z3_zr2;
      const float r_v = cam.fv * (abs_y * r2 + rz * sqrtf(z2_r2 + y2)) / z3_zr2;
      const float center_u = x * cam.fu / z + cam.ppu;
      const float center_v = y * cam.fv / z + cam.ppv;
      const float u_min_body = center_u - r_u, u_max_body = center_u + r_u;
      const float v_min_body = center_v - r_v, v_max_body = center_v + r_v;
      if (!(u_min_body > float(cam.width) || u_max_body < 0.0f || v_min_body > float(cam.height) || v_max_body < 0.0f)) {
        u_min = u_min_body < u_min ? u_min_body : u_min;  // std::min(a, b) = b < a ? b : a
        u_max = u_max < u_max_body ? u_max_body : u_max;  // std::max(a, b) = a < b ? b : a
        v_min = v_min_body < v_min ? v_min_body : v_min;
        v_max = v_max < v_max_body ? v_max_body : v_max;
        vis = 1;
        any = true;
      }
    }
    visible[k] = vis;
  }
  const float du = u_max - u_min, dv = v_max - v_min;
  const float d = (du < dv ? dv : du) * 1.05f;  // kImageSizeSafetyMargin
  o.corner_u = 0.5f * (u_min + u_max - d);
  o.corner_v = 0.5f * (v_min + v_max - d);
  o.scale = float(S) / d;
  o.projection_term_a = z_max * z_min * 65535.0f / (z_max - z_min);  // renderer.cpp:567-570
  o.projection_term_b = z_max * 65535.0f / (z_max - z_min);
  const float ppu_scaled = (cam.ppu - o.corner_u) * o.scale;
  const float ppv_scaled = (cam.ppv - o.corner_v) * o.scale;
  P[0] = 2.0f * cam.fu / d;
  P[1] = 2.0f * (ppu_scaled + 0.5f) / float(S) - 1.0f;
  P[2] = 2.0f * cam.fv / d;
  P[3] = 2.0f * (ppv_scaled + 0.5f) / float(S) - 1.0f;
  P[4] = (z_max + z_min) / (z_max - z_min);
  P[5] = -2.0f * z_max * z_min / (z_max - z_min);
  return any;
}

struct RenderArgs {
  const RendererDev* renderers;
  const int* render_list;      // [gridDim.x] renderer of each CTA
  const GeometryDev* geometry; // [max_bodies]
  const int* geometry_bodies;
  const int* referenced_bodies;
  const float* poses;          // body2world [max_bodies][12]
  const CameraDev* color_cams;
  const CameraDev* depth_cams;
  RenderOutDev* out;           // [n_renderers]
  int* visible;                // parallel to referenced_bodies: FocusedRenderer::IsBodyVisible
  BodyDev* bodies;             // renderer-image records of attached slots are written here
  const RenderAttachDev* attach;
  int n_attach;
};

__global__ void k_render(const __grid_constant__ RenderArgs a);

}  // namespace m3tb
