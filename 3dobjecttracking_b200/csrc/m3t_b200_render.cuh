// m3t_b200_render.cuh — focused depth / silhouette rendering on the device (FocusedRenderer::CalculateProjectionMatrix,
// FocusedBasicDepthRenderer / FocusedSilhouetteRenderer::StartRendering). The rasterisation contract is DESIGN.md §3
// "k_render"; tests/render_reference.py restates it operation for operation.
#pragma once

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
