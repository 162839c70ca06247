// m3t_b200_view.cuh — NormalColorViewer / NormalDepthViewer on the device (normal_viewer.cpp, normal_renderer.cpp):
// every viewer's FullNormalRenderer draws its geometry bodies over the whole camera image (W x H) into a global-memory
// z-buffer, and the normal image is alpha-blended over the camera frame. DESIGN.md §3 "k_view_setup / k_view_raster /
// k_view_resolve" states the contract; tests/viewer_reference.py restates it.
#pragma once

#include <stdint.h>

#include <cuda_runtime.h>

#include "m3t_b200_render.cuh"

namespace m3tb {

constexpr int kViewThreads = 256;
constexpr int kViewTile = 32;                  // k_view_raster: one warp per (triangle, 32 x 32 screen tile)
constexpr uint64_t kViewClear = ~uint64_t(0);  // glClear: depth 1.0, no triangle
constexpr int kViewFanShift = 40;              // allocation counter of k_view_setup: triangles << 40 | tiles
constexpr uint64_t kViewTileMask = (uint64_t(1) << kViewFanShift) - 1;
// m3tb_set_focused_normal_renderer: the z-buffer of an S x S renderer is S * S * 8 bytes of global memory
constexpr int kFocusedNormalMaxImageSize = 4096;

// VK_FULL: a full renderer (m3tb_set_full_renderer: FullBasicDepthRenderer / FullSilhouetteRenderer /
// FullNormalRenderer), whose resolve writes depth, silhouette and normal images and blends nothing. VK_FOCUSED: a
// focused normal renderer (m3tb_set_focused_normal_renderer: FocusedNormalRenderer), S x S, whose projection
// k_view_focus sets from the current poses and whose resolve writes the depth and normal images.
enum ViewerKind { VK_COLOR = 0, VK_DEPTH = 1, VK_FULL = 2, VK_FOCUSED = 3 };

// One viewer (or full renderer) of an update: its renderer's projection, the camera frame it blends over and its images
struct ViewerDev {
  int width, height;
  int kind;                    // ViewerKind
  float P00, P02, P11, P12, P22, P23;  // FullRenderer::CalculateProjectionMatrix (renderer.cpp:257-264)
  float w2c[12];               // the camera's world2camera pose
  const uint8_t* frame;        // BGR8 or u16 frame: the device copy, or the device-visible alias of a pinned frame
  unsigned frame_pitch;        // bytes
  float opacity;
  float depth_alpha, depth_beta;  // DepthCamera::NormalizedDepthImage: convertTo scale and shift
  uint64_t* zbuf;              // [H][W] depth16 << 48 | draw << 32 | triangle; kViewClear between updates
  uint8_t* normal;             // [H][W][4] FullNormalRenderer::normal_image() (GL_BGRA read-back order)
  uint8_t* image;              // [H][W][3] the blended BGR8 viewer image
  uint16_t* depth;             // VK_FULL, VK_FOCUSED: [H][W] depth image (DEPTH_COMPONENT16, 65535 = clear)
  uint8_t* silhouette;         // VK_FULL: [H][W] FullSilhouetteRenderer::silhouette_image() (0 = background)
  int first_draw, n_draws;     // the viewer's bodies in ViewArgs::draws, in draw order
};

// One body drawn by one viewer (RendererGeometry::render_data_bodies)
struct ViewDrawDev {
  const float* triangles;      // [n_triangles][3][3], geometry frame
  int n_triangles;
  int enable_culling;
  int viewer;
  int draw;                    // index among the viewer's draws (the z-buffer key's draw field)
  int body;                    // index of the body2world pose
  int silhouette_id;           // VK_FULL: Body::body_id() or region_id() by the renderer's id type
  float geometry2body[12];
};

// One triangle of the fan of a clipped polygon, oriented and boxed (OrientTriangle, PixelBox), tagged with its key
struct ViewFanDev {
  float v[9];                  // window-space v0, v1, v2 (x, y, z) after orientation
  float A;
  int i0, j0, nx, ny;
  int viewer;
  uint64_t tag;                // draw << 32 | triangle
};

// One focused normal renderer of a render (FocusedRenderer::CalculateProjectionMatrix): its camera, size, z range and
// referenced bodies
struct FocusDev {
  CameraDev cam;               // intrinsics and world2camera
  int image_size;
  float z_min, z_max;
  int viewer;                  // its slot in ViewArgs::viewers
  int first_referenced, n_referenced;  // range of FocusArgs::referenced / radius / visible
};

struct FocusArgs {
  const FocusDev* focus;
  int n_focus;
  const int* referenced;       // body index of every referenced body
  const float* radius;         // 0.5f * Body::maximum_body_diameter() of each
  const float* poses;          // [body][12] body2world
  int* visible;                // parallel to referenced: FocusedRenderer::IsBodyVisible
  RenderOutDev* out;           // [n_focus] corner, scale, projection terms
  ViewerDev* viewers;          // the projections are written here
  ViewDrawDev* draws;          // a renderer that sees no referenced body draws nothing: its draws get no triangles
};

// NormalizedDepthImage of a depth camera's frame (DepthCamera, camera.cpp:108-115) or of a full renderer's depth image
// (FullDepthRenderer, renderer.cpp:407-427) into a W x H u8 image
struct NormalizedDepthArgs {
  const uint8_t* src;          // u16 rows, src_pitch bytes apart
  unsigned src_pitch;
  int width, height;
  int renderer;                // 0: camera frame (alpha, beta), 1: full renderer (a, b, min_depth, delta, scale)
  float alpha, beta;           // convertTo scale and shift
  float a, b, min_depth, delta, scale;  // projection terms, max_depth - min_depth, 255 / delta
  uint8_t* dst;
  size_t dst_pitch;
};

struct ViewArgs {
  const ViewerDev* viewers;
  int n_viewers;
  const ViewDrawDev* draws;
  int n_draws;
  const float* poses;          // [body][12] body2world
  float* rot;                  // [n_draws][9] rotation block of world2camera * geometry2world (k_view_setup)
  ViewFanDev* fans;            // [fan_cap], in allocation order
  uint64_t* fan_tile;          // [fan_cap] index of each fan's first (triangle, tile) work item
  int fan_cap;                 // 2 x the triangles of all draws: the fan of a clipped triangle has at most two
  unsigned long long* counter; // fans << kViewFanShift | tiles; 0 between updates
};

// one thread per focused normal renderer, before k_view_setup: FocusProjection from the current poses into its slot
__global__ void k_view_focus(const __grid_constant__ FocusArgs a);
// grid (triangle blocks, draws): transform, near-plane clipping, window mapping, culling and bounding box of every
// triangle; each fan triangle takes a slot and a range of work items, one per 32 x 32 tile its box touches
__global__ void k_view_setup(const __grid_constant__ ViewArgs a);
// persistent warps over the work items of k_view_setup: the covered pixels of one tile of one triangle, atomicMin
// into the viewer's z-buffer
__global__ void k_view_raster(const __grid_constant__ ViewArgs a);
// grid (pixel blocks, viewers): normal image, frame pixel (or normalised depth), alpha blend; for VK_FULL the depth,
// silhouette and normal images instead (VK_FOCUSED: depth and normal). Clears the z-buffer and the counter for the next
// update.
__global__ void k_view_resolve(const __grid_constant__ ViewArgs a);
// grid (pixel blocks): one NormalizedDepthImage
__global__ void k_normalized_depth(const __grid_constant__ NormalizedDepthArgs a);

}  // namespace m3tb
