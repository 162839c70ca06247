// m3t_b200_model.cuh — depth sparse-viewpoint-model generation on the device (DepthModel::GenerateModel,
// depth_model.cpp:144-213,302-351, Model::CalculateDepthOffsets, model.cpp:338-384). DESIGN.md §3 "k_model_raster /
// k_model_points" states the contract; tests/model_generation_reference.py restates it.
#pragma once

#include <stdint.h>

#include <cuda_runtime.h>

namespace m3tb {

constexpr int kModelThreads = 256;
constexpr int kModelMaxOffsets = 30;               // Model::kMaxNDepthOffsets
constexpr int kModelTrianglesPerCta = 64;          // k_model_raster: triangles one CTA walks per body
constexpr uint64_t kModelClear = ~uint64_t(0);     // glClear: depth 1.0, no triangle
// upper bound of the z-buffer scratch of one generation call; the view batch is sized to stay below it
constexpr size_t kModelScratchBytes = size_t(1) << 30;

constexpr int kModelMaxRenderers = 5;              // region: main, same-region, occlusion, foreground, background

// One draw of a full renderer (RendererGeometry::AddBody with body2world = I): a body and its silhouette id
struct ModelBodyDev {
  const float* triangles;  // [n_triangles][3][3], geometry frame
  int n_triangles;
  int enable_culling;
  int id;                  // silhouette value where this draw wins (BodyID: 0, 120 or 255)
};

// z-buffer key: depth16 << 48 | draw index << 32 | triangle index. The minimum is what GL_LESS keeps when the
// bodies and their triangles are drawn in order: the nearer quantised depth, then the body drawn first, then the
// triangle drawn first.
__host__ __device__ __forceinline__ uint64_t ModelKey(unsigned d16, unsigned draw, unsigned tri) {
  return (uint64_t(d16) << 48) | (uint64_t(draw) << 32) | uint64_t(tri);
}

// The renderer table of one generation: renderer r draws draws[first[r] .. first[r + 1]) in that order, each with
// its own clip-space matrix (the renderer's z range is widened over its bodies). Depth models: renderer 0 is the main
// FullNormalRenderer (the body alone), renderer 1 the occlusion FullSilhouetteRenderer (the body, then the occlusion
// bodies). Region models: main (body 255, fixed bodies 120), then same-region, occlusion, foreground, background.
struct ModelRenderers {
  const ModelBodyDev* draws;   // [n_draws]
  int first[kModelMaxRenderers + 1];
  int n_renderers;
};

// silhouette value of a z-buffer key of renderer r: the id of the winning draw, 0 where nothing was drawn
__device__ __forceinline__ unsigned SilhouetteId(const ModelRenderers& R, int r, uint64_t key) {
  return key == kModelClear ? 0u : unsigned(R.draws[R.first[r] + int((key >> 32) & 0xffffu)].id);
}

// k_model_raster: grid (triangle chunks, views of the batch, renderers)
struct ModelRasterArgs {
  ModelRenderers R;
  int n_draws;                 // first[n_renderers]
  const float* M;              // [view][n_draws][16]
  uint64_t* zbuf;              // [view][renderer][S][S]
  int image_size;
};

// k_model_points: one CTA per view of the batch
struct ModelPointArgs {
  const uint64_t* zbuf;        // as in ModelRasterArgs
  int n_renderers;
  int image_size;
  const float* face_normals;   // [n_triangles][3] of the body, geometry frame (RendererGeometry::AssembleVertexData)
  const float* rot;            // [view][9] linear block of world2camera * geometry2world (main renderer)
  const float* camera2body;    // [view][12]
  float fu, ppu, ppv, fv;
  float projection_term_a, projection_term_b;  // main renderer
  float sphere_radius, stride_depth_offset;
  int n_values;                // int(max_radius_depth_offset / stride_depth_offset + 1.0f) <= kModelMaxOffsets
  int n_points;
  unsigned seed;               // std::mt19937 seed of every view (7)
  int* coords;                 // scratch [view][n_points] sampled pixel (row * S + column)
  float* points;               // [view][n_points][36] DataPoints of the batch
  float* surface_area;         // [view]
};

// k_region_contours / k_region_points: region-model generation, one CTA per view of the batch (DESIGN.md §3
// "k_region_contours / k_region_points"; tests/region_model_generation_reference.py restates it)
constexpr int kRegionMinContourLength = 15;        // RegionModel::kMinContourLength
constexpr int kRegionNormalApproxRadius = 3;       // RegionModel::kContourNormalApproxRadius
constexpr int kRegionMaxSamplingTries = 100;       // RegionModel::kMaxPointSamplingTries
constexpr float kRegionMaxSurfaceGradient = 10.0f; // RegionModel::kMaxSurfaceGradient
constexpr int kRegionContourCapPerPixel = 64;      // contour points one view may hold: 64 * image_size
constexpr int kRegionPointFloats = 38;             // RegionModel::DataPoint, 152 B

struct RegionContourArgs {
  const uint64_t* zbuf;        // [view][renderer][S][S]; renderer 0 is the main renderer
  ModelRenderers R;
  int image_size;
  int8_t* label;               // scratch [view][(S + 2)^2]: the zero-padded mask, then Suzuki's marks
  uint32_t* raw;               // scratch [view][cap]: kept contours in discovery order, x | y << 16
  int* raw_start;              // scratch [view][cap / 15 + 2]
  uint32_t* contour;           // [view][cap]: kept contours in cv::findContours order
  int* contour_start;          // [view][cap / 15 + 2]: offsets of the contours in `contour`, n_contours + 1 entries
  int* counts;                 // [view][2]: n_contours, n_contour_points
  int cap;
  int* overflow;               // set to 1 when a view's contours do not fit in cap points (the call then fails)
};

struct RegionPointArgs {
  const uint64_t* zbuf;
  ModelRenderers R;
  int r_same, r_occ, r_fg, r_bg;  // renderer indices, -1 when not used
  int image_size;
  const uint32_t* contour;
  const int* contour_start;
  const int* counts;
  int cap;
  uint32_t* valid;             // scratch [view][cap]: valid contour points in contour order
  int* coords;                 // scratch [view][n_points]: sampled centres (row * S + column)
  float* normals;              // scratch [view][n_points][2]
  const float* camera2body;    // [view][12]
  float fu, ppu, ppv, fv;
  float projection_term_a, projection_term_b;  // main renderer
  float sphere_radius, stride_depth_offset;
  int n_values;
  int n_points;
  unsigned seed;
  float* points;               // [view][n_points][38]
  float* contour_length;       // [view]
};

__global__ void k_model_raster(const __grid_constant__ ModelRasterArgs a);
__global__ void k_region_contours(const __grid_constant__ RegionContourArgs a);
__global__ void k_region_points(const __grid_constant__ RegionPointArgs a);
// debug read-back of one view: the silhouette of every renderer and the main depth image
__global__ void k_region_images(const uint64_t* zbuf, ModelRenderers R, int image_size, uint8_t* silhouettes,
                                uint16_t* depth);
__global__ void k_model_points(const __grid_constant__ ModelPointArgs a);
// debug read-back of one view: normal (BGRA u8), depth (u16) and occlusion silhouette (u8) images
__global__ void k_model_images(const __grid_constant__ ModelPointArgs a, int view, uint8_t* normal, uint16_t* depth,
                               uint8_t* silhouette);

}  // namespace m3tb
