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

// One body of a full renderer (RendererGeometry::AddBody with body2world = I)
struct ModelBodyDev {
  const float* triangles;  // [n_triangles][3][3], geometry frame
  int n_triangles;
  int enable_culling;
};

// z-buffer key: depth16 << 48 | draw index << 32 | triangle index. The minimum is what GL_LESS keeps when the
// bodies and their triangles are drawn in order: the nearer quantised depth, then the body drawn first, then the
// triangle drawn first.
__host__ __device__ __forceinline__ uint64_t ModelKey(unsigned d16, unsigned draw, unsigned tri) {
  return (uint64_t(d16) << 48) | (uint64_t(draw) << 32) | uint64_t(tri);
}

// k_model_raster: grid (triangle chunks, views of the batch, renderers). Renderer 0 is the main FullNormalRenderer
// (the body alone), renderer 1 the occlusion FullSilhouetteRenderer (the body, then the occlusion bodies).
struct ModelRasterArgs {
  const ModelBodyDev* bodies;  // [1 + n_occlusion]: the body, then the occlusion bodies
  int n_occlusion;
  const float* M;              // [view][1 + 1 + n_occlusion][16]: renderer 0 body 0, renderer 1 bodies 0..n_occlusion
  uint64_t* zbuf;              // [view][renderer][S][S]
  int n_renderers;             // 1 (no occlusion body: the silhouette is the main coverage) or 2
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

__global__ void k_model_raster(const __grid_constant__ ModelRasterArgs a);
__global__ void k_model_points(const __grid_constant__ ModelPointArgs a);
// debug read-back of one view: normal (BGRA u8), depth (u16) and occlusion silhouette (u8) images
__global__ void k_model_images(const __grid_constant__ ModelPointArgs a, int view, uint8_t* normal, uint16_t* depth,
                               uint8_t* silhouette);

}  // namespace m3tb
