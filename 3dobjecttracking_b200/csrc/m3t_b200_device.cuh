// m3t_b200_device.cuh — device-side data layout and math of the H100 pose-optimisation path.
//
// One CTA owns one body for a whole tracking step (all correspondence iterations x update
// iterations); warps own groups of correspondence lines / surface points, lanes own lines.
// Per-line state (RegionModality::DataLine, region_modality.h:150-165) lives in shared memory
// between CalculateCorrespondences and the n_update gradient passes. All arithmetic is float32
// with -fmad=false: every operation rounds once, in the order the reference writes it, so that
// control flow (int truncation, validity tests, branch selection) is bit-identical to a CPU
// evaluation of the same expressions (SURVEY.md App. B).
#pragma once

#include <cuda.h>  // CUtensorMap (type only; the encoder is fetched through cudaGetDriverEntryPoint)
#include <cuda_runtime.h>
#include <stdint.h>

namespace m3tb {

constexpr int kFunctionLength = 8;       // region_modality.h:415
constexpr int kDistributionLength = 12;  // region_modality.h:416
constexpr int kLineSegments = kFunctionLength + kDistributionLength - 1;  // 19, region_modality.cpp:926
constexpr int kMaxSchedule = 8;
constexpr int kTileWidths = 7;    // tile widths 64, 96, .. 256 pixels (tensor-map box widths)
constexpr int kTileBoxRows = 16;  // rows per TMA box
__host__ __device__ constexpr int TileWidth(int i) { return 64 + 32 * i; }
constexpr int kPhaseSlots = 256;

// Where bin `idx` of the colour histograms lives in the posterior lookup table (float2 per bin). A table entry is 8
// bytes, so its shared-memory bank pair is the slot's low four bits - in index order the RED bin alone, and the 32 lanes
// of a warp, looking at two colour blobs a few bins wide, land on three or four bank pairs (measured: 7.9 wavefronts
// per LDS.64 of the table, 4.9 M of the kernel's 10.7 M shared-memory wavefronts). XOR-ing the green and blue bins into
// the low bits spreads neighbouring colours over the banks. A bijection on [0, n_bins^3) for 16 and 32 bins (bits >= 4
// are untouched); every writer and reader of the table goes through it, and the bin-index images store slots.
__host__ __device__ __forceinline__ unsigned LutSlot(unsigned idx) { return idx ^ ((idx >> 4) & 15u) ^ ((idx >> 8) & 15u); }
constexpr int kBlockThreads = 256;
constexpr int kWarps = kBlockThreads / 32;

// per-line state fields (SoA, [field][line])
enum RegionField {
  RF_CBX = 0, RF_CBY, RF_CBZ, RF_CU, RF_CV, RF_NU, RF_NV, RF_DR, RF_NCTS, RF_MEAN, RF_VAR, RF_VALID,
  RF_DIST0,  // 12 values
  RF_COUNT = RF_DIST0 + kDistributionLength
};
enum DepthField { DF_CBX = 0, DF_CBY, DF_CBZ, DF_NX, DF_NY, DF_NZ, DF_YX, DF_YY, DF_YZ, DF_VALID, DF_COUNT };

// phases of k_track
enum Phase : unsigned {
  PH_REGION_CORR = 1u, PH_DEPTH_CORR = 2u, PH_REGION_GH = 4u, PH_DEPTH_GH = 8u, PH_SOLVE = 16u,
  PH_LOAD_REGION = 32u, PH_LOAD_DEPTH = 64u, PH_STORE_REGION = 128u, PH_STORE_DEPTH = 256u,
  PH_STORE_GH = 512u, PH_LOAD_GH = 1024u,
  PH_STORE_LINK_GH = 2048u,  // sum over the body's modalities -> gh_link (input of k_structure)
  PH_TEXTURE_GH = 8192u      // TextureModality::CalculateGradientAndHessian of the bodies with a texture modality
};

struct CameraDev {
  float fu, fv, ppu, ppv;
  int width, height;
  float w2c[12];
  float depth_scale;
  const uint8_t* image;  // BGR8 or U16, device copy (complete, or valid only inside each body's ROI, see FrameView)
  unsigned pitch;        // bytes
  const uint8_t* host_src;  // device-visible alias of the caller's pinned frame (zero-copy ROI ingest), or null
  unsigned host_pitch;
  int generation;        // bumped by every upload; k_ingest refreshes a body's ROI when it differs from the ROI's
  int set;
  // colour cameras in the pool: histogram BIN-INDEX image (u16 per pixel, ColorHistograms::GetProbabilities index,
  // color_histograms.cpp:97-99) written once per frame by k_bin / k_ingest; the source of k_track2's colour tiles
  uint16_t* bins;
  unsigned bin_pitch;    // bytes
};

// How one body sees one camera frame. The device copy is valid inside [x0,x1) x [y0,y1); everything else is read
// straight from the caller's pinned frame over PCIe (always correct, just slower), so the ROI is purely a transfer
// optimisation. Without a pinned source the rectangle is the whole frame.
struct FrameView {
  const uint8_t* dev;
  const uint8_t* host;
  unsigned dev_pitch, host_pitch;
  int x0, y0, x1, y1;
};
struct RoiRecord {  // per body, per camera kind
  int x0, y0, x1, y1, generation, pad0, pad1, pad2;
};

struct ModelDev {
  int n_views, n_points;
  const float4* orientations4; // [n_views] (x, y, z, 0): one 16-byte load per view in the closest-view scan
  const float* view_scalars;  // [n_views] contour_length | surface_area
  const float4* points;       // [n_views][n_points][2]: region (cx,cy,cz,nx)(ny,nz,fg,bg); depth (cx,cy,cz,nx)(ny,nz,0,0)
  float max_view_scalar;
  float radius;               // max |center_f_body| over all points: bounding sphere used for the ROI tiles
  int set;
  const float* depth_offsets; // [n_views][n_points][30]: DataPoint::depth_offsets (measured occlusion handling)
  float stride_depth_offset, max_radius_depth_offset;  // Model::stride_depth_offset / max_radius_depth_offset
  // pruned GetClosestView (m3t_b200_views.cuh): cluster bounds [n_clusters][2] and the views in cluster order
  const float4* cluster_info;
  const float4* sorted_views;
  int n_clusters;
};

struct RegionParamsDev {
  int n_lines_max, use_adaptive_coverage;
  float reference_contour_length, min_continuous_distance;
  float learning_rate;
  int n_global_iterations;
  int n_scales, scales[kMaxSchedule];
  int n_standard_deviations;
  float standard_deviations[kMaxSchedule];
  int n_bins, bitshift;
  float learning_rate_f, learning_rate_b, unconsidered_line_length, max_considered_line_length;
  float lookup_f[kFunctionLength], lookup_b[kFunctionLength];  // PrecalculateFunctionLookup
  float min_expected_variance;                                  // PrecalculateDistributionVariables
  // measured occlusion handling (region_modality.h:432-443)
  int measure_occlusions, n_unoccluded_iterations, min_n_unoccluded_lines;
  float measured_depth_offset_radius, measured_occlusion_radius, measured_occlusion_threshold;
  // checks on renderer images (region_modality.h:424-431)
  int model_occlusions, use_region_checking;
  float modeled_depth_offset_radius, modeled_occlusion_radius, modeled_occlusion_threshold;
};

struct DepthParamsDev {
  int n_points_max, use_adaptive_coverage, use_depth_scaling;
  float reference_surface_area, stride_length;
  int n_considered_distances;
  float considered_distances[kMaxSchedule];
  int n_standard_deviations;
  float standard_deviations[kMaxSchedule];
  // measured occlusion handling (depth_modality.h:313-321)
  int measure_occlusions, n_unoccluded_iterations, min_n_unoccluded_points;
  float measured_depth_offset_radius, measured_occlusion_radius, measured_occlusion_threshold;
  // checks on renderer images (depth_modality.h:305-312)
  int model_occlusions, use_silhouette_checking;
  float modeled_depth_offset_radius, modeled_occlusion_radius, modeled_occlusion_threshold;
};

// One FocusedRenderer output of one body (renderer.h:156-230), device copy: focused depth image (u16) or focused
// silhouette image (u8)
struct RenderingDev {
  const uint8_t* image;  // null: not uploaded
  int image_size;
  unsigned pitch;        // bytes
  float corner_u, corner_v, scale;
  float projection_term_a, projection_term_b;
  int id;
  int visible;
};
// The texture modality's silhouette renderer feeds two slots: its silhouette image and the focused depth image that
// Reconstruct3DPoint reads beside it (texture_modality.cpp:987-1006).
enum RenderingSlot {
  RS_REGION_DEPTH = 0, RS_REGION_SILHOUETTE, RS_DEPTH_DEPTH, RS_DEPTH_SILHOUETTE,
  RS_TEXTURE_SILHOUETTE, RS_TEXTURE_SILHOUETTE_DEPTH, RS_TEXTURE_DEPTH, RS_COUNT
};
constexpr int kNRegionStride = 5;      // region_modality.h:146
constexpr float kRegionOffset = 2.0f;  // region_modality.h:147

constexpr int kDepthOffsets = 30;        // DataPoint::depth_offsets (region_model.h:97, depth_model.h:74)
constexpr int kMaxNOcclusionStrides = 5; // region_modality.h:145, depth_modality.h:113

// Whether an occlusion window of this diameter [px] is scanned. A NaN diameter or one in (-5, 0) gives a stride of 0
// (float-to-int conversion maps NaN to 0), so the reference's scan would never end; a non-finite or negative diameter
// comes from an item behind or level with the camera or from a non-finite pose. Such a window scans nothing and counts
// as unoccluded (DESIGN.md §3).
__device__ __forceinline__ bool ScanDiameterValid(float diameter) { return diameter >= 0.0f && diameter <= 3.40282347e38f; }

// Parameters of m3t::TextureModality (texture_modality.h:400-436)
struct TextureParamsDev {
  int focused_image_size;
  float descriptor_distance_threshold, tukey_norm_constant;
  int n_standard_deviations;
  float standard_deviations[kMaxSchedule];
  float max_keyframe_rotation_difference;
  int max_keyframe_age, n_keyframes;
  int measure_occlusions;
  float measured_occlusion_radius, measured_occlusion_threshold;
  int model_occlusions;
  float modeled_occlusion_radius, modeled_occlusion_threshold;
  // descriptor_type: M3TB_DESCRIPTOR_*, whose table, row width and distance m3t_b200_texture.cuh states (TexWideRows,
  // TexRowWords, TexHamming); descriptor_length: the floats of a SIFT / DAISY descriptor, fixed by the first upload
  // after m3tb_set_texture_modality (0 before it, and for binary types)
  int descriptor_type, descriptor_length;
  // m3tb_texture_params::n_features_max: a body above kTexMaxFeatures matches ORB descriptors with
  // k_texture_knn_hamming instead of k_texture_match's in-CTA scan
  int n_features_max;
  int pad[4];  // keeps BodyDev::rend 16-byte aligned
};

struct BodyDev {
  int has_region, has_depth;
  int region_model, depth_model, color_camera, depth_camera;
  float tikhonov_rotation, tikhonov_translation;
  int first_iteration;
  int set;
  RegionParamsDev rp;
  DepthParamsDev dp;
  int has_texture, texture_camera;  // TextureModality: its colour camera
  TextureParamsDev tp;
  RenderingDev rend[RS_COUNT];
};

struct TrackArgs {
  const BodyDev* bodies;
  float* poses;                 // [n_bodies][12] body2world
  const CameraDev* color_cams;
  const CameraDev* depth_cams;
  const ModelDev* region_models;
  const ModelDev* depth_models;
  const float2* lut;            // [n_bodies][lut_stride] normalised (pf, pb) per bin
  size_t lut_stride;
  float* region_state;          // [n_bodies][RF_COUNT][line_cap]
  float* depth_state;           // [n_bodies][DF_COUNT][point_cap]
  int line_cap, point_cap;
  int* counts;                  // [n_bodies][4]: n_lines, n_points, region_view, depth_view
  float* gh_region;             // [n_bodies][27]: g[6], H lower [21]
  float* gh_depth;              // [n_bodies][27]
  float* gh_link;               // [n_bodies][27]: Link::CalculateGradientAndHessian (region + depth)
  int iteration, corr_begin, corr_end, n_update, opt_base;
  unsigned phases;
  int tile_bytes;               // dynamic shared memory available for the colour / depth ROI tiles (0: no tiling)
  RoiRecord* roi;               // [n_bodies][2]: colour, depth
  long long* phase_clock;       // optional [n_bodies][kPhaseSlots] clock64() stamps of thread 0 (profiling aid), or null
  // k_track2: TMA tensor maps over the image pools ([camera][row][column] u16), one per tile width; the box is
  // kTileBoxRows rows high. tma_ok = 0: the pools cannot be described (private images): k_track2 is not launched.
  CUtensorMap bin_maps[kTileWidths];
  CUtensorMap depth_maps[kTileWidths];
  const CUtensorMap* tmaps_global;  // the same 2 x kTileWidths maps in global memory (tma_mode 2)
  int tma_max_w;                    // widest tile (debug knob M3TB_TMA_MAXW; 256)
  int tma_mode;                     // 0: legacy staging without tensor maps, 1: maps in the kernel parameters, 2: in global memory
  // k_track2: RegionModality::PrecalculateFunctionLookup tables, identical for every region body of the launch
  // (checked by the host), so that they are kernel-parameter constants instead of per-thread registers
  float lookup_f[kFunctionLength], lookup_b[kFunctionLength];
  // texture modality (PH_TEXTURE_GH): data points [n_bodies][TF_COUNT][tex_point_cap] and their counts from
  // k_texture_match, the pose of each gradient pass (tex_pose [n_bodies][12]) and the sums (gh_texture [n_bodies][27])
  float* tex_points;
  const int* tex_counts;
  float* tex_pose;
  float* gh_texture;
  int tex_point_cap;            // kTexMaxKeyframes x the context's feature capacity (TextureArgs::cap)
};

// ---------------------------------------------------------------------------------------------
// pose helpers: float[12] row-major 3x4, same expressions as the reference's Eigen calls
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ void PoseMul(const float* a, const float* b, float* o) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j)
      o[4 * i + j] = a[4 * i + 0] * b[0 + j] + a[4 * i + 1] * b[4 + j] + a[4 * i + 2] * b[8 + j];
    o[4 * i + 3] = a[4 * i + 0] * b[3] + a[4 * i + 1] * b[7] + a[4 * i + 2] * b[11] + a[4 * i + 3];
  }
}

__device__ __forceinline__ void PoseApply(const float* p, float vx, float vy, float vz, float& x, float& y, float& z) {
  x = p[0] * vx + p[1] * vy + p[2] * vz + p[3];
  y = p[4] * vx + p[5] * vy + p[6] * vz + p[7];
  z = p[8] * vx + p[9] * vy + p[10] * vz + p[11];
}

// Transform3fA::inverse() (Affine): 3x3 cofactor inverse, translation = -inv * t  (depth_modality.cpp:644)
__host__ __device__ __forceinline__ void PoseInverse(const float* p, float* o) {
  float m[9] = {p[0], p[1], p[2], p[4], p[5], p[6], p[8], p[9], p[10]};
  float inv[9];
#define M3TB_COF(i, j) (m[3 * (((i) + 1) % 3) + (((j) + 1) % 3)] * m[3 * (((i) + 2) % 3) + (((j) + 2) % 3)] - \
                        m[3 * (((i) + 1) % 3) + (((j) + 2) % 3)] * m[3 * (((i) + 2) % 3) + (((j) + 1) % 3)])
  float c00 = M3TB_COF(0, 0), c10 = M3TB_COF(1, 0), c20 = M3TB_COF(2, 0);
  float det = c00 * m[0] + c10 * m[3] + c20 * m[6];
  float invdet = 1.0f / det;
  inv[0] = c00 * invdet; inv[1] = c10 * invdet; inv[2] = c20 * invdet;
  inv[3] = M3TB_COF(0, 1) * invdet; inv[4] = M3TB_COF(1, 1) * invdet; inv[5] = M3TB_COF(2, 1) * invdet;
  inv[6] = M3TB_COF(0, 2) * invdet; inv[7] = M3TB_COF(1, 2) * invdet; inv[8] = M3TB_COF(2, 2) * invdet;
#undef M3TB_COF
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    o[4 * i + 0] = inv[3 * i + 0]; o[4 * i + 1] = inv[3 * i + 1]; o[4 * i + 2] = inv[3 * i + 2];
    o[4 * i + 3] = (-inv[3 * i + 0]) * p[3] + (-inv[3 * i + 1]) * p[7] + (-inv[3 * i + 2]) * p[11];
  }
}

// Vector2Skewsymmetric(w).exp() in closed form (Rodrigues), row-major 3x3; the reference uses Eigen's Pade approximant
// (link.cpp:224), the two agree to < 1e-7 for |w| <= 1 (tests/test_oracle_math.py). Rigid bodies and kinematic
// structures share it.
__device__ __forceinline__ void ExpSkew(const float* w, float* r) {
  float t2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  float a, b;
  if (t2 < 0.01f) {
    // |w| < 0.1 rad (every realistic Gauss-Newton step): truncated series, remainder < 3e-14 relative
    a = 1.0f + t2 * (-1.0f / 6.0f + t2 * (1.0f / 120.0f + t2 * (-1.0f / 5040.0f)));
    b = 0.5f + t2 * (-1.0f / 24.0f + t2 * (1.0f / 720.0f + t2 * (-1.0f / 40320.0f)));
  } else {
    float t = sqrtf(t2);
    float sh = sinf(0.5f * t);
    a = sinf(t) / t;
    b = 2.0f * sh * sh / t2;
  }
  float A[9] = {0.0f, -w[2], w[1], w[2], 0.0f, -w[0], -w[1], w[0], 0.0f};
  float A2[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) A2[3 * i + j] = A[3 * i + 0] * A[0 + j] + A[3 * i + 1] * A[3 + j] + A[3 * i + 2] * A[6 + j];
#pragma unroll
  for (int k = 0; k < 9; ++k) r[k] = ((k % 4 == 0) ? 1.0f : 0.0f) + a * A[k] + b * A2[k];
}

template <typename T>
__device__ __forceinline__ T LastValid(const T* v, int n, int idx) {  // common.h:170-176
  return idx < n ? v[idx] : v[n - 1];
}

__device__ __forceinline__ int AdaptiveCount(int n_max, int use_adaptive, float reference, float view_scalar,
                                             float max_scalar, int n_model) {
  int n = n_max;  // region_modality.cpp:414-430, depth_modality.cpp:281-293
  if (use_adaptive) {
    if (reference > 0.0f)
      n = int(float(n_max) * fminf(1.0f, view_scalar / reference));
    else
      n = int(float(n_max) * view_scalar / max_scalar);
  }
  if (n > n_model) n = n_model;
  return n;
}

}  // namespace m3tb
