// m3t_b200.cu — host side of libm3t_b200.so: context, device memory, launches; implements include/m3t_b200.h.
// No CPU fallback anywhere: if CUDA is unusable every compute entry point returns M3TB_ERR_CUDA.
#include "m3t_b200.h"

#include <cudaTypedefs.h>  // PFN_cuTensorMapEncodeTiled

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <array>
#include <set>
#include <cstring>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include "m3t_b200_owned.h"
#include "m3t_b200_model.cuh"
#include "m3t_b200_render.cuh"
#include "m3t_b200_structures.cuh"
#include "m3t_b200_kernels.cuh"
#include "m3t_b200_views.cuh"
#include "m3t_b200_view.cuh"
#include "m3t_b200_undistort.cuh"
#include "m3t_b200_texture.cuh"
#include "m3t_b200_score.cuh"

#include "m3t_b200_track_variants.h"
#include "m3t_b200_track2.cuh"

namespace m3tb {
extern template __global__ void k_track2<512, true>(const __grid_constant__ TrackArgs);
extern template __global__ void k_track2<512, false>(const __grid_constant__ TrackArgs);
extern template __global__ void k_track2<1024, true>(const __grid_constant__ TrackArgs);
extern template __global__ void k_track2<1024, false>(const __grid_constant__ TrackArgs);
// the fused kernel's variants are compiled in m3t_b200_track_<g>.cu
#define M3TB_DECLARE(T_, K_, L_, O_) extern template __global__ void k_track<T_, K_, L_, O_>(const __grid_constant__ TrackArgs);
M3TB_TRACK_ALL(M3TB_DECLARE)
#undef M3TB_DECLARE
}  // namespace m3tb

using namespace m3tb;

namespace {

struct ImagePool {
  DeviceBuffer<uint8_t> base;
  size_t frame_bytes = 0;
  unsigned pitch = 0;
  int width = 0, height = 0, capacity = 0;
  // colour pools: the bin-index images (u16 per pixel), same slot order
  DeviceBuffer<uint8_t> bins;
  size_t bin_frame_bytes = 0;
  unsigned bin_pitch = 0;

  uint16_t* BinImage(int slot) const { return reinterpret_cast<uint16_t*>(bins.get() + bin_frame_bytes * slot); }
};

// what a colour camera's bin-index image holds besides a bit shift (m3tb_ctx::bin_shift)
constexpr int kBinsNone = -1;      // nothing that matches the frame copy
constexpr int kBinsAtIngest = -2;  // a pinned frame whose bin indices the next k_ingest writes

// TMA tensor maps over one pool ([camera][row][column] u16), one per tile width; cached per pool base address
struct PoolMaps {
  const void* base = nullptr;
  bool ok = false;
  CUtensorMap maps[kTileWidths];
};

// One m3t::Optimizer with more than a single free root link (host image; flattened into the device tables on demand)
struct StructureHost {
  std::vector<LinkDev> links;
  std::vector<LinkDev> default_links;  // Link::default_body2joint_pose_ / default_joint2parent_pose_: as handed to m3tb_set_structure
  std::vector<ConstraintDev> constraints;
  float tikhonov_rotation = 1000.0f, tikhonov_translation = 30000.0f;
  bool set = false;
};

struct ModelAlloc {
  DeviceBuffer<float4> orientations;
  DeviceBuffer<float> view_scalars, points, depth_offsets, cluster_info, sorted_views;
};

// Made by the first m3tb_prefetch_frames
struct PrefetchResources {
  Stream ingest_stream;
  Stream table_stream;  // camera tables + counter reset of a prefetch: beside the ingest in flight, not behind it
  PinnedBuffer<CameraDev> cam_stage[2][2];  // pinned staging [parity][colour | depth]
  Event ev_ingest_done, ev_poses_snap, ev_tables;
  Event ev_stage[2];  // the table copies out of cam_stage[parity] have run
  DeviceBuffer<CameraDev> ccams_alt, dcams_alt;  // second set of camera tables / ROI records
  DeviceBuffer<RoiRecord> roi_alt;
  DeviceBuffer<float> poses_snap[2];  // poses at the start of the last two tracking launches (snap_parity)
};

// which device renderers one k_render launch draws
enum RenderList { kRenderAll = 0, kRenderAttached, kRenderRegion, kRenderLists };

// What one m3tb_refine_poses launches on: lists in m3tb_ctx::d_refine and their lengths. m3tb_ctx::refine points at it
// while the refinement runs and is null otherwise, so every other entry point launches over the whole context.
struct RefineSelection {
  const int* bodies = nullptr;          // k_histogram, k_ingest: the refined bodies with the bodies of the
  int n_bodies = 0;                     //   refined structures (links and extra bodies)
  const int* structures = nullptr;      // k_structure: the refined structures and the implicit one-link structures of
  int n_structures = 0;                 //   the refined rigid bodies (contexts with kinematic structures only)
  const int* renderers[kRenderLists] = {};  // k_render: the renderers attached to the refined bodies (kRenderAttached:
  int n_renderers[kRenderLists] = {};       //   every slot that feeds correspondences, kRenderRegion: the region slots)
  size_t render_smem[kRenderLists] = {};
  std::vector<int> renderer_ids[kRenderLists];  // host copies
  const int* hist_groups = nullptr;     // shared ColorHistograms objects with a refined member:
  int n_hist_groups = 0;                //   owner[n] | first[n + 1] | summed[n] | members (refined ones first)
  bool ingested = false;                // k_ingest ran for the refined bodies
  std::vector<std::pair<int, int>> runs;  // k_track: (first body, count) of each run of consecutive refined bodies
  const int* texture = nullptr;         // k_texture_keyframe / _match / _knn_*: the refined texture bodies
  int n_texture = 0;                    //   (m3tb_refine_poses_orb only)
  std::vector<int> texture_ids;         // host copy
};

}  // namespace

struct m3tb_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  int max_bodies = 0, max_cameras = 0, max_models = 0;
  int n_bodies = 0;
  std::string err;
  int64_t launches = 0;

  std::vector<BodyDev> h_bodies;
  std::vector<CameraDev> h_ccams, h_dcams;
  std::vector<ModelDev> h_rmodels, h_dmodels;
  std::vector<ModelAlloc> rmodel_alloc, dmodel_alloc;
  std::vector<DeviceBuffer<uint8_t>> private_color, private_depth;  // images that do not fit the pools
  bool bodies_dirty = true, cams_dirty = true, models_dirty = true;

  DeviceBuffer<BodyDev> d_bodies;
  DeviceBuffer<CameraDev> d_ccams, d_dcams;
  DeviceBuffer<ModelDev> d_rmodels, d_dmodels;
  DeviceBuffer<float> d_poses;
  ImagePool color_pool, depth_pool;

  DeviceBuffer<float> d_hist_f, d_hist_b, d_mem_f, d_mem_b;
  DeviceBuffer<float2> d_lut;
  size_t hist_stride = 0;

  DeviceBuffer<float> d_rstate, d_dstate;
  int line_cap = 0, point_cap = 0;
  DeviceBuffer<int> d_counts;
  DeviceBuffer<float> d_gh_region, d_gh_depth;
  size_t max_dyn_smem = 0;
  DeviceBuffer<RoiRecord> d_roi;          // [max_bodies][2]
  DeviceBuffer<unsigned long long> d_ingest_bytes;  // [2]: one counter per ingest launch in flight
  int ingest_bytes_slot = 0;              // the counter of the last ingest launch
  int sm_count = 132;
  bool ingest_pending = false;            // a pinned frame was handed over since the last k_ingest launch
  // frame prefetch (m3tb_prefetch_frames): second set of image pools / camera tables / ROI records, side stream
  ImagePool color_pool_alt, depth_pool_alt;
  PrefetchResources pf;
  int snap_parity = 0;  // pf.poses_snap[snap_parity] is what the next prefetch projects with, the other one may still be
                        //   read by the ingest in flight
  int stage_parity = 0;
  bool prefetch_enabled = false;          // set by the first m3tb_prefetch_frames
  bool prefetched = false;                // the next consumer launch has to wait for ev_ingest_done
  bool poses_snap_valid = false;
  bool roi_ingest = true;                 // M3TB_NO_ROI_INGEST=1 forces full-frame copies
  DeviceBuffer<long long> d_phase_clock;  // allocated when M3TB_TIMING=1
  bool use_tiles = true;  // stage ROI tiles in shared memory (M3TB_NO_TILES=1 in the environment disables it)
  bool use_track2 = true; // second-generation fused kernel where it applies (M3TB_KERNEL=1 forces k_track)
  m3tb_launch_info last_launch = {};      // variant of the last tracking launch (m3tb_debug_last_launch)
  // per colour camera: the histogram bit shift its bin-index image was written with, kBinsNone when it holds none that
  // matches the frame copy, kBinsAtIngest while a pinned frame waits for the k_ingest that writes them (NoteIngestBins)
  std::vector<int> bin_shift;
  DeviceBuffer<int> d_bin_ids;            // staging for k_bin
  // device copies of the renderer images (m3tb_upload_*_rendering), per body and renderer slot
  std::vector<std::array<DeviceBuffer<uint8_t>, RS_COUNT>> rendering_images;
  std::vector<PoolMaps> pool_maps;        // tensor maps of the pools seen so far (current / alternate x bins / depth)
  int tma_mode = 1;                       // M3TB_TMA: 0 legacy staging, 1 tensor maps in the kernel parameters, 2 in global memory
  DeviceBuffer<CUtensorMap> d_tmaps;      // tma_mode 2: [2][kTileWidths]
  const void* d_tmaps_bases[2] = {nullptr, nullptr};  // the pools d_tmaps currently describes

  // kinematic structures (empty: every body is its own rigid-body optimiser inside k_track)
  // shared ColorHistograms objects (m3tb_share_color_histograms): per body the owner of the object it uses, -1 = its own
  std::vector<int> hist_owner;
  std::vector<int> hist_table_uploaded;  // what d_hist_owner / d_hist_groups hold
  int n_hist_groups = 0;
  DeviceBuffer<int> d_hist_owner;  // [max_bodies]
  DeviceBuffer<int> d_hist_groups; // group_owner[n] | group_first[n + 1] | members[...]
  std::vector<StructureHost> structures;
  bool structures_dirty = false;
  int n_struct_launch = 0;                 // user structures + one implicit structure per unreferenced body
  std::vector<int> h_link_bodies;          // body index of every launched link
  std::vector<StructureDev> h_structures;
  DeviceBuffer<StructureDev> d_structures;
  DeviceBuffer<LinkDev> d_links;
  DeviceBuffer<LinkDev> d_links_default;   // Link::default_body2joint_pose_ / default_joint2parent_pose_
  int n_links_total = 0;
  bool defaults_valid = false;
  std::vector<LinkDev> h_links_default;
  DeviceBuffer<ConstraintDev> d_constraints;
  DeviceBuffer<float> d_gh_link;
  DeviceBuffer<float> d_theta;             // [d_structures.size()][kMaxSystem]
  DeviceBuffer<int> d_struct_status;
  size_t struct_smem = 0;

  // device renderers (m3tb_set_body_geometry / m3tb_set_focused_renderer / m3tb_attach_renderer, k_render)
  std::vector<GeometryDev> h_geometry;       // [max_bodies]
  std::vector<DeviceBuffer<float>> geometry_alloc;  // [max_bodies] device triangle soups
  DeviceBuffer<GeometryDev> d_geometry;
  struct RendererHost {
    RendererDev dev;  // dev.depth / dev.silhouette view the two images below
    DeviceBuffer<uint16_t> depth;
    DeviceBuffer<uint8_t> silhouette;
    std::vector<int> geometry, referenced;
    bool rendered = false;  // images / records exist (m3tb_get_rendering)
  };
  std::vector<RendererHost> renderers;       // dense ids
  std::vector<std::array<int, RS_COUNT>> attached;  // per body and renderer slot: the device renderer feeding it, or -1
  std::vector<std::array<char, RS_COUNT>> attach_uploaded;  // the slot's record went to d_bodies once (k_render owns it)
  bool render_dirty = true;                  // the renderer / geometry / attachment tables changed
  DeviceBuffer<RendererDev> d_renderers;
  DeviceBuffer<int> d_render_lists;          // geometry_bodies | referenced_bodies | render_list
  DeviceBuffer<int> d_visible;
  DeviceBuffer<RenderOutDev> d_render_out;
  DeviceBuffer<RenderAttachDev> d_attach;
  int n_attached = 0;                        // slots with a device renderer (0: every launch is as without renderers)
  int n_attach = 0, n_geometry_list = 0, n_referenced_list = 0;
  int render_n[kRenderLists] = {};           // renderers in each RenderList
  size_t render_smem[kRenderLists] = {};     // z-buffer bytes of the largest renderer of each list
  std::vector<int> render_list[kRenderLists];  // host copies of the lists

  // host copies of the models made by m3tb_generate_depth_model / m3tb_generate_region_model (m3tb_get_depth_model,
  // m3tb_get_region_model); empty: not generated. view_scalars are surface areas or contour lengths.
  struct GeneratedModel {
    int n_views = 0, n_points = 0;
    float stride_depth_offset = 0.0f, max_radius_depth_offset = 0.0f;
    std::vector<float> orientations, view_scalars, points;
  };
  std::vector<GeneratedModel> dmodel_generated, rmodel_generated;

  // camera-image renderers drawn by k_view_*: viewers (m3tb_set_viewer / m3tb_update_viewers) and full renderers
  // (m3tb_set_full_renderer / m3tb_render_full, VK_FULL), one table each with dense ids of its own
  struct ViewImages {                     // a kind leaves empty what it does not produce
    DeviceBuffer<uint64_t> zbuf;          // cleared; k_view_resolve clears it again after each draw
    DeviceBuffer<uint8_t> normal;
    DeviceBuffer<uint8_t> image;          // viewers: the frame blended with the normal image
    DeviceBuffer<uint16_t> depth;         // VK_FULL, VK_FOCUSED
    DeviceBuffer<uint8_t> silhouette;     // VK_FULL
  };
  struct ViewSlotHost {
    int kind = VK_COLOR;                  // ViewerKind
    int camera_kind = 0, camera = 0;      // a viewer looks through the camera of its kind
    std::vector<int> geometry;
    float opacity = 0.0f, min_depth = 0.0f, max_depth = 0.0f;  // viewers
    int id_type = 0;                                           // VK_FULL
    float z_min = 0.0f, z_max = 0.0f;                          // VK_FULL, VK_FOCUSED
    int image_size = 0;                                        // VK_FOCUSED
    std::vector<int> referenced;                               // VK_FOCUSED
    int first_referenced = 0;             // VK_FOCUSED: where its visible flags are in d_focus_visible after a render
    int width = 0, height = 0;            // of the images (the camera's size when they were made; VK_FOCUSED: S x S)
    ViewImages images;
    bool drawn = false;                   // the images hold a result (m3tb_get_viewer_image / m3tb_get_full_rendering)
  };
  std::vector<ViewSlotHost> viewers, full_renderers;
  // focused normal renderers (m3tb_set_focused_normal_renderer / m3tb_render_focused_normals, VK_FOCUSED), dense ids of
  // their own, and the k_view_focus tables of their last render, grown lazily, each set all or nothing
  std::vector<ViewSlotHost> focused_normal_renderers;
  std::vector<FocusDev> h_focus;
  std::vector<int> h_focus_referenced;
  std::vector<float> h_focus_radius;
  DeviceBuffer<FocusDev> d_focus;
  DeviceBuffer<int> d_focus_referenced, d_focus_visible;
  DeviceBuffer<float> d_focus_radius;
  DeviceBuffer<RenderOutDev> d_focus_out;
  DeviceBuffer<uint8_t> d_normalized_depth;  // m3tb_get_normalized_depth_image into host memory, grown lazily
  // tables of one update (or one full render), grown lazily, each set all or nothing
  std::vector<ViewerDev> h_view_viewers;
  std::vector<ViewDrawDev> h_view_draws;
  DeviceBuffer<ViewerDev> d_view_viewers;
  DeviceBuffer<ViewDrawDev> d_view_draws;
  DeviceBuffer<float> d_view_rot;
  DeviceBuffer<ViewFanDev> d_view_fans;
  DeviceBuffer<uint64_t> d_view_fan_tile;
  DeviceBuffer<unsigned long long> d_view_counter;  // 0 between updates

  // undistortion of raw frames as they are uploaded (m3tb_set_camera_undistortion, k_undistort)
  struct UndistortHost {
    DeviceBuffer<int16_t> map;  // [height][map_pitch / 2] (x, y) pairs; empty: frames are uploaded as they are
    unsigned map_pitch = 0;     // bytes, a multiple of 16
    int channels = 0;           // bytes per raw colour pixel (3 or 4); 1 for depth
    int offset = 0;             // depth only
  };
  std::vector<UndistortHost> undistort[2];  // [colour | depth][max_cameras]
  DeviceBuffer<uint8_t> undistort_staging;  // the raw host frames of one upload call, grown lazily

  // texture modality (m3tb_set_texture_modality, k_texture_keyframe / k_texture_match): tables for max_bodies, made by
  // the first m3tb_set_texture_modality (TextureArgs for the layouts)
  int n_texture = 0;                    // bodies with a texture modality
  int tex_cap = 0;                      // features per body of the tables (TextureArgs::cap); 0 before they exist
  std::vector<int> tex_feat_gen;        // per body: colour-frame generation its features belong to, -1: none
  DeviceBuffer<float2> d_tex_xy;
  DeviceBuffer<uint32_t> d_tex_desc, d_tex_kf_desc;
  DeviceBuffer<int> d_tex_nfeat, d_tex_kf_n, d_tex_counts;
  DeviceBuffer<float> d_tex_kf_points, d_tex_points, d_tex_pose, d_gh_texture;
  DeviceBuffer<TexKeyframeState> d_tex_kf_state;
  // the wide descriptor tables (TexWideRows: SIFT / DAISY floats, BRISK / FREAK 64-byte rows): made by the first
  // m3tb_set_texture_modality with such a type; the matches of k_texture_knn_l2 / _hamming: made with them or by the
  // first ORB body above kTexMaxFeatures. Contexts whose ORB bodies keep the default n_features_max have neither.
  DeviceBuffer<float> d_tex_fdesc, d_tex_kf_fdesc;
  DeviceBuffer<int> d_tex_knn;
  // device front end (m3tb_texture_crop / m3tb_upload_texture_features_device): per body, the focus of its last crop
  // and the colour-frame generation it was cropped from (-1: none); the non-finite flags of k_texture_features, made by
  // the first device upload
  struct TexCrop {
    int roi_x = 0, roi_y = 0, gen = -1;
    float scale = 0.0f;
  };
  std::vector<TexCrop> tex_crop;
  DeviceBuffer<int> d_tex_nonfinite;
  // device ORB (m3tb_texture_detect_orb, k_texture_orb): scratch for up to kTexJobs bodies, grown on demand; the
  // parity tables [max_bodies][orb_cap] (keypoints and descriptors, apart from the feature slot, which later uploads
  // replace) and the kept counts [max_bodies]; per body, the n_features_max of its last detection (-1: none since the
  // tables were made or its texture modality was set)
  DeviceBuffer<uint8_t> d_orb_scratch;
  DeviceBuffer<float2> d_orb_xy;
  DeviceBuffer<float> d_orb_angle, d_orb_response;
  DeviceBuffer<int> d_orb_octave, d_orb_found;
  DeviceBuffer<uint32_t> d_orb_desc;
  int orb_cap = 0;
  std::vector<int> orb_nmax;

  // pose refinement (m3tb_refine_poses): the lists of RefineSelection, grown on demand; `refine` is set while it runs
  DeviceBuffer<int> d_refine;
  RefineSelection* refine = nullptr;

  // pose scoring (m3tb_set_evaluation_model / m3tb_score_poses / m3tb_calculate_diameters, k_score / k_diameter):
  // evaluation models with dense ids, per body its model (-1: none) and geometry2body term; the device tables are
  // uploaded by the next scoring call after a change, the per-call scratch grows lazily, each all or nothing
  struct EvalModelHost {
    DeviceBuffer<float4> full, reduced;
    int n_full = 0, n_reduced = 0;
  };
  std::vector<EvalModelHost> eval_models;
  std::vector<EvalBodyDev> h_eval_bodies;  // [max_bodies]
  bool eval_dirty = true;
  DeviceBuffer<EvalModelDev> d_eval_models;
  DeviceBuffer<EvalBodyDev> d_eval_bodies;
  DeviceBuffer<int> d_score_ids;           // bodies or models of the call
  DeviceBuffer<float> d_score_gt, d_score_partial, d_score_curves;
  DeviceBuffer<m3tb_pose_score> d_score_out;
  DeviceBuffer<unsigned> d_diameter;
};

namespace {

int Fail(m3tb_ctx* ctx, int code, const std::string& msg) {
  if (ctx) ctx->err = msg;
  return code;
}

// TextureModality::DescriptorType's names, for refusals
const char* DescriptorName(int type) {
  static const char* const names[] = {"BRISK", "DAISY", "FREAK", "SIFT", "ORB", "ORB_CUDA"};
  return type >= 0 && type < 6 ? names[type] : "unknown";
}

#define CU(call)                                                                                       \
  do {                                                                                                 \
    cudaError_t e_ = (call);                                                                           \
    if (e_ != cudaSuccess)                                                                             \
      return Fail(ctx, M3TB_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));             \
  } while (0)

#define CHECK_CTX()                                          \
  do {                                                       \
    if (!ctx) return M3TB_ERR_INVALID;                       \
    cudaError_t e0_ = cudaSetDevice(ctx->device);            \
    if (e0_ != cudaSuccess) return Fail(ctx, M3TB_ERR_CUDA, std::string("cudaSetDevice: ") + cudaGetErrorString(e0_)); \
  } while (0)

int Bitshift(int n_bins) {  // color_histograms.cpp:131-159
  switch (n_bins) {
    case 2: return 7;
    case 4: return 6;
    case 8: return 5;
    case 16: return 4;
    case 32: return 3;
    case 64: return 2;
    default: return -1;
  }
}

size_t Align(size_t v, size_t a) { return (v + a - 1) / a * a; }

// The host record of colour (camera kind 0) or depth (camera kind 1) camera `cam`, which the caller has checked
CameraDev& CameraOf(m3tb_ctx* ctx, bool color, int cam) { return (color ? ctx->h_ccams : ctx->h_dcams)[cam]; }

// A renderer's camera: (camera_kind, camera) names a camera that is set. The caller has checked camera_kind.
int CheckCameraSet(m3tb_ctx* ctx, int camera_kind, int camera) {
  if (camera < 0 || camera >= ctx->max_cameras || !CameraOf(ctx, camera_kind == 0, camera).set)
    return Fail(ctx, M3TB_ERR_INVALID, "camera not set");
  return M3TB_OK;
}

// A renderer's body list: every body in range and with geometry, none twice. The caller has checked `bodies` and `n`.
int CheckBodyList(m3tb_ctx* ctx, const int* bodies, int n) {
  for (int k = 0; k < n; ++k) {
    const int b = bodies[k];
    if (b < 0 || b >= ctx->max_bodies || !ctx->h_geometry[b].set)
      return Fail(ctx, M3TB_ERR_INVALID, "body " + std::to_string(b) + " has no geometry (m3tb_set_body_geometry)");
    for (int q = 0; q < k; ++q)
      if (bodies[q] == b) return Fail(ctx, M3TB_ERR_INVALID, "body listed twice");
  }
  return M3TB_OK;
}

int EnsureHist(m3tb_ctx* ctx, size_t stride) {
  if (stride <= ctx->hist_stride) return M3TB_OK;
  const size_t nb = size_t(ctx->max_bodies);
  DeviceBuffer<float> nf[4];
  DeviceBuffer<float2> nl;
  for (int k = 0; k < 4; ++k) {
    CU(nf[k].create(nb * stride));
    CU(cudaMemsetAsync(nf[k], 0, nb * stride * sizeof(float), ctx->stream));
  }
  CU(nl.create(nb * stride));
  CU(cudaMemsetAsync(nl, 0, nb * stride * sizeof(float2), ctx->stream));
  DeviceBuffer<float>* old[4] = {&ctx->d_hist_f, &ctx->d_hist_b, &ctx->d_mem_f, &ctx->d_mem_b};
  if (ctx->hist_stride) {
    for (int k = 0; k < 4; ++k)
      CU(cudaMemcpy2DAsync(nf[k], stride * sizeof(float), *old[k], ctx->hist_stride * sizeof(float),
                           ctx->hist_stride * sizeof(float), nb, cudaMemcpyDeviceToDevice, ctx->stream));
    CU(cudaMemcpy2DAsync(nl, stride * sizeof(float2), ctx->d_lut, ctx->hist_stride * sizeof(float2),
                         ctx->hist_stride * sizeof(float2), nb, cudaMemcpyDeviceToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  for (int k = 0; k < 4; ++k) *old[k] = std::move(nf[k]);
  ctx->d_lut = std::move(nl);
  ctx->hist_stride = stride;
  return M3TB_OK;
}

int EnsureState(m3tb_ctx* ctx) {
  int lc = 0, pc = 0;
  for (int b = 0; b < ctx->n_bodies; ++b) {
    const BodyDev& B = ctx->h_bodies[b];
    if (!B.set) continue;
    if (B.has_region) lc = std::max(lc, B.rp.n_lines_max);
    if (B.has_depth) pc = std::max(pc, B.dp.n_points_max);
  }
  lc = int(Align(size_t(std::max(lc, 1)), 32));
  pc = int(Align(size_t(std::max(pc, 1)), 32));
  const bool grow_r = lc > ctx->line_cap || !ctx->d_rstate, grow_d = pc > ctx->point_cap || !ctx->d_dstate;
  if (!grow_r && !grow_d) return M3TB_OK;
  DeviceBuffer<float> rs, ds;
  if (grow_r) {
    CU(rs.create(size_t(ctx->max_bodies) * RF_COUNT * lc));
    CU(cudaMemsetAsync(rs, 0, size_t(ctx->max_bodies) * RF_COUNT * lc * sizeof(float), ctx->stream));
  }
  if (grow_d) {
    CU(ds.create(size_t(ctx->max_bodies) * DF_COUNT * pc));
    CU(cudaMemsetAsync(ds, 0, size_t(ctx->max_bodies) * DF_COUNT * pc * sizeof(float), ctx->stream));
  }
  // the stored correspondences are gone: a load-state call before the next CalculateCorrespondences sees 0 lines
  CU(cudaMemsetAsync(ctx->d_counts, 0, sizeof(int) * 4 * ctx->max_bodies, ctx->stream));
  if (grow_r) {
    ctx->d_rstate = std::move(rs);
    ctx->line_cap = lc;
  }
  if (grow_d) {
    ctx->d_dstate = std::move(ds);
    ctx->point_cap = pc;
  }
  return M3TB_OK;
}

int SyncTables(m3tb_ctx* ctx) {
  if (ctx->bodies_dirty && ctx->n_attached == 0) {
    CU(cudaMemcpyAsync(ctx->d_bodies, ctx->h_bodies.data(), sizeof(BodyDev) * ctx->max_bodies, cudaMemcpyHostToDevice,
                       ctx->stream));
    ctx->bodies_dirty = false;
  } else if (ctx->bodies_dirty) {
    // k_render writes the records of the slots a device renderer feeds: after their first upload (image pointer, size,
    // pitch; visible = 0 until rendered) the host copy, which never learns corner / scale / visible, must not replace them
    for (int b = 0; b < ctx->max_bodies; ++b) {
      const auto& at = ctx->attached[b];
      auto& up = ctx->attach_uploaded[b];
      bool keep_any = false;
      for (int s = 0; s < RS_COUNT; ++s) keep_any = keep_any || (at[s] >= 0 && up[s]);
      BodyDev* dst = ctx->d_bodies + b;
      const BodyDev* src = ctx->h_bodies.data() + b;
      if (!keep_any) {
        CU(cudaMemcpyAsync(dst, src, sizeof(BodyDev), cudaMemcpyHostToDevice, ctx->stream));
      } else {
        CU(cudaMemcpyAsync(dst, src, offsetof(BodyDev, rend), cudaMemcpyHostToDevice, ctx->stream));
        for (int s = 0; s < RS_COUNT; ++s)
          if (!(at[s] >= 0 && up[s]))
            CU(cudaMemcpyAsync(&dst->rend[s], &src->rend[s], sizeof(RenderingDev), cudaMemcpyHostToDevice, ctx->stream));
      }
      for (int s = 0; s < RS_COUNT; ++s) up[s] = at[s] >= 0;
    }
    ctx->bodies_dirty = false;
  }
  if (ctx->cams_dirty) {
    CU(cudaMemcpyAsync(ctx->d_ccams, ctx->h_ccams.data(), sizeof(CameraDev) * ctx->max_cameras, cudaMemcpyHostToDevice,
                       ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_dcams, ctx->h_dcams.data(), sizeof(CameraDev) * ctx->max_cameras, cudaMemcpyHostToDevice,
                       ctx->stream));
    ctx->cams_dirty = false;
  }
  if (ctx->models_dirty) {
    CU(cudaMemcpyAsync(ctx->d_rmodels, ctx->h_rmodels.data(), sizeof(ModelDev) * ctx->max_models, cudaMemcpyHostToDevice,
                       ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_dmodels, ctx->h_dmodels.data(), sizeof(ModelDev) * ctx->max_models, cudaMemcpyHostToDevice,
                       ctx->stream));
    ctx->models_dirty = false;
  }
  return M3TB_OK;
}

// An occlusion or depth-offset radius the window scans and the depth-offset table can take: a negative or NaN one gives
// a stride of 0 (a scan that never ends, in the reference too) or a negative offset index
bool RadiusValid(float r) { return r >= 0.0f && std::isfinite(r); }

// The region modality's depth-offset id (region_modality.cpp:975-976, 985-986) as the kernels compute it. The reference
// checks only radius <= max_radius; when max_radius / stride lies in [29.5, 30) a radius near the maximum rounds to
// id 30, one past the table, so ValidateBodies refuses any id of 30 or more.
int RegionOffsetId(float radius, const ModelDev& m) { return int(radius / m.stride_depth_offset + 0.5f); }

// Checks that every set body references set-up objects ("Set up ... first").
int ValidateBodies(m3tb_ctx* ctx) {
  if (ctx->n_bodies == 0) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "no body set");
  for (int b = 0; b < ctx->n_bodies; ++b) {
    const BodyDev& B = ctx->h_bodies[b];
    if (!B.set) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "body " + std::to_string(b) + " not set (bodies must be dense)");
    if (B.has_region) {
      if (!ctx->h_rmodels[B.region_model].set) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "region model not set");
      const CameraDev& c = ctx->h_ccams[B.color_camera];
      if (!c.set || !c.image) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "color camera not set / no image uploaded");
      const ModelDev& m = ctx->h_rmodels[B.region_model];
      if (B.rp.measure_occlusions) {  // RegionModality::SetUp / PrecalculateModelVariables (region_modality.cpp:965-977)
        const CameraDev& d = ctx->h_dcams[B.depth_camera];
        if (!d.set || !d.image) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "measure_occlusions: depth camera not set / no image uploaded");
        if (B.rp.measured_depth_offset_radius > m.max_radius_depth_offset)
          return Fail(ctx, M3TB_ERR_INVALID, "Measured depth offset radius too large");
        if (RegionOffsetId(B.rp.measured_depth_offset_radius, m) >= kDepthOffsets)
          return Fail(ctx, M3TB_ERR_INVALID, "Measured depth offset radius rounds past the model's 30 depth offsets");
      }
      if (B.rp.model_occlusions) {  // region_modality.cpp:979-991
        if (B.rp.modeled_depth_offset_radius > m.max_radius_depth_offset)
          return Fail(ctx, M3TB_ERR_INVALID, "Modeled depth offset radius too large");
        if (RegionOffsetId(B.rp.modeled_depth_offset_radius, m) >= kDepthOffsets)
          return Fail(ctx, M3TB_ERR_INVALID, "Modeled depth offset radius rounds past the model's 30 depth offsets");
      }
    }
    if (B.has_depth) {
      if (!ctx->h_dmodels[B.depth_model].set) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "depth model not set");
      const CameraDev& c = ctx->h_dcams[B.depth_camera];
      if (!c.set || !c.image) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "depth camera not set / no image uploaded");
    }
  }
  return M3TB_OK;
}

// k_ingest writes the bin indices of the colour rectangles it fetches with the bit shift of the body that fetches them,
// and none for bodies above 32 bins. Records, for every colour camera it is about to fetch from, the bit shift its
// bin-index image will hold (kBinsNone where its region bodies disagree or write none). Called before each k_ingest.
void NoteIngestBins(m3tb_ctx* ctx) {
  for (int i = 0; i < ctx->max_cameras; ++i) {
    if (ctx->bin_shift[i] != kBinsAtIngest) continue;
    int shift = kBinsNone;
    bool first = true;
    for (int b = 0; b < ctx->n_bodies; ++b) {
      const BodyDev& B = ctx->h_bodies[b];
      if (!B.set || !B.has_region || B.color_camera != i) continue;
      const int s = B.rp.n_bins <= 32 ? B.rp.bitshift : kBinsNone;
      if (first) shift = s;
      else if (s != shift) shift = kBinsNone;
      first = false;
    }
    ctx->bin_shift[i] = shift;
  }
}

// Frame ingest for pinned host frames: fetch every body's ROI (k_ingest) before the first consumer of the new frame.
int LaunchIngestIfPending(m3tb_ctx* ctx) {
  if (ctx->prefetched) {  // the frames were prefetched on the side stream: order the consumers behind that ingest
    CU(cudaStreamWaitEvent(ctx->stream, ctx->pf.ev_ingest_done, 0));
    ctx->prefetched = false;
  }
  if (!ctx->ingest_pending) return M3TB_OK;
  // a refinement fetches the ROIs of its bodies only; the others are fetched by the next launch over the whole context
  RefineSelection* sel = ctx->refine;
  if (sel && sel->ingested) return M3TB_OK;
  IngestArgs a;
  a.bodies = ctx->d_bodies;
  a.poses = ctx->d_poses;
  a.color_cams = ctx->d_ccams;
  a.depth_cams = ctx->d_dcams;
  a.region_models = ctx->d_rmodels;
  a.depth_models = ctx->d_dmodels;
  a.roi = ctx->d_roi;
  ctx->ingest_bytes_slot ^= 1;
  a.bytes = ctx->d_ingest_bytes + ctx->ingest_bytes_slot;
  a.n_bodies = sel ? sel->n_bodies : ctx->n_bodies;
  a.body_list = sel ? sel->bodies : nullptr;
  CU(cudaMemsetAsync(a.bytes, 0, sizeof(unsigned long long), ctx->stream));
  if (!sel) NoteIngestBins(ctx);  // the bin-index images are complete once every body's rectangles are fetched
  k_ingest<<<a.n_bodies, kBlockThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  if (sel) sel->ingested = true;
  else ctx->ingest_pending = false;
  return M3TB_OK;
}

int SyncStructures(m3tb_ctx* ctx);
int LaunchRender(m3tb_ctx* ctx, int which);
int LaunchTexture(m3tb_ctx* ctx, bool keyframe, int mode);
int ValidateTexture(m3tb_ctx* ctx);
int ValidateTextureBody(m3tb_ctx* ctx, int b);
int CheckOrbDetection(m3tb_ctx* ctx, int b, const m3tb_orb_params& p);
int DetectOrb(m3tb_ctx* ctx, const int* bodies, int count, const m3tb_orb_params* params);

// cuTensorMapEncodeTiled through the runtime (libcuda is not linked: the library must load on machines without a driver)
PFN_cuTensorMapEncodeTiled_v12000 TensorMapEncoder() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = []() -> PFN_cuTensorMapEncodeTiled_v12000 {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }();
  return fn;
}

// Tensor maps of a u16 image pool viewed as [n_frames][height][width], boxes of TileWidth(i) x kTileBoxRows x 1.
const PoolMaps* GetPoolMaps(m3tb_ctx* ctx, void* base, int width, int height, unsigned pitch_bytes, size_t frame_bytes,
                            int n_frames) {
  for (const PoolMaps& m : ctx->pool_maps)
    if (m.base == base) return m.ok ? &m : nullptr;
  PoolMaps pm;
  pm.base = base;
  pm.ok = false;
  auto encode = TensorMapEncoder();
  if (encode && base && width >= 64 && height >= kTileBoxRows && (pitch_bytes & 15u) == 0 && (frame_bytes & 15u) == 0) {
    pm.ok = true;
    for (int i = 0; i < kTileWidths && pm.ok; ++i) {
      const cuuint64_t dims[3] = {cuuint64_t(width), cuuint64_t(height), cuuint64_t(n_frames)};
      const cuuint64_t strides[2] = {cuuint64_t(pitch_bytes), cuuint64_t(frame_bytes)};
      const cuuint32_t box[3] = {cuuint32_t(TileWidth(i)), cuuint32_t(kTileBoxRows), 1u};
      const cuuint32_t estr[3] = {1u, 1u, 1u};
      const CUresult r = encode(&pm.maps[i], CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, base, dims, strides, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) pm.ok = false;
    }
  }
  if (ctx->pool_maps.size() >= 8) ctx->pool_maps.erase(ctx->pool_maps.begin());
  ctx->pool_maps.push_back(pm);
  return pm.ok ? &ctx->pool_maps.back() : nullptr;
}

// Can k_track2 stage its tiles with TMA for this batch? Every camera in use sits in its pool, the region bodies share one
// histogram resolution (<= 32 bins: the index fits 16 bits); refreshes the bin-index images of frames that were copied in
// full (k_bin) and fills the tensor maps of `a`. A pinned frame's device copy is valid only inside the ROIs k_ingest
// fetched, so its bin indices cannot be rebuilt: when they were written with another bit shift (the resolution changed
// since the ingest) or none, the launch uses the legacy staging, which bins from the frame itself.
int PrepareTensorTiles(m3tb_ctx* ctx, TrackArgs& a, bool& usable) {
  a.tma_mode = ctx->tma_mode;
  a.tma_max_w = 256;
  if (const char* e = std::getenv("M3TB_TMA_MAXW")) a.tma_max_w = std::max(64, std::min(256, std::atoi(e) / 32 * 32));
  a.tmaps_global = ctx->d_tmaps;
  if (ctx->tma_mode == 0) { usable = true; return M3TB_OK; }  // legacy staging needs neither maps nor bin images
  usable = false;
  int bitshift = -1, n_bins = 0;
  bool any_region = false, any_depth = false;
  for (int b = 0; b < ctx->n_bodies; ++b) {
    const BodyDev& B = ctx->h_bodies[b];
    if (B.has_region) {
      any_region = true;
      if (bitshift >= 0 && B.rp.bitshift != bitshift) return M3TB_OK;
      bitshift = B.rp.bitshift;
      n_bins = B.rp.n_bins;
      if (n_bins > 32) return M3TB_OK;
      const CameraDev& c = ctx->h_ccams[B.color_camera];
      if (!ctx->color_pool.base || !ctx->color_pool.bins ||
          c.image != ctx->color_pool.base + ctx->color_pool.frame_bytes * B.color_camera || !c.bins)
        return M3TB_OK;
    }
    if (B.has_depth) {
      any_depth = true;
      const CameraDev& c = ctx->h_dcams[B.depth_camera];
      if (!ctx->depth_pool.base || c.image != ctx->depth_pool.base + ctx->depth_pool.frame_bytes * B.depth_camera)
        return M3TB_OK;
    }
  }
  if (any_region) {
    const ImagePool& p = ctx->color_pool;
    const PoolMaps* m = GetPoolMaps(ctx, p.bins, p.width, p.height, p.bin_pitch, p.bin_frame_bytes, p.capacity);
    if (!m) return M3TB_OK;
    std::memcpy(a.bin_maps, m->maps, sizeof(a.bin_maps));
    for (int b = 0; b < ctx->n_bodies; ++b) {
      const BodyDev& B = ctx->h_bodies[b];
      if (B.has_region && ctx->h_ccams[B.color_camera].host_src && ctx->bin_shift[B.color_camera] != bitshift) {
        a.tma_mode = 0;
        usable = true;
        return M3TB_OK;
      }
    }
    // frames that arrived by full copy: (re)build their bin-index images
    std::vector<int> ids;
    for (int i = 0; i < ctx->max_cameras; ++i) {
      const CameraDev& c = ctx->h_ccams[i];
      if (c.set && c.image && c.bins && !c.host_src && ctx->bin_shift[i] != bitshift) ids.push_back(i);
    }
    if (!ids.empty()) {
      CU(cudaMemcpyAsync(ctx->d_bin_ids, ids.data(), sizeof(int) * ids.size(), cudaMemcpyHostToDevice, ctx->stream));
      CU(cudaStreamSynchronize(ctx->stream));  // `ids` is a temporary (set-up path, not per step)
      BinArgs ba;
      ba.cams = ctx->d_ccams;
      ba.cam_ids = ctx->d_bin_ids;
      ba.bitshift = bitshift;
      ba.n_bins = n_bins;
      k_bin<<<dim3(unsigned(std::min(p.height, 120)), unsigned(ids.size())), kBlockThreads, 0, ctx->stream>>>(ba);
      CU(cudaGetLastError());
      ctx->launches++;
      for (int i : ids) ctx->bin_shift[i] = bitshift;
    }
  }
  if (any_depth) {
    const ImagePool& p = ctx->depth_pool;
    const PoolMaps* m = GetPoolMaps(ctx, p.base, p.width, p.height, p.pitch, p.frame_bytes, p.capacity);
    if (!m) return M3TB_OK;
    std::memcpy(a.depth_maps, m->maps, sizeof(a.depth_maps));
  }
  if (ctx->tma_mode == 2) {  // descriptors in global memory: refresh when the pools behind them changed (prefetch swaps)
    const void* bases[2] = {any_region ? static_cast<const void*>(ctx->color_pool.bins) : nullptr,
                            any_depth ? static_cast<const void*>(ctx->depth_pool.base) : nullptr};
    if (bases[0] != ctx->d_tmaps_bases[0] || bases[1] != ctx->d_tmaps_bases[1]) {
      CU(cudaMemcpyAsync(ctx->d_tmaps, a.bin_maps, sizeof(CUtensorMap) * kTileWidths, cudaMemcpyHostToDevice, ctx->stream));
      CU(cudaMemcpyAsync(ctx->d_tmaps + kTileWidths, a.depth_maps, sizeof(CUtensorMap) * kTileWidths, cudaMemcpyHostToDevice,
                         ctx->stream));
      CU(cudaStreamSynchronize(ctx->stream));  // `a` is a stack object
      ctx->d_tmaps_bases[0] = bases[0];
      ctx->d_tmaps_bases[1] = bases[1];
    }
  }
  usable = true;
  return M3TB_OK;
}

// The arguments of a k_track launch over bodies [first, first + gridDim.x): every per-body table starts at body `first`,
// so that the kernel, which indexes them by blockIdx.x, runs unchanged on a run of refined bodies (m3tb_refine_poses)
TrackArgs RunArgs(const TrackArgs& a, int first) {
  if (first == 0) return a;
  TrackArgs r = a;
  const size_t f = size_t(first);
  r.bodies += f;
  r.poses += 12 * f;
  r.lut += f * a.lut_stride;
  r.region_state += f * RF_COUNT * size_t(a.line_cap);
  r.depth_state += f * DF_COUNT * size_t(a.point_cap);
  r.counts += 4 * f;
  r.roi += 2 * f;
  auto shift = [](auto* p, size_t n) { return p ? p + n : p; };  // tables a context may not have made
  r.gh_region = shift(a.gh_region, 27 * f);
  r.gh_depth = shift(a.gh_depth, 27 * f);
  r.gh_link = shift(a.gh_link, 27 * f);
  r.gh_texture = shift(a.gh_texture, 27 * f);
  r.tex_points = shift(a.tex_points, f * TF_COUNT * size_t(a.tex_point_cap));
  r.tex_counts = shift(a.tex_counts, f);
  r.tex_pose = shift(a.tex_pose, 12 * f);
  r.phase_clock = shift(a.phase_clock, f * kPhaseSlots);
  return r;
}

int LaunchTrack(m3tb_ctx* ctx, int iteration, int corr_begin, int corr_end, int n_update, int opt_base,
                unsigned phases) {
  int rc = ValidateBodies(ctx);
  if (!rc && (phases & PH_TEXTURE_GH)) rc = ValidateTexture(ctx);
  if (rc) return rc;
  rc = EnsureState(ctx);
  if (rc) return rc;
  rc = SyncTables(ctx);
  if (rc) return rc;
  if (ctx->prefetch_enabled && (phases & (PH_REGION_CORR | PH_DEPTH_CORR))) {
    // What the next prefetch projects the ROIs with: the poses this launch starts from (the side stream must not read
    // d_poses while this launch writes them). Taken BEFORE this launch is ordered behind the ingest of its own frames,
    // so the next ingest never waits for it; two buffers, because the ingest in flight may still be reading the
    // snapshot of the launch before (it is finished before this buffer's turn comes again: the launch in between
    // waits for it).
    ctx->snap_parity ^= 1;
    CU(cudaMemcpyAsync(ctx->pf.poses_snap[ctx->snap_parity], ctx->d_poses, sizeof(float) * 12 * ctx->n_bodies,
                       cudaMemcpyDeviceToDevice, ctx->stream));
    CU(cudaEventRecord(ctx->pf.ev_poses_snap, ctx->stream));
    ctx->poses_snap_valid = true;
  }
  rc = LaunchIngestIfPending(ctx);
  if (rc) return rc;
  TrackArgs a = {};
  a.bodies = ctx->d_bodies;
  a.poses = ctx->d_poses;
  a.color_cams = ctx->d_ccams;
  a.depth_cams = ctx->d_dcams;
  a.region_models = ctx->d_rmodels;
  a.depth_models = ctx->d_dmodels;
  a.lut = ctx->d_lut;
  a.lut_stride = ctx->hist_stride;
  a.region_state = ctx->d_rstate;
  a.depth_state = ctx->d_dstate;
  a.line_cap = ctx->line_cap;
  a.point_cap = ctx->point_cap;
  a.counts = ctx->d_counts;
  a.gh_region = ctx->d_gh_region;
  a.gh_depth = ctx->d_gh_depth;
  a.gh_link = ctx->d_gh_link;
  a.tex_points = ctx->d_tex_points;
  a.tex_counts = ctx->d_tex_counts;
  a.tex_pose = ctx->d_tex_pose;
  a.gh_texture = ctx->d_gh_texture;
  a.tex_point_cap = kTexMaxKeyframes * ctx->tex_cap;
  a.iteration = iteration;
  a.corr_begin = corr_begin;
  a.corr_end = corr_end;
  a.n_update = n_update;
  a.opt_base = opt_base;
  a.phases = phases;
  a.phase_clock = ctx->d_phase_clock;
  a.roi = ctx->d_roi;
  // thread <-> line mapping: T threads per body, K lines and K points per thread (state in registers)
  const int items = std::max(ctx->line_cap, ctx->point_cap);
  bool lut_smem = true;  // normalised LUT staged in shared memory when every region body has <= 16 bins (32 KB)
  for (int b = 0; b < ctx->n_bodies; ++b)
    if (ctx->h_bodies[b].has_region && ctx->h_bodies[b].rp.n_bins > 16) lut_smem = false;
  // dynamic shared memory: [normalised LUT 32 KB (16 bins)] [colour bin-index tile] [depth tile]
  const size_t lut_bytes = lut_smem ? size_t(16 * 16 * 16) * sizeof(float2) : 0;
  bool bins_fit_u16 = true;  // the colour tile holds 16-bit bin indices: 64 bins (18 bits) go without tiles
  for (int b = 0; b < ctx->n_bodies; ++b)
    if (ctx->h_bodies[b].has_region && ctx->h_bodies[b].rp.n_bins > 32) bins_fit_u16 = false;
  const bool tiles = ctx->use_tiles && bins_fit_u16;
  const size_t dyn = tiles ? size_t(kDynSmemBytes) : lut_bytes;
  a.tile_bytes = tiles ? int(dyn - lut_bytes) : 0;
  bool occ = false;  // measured occlusion handling anywhere: the kernel variant that carries the depth-window scans
  for (int b = 0; b < ctx->n_bodies; ++b) {
    const BodyDev& B = ctx->h_bodies[b];
    occ = occ || (B.has_region && B.rp.measure_occlusions) || (B.has_depth && B.dp.measure_occlusions);
    // the renderer-image checks live in the same kernel variants
    occ = occ || (B.has_region && (B.rp.model_occlusions || B.rp.use_region_checking)) ||
          (B.has_depth && (B.dp.model_occlusions || B.dp.use_silhouette_checking));
  }
  // ---- k_track2: rigid bodies, <= 512 items per modality, <= 32 histogram bins (its colour tile holds 16-bit bin indices
  //      under every staging mode), no measured occlusion handling, correspondence / fused phases, one function lookup
  //      for the whole batch (m3t_b200_track2.cuh) --------------------------------------------------------------------
  {
    const unsigned k2_phases = PH_REGION_CORR | PH_DEPTH_CORR | PH_REGION_GH | PH_DEPTH_GH | PH_SOLVE | PH_STORE_REGION |
                               PH_STORE_DEPTH;
    bool ok = ctx->use_track2 && !ctx->refine && bins_fit_u16 && !occ && items <= kGroup && (phases & ~k2_phases) == 0 &&
              (n_update == 0 || (phases & PH_SOLVE));
    bool both = false, have_lookup = false;
    for (int b = 0; b < ctx->n_bodies && ok; ++b) {
      const BodyDev& B = ctx->h_bodies[b];
      both = both || (B.has_region && B.has_depth);
      if (!B.has_region) continue;
      if (!have_lookup) {
        std::memcpy(a.lookup_f, B.rp.lookup_f, sizeof(a.lookup_f));
        std::memcpy(a.lookup_b, B.rp.lookup_b, sizeof(a.lookup_b));
        have_lookup = true;
      } else if (std::memcmp(a.lookup_f, B.rp.lookup_f, sizeof(a.lookup_f)) != 0 ||
                 std::memcmp(a.lookup_b, B.rp.lookup_b, sizeof(a.lookup_b)) != 0) {
        ok = false;
      }
    }
    if (!have_lookup) { std::memset(a.lookup_f, 0, sizeof(a.lookup_f)); std::memset(a.lookup_b, 0, sizeof(a.lookup_b)); }
    if (ok) {
      int trc = PrepareTensorTiles(ctx, a, ok);
      if (trc) return trc;
    }
    if (ok) {
      const size_t fixed = lut_bytes + size_t(kFixedDynBytes);
      const size_t dyn2 = ctx->use_tiles ? size_t(kDynSmemBytes) : fixed;
      a.tile_bytes = ctx->use_tiles ? int(dyn2 - fixed) : 0;
#define M3TB_LAUNCH2(T_, L_)                                                                                     \
  do {                                                                                                           \
    CU(cudaFuncSetAttribute(k_track2<T_, L_>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(dyn2)));          \
    k_track2<T_, L_><<<ctx->n_bodies, T_, dyn2, ctx->stream>>>(a);                                               \
  } while (0)
      if (both) { if (lut_smem) M3TB_LAUNCH2(1024, true); else M3TB_LAUNCH2(1024, false); }
      else { if (lut_smem) M3TB_LAUNCH2(512, true); else M3TB_LAUNCH2(512, false); }
#undef M3TB_LAUNCH2
      CU(cudaGetLastError());
      ctx->launches++;
      ctx->last_launch = {M3TB_KERNEL_TRACK2, both ? 1024 : 512, 1, lut_smem ? 1 : 0, 0, a.tile_bytes > 0 ? 1 : 0, a.tma_mode};
      return M3TB_OK;
    }
  }
#define M3TB_LAUNCH1(T_, K_, L_, O_)                                                                                   \
  do {                                                                                                                 \
    CU(cudaFuncSetAttribute(k_track<T_, K_, L_, O_>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(dyn)));           \
    for (size_t r_ = 0; r_ < n_runs; ++r_)                                                                             \
      k_track<T_, K_, L_, O_><<<runs_begin[r_].second, T_, dyn, ctx->stream>>>(RunArgs(a, runs_begin[r_].first));       \
    n_launches = int(n_runs);                                                                                          \
    info = {M3TB_KERNEL_TRACK, T_, K_, L_ ? 1 : 0, O_ ? 1 : 0, tiles ? 1 : 0, -1};                                     \
  } while (0)
#define M3TB_LAUNCH(T_, K_)                                       \
  do {                                                            \
    if (lut_smem && !occ) M3TB_LAUNCH1(T_, K_, true, false);      \
    else if (lut_smem) M3TB_LAUNCH1(T_, K_, true, true);          \
    else if (!occ) M3TB_LAUNCH1(T_, K_, false, false);            \
    else M3TB_LAUNCH1(T_, K_, false, true);                       \
  } while (0)
  m3tb_launch_info info = {};
  int n_launches = 1;
  // a refinement launches k_track once per run of consecutive refined bodies (RunArgs), one CTA per body
  const std::pair<int, int> all_bodies(0, ctx->n_bodies);
  const std::pair<int, int>* runs_begin = ctx->refine ? ctx->refine->runs.data() : &all_bodies;
  const size_t n_runs = ctx->refine ? ctx->refine->runs.size() : 1;
  if (items <= 256) M3TB_LAUNCH(256, 1);
  else if (items <= 512) M3TB_LAUNCH(512, 1);
  else if (items <= 1024) M3TB_LAUNCH(512, 2);
  else if (items <= 2048) M3TB_LAUNCH(512, 4);
  else return Fail(ctx, M3TB_ERR_UNSUPPORTED, "n_lines_max / n_points_max above 2048");
#undef M3TB_LAUNCH
#undef M3TB_LAUNCH1
  CU(cudaGetLastError());
  ctx->launches += n_launches;
  ctx->last_launch = info;
  return M3TB_OK;
}


// ---- kinematic structures -------------------------------------------------------------------------------------
bool HasStructures(const m3tb_ctx* ctx) {
  for (const auto& s : ctx->structures)
    if (s.set) return true;
  return false;
}

// The joint poses live on the device while tracking runs; bring them back before the host tables are edited.
int PullLinks(m3tb_ctx* ctx) {
  if (ctx->structures_dirty || !ctx->d_links || ctx->n_struct_launch == 0) return M3TB_OK;
  int total = 0;
  for (const auto& s : ctx->structures) total += int(s.links.size());
  if (total == 0) return M3TB_OK;
  std::vector<LinkDev> tmp(total);
  CU(cudaMemcpyAsync(tmp.data(), ctx->d_links, sizeof(LinkDev) * total, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  int o = 0;
  for (auto& s : ctx->structures)
    for (auto& l : s.links) l = tmp[o++];
  return M3TB_OK;
}

// Flatten the user structures, append one implicit single-link structure (free root link, body2joint = identity:
// the rigid-body optimiser) per body that no structure references, upload.
int SyncStructures(m3tb_ctx* ctx) {
  if (!ctx->structures_dirty) return M3TB_OK;
  std::vector<LinkDev> links;
  std::vector<ConstraintDev> cons;
  std::vector<StructureDev> sts;
  std::vector<char> used(ctx->n_bodies, 0);
  size_t smem = 0;
  auto push = [&](const std::vector<LinkDev>& L, const std::vector<ConstraintDev>& C, float lr, float lt) {
    StructureDev d;
    d.first_link = int(links.size());
    d.n_links = int(L.size());
    d.first_constraint = int(cons.size());
    d.n_constraints = int(C.size());
    d.dof = 0;
    for (const auto& l : L) d.dof += l.dof;
    d.n_rows = 0;
    for (const auto& c : C) d.n_rows += c.soft ? 0 : c.n_rows;
    d.tikhonov_rotation = lr;
    d.tikhonov_translation = lt;
    links.insert(links.end(), L.begin(), L.end());
    cons.insert(cons.end(), C.begin(), C.end());
    sts.push_back(d);
    smem = std::max(smem, StructSmemFloats(d.n_links, d.dof, d.dof + d.n_rows, d.n_constraints) * sizeof(float));
  };
  for (size_t si = 0; si < ctx->structures.size(); ++si) {
    const StructureHost& s = ctx->structures[si];
    if (!s.set) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "structure " + std::to_string(si) + " not set (structure ids must be dense)");
    for (const auto& l : s.links) {
      if (l.body >= ctx->n_bodies) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "structure references a body that is not set");
      if (l.body >= 0) {
        if (used[l.body]) return Fail(ctx, M3TB_ERR_INVALID, "body " + std::to_string(l.body) + " is referenced by two links");
        used[l.body] = 1;
      }
      for (int x = 0; x < l.n_extra; ++x) {
        if (l.extra[x] < 0 || l.extra[x] >= ctx->n_bodies) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "structure references a body that is not set");
        if (used[l.extra[x]]) return Fail(ctx, M3TB_ERR_INVALID, "body " + std::to_string(l.extra[x]) + " is referenced twice");
        used[l.extra[x]] = 1;
      }
    }
    push(s.links, s.constraints, s.tikhonov_rotation, s.tikhonov_translation);
  }
  for (int b = 0; b < ctx->n_bodies; ++b) {
    if (used[b]) continue;
    LinkDev l;
    std::memset(&l, 0, sizeof(l));
    l.body = b; l.parent = -1; l.first_index = 0; l.dof = 6; l.fixed_body2joint = 1;
    for (int d = 0; d < 6; ++d) l.free_directions[d] = 1;
    for (int k = 0; k < 3; ++k) l.body2joint[5 * k] = l.joint2parent[5 * k] = l.link2world[5 * k] = 1.0f;
    push(std::vector<LinkDev>{l}, std::vector<ConstraintDev>{}, ctx->h_bodies[b].tikhonov_rotation,
         ctx->h_bodies[b].tikhonov_translation);
  }
  const int ns = int(sts.size()), nl = int(links.size()), nc = int(std::max<size_t>(cons.size(), 1));
  // grow the tables: every new one is made before any old one is replaced
  DeviceBuffer<StructureDev> structures;
  DeviceBuffer<float> theta;
  DeviceBuffer<int> status;
  DeviceBuffer<LinkDev> dlinks, dlinks_default;
  DeviceBuffer<ConstraintDev> constraints;
  const bool grow_s = size_t(ns) > ctx->d_structures.size(), grow_l = size_t(nl) > ctx->d_links.size(),
             grow_c = size_t(nc) > ctx->d_constraints.size();
  if (grow_s) {
    CU(structures.create(ns));
    CU(theta.create(size_t(kMaxSystem) * ns));
    CU(status.create(ns));
  }
  if (grow_l) {
    CU(dlinks.create(nl));
    CU(dlinks_default.create(nl));
  }
  if (grow_c) CU(constraints.create(nc));
  if (grow_s) {
    ctx->d_structures = std::move(structures);
    ctx->d_theta = std::move(theta);
    ctx->d_struct_status = std::move(status);
  }
  if (grow_l) {
    ctx->d_links = std::move(dlinks);
    ctx->d_links_default = std::move(dlinks_default);
  }
  if (grow_c) ctx->d_constraints = std::move(constraints);
  CU(cudaMemsetAsync(ctx->d_theta, 0, sizeof(float) * kMaxSystem * ns, ctx->stream));
  CU(cudaMemsetAsync(ctx->d_struct_status, 0, sizeof(int) * ns, ctx->stream));
  CU(cudaMemcpyAsync(ctx->d_structures, sts.data(), sizeof(StructureDev) * ns, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(ctx->d_links, links.data(), sizeof(LinkDev) * nl, cudaMemcpyHostToDevice, ctx->stream));
  {
    // Defaults are per link and change only through that link's own setters (link.cpp:131-139): the default table is the
    // concatenation of what each m3tb_set_structure call was given (implicit one-link structures: identity joints), NOT
    // the current - possibly already tracked - joint poses of the other structures.
    std::vector<LinkDev> d = links;
    size_t o = 0;
    for (const StructureHost& sh : ctx->structures) {
      for (size_t k = 0; k < sh.default_links.size() && o + k < d.size(); ++k) d[o + k] = sh.default_links[k];
      o += sh.links.size();
    }
    CU(cudaMemcpyAsync(ctx->d_links_default, d.data(), sizeof(LinkDev) * nl, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->h_links_default = d;
    ctx->defaults_valid = true;
  }
  ctx->n_links_total = nl;
  if (!cons.empty())
    CU(cudaMemcpyAsync(ctx->d_constraints, cons.data(), sizeof(ConstraintDev) * cons.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));  // staging vectors go out of scope
  ctx->h_structures = sts;
  ctx->h_link_bodies.resize(links.size());
  for (size_t k = 0; k < links.size(); ++k) ctx->h_link_bodies[k] = links[k].body;
  ctx->n_struct_launch = ns;
  ctx->struct_smem = smem;
  ctx->structures_dirty = false;
  return M3TB_OK;
}

// Optimizer::CalculateOptimization (mode 0) / CalculateConsistentPoses (mode 1) for every structure
int LaunchStructure(m3tb_ctx* ctx, int mode, bool from_modalities) {
  if (ctx->n_bodies == 0) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "no body set");
  int rc = SyncStructures(ctx);
  if (rc) return rc;
  StructArgs a;
  a.structures = ctx->d_structures;
  a.links = ctx->d_links;
  a.constraints = ctx->d_constraints;
  a.poses = ctx->d_poses;
  a.gh_link = from_modalities ? nullptr : ctx->d_gh_link.get();
  a.gh_region = ctx->d_gh_region;
  a.gh_depth = ctx->d_gh_depth;
  // the texture sums of the fine-grained calls; the kernel reads has_texture from the device body table
  a.gh_texture = from_modalities && ctx->n_texture > 0 ? ctx->d_gh_texture.get() : nullptr;
  a.bodies = ctx->d_bodies;
  if (a.gh_texture) {
    rc = SyncTables(ctx);
    if (rc) return rc;
  }
  a.mode = mode;
  a.theta_out = ctx->d_theta;
  a.status = ctx->d_struct_status;
  a.list = ctx->refine ? ctx->refine->structures : nullptr;
  const int n = ctx->refine ? ctx->refine->n_structures : ctx->n_struct_launch;
  if (n == 0) return M3TB_OK;
  if (ctx->struct_smem > 48 * 1024)
    CU(cudaFuncSetAttribute(k_structure, cudaFuncAttributeMaxDynamicSharedMemorySize, int(ctx->struct_smem)));
  k_structure<<<n, kStructThreads, ctx->struct_smem, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  return M3TB_OK;
}

// Tracker::ExecuteTrackingStep's loop nest (tracker.cpp:344-361) when the optimisers are kinematic structures: the
// per-body work stays in k_track (correspondences, gradient / Hessian of region, depth and texture -> gh_link), every
// Optimizer::CalculateOptimization is one k_structure launch over all structures. Texture matching runs once per frame,
// at correspondence iteration 0, as in the rigid path.
int StructureStep(m3tb_ctx* ctx, int iteration, int corr_begin, int corr_end, int n_update) {
  int rc0 = SyncStructures(ctx);
  // TextureModality::SetUp's conditions first: a texture modality then has its silhouette renderer attached, so a
  // textured context renders (below)
  if (!rc0 && ctx->n_texture > 0) rc0 = ValidateTexture(ctx);
  if (rc0) return rc0;
  // device renderers refresh their images before every correspondence iteration
  const bool render = ctx->n_attached > 0;
  const unsigned tex = ctx->n_texture > 0 ? unsigned(PH_TEXTURE_GH) : 0u;
  for (int corr = corr_begin; corr < corr_end; ++corr) {
    if (render) {
      int rc = LaunchRender(ctx, kRenderAttached);
      if (!rc && corr == 0) rc = LaunchTexture(ctx, false, 1);  // texture matches of this frame (no-op without texture)
      if (rc) return rc;
    }
    if (n_update == 0) {
      int rc = LaunchTrack(ctx, iteration, corr, corr + 1, 0, 0, PH_REGION_CORR | PH_DEPTH_CORR | PH_STORE_REGION | PH_STORE_DEPTH);
      if (rc) return rc;
      continue;
    }
    int rc = LaunchTrack(ctx, iteration, corr, corr + 1, 1, 0,
                         PH_REGION_CORR | PH_DEPTH_CORR | PH_REGION_GH | PH_DEPTH_GH | PH_STORE_LINK_GH | PH_STORE_REGION |
                             PH_STORE_DEPTH | tex);
    if (rc) return rc;
    rc = LaunchStructure(ctx, 0, false);
    if (rc) return rc;
    for (int upd = 1; upd < n_update; ++upd) {
      rc = LaunchTrack(ctx, iteration, corr, corr + 1, 1, upd,
                       PH_LOAD_REGION | PH_LOAD_DEPTH | PH_REGION_GH | PH_DEPTH_GH | PH_STORE_LINK_GH | tex);
      if (rc) return rc;
      rc = LaunchStructure(ctx, 0, false);
      if (rc) return rc;
    }
  }
  return M3TB_OK;
}

int LaunchHistogram(m3tb_ctx* ctx, int mode, int iteration) {
  int rc = ValidateBodies(ctx);
  if (rc) return rc;
  rc = SyncTables(ctx);
  if (rc) return rc;
  rc = LaunchIngestIfPending(ctx);
  if (rc) return rc;
  if (!ctx->hist_stride) return M3TB_OK;  // no region modality anywhere
  HistArgs a;
  a.bodies = ctx->d_bodies;
  a.poses = ctx->d_poses;
  a.color_cams = ctx->d_ccams;
  a.region_models = ctx->d_rmodels;
  a.hist_f = ctx->d_hist_f;
  a.hist_b = ctx->d_hist_b;
  a.mem_f = ctx->d_mem_f;
  a.mem_b = ctx->d_mem_b;
  a.lut = ctx->d_lut;
  a.stride = ctx->hist_stride;
  a.mode = mode;
  a.roi = ctx->d_roi;
  a.depth_cams = ctx->d_dcams;
  a.iteration = iteration;
  a.shared_owner = nullptr;
  const RefineSelection* sel = ctx->refine;
  a.body_list = sel ? sel->bodies : nullptr;
  // shared ColorHistograms objects: group tables (owner first), checked against the bodies as they are now
  std::vector<int> group_owner, group_first, members;
  bool any_shared = false;
  for (int b = 0; b < ctx->n_bodies && b < int(ctx->hist_owner.size()); ++b) any_shared = any_shared || ctx->hist_owner[b] >= 0;
  if (any_shared) {
    for (int o = 0; o < ctx->n_bodies; ++o) {
      if (ctx->hist_owner[o] != o) continue;
      group_owner.push_back(o);
      group_first.push_back(int(members.size()));
      members.push_back(o);
      for (int b = 0; b < ctx->n_bodies; ++b)
        if (b != o && ctx->hist_owner[b] == o) members.push_back(b);
    }
    group_first.push_back(int(members.size()));
    for (int b = 0; b < ctx->n_bodies; ++b) {
      const int o = ctx->hist_owner[b];
      if (o < 0) continue;
      const BodyDev &B = ctx->h_bodies[b], &O = ctx->h_bodies[o];
      if (o >= ctx->n_bodies || ctx->hist_owner[o] != o || !B.set || !O.set || !B.has_region || !O.has_region ||
          B.rp.n_bins != O.rp.n_bins)
        return Fail(ctx, M3TB_ERR_NOT_SET_UP, "shared colour histograms: owner and member need region modalities with the same number of bins");
    }
    const int n_groups = int(group_owner.size());
    std::vector<int> table(group_owner);
    table.insert(table.end(), group_first.begin(), group_first.end());
    table.insert(table.end(), members.begin(), members.end());
    DeviceBuffer<int> owner, groups;
    if (!ctx->d_hist_owner) CU(owner.create(ctx->max_bodies));
    if (table.size() > ctx->d_hist_groups.size()) {
      CU(groups.create(table.size()));
      CU(cudaStreamSynchronize(ctx->stream));
      ctx->d_hist_groups = std::move(groups);
    }
    if (owner) ctx->d_hist_owner = std::move(owner);
    std::vector<int> key(table);  // groups + the per-body owners of the bodies that exist now
    key.insert(key.end(), ctx->hist_owner.begin(), ctx->hist_owner.begin() + ctx->n_bodies);
    if (key != ctx->hist_table_uploaded) {
      CU(cudaStreamSynchronize(ctx->stream));  // the tables may still be read by the launch before; they change rarely
      CU(cudaMemcpy(ctx->d_hist_owner, ctx->hist_owner.data(), sizeof(int) * ctx->n_bodies, cudaMemcpyHostToDevice));
      CU(cudaMemcpy(ctx->d_hist_groups, table.data(), sizeof(int) * table.size(), cudaMemcpyHostToDevice));
      ctx->hist_table_uploaded = key;
      ctx->n_hist_groups = n_groups;
    }
    a.shared_owner = ctx->d_hist_owner;
  }
  k_histogram<<<sel ? sel->n_bodies : ctx->n_bodies, kBlockThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  if (any_shared && (!sel || sel->n_hist_groups > 0)) {
    SharedHistArgs s;
    s.bodies = ctx->d_bodies;
    s.hist_f = ctx->d_hist_f; s.hist_b = ctx->d_hist_b; s.mem_f = ctx->d_mem_f; s.mem_b = ctx->d_mem_b; s.lut = ctx->d_lut;
    s.stride = ctx->hist_stride;
    s.mode = mode;
    s.group_owner = ctx->d_hist_groups;
    s.group_first = ctx->d_hist_groups + ctx->n_hist_groups;
    s.members = ctx->d_hist_groups + 2 * ctx->n_hist_groups + 1;
    s.group_summed = nullptr;
    int n_groups = ctx->n_hist_groups;
    if (sel) {  // the objects a refined body uses, from the refined members' line pixels only (Refiner::StartModalities)
      n_groups = sel->n_hist_groups;
      s.group_owner = sel->hist_groups;
      s.group_first = sel->hist_groups + n_groups;
      s.group_summed = sel->hist_groups + 2 * n_groups + 1;
      s.members = sel->hist_groups + 3 * n_groups + 1;
    }
    k_histogram_shared<<<n_groups, kBlockThreads, 0, ctx->stream>>>(s);
    CU(cudaGetLastError());
    ctx->launches++;
  }
  return M3TB_OK;
}

// A device table of at least `n` elements: `table` itself when it is large enough, else a new one in `grown` (contents
// are rewritten by the caller).
template <typename T>
int GrowTable(m3tb_ctx* ctx, const DeviceBuffer<T>& table, DeviceBuffer<T>& grown, size_t n) {
  if (n <= table.size()) return M3TB_OK;
  CU(grown.create(std::max<size_t>(n, 16)));
  return M3TB_OK;
}

// Flattens the renderer, list and attachment tables and uploads them with the geometry table.
int SyncRenderTables(m3tb_ctx* ctx) {
  if (!ctx->render_dirty) return M3TB_OK;
  const int nr = int(ctx->renderers.size());
  std::vector<RendererDev> devs(nr);
  std::vector<int> geo, ref;
  for (int r = 0; r < nr; ++r) {
    const auto& h = ctx->renderers[r];
    devs[r] = h.dev;
    devs[r].first_geometry = int(geo.size());
    devs[r].n_geometry = int(h.geometry.size());
    devs[r].first_referenced = int(ref.size());
    devs[r].n_referenced = int(h.referenced.size());
    geo.insert(geo.end(), h.geometry.begin(), h.geometry.end());
    ref.insert(ref.end(), h.referenced.begin(), h.referenced.end());
  }
  std::vector<RenderAttachDev> att;
  for (int b = 0; b < ctx->max_bodies; ++b)
    for (int s = 0; s < RS_COUNT; ++s) {
      const int r = ctx->attached[b][s];
      if (r < 0) continue;
      const auto& L = ctx->renderers[r].referenced;
      const int k = int(std::find(L.begin(), L.end(), b) - L.begin());
      att.push_back({b, s, r, k});
    }
  // lists: geometry_bodies | referenced_bodies | the three render lists (RenderList)
  std::vector<int> lists(geo);
  lists.insert(lists.end(), ref.begin(), ref.end());
  for (int pass = 0; pass < kRenderLists; ++pass) {
    ctx->render_smem[pass] = 0;
    ctx->render_n[pass] = 0;
    ctx->render_list[pass].clear();
  }
  for (int pass = 0; pass < kRenderLists; ++pass)
    for (int r = 0; r < nr; ++r) {
      bool use = pass == kRenderAll;
      for (const auto& x : att)
        // the texture modality has no correspondence renderers (TextureModality::correspondence_renderer_ptrs is empty):
        // its renderers draw only for StartModality and CalculateResults
        use = use || (x.renderer == r && ((pass == kRenderAttached && x.slot < RS_TEXTURE_SILHOUETTE) ||
                                          x.slot == RS_REGION_DEPTH || x.slot == RS_REGION_SILHOUETTE ||
                                          x.slot >= RS_TEXTURE_SILHOUETTE));
      if (!use) continue;
      lists.push_back(r);
      ctx->render_list[pass].push_back(r);
      ctx->render_n[pass]++;
      ctx->render_smem[pass] = std::max(ctx->render_smem[pass], size_t(devs[r].image_size) * devs[r].image_size * sizeof(uint32_t));
    }
  DeviceBuffer<RendererDev> renderers;
  DeviceBuffer<int> render_lists, visible;
  DeviceBuffer<RenderAttachDev> attach;
  DeviceBuffer<RenderOutDev> render_out;
  DeviceBuffer<GeometryDev> geometry;
  int rc = GrowTable(ctx, ctx->d_renderers, renderers, size_t(std::max(nr, 1)));
  if (!rc) rc = GrowTable(ctx, ctx->d_render_lists, render_lists, std::max<size_t>(lists.size(), 1));
  if (!rc) rc = GrowTable(ctx, ctx->d_attach, attach, std::max<size_t>(att.size(), 1));
  if (!rc) rc = GrowTable(ctx, ctx->d_visible, visible, std::max<size_t>(ref.size(), 1));
  if (rc) return rc;
  if (!ctx->d_render_out) CU(render_out.create(4 * size_t(ctx->max_bodies)));
  if (!ctx->d_geometry) CU(geometry.create(ctx->max_bodies));
  // the host vectors below are temporaries (set-up path, not per step), and a launch in flight may still read the
  // tables that are replaced
  CU(cudaStreamSynchronize(ctx->stream));
  if (renderers) ctx->d_renderers = std::move(renderers);
  if (render_lists) ctx->d_render_lists = std::move(render_lists);
  if (attach) ctx->d_attach = std::move(attach);
  if (visible) ctx->d_visible = std::move(visible);
  if (render_out) ctx->d_render_out = std::move(render_out);
  if (geometry) ctx->d_geometry = std::move(geometry);
  if (nr) CU(cudaMemcpy(ctx->d_renderers, devs.data(), sizeof(RendererDev) * nr, cudaMemcpyHostToDevice));
  if (!lists.empty()) CU(cudaMemcpy(ctx->d_render_lists, lists.data(), sizeof(int) * lists.size(), cudaMemcpyHostToDevice));
  if (!att.empty()) CU(cudaMemcpy(ctx->d_attach, att.data(), sizeof(RenderAttachDev) * att.size(), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(ctx->d_geometry, ctx->h_geometry.data(), sizeof(GeometryDev) * ctx->max_bodies, cudaMemcpyHostToDevice));
  ctx->n_attach = int(att.size());
  for (int r = 0; r < nr; ++r) {
    ctx->renderers[r].dev = devs[r];
    ctx->renderers[r].rendered = false;  // offsets / visible flags moved: read-back waits for the next render
  }
  ctx->n_geometry_list = int(geo.size());
  ctx->n_referenced_list = int(ref.size());
  ctx->render_dirty = false;
  return M3TB_OK;
}

// FocusedRenderer::StartRendering of the renderers of one RenderList: every device renderer (m3tb_render), those attached
// to a modality (Modality::correspondence_renderer_ptrs, before each correspondence iteration) or those attached to a
// region modality (RegionModality::start_modality_renderer_ptrs / results_renderer_ptrs; DepthModality has none there).
// One k_render launch; the images and the attached slots' records are current when the launch has run.
int LaunchRender(m3tb_ctx* ctx, int which) {
  int rc = SyncTables(ctx);  // pending body-table uploads go first: k_render then owns the attached records
  if (!rc) rc = SyncRenderTables(ctx);
  if (rc) return rc;
  const RefineSelection* sel = ctx->refine;
  const int n = sel ? sel->n_renderers[which] : ctx->render_n[which];
  const size_t smem = sel ? sel->render_smem[which] : ctx->render_smem[which];
  if (n == 0) return M3TB_OK;
  const int* d_list = ctx->d_render_lists + ctx->n_geometry_list + ctx->n_referenced_list;
  for (int k = 0; k < which; ++k) d_list += ctx->render_n[k];
  if (sel) d_list = sel->renderers[which];
  RenderArgs a;
  a.renderers = ctx->d_renderers;
  a.render_list = d_list;
  a.geometry = ctx->d_geometry;
  a.geometry_bodies = ctx->d_render_lists;
  a.referenced_bodies = ctx->d_render_lists + ctx->n_geometry_list;
  a.poses = ctx->d_poses;
  a.color_cams = ctx->d_ccams;
  a.depth_cams = ctx->d_dcams;
  a.out = ctx->d_render_out;
  a.visible = ctx->d_visible;
  a.bodies = ctx->d_bodies;
  a.attach = ctx->d_attach;
  a.n_attach = ctx->n_attach;
  CU(cudaFuncSetAttribute(k_render, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  k_render<<<unsigned(n), kRenderThreads, smem, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  for (int r : sel ? sel->renderer_ids[which] : ctx->render_list[which]) ctx->renderers[r].rendered = true;
  return M3TB_OK;
}

int SetModel(m3tb_ctx* ctx, bool region, int model_id, int n_views, int n_points, const float* orientations,
             const float* scalars, const void* points, float stride_depth_offset, float max_radius_depth_offset) {
  if (model_id < 0 || model_id >= ctx->max_models || n_views <= 0 || n_points <= 0 || !orientations || !points)
    return Fail(ctx, M3TB_ERR_INVALID, "bad model arguments");
  // what model generation refuses (CheckModelParams), and an infinite stride besides: a stride of 0, a negative or
  // non-finite one, or more than 30 depth offsets would give depth-offset ids outside the table
  if (!(stride_depth_offset > 0.0f) || !std::isfinite(stride_depth_offset) || !(max_radius_depth_offset >= 0.0f) ||
      !std::isfinite(max_radius_depth_offset) || int(max_radius_depth_offset / stride_depth_offset + 1.0f) > kDepthOffsets)
    return Fail(ctx, M3TB_ERR_INVALID, "bad model depth-offset parameters");
  // Repack the .bin AoS DataPoints (152 B / 144 B) into the 32 B records the kernels read:
  // region (cx,cy,cz,nx)(ny,nz,fg,bg), depth (cx,cy,cz,nx)(ny,nz,0,0). One-time setup, not on the hot path.
  const int fl = region ? M3TB_REGION_POINT_BYTES / 4 : M3TB_DEPTH_POINT_BYTES / 4;
  const float* src = static_cast<const float*>(points);
  std::vector<float> packed(size_t(n_views) * n_points * 8);
  for (size_t k = 0; k < size_t(n_views) * n_points; ++k) {
    const float* s = src + k * fl;
    float* d = packed.data() + k * 8;
    d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; d[3] = s[3]; d[4] = s[4]; d[5] = s[5];
    d[6] = region ? s[6] : 0.0f;
    d[7] = region ? s[7] : 0.0f;
  }
  // DataPoint::depth_offsets (30 floats per point) for the measured occlusion handling, kept as a separate table
  std::vector<float> offsets(size_t(n_views) * n_points * kDepthOffsets);
  for (size_t k = 0; k < size_t(n_views) * n_points; ++k)
    std::memcpy(offsets.data() + k * kDepthOffsets, src + k * fl + (region ? 8 : 6), sizeof(float) * kDepthOffsets);
  float radius2 = 0.0f;
  for (size_t k = 0; k < size_t(n_views) * n_points; ++k) {
    const float* d = packed.data() + k * 8;
    radius2 = std::max(radius2, d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  }
  std::vector<float> sc(n_views, 0.0f);
  float max_scalar = 0.0f;
  for (int v = 0; v < n_views; ++v) {
    if (scalars) sc[v] = scalars[v];
    max_scalar = std::max(max_scalar, sc[v]);
  }
  std::vector<float> ori4(size_t(n_views) * 4, 0.0f);
  for (int v = 0; v < n_views; ++v)
    for (int c = 0; c < 3; ++c) ori4[size_t(v) * 4 + c] = orientations[3 * v + c];
  // the new model is complete on the device before it replaces the old one (both exist for a moment)
  ModelAlloc al;
  CU(al.orientations.create(n_views));
  CU(al.view_scalars.create(n_views));
  CU(al.points.create(packed.size()));
  CU(al.depth_offsets.create(offsets.size()));
  CU(cudaMemcpyAsync(al.depth_offsets, offsets.data(), sizeof(float) * offsets.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(al.orientations, ori4.data(), sizeof(float4) * n_views, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(al.view_scalars, sc.data(), sizeof(float) * n_views, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(al.points, packed.data(), sizeof(float) * packed.size(), cudaMemcpyHostToDevice, ctx->stream));
  // cluster tables of the pruned closest-view search (one-time, host)
  ViewClustersHost vc;
  BuildViewClusters(orientations, n_views, vc);
  CU(al.cluster_info.create(std::max<size_t>(vc.info.size(), 8)));
  CU(al.sorted_views.create(vc.sorted.size()));
  CU(cudaMemcpyAsync(al.cluster_info, vc.info.data(), sizeof(float) * vc.info.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(al.sorted_views, vc.sorted.data(), sizeof(float) * vc.sorted.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));  // staging vectors go out of scope
  ModelDev& m = (region ? ctx->h_rmodels : ctx->h_dmodels)[model_id];
  m.n_views = n_views;
  m.n_points = n_points;
  m.orientations4 = al.orientations;
  m.view_scalars = al.view_scalars;
  m.points = reinterpret_cast<const float4*>(al.points.get());
  m.max_view_scalar = max_scalar;
  m.radius = std::sqrt(radius2);
  m.depth_offsets = al.depth_offsets;
  m.stride_depth_offset = stride_depth_offset;
  m.max_radius_depth_offset = max_radius_depth_offset;
  m.cluster_info = reinterpret_cast<const float4*>(al.cluster_info.get());
  m.sorted_views = reinterpret_cast<const float4*>(al.sorted_views.get());
  m.n_clusters = vc.n_clusters;
  m.set = 1;
  (region ? ctx->rmodel_alloc : ctx->dmodel_alloc)[model_id] = std::move(al);  // releases the old model
  ctx->models_dirty = true;
  return M3TB_OK;
}

int SetCamera(m3tb_ctx* ctx, bool color, int cam, const m3tb_intrinsics* in, const float* w2c, float depth_scale) {
  if (cam < 0 || cam >= ctx->max_cameras || !in || !w2c || in->width <= 0 || in->height <= 0)
    return Fail(ctx, M3TB_ERR_INVALID, "bad camera arguments");
  CameraDev& c = CameraOf(ctx, color, cam);
  const bool dims_changed = c.set && (c.width != in->width || c.height != in->height);
  c.fu = in->fu; c.fv = in->fv; c.ppu = in->ppu; c.ppv = in->ppv;
  c.width = in->width; c.height = in->height;
  std::memcpy(c.w2c, w2c, sizeof(float) * 12);
  c.depth_scale = depth_scale;
  if (dims_changed) {
    c.image = nullptr;
    ctx->undistort[color ? 0 : 1][cam] = {};  // the map was made for the old size
  }
  c.set = 1;
  ctx->cams_dirty = true;
  return M3TB_OK;
}

// Device storage of the frames of cameras [first, first + count): a slot of the shared pool when the dimensions match
// the pool's (so that a batch of frames is one contiguous copy), a private allocation otherwise. The first frame sets
// the pool's dimensions. The cameras change only once every allocation has succeeded.
int EnsureImages(m3tb_ctx* ctx, bool color, int first, int count) {
  std::vector<CameraDev>& cams = color ? ctx->h_ccams : ctx->h_dcams;
  ImagePool& pool = color ? ctx->color_pool : ctx->depth_pool;
  auto pitch_of = [&](const CameraDev& c) { return unsigned(Align(size_t(c.width) * (color ? 3 : 2), 16)); };
  ImagePool new_pool;
  const ImagePool* p = &pool;
  std::vector<DeviceBuffer<uint8_t>> priv(count);
  for (int k = 0; k < count; ++k) {
    const CameraDev& c = cams[first + k];
    if (!c.set) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "set the camera before uploading images");
    if (c.image) continue;
    if (!p->base) {
      new_pool.width = c.width; new_pool.height = c.height; new_pool.pitch = pitch_of(c);
      new_pool.frame_bytes = size_t(new_pool.pitch) * c.height;
      new_pool.capacity = ctx->max_cameras;
      CU(new_pool.base.create(new_pool.frame_bytes * new_pool.capacity));
      if (color && (c.width & 3) == 0) {
        new_pool.bin_pitch = unsigned(Align(size_t(c.width) * 2, 16));
        new_pool.bin_frame_bytes = size_t(new_pool.bin_pitch) * c.height;
        CU(new_pool.bins.create(new_pool.bin_frame_bytes * new_pool.capacity));
      }
      p = &new_pool;
    }
    if (p->width != c.width || p->height != c.height) CU(priv[k].create(size_t(pitch_of(c)) * c.height));
  }
  if (new_pool.base) pool = std::move(new_pool);
  for (int k = 0; k < count; ++k) {
    const int cam = first + k;
    CameraDev& c = cams[cam];
    if (c.image) continue;
    if (!priv[k]) {
      c.image = pool.base + pool.frame_bytes * cam;
      c.pitch = pool.pitch;
      if (color && pool.bins) {
        c.bins = pool.BinImage(cam);
        c.bin_pitch = pool.bin_pitch;
      }
    } else {
      c.bins = nullptr;
      c.bin_pitch = 0;
      c.image = priv[k];
      c.pitch = pitch_of(c);
      (color ? ctx->private_color : ctx->private_depth)[cam] = std::move(priv[k]);
    }
    ctx->cams_dirty = true;
  }
  return M3TB_OK;
}

// Device-visible alias of a pinned (page-locked, mapped) host pointer, or null for pageable / foreign memory.
const uint8_t* PinnedAlias(m3tb_ctx* ctx, const void* host) {
  if (!ctx->roi_ingest) return nullptr;
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, host) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  if (attr.type != cudaMemoryTypeHost || !attr.devicePointer) return nullptr;
  return static_cast<const uint8_t*>(attr.devicePointer);
}

// Camera::UpdateImage. Pinned host frames are NOT copied here: the camera records the frame (zero-copy alias) and
// the next consumer launch first runs k_ingest, which fetches only each body's ROI. The caller keeps the frame
// unchanged until the work that uses it has completed (m3tb_synchronize / m3tb_get_poses), exactly as for any
// asynchronous copy from pinned memory. Pageable frames and device frames are copied in full.
int UploadUndistorted(m3tb_ctx* ctx, bool color, const int* cams, const void* const* srcs, int n, size_t pitch,
                      bool on_device);

int Upload(m3tb_ctx* ctx, bool color, int cam, const void* src, size_t pitch, cudaMemcpyKind kind,
           const uint8_t* pinned_alias) {
  if (cam < 0 || cam >= ctx->max_cameras || !src) return Fail(ctx, M3TB_ERR_INVALID, "bad upload arguments");
  if (ctx->undistort[color ? 0 : 1][cam].map)
    return UploadUndistorted(ctx, color, &cam, &src, 1, pitch, kind == cudaMemcpyDeviceToDevice);
  int rc = EnsureImages(ctx, color, cam, 1);
  if (rc) return rc;
  CameraDev& c = CameraOf(ctx, color, cam);
  const size_t row = size_t(c.width) * (color ? 3 : 2);
  if (pitch < row) return Fail(ctx, M3TB_ERR_INVALID, "pitch smaller than a row");
  c.generation = (c.generation + 1) & 0x3fffffff;
  ctx->cams_dirty = true;
  if (pinned_alias) {
    c.host_src = pinned_alias;
    c.host_pitch = unsigned(pitch);
    ctx->ingest_pending = true;
    if (color) ctx->bin_shift[cam] = kBinsAtIngest;  // k_ingest writes the bin indices of every rectangle it fetches
    return M3TB_OK;
  }
  c.host_src = nullptr;
  c.host_pitch = 0;
  if (color) ctx->bin_shift[cam] = kBinsNone;
  CU(cudaMemcpy2DAsync(const_cast<uint8_t*>(c.image), c.pitch, src, pitch, row, c.height, kind, ctx->stream));
  return M3TB_OK;
}

int UploadBatch(m3tb_ctx* ctx, bool color, int first, int count, const void* src, size_t frame_stride, size_t pitch) {
  if (first < 0 || count <= 0 || first + count > ctx->max_cameras || !src)
    return Fail(ctx, M3TB_ERR_INVALID, "bad batch upload arguments");
  const uint8_t* s = static_cast<const uint8_t*>(src);
  {  // cameras with an undistortion: all of them in one k_undistort launch; the others as single uploads
    std::vector<int> und;
    std::vector<const void*> und_src;
    for (int k = 0; k < count; ++k)
      if (ctx->undistort[color ? 0 : 1][first + k].map) {
        und.push_back(first + k);
        und_src.push_back(s + frame_stride * k);
      }
    if (!und.empty()) {
      int rc = UploadUndistorted(ctx, color, und.data(), und_src.data(), int(und.size()), pitch, false);
      if (rc) return rc;
      for (int k = 0; k < count; ++k) {
        if (ctx->undistort[color ? 0 : 1][first + k].map) continue;
        const uint8_t* f = s + frame_stride * k;
        rc = Upload(ctx, color, first + k, f, pitch, cudaMemcpyHostToDevice, PinnedAlias(ctx, f));
        if (rc) return rc;
      }
      return M3TB_OK;
    }
  }
  ImagePool& pool = color ? ctx->color_pool : ctx->depth_pool;
  int rc = EnsureImages(ctx, color, first, count);
  if (rc) return rc;
  bool pooled = true;
  for (int k = 0; k < count; ++k) {
    const CameraDev& c = CameraOf(ctx, color, first + k);
    pooled = pooled && pool.base && c.image == pool.base + pool.frame_bytes * (first + k);
  }
  if (const uint8_t* alias = PinnedAlias(ctx, src)) {
    for (int k = 0; k < count; ++k) {
      int rc = Upload(ctx, color, first + k, s + frame_stride * k, pitch, cudaMemcpyHostToDevice, alias + frame_stride * k);
      if (rc) return rc;
    }
    return M3TB_OK;
  }
  for (int k = 0; k < count; ++k) {
    CameraDev& c = CameraOf(ctx, color, first + k);
    c.host_src = nullptr; c.host_pitch = 0; c.generation = (c.generation + 1) & 0x3fffffff;
    if (color) ctx->bin_shift[first + k] = kBinsNone;
  }
  ctx->cams_dirty = true;
  if (pooled && frame_stride == pitch * size_t(pool.height)) {
    const size_t row = size_t(pool.width) * (color ? 3 : 2);
    uint8_t* dst = pool.base + pool.frame_bytes * first;
    if (pitch == pool.pitch) {
      CU(cudaMemcpyAsync(dst, s, pool.frame_bytes * count, cudaMemcpyHostToDevice, ctx->stream));
    } else {
      CU(cudaMemcpy2DAsync(dst, pool.pitch, s, pitch, row, size_t(pool.height) * count, cudaMemcpyHostToDevice,
                           ctx->stream));
    }
    return M3TB_OK;
  }
  for (int k = 0; k < count; ++k) {
    int rc = Upload(ctx, color, first + k, s + frame_stride * k, pitch, cudaMemcpyHostToDevice, nullptr);
    if (rc) return rc;
  }
  return M3TB_OK;
}

// Camera::UpdateImage of an AzureKinect camera: the raw frames of cameras cams[0..n) (srcs[k], `pitch` bytes per row)
// are rectified into the cameras' device copies by one k_undistort launch (one per kUndistortMaxJobs frames). Device
// frames are read where they are. Host frames, pageable or pinned, first go to a staging buffer by DMA: k_undistort's
// gather would otherwise cross PCIe in small scattered reads (scripts/undistortion_timing.py measures both). Afterwards
// the cameras refer to no host memory, as after a pageable copy.
int UploadUndistorted(m3tb_ctx* ctx, bool color, const int* cams, const void* const* srcs, int n, size_t pitch,
                      bool on_device) {
  auto& U = ctx->undistort[color ? 0 : 1];
  std::vector<CameraDev>& C = color ? ctx->h_ccams : ctx->h_dcams;
  std::vector<size_t> offset(n, 0);
  size_t staging = 0;
  for (int k = 0; k < n; ++k) {
    const CameraDev& c = C[cams[k]];
    const size_t row = size_t(c.width) * (color ? U[cams[k]].channels : 2);
    if (pitch < row) return Fail(ctx, M3TB_ERR_INVALID, "pitch smaller than a raw row");
    if (!color && ((reinterpret_cast<uintptr_t>(srcs[k]) | pitch) & 1))
      return Fail(ctx, M3TB_ERR_INVALID, "depth frame not aligned to 2 bytes");
    offset[k] = staging;
    if (!on_device) staging += Align(row, 16) * size_t(c.height);
  }
  // staging first: a failed allocation leaves the cameras as they were
  if (staging > ctx->undistort_staging.size()) CU(ctx->undistort_staging.create(staging));
  for (int k = 0; k < n; ++k) {
    int rc = EnsureImages(ctx, color, cams[k], 1);
    if (rc) return rc;
  }
  // a prefetched ingest may still write the device copies
  if (ctx->prefetched) CU(cudaStreamWaitEvent(ctx->stream, ctx->pf.ev_ingest_done, 0));
  UndistortArgs a;
  a.n_jobs = 0;
  unsigned blocks = 0;
  auto launch = [&]() -> int {
    k_undistort<<<dim3(blocks, unsigned(a.n_jobs)), kUndistortThreads, 0, ctx->stream>>>(a);
    CU(cudaGetLastError());
    ctx->launches++;
    a.n_jobs = 0;
    blocks = 0;
    return M3TB_OK;
  };
  for (int k = 0; k < n; ++k) {
    const int cam = cams[k];
    CameraDev& c = C[cam];
    const auto& u = U[cam];
    UndistortJob& j = a.jobs[a.n_jobs++];
    j.map = u.map;
    j.map_pitch = u.map_pitch;
    j.width = c.width;
    j.height = c.height;
    j.channels = u.channels;
    j.offset = u.offset;
    j.dst = const_cast<uint8_t*>(c.image);
    j.dst_pitch = c.pitch;
    if (on_device) {
      j.src = static_cast<const uint8_t*>(srcs[k]);
      j.src_pitch = unsigned(pitch);
    } else {
      const size_t row = size_t(c.width) * (color ? u.channels : 2);
      j.src = ctx->undistort_staging + offset[k];
      j.src_pitch = unsigned(Align(row, 16));
      CU(cudaMemcpy2DAsync(const_cast<uint8_t*>(j.src), j.src_pitch, srcs[k], pitch, row, c.height,
                           cudaMemcpyHostToDevice, ctx->stream));
    }
    const size_t threads = size_t((c.width + kUndistortPixels - 1) / kUndistortPixels) * size_t(c.height);
    blocks = std::max(blocks, unsigned((threads + kUndistortThreads - 1) / kUndistortThreads));
    c.host_src = nullptr;
    c.host_pitch = 0;
    c.generation = (c.generation + 1) & 0x3fffffff;
    if (color) ctx->bin_shift[cam] = kBinsNone;  // k_bin rebuilds the bin indices, as after a pageable copy
    if (a.n_jobs == kUndistortMaxJobs) {
      int rc = launch();
      if (rc) return rc;
    }
  }
  ctx->cams_dirty = true;
  if (a.n_jobs) return launch();
  return M3TB_OK;
}

// ---- depth-model generation (m3tb_generate_depth_model) -------------------------------------------------------------
// Host side: parameters, geodesic views and the per-view transforms, in float32 with the reference's expressions.

constexpr int kImageSizeSafetyBoundary = 20;    // model.h:57
constexpr float kMinimumClipSpaceRatio = 0.2f;  // model.h:59
constexpr unsigned kModelSeed = 7;              // std::mt19937 generator{7} (depth_model.cpp:317, region_model.cpp:513)
constexpr int kRegionBackgroundID = 0, kRegionDifferentBodyID = 120, kRegionMainBodyID = 255;  // region_model.h:67-70
constexpr int kModelMaxImageSize = 8192;        // two 8192^2 z-buffers of 8 B are the whole scratch bound of a depth
                                                // view; region generation refuses views that need more
constexpr int kModelMaxDivides = 8;
constexpr float kViewerZMin = 0.02f, kViewerZMax = 10.0f;  // FullNormalRenderer defaults (normal_renderer.h:84-93)

using Vec3 = std::array<float, 3>;

struct SmallerVec3 {  // Model::CompareSmallerVector3f (model.h:62-67)
  bool operator()(const Vec3& a, const Vec3& b) const {
    return a[0] < b[0] || (a[0] == b[0] && a[1] < b[1]) || (a[0] == b[0] && a[1] == b[1] && a[2] < b[2]);
  }
};

Vec3 Normalized(const Vec3& v) {  // Eigen normalized(): v / sqrt(squaredNorm), unchanged if the norm is 0
  const float n = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  if (!(n > 0.0f)) return v;
  const float s = std::sqrt(n);
  return {v[0] / s, v[1] / s, v[2] / s};
}

Vec3 Cross(const Vec3& a, const Vec3& b) {
  return {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
}

void SubdivideTriangle(const Vec3& v1, const Vec3& v2, const Vec3& v3, int n, std::set<Vec3, SmallerVec3>& points) {
  if (n == 0) {
    points.insert(v1);
    points.insert(v2);
    points.insert(v3);
    return;
  }
  const Vec3 v12 = Normalized({v1[0] + v2[0], v1[1] + v2[1], v1[2] + v2[2]});
  const Vec3 v13 = Normalized({v1[0] + v3[0], v1[1] + v3[1], v1[2] + v3[2]});
  const Vec3 v23 = Normalized({v2[0] + v3[0], v2[1] + v3[1], v2[2] + v3[2]});
  SubdivideTriangle(v1, v12, v13, n - 1, points);
  SubdivideTriangle(v2, v12, v23, n - 1, points);
  SubdivideTriangle(v3, v13, v23, n - 1, points);
  SubdivideTriangle(v12, v13, v23, n - 1, points);
}

// Model::GenerateGeodesicPoints / GenerateGeodesicPoses (model.cpp:386-454): camera2body [n][12], row-major 3x4
std::vector<float> GeodesicPoses(int n_divides, float sphere_radius) {
  const float x = 0.525731112119133606f, z = 0.850650808352039932f;
  const Vec3 ico[12] = {{-x, 0.0f, z}, {x, 0.0f, z},  {-x, 0.0f, -z}, {x, 0.0f, -z}, {0.0f, z, x},  {0.0f, z, -x},
                        {0.0f, -z, x}, {0.0f, -z, -x}, {z, x, 0.0f},  {-z, x, 0.0f}, {z, -x, 0.0f}, {-z, -x, 0.0f}};
  const int ids[20][3] = {{0, 4, 1},  {0, 9, 4},  {9, 5, 4},  {4, 5, 8},  {4, 8, 1},  {8, 10, 1}, {8, 3, 10},
                          {5, 3, 8},  {5, 2, 3},  {2, 7, 3},  {7, 10, 3}, {7, 6, 10}, {7, 11, 6}, {11, 0, 6},
                          {0, 1, 6},  {6, 1, 10}, {9, 0, 11}, {9, 11, 2}, {9, 2, 5},  {7, 2, 11}};
  std::set<Vec3, SmallerVec3> points;
  for (const auto& t : ids) SubdivideTriangle(ico[t[0]], ico[t[1]], ico[t[2]], n_divides, points);
  std::vector<float> poses;
  poses.reserve(points.size() * 12);
  for (const Vec3& p : points) {
    const Vec3 c2 = {-p[0], -p[1], -p[2]};
    const Vec3 c0 = (p[0] == 0.0f && p[2] == 0.0f) ? Vec3{1.0f, 0.0f, 0.0f} : Normalized(Cross({0.0f, 1.0f, 0.0f}, c2));
    const Vec3 c1 = Cross(c2, c0);
    for (int r = 0; r < 3; ++r) {
      const float row[4] = {c0[r], c1[r], c2[r], p[r] * sphere_radius};
      poses.insert(poses.end(), row, row + 4);
    }
  }
  return poses;
}

// Checks the model parameters (Model::DepthOffsetVariablesValid, model.cpp:325-336)
int CheckModelParams(m3tb_ctx* ctx, const m3tb_model_params* p) {
  if (!p) return Fail(ctx, M3TB_ERR_INVALID, "null model parameters");
  if (p->use_random_seed) return Fail(ctx, M3TB_ERR_UNSUPPORTED, "use_random_seed: the reference seeds from the clock");
  if (!(p->sphere_radius > 0.0f) || !std::isfinite(p->sphere_radius) || p->n_divides < 0 ||
      p->n_divides > kModelMaxDivides || p->n_points < 1 || !(p->stride_depth_offset > 0.0f) ||
      !(p->max_radius_depth_offset >= 0.0f) || !std::isfinite(p->max_radius_depth_offset) ||
      p->image_size <= kImageSizeSafetyBoundary || p->image_size > kModelMaxImageSize)
    return Fail(ctx, M3TB_ERR_INVALID, "bad model parameters");
  if (int(p->max_radius_depth_offset / p->stride_depth_offset + 1.0f) > kModelMaxOffsets)
    return Fail(ctx, M3TB_ERR_INVALID, "max_radius_depth_offset / stride_depth_offset is above 30");
  return M3TB_OK;
}

// What one generation renders: the full renderers' intrinsics and projection, the renderer table, and per view the
// camera2body pose, the clip-space matrix of every draw and the main body's world2camera * geometry2world rotation.
struct ModelSetup {
  int S = 0, n_views = 0, n_renderers = 1, n_draws = 1, max_triangles = 0;
  int first[kModelMaxRenderers + 1] = {};
  int r_same = -1, r_occ = -1, r_fg = -1, r_bg = -1;  // region renderers, -1 when not used
  float fu = 0.0f, pp = 0.0f, projection_term_a = 0.0f, projection_term_b = 0.0f;
  std::vector<float> camera2body, M, rot, face_normals;
  std::vector<ModelBodyDev> draws;
};

struct ModelDraw {
  int body, id;
};

// Model::SetUpRenderer / AddBodiesToRenderer (model.cpp:120-196) for a table of full renderers. Every renderer is set
// up for `body` (its intrinsics, and a z range that starts from it) and widened over the bodies it draws; renderer 0
// gives the depth image and the normal rotation. The parameters and `body` have been checked by the caller.
int PrepareRenderers(m3tb_ctx* ctx, int body, const std::vector<std::vector<ModelDraw>>& renderers,
                     const m3tb_model_params* p, ModelSetup& st) {
  // the radius is 0.5f * diameter, exactly
  const float r = p->sphere_radius;
  const GeometryDev& G = ctx->h_geometry[body];
  const float z_min = r - G.radius, z_max = r + G.radius;
  if (z_min < r * kMinimumClipSpaceRatio) return Fail(ctx, M3TB_ERR_INVALID, "z_min of the body below 0.2 * sphere_radius");
  const int n_renderers = int(renderers.size());
  std::vector<float> P22(n_renderers), P23(n_renderers);
  st.draws.clear();
  for (int q = 0; q < n_renderers; ++q) {
    float lo_min = z_min, hi_max = z_max;
    st.first[q] = int(st.draws.size());
    for (const ModelDraw& d : renderers[q]) {
      const GeometryDev& B = ctx->h_geometry[d.body];
      const float lo = r - B.radius, hi = r + B.radius;
      if (lo < r * kMinimumClipSpaceRatio)
        return Fail(ctx, M3TB_ERR_INVALID, "z_min of body " + std::to_string(d.body) + " below 0.2 * sphere_radius");
      lo_min = std::min(lo, lo_min);
      hi_max = std::max(hi, hi_max);
      st.draws.push_back({B.triangles, B.n_triangles, B.enable_culling, d.id});
      st.max_triangles = std::max(st.max_triangles, B.n_triangles);
    }
    // FullRenderer::CalculateProjectionMatrix (renderer.cpp:257-263)
    P22[q] = (hi_max + lo_min) / (hi_max - lo_min);
    P23[q] = -2.0f * hi_max * lo_min / (hi_max - lo_min);
    if (q == 0) {  // FullDepthRenderer (renderer.cpp:476-477) of the main renderer
      st.projection_term_a = hi_max * lo_min * 65535.0f / (hi_max - lo_min);
      st.projection_term_b = hi_max * 65535.0f / (hi_max - lo_min);
    }
  }
  st.first[n_renderers] = int(st.draws.size());
  st.S = p->image_size;
  st.n_renderers = n_renderers;
  st.n_draws = int(st.draws.size());
  st.fu = 0.5f * float(st.S - kImageSizeSafetyBoundary) / tanf(asinf(G.radius / r));
  st.pp = float(st.S) / 2.0f;
  const float fS = float(st.S);
  const float P00 = 2.0f * st.fu / fS, P02 = 2.0f * (st.pp + 0.5f) / fS - 1.0f;
  const float P11 = P00, P12 = P02;  // fv = fu, ppv = ppu, height = width

  // face normals of the body (RendererGeometry::AssembleVertexData, renderer_geometry.cpp:199-200)
  std::vector<float> tri(size_t(G.n_triangles) * 9);
  CU(cudaMemcpy(tri.data(), G.triangles, sizeof(float) * tri.size(), cudaMemcpyDeviceToHost));
  st.face_normals.resize(size_t(G.n_triangles) * 3);
  for (int t = 0; t < G.n_triangles; ++t) {
    const float* v = tri.data() + 9 * size_t(t);
    const Vec3 a = {v[6] - v[3], v[7] - v[4], v[8] - v[5]}, b = {v[0] - v[3], v[1] - v[4], v[2] - v[5]};
    const Vec3 n = Normalized(Cross(a, b));
    std::memcpy(st.face_normals.data() + 3 * size_t(t), n.data(), sizeof(float) * 3);
  }

  st.camera2body = GeodesicPoses(p->n_divides, r);
  st.n_views = int(st.camera2body.size() / 12);
  st.M.assign(size_t(st.n_views) * st.n_draws * 16, 0.0f);
  st.rot.assign(size_t(st.n_views) * 9, 0.0f);
  for (int v = 0; v < st.n_views; ++v) {
    float w2c[12];
    PoseInverse(st.camera2body.data() + 12 * size_t(v), w2c);  // Renderer::set_camera2world_pose, body2world = I
    for (int q = 0; q < n_renderers; ++q)
      for (int k = 0; k < int(renderers[q].size()); ++k) {
        const int d = st.first[q] + k;
        float T[12];
        PoseMul(w2c, ctx->h_geometry[renderers[q][k].body].geometry2body, T);  // world2camera * geometry2world
        float* M = st.M.data() + (size_t(v) * st.n_draws + d) * 16;
        for (int c = 0; c < 4; ++c) {  // P * [T; 0 0 0 1] without the products with P's zero entries, as k_render
          M[c] = P00 * T[c] + P02 * T[8 + c];
          M[4 + c] = P11 * T[4 + c] + P12 * T[8 + c];
          M[8 + c] = P22[q] * T[8 + c];
          M[12 + c] = T[8 + c];
        }
        M[11] = M[11] + P23[q];
        if (d == 0)
          for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) st.rot[9 * size_t(v) + 3 * i + j] = T[4 * i + j];
      }
  }
  return M3TB_OK;
}

// DepthModel::GenerateModel's renderers: the body alone (main), and the body in front of the occlusion bodies
int PrepareModel(m3tb_ctx* ctx, int body, const int* occlusion_bodies, int n_occlusion, const m3tb_model_params* p,
                 ModelSetup& st) {
  int rc = CheckModelParams(ctx, p);
  if (rc) return rc;
  if (body < 0 || body >= ctx->max_bodies || !ctx->h_geometry[body].set)
    return Fail(ctx, M3TB_ERR_INVALID, "body has no geometry (m3tb_set_body_geometry)");
  if (n_occlusion < 0 || (n_occlusion > 0 && !occlusion_bodies) || n_occlusion >= 65535)
    return Fail(ctx, M3TB_ERR_INVALID, "bad occlusion body list");
  for (int k = 0; k < n_occlusion; ++k) {
    const int b = occlusion_bodies[k];
    if (b < 0 || b >= ctx->max_bodies || !ctx->h_geometry[b].set)
      return Fail(ctx, M3TB_ERR_INVALID, "occlusion body " + std::to_string(b) + " has no geometry");
    if (b == body) return Fail(ctx, M3TB_ERR_INVALID, "the body is its own occlusion body");
    for (int q = 0; q < k; ++q)
      if (occlusion_bodies[q] == b) return Fail(ctx, M3TB_ERR_INVALID, "occlusion body listed twice");
  }
  std::vector<std::vector<ModelDraw>> renderers = {{{body, kRegionMainBodyID}}};
  if (n_occlusion > 0) {  // depth_model.cpp:171-178
    renderers.push_back({{body, kRegionMainBodyID}});
    for (int k = 0; k < n_occlusion; ++k) renderers[1].push_back({occlusion_bodies[k], kRegionBackgroundID});
  }
  return PrepareRenderers(ctx, body, renderers, p, st);
}

int RegionCap(int S) { return kRegionContourCapPerPixel * S; }

size_t RegionViewBytes(int S, int n_points) {
  const size_t cap = size_t(RegionCap(S)), starts = cap / kRegionMinContourLength + 2;
  return size_t(S + 2) * (S + 2) + 3 * cap * sizeof(uint32_t) + 2 * starts * sizeof(int) + 2 * sizeof(int) +
         size_t(n_points) * 3 * sizeof(float);
}

// RegionModel::GenerateModel's renderers (region_model.cpp:187-257,365-464): main (body 255, fixed bodies 120), then,
// each only when used, same-region, occlusion, foreground and background. The associated bodies keep their insertion
// order within each of the four groups (RegionModel::AddAssociatedBody).
int PrepareRegionModel(m3tb_ctx* ctx, int body, const m3tb_associated_body* associated, int n_associated,
                       const m3tb_model_params* p, ModelSetup& st) {
  int rc = CheckModelParams(ctx, p);
  if (rc) return rc;
  if (body < 0 || body >= ctx->max_bodies || !ctx->h_geometry[body].set)
    return Fail(ctx, M3TB_ERR_INVALID, "body has no geometry (m3tb_set_body_geometry)");
  if (n_associated < 0 || (n_associated > 0 && !associated) || n_associated >= 65535)
    return Fail(ctx, M3TB_ERR_INVALID, "bad associated body list");
  std::vector<ModelDraw> fixed, fixed_same, movable, movable_same;
  for (int k = 0; k < n_associated; ++k) {
    const int b = associated[k].body;
    if (b < 0 || b >= ctx->max_bodies || !ctx->h_geometry[b].set)
      return Fail(ctx, M3TB_ERR_INVALID, "associated body " + std::to_string(b) + " has no geometry");
    if (b == body) return Fail(ctx, M3TB_ERR_INVALID, "the body is its own associated body");
    for (int q = 0; q < k; ++q)
      if (associated[q].body == b) return Fail(ctx, M3TB_ERR_INVALID, "associated body listed twice");
    auto& group = associated[k].movable ? (associated[k].same_region ? movable_same : movable)
                                        : (associated[k].same_region ? fixed_same : fixed);
    group.push_back({b, 0});
  }
  auto add = [](std::vector<ModelDraw>& r, const std::vector<ModelDraw>& bodies, int id) {
    for (const ModelDraw& d : bodies) r.push_back({d.body, id});
  };
  const int B = kRegionBackgroundID, M = kRegionMainBodyID;
  std::vector<std::vector<ModelDraw>> renderers(1);
  renderers[0].push_back({body, M});
  add(renderers[0], fixed, kRegionDifferentBodyID);
  if (!fixed_same.empty() || !movable_same.empty()) {
    st.r_same = int(renderers.size());
    std::vector<ModelDraw> r = {{body, B}};
    add(r, fixed, B);
    add(r, fixed_same, M);
    add(r, movable_same, M);
    renderers.push_back(r);
  }
  if (!movable.empty()) {
    st.r_occ = int(renderers.size());
    std::vector<ModelDraw> r = {{body, B}};
    add(r, fixed, B);
    add(r, movable, M);
    renderers.push_back(r);
  }
  if (!movable.empty() || !fixed_same.empty() || !movable_same.empty()) {
    st.r_fg = int(renderers.size());
    std::vector<ModelDraw> f = {{body, M}};
    add(f, fixed, B);
    add(f, movable, B);
    add(f, fixed_same, M);
    renderers.push_back(f);
    st.r_bg = int(renderers.size());
    std::vector<ModelDraw> g = {{body, M}};
    add(g, fixed, B);
    add(g, fixed_same, M);
    add(g, movable_same, M);
    renderers.push_back(g);
  }
  rc = PrepareRenderers(ctx, body, renderers, p, st);
  if (rc) return rc;
  // one view's z-buffers and contour scratch must fit the scratch bound (a batch holds at least one view)
  const size_t view_bytes = size_t(st.n_renderers) * st.S * st.S * sizeof(uint64_t) + RegionViewBytes(st.S, p->n_points);
  if (view_bytes > kModelScratchBytes)
    return Fail(ctx, M3TB_ERR_INVALID, "one view of " + std::to_string(st.n_renderers) + " renderers at image_size " +
                                           std::to_string(st.S) + " needs more than 1 GiB of scratch");
  return M3TB_OK;
}

ModelRenderers RendererTable(const ModelSetup& st, const ModelBodyDev* d_draws) {
  ModelRenderers R;
  R.draws = d_draws;
  for (int q = 0; q <= kModelMaxRenderers; ++q) R.first[q] = q <= st.n_renderers ? st.first[q] : st.first[st.n_renderers];
  R.n_renderers = st.n_renderers;
  return R;
}

// Device buffers of one generation call, released when it returns
struct ModelBuffers {
  DeviceBuffer<uint64_t> zbuf;
  DeviceBuffer<float> M, rot, camera2body, face_normals, points, surface_area;
  DeviceBuffer<int> coords;
  DeviceBuffer<ModelBodyDev> bodies;
  int batch = 0;
};

// Allocates the buffers for views [first, first + n_views) of `st` (points only when n_points > 0) and uploads their
// tables; view k of the buffers is view first + k of `st`. extra_view_bytes is the caller's own scratch per view of a
// batch, counted against the same bound as the z-buffers.
int AllocModel(m3tb_ctx* ctx, const ModelSetup& st, int first, int n_views, int n_points, ModelBuffers& b,
               size_t extra_view_bytes = 0) {
  const size_t view_bytes = size_t(st.n_renderers) * st.S * st.S * sizeof(uint64_t);
  b.batch = int(std::max<size_t>(
      1, std::min<size_t>({size_t(n_views), kModelScratchBytes / (view_bytes + extra_view_bytes), 65535})));
  const size_t nm = size_t(n_views) * st.n_draws * 16, nr = size_t(n_views) * 9, nc = size_t(n_views) * 12;
  CU(b.zbuf.create(view_bytes / sizeof(uint64_t) * b.batch));
  CU(b.M.create(nm));
  CU(b.rot.create(nr));
  CU(b.camera2body.create(nc));
  CU(b.face_normals.create(st.face_normals.size()));
  CU(b.bodies.create(st.draws.size()));
  CU(cudaMemcpy(b.M, st.M.data() + size_t(first) * st.n_draws * 16, sizeof(float) * nm, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(b.rot, st.rot.data() + size_t(first) * 9, sizeof(float) * nr, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(b.camera2body, st.camera2body.data() + size_t(first) * 12, sizeof(float) * nc, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(b.face_normals, st.face_normals.data(), sizeof(float) * st.face_normals.size(), cudaMemcpyHostToDevice));
  CU(cudaMemcpy(b.bodies, st.draws.data(), sizeof(ModelBodyDev) * st.draws.size(), cudaMemcpyHostToDevice));
  if (n_points > 0) {
    CU(b.coords.create(size_t(b.batch) * n_points));
    CU(b.points.create(36 * size_t(n_views) * n_points));
    CU(b.surface_area.create(n_views));
  }
  return M3TB_OK;
}

// Renders views [first, first + count) into the z-buffers (k_model_raster)
int RenderModelViews(m3tb_ctx* ctx, const ModelSetup& st, const ModelBuffers& b, int first, int count) {
  const size_t view_bytes = size_t(st.n_renderers) * st.S * st.S * sizeof(uint64_t);
  CU(cudaMemsetAsync(b.zbuf, 0xff, view_bytes * count, ctx->stream));  // glClear
  ModelRasterArgs ra;
  ra.R = RendererTable(st, b.bodies);
  ra.n_draws = st.n_draws;
  ra.M = b.M + size_t(first) * st.n_draws * 16;
  ra.zbuf = b.zbuf;
  ra.image_size = st.S;
  const dim3 grid(unsigned((st.max_triangles + kModelTrianglesPerCta - 1) / kModelTrianglesPerCta), unsigned(count),
                  unsigned(st.n_renderers));
  k_model_raster<<<grid, kModelThreads, 0, ctx->stream>>>(ra);
  CU(cudaGetLastError());
  ctx->launches++;
  return M3TB_OK;
}

ModelPointArgs PointArgs(const ModelSetup& st, const ModelBuffers& b, const m3tb_model_params* p, int first) {
  ModelPointArgs a;
  a.zbuf = b.zbuf;
  a.n_renderers = st.n_renderers;
  a.image_size = st.S;
  a.face_normals = b.face_normals;
  a.rot = b.rot + 9 * size_t(first);
  a.camera2body = b.camera2body + 12 * size_t(first);
  a.fu = a.fv = st.fu;
  a.ppu = a.ppv = st.pp;
  a.projection_term_a = st.projection_term_a;
  a.projection_term_b = st.projection_term_b;
  a.sphere_radius = p->sphere_radius;
  a.stride_depth_offset = p->stride_depth_offset;
  a.n_values = int(p->max_radius_depth_offset / p->stride_depth_offset + 1.0f);  // model.cpp:343
  a.n_points = p->n_points;
  a.seed = kModelSeed;
  a.coords = b.coords;
  a.points = b.points ? b.points + 36 * size_t(first) * p->n_points : nullptr;
  a.surface_area = b.surface_area ? b.surface_area + first : nullptr;
  return a;
}


// Scratch of region-model generation for one batch (k_region_contours / k_region_points)
struct RegionBuffers {
  DeviceBuffer<int8_t> label;
  DeviceBuffer<uint32_t> raw, contour, valid;
  DeviceBuffer<int> raw_start, contour_start, counts, coords, overflow;
  DeviceBuffer<float> normals, points, contour_length;
  int cap = 0;
};

int AllocRegion(m3tb_ctx* ctx, const ModelSetup& st, int batch, int n_views, int n_points, RegionBuffers& rb) {
  rb.cap = RegionCap(st.S);
  const size_t cap = size_t(rb.cap), starts = cap / kRegionMinContourLength + 2;
  CU(rb.label.create(size_t(batch) * (st.S + 2) * (st.S + 2)));
  CU(rb.raw.create(size_t(batch) * cap));
  CU(rb.contour.create(size_t(batch) * cap));
  CU(rb.valid.create(size_t(batch) * cap));
  CU(rb.raw_start.create(size_t(batch) * starts));
  CU(rb.contour_start.create(size_t(batch) * starts));
  CU(rb.counts.create(2 * size_t(batch)));
  CU(rb.overflow.create(1));
  CU(cudaMemset(rb.overflow, 0, sizeof(int)));
  if (n_points > 0) {
    CU(rb.coords.create(size_t(batch) * n_points));
    CU(rb.normals.create(2 * size_t(batch) * n_points));
    CU(rb.points.create(size_t(kRegionPointFloats) * n_views * n_points));
    CU(rb.contour_length.create(n_views));
  }
  return M3TB_OK;
}

RegionContourArgs ContourArgs(const ModelSetup& st, const ModelBuffers& b, const RegionBuffers& rb) {
  RegionContourArgs a;
  a.zbuf = b.zbuf;
  a.R = RendererTable(st, b.bodies);
  a.image_size = st.S;
  a.label = rb.label;
  a.raw = rb.raw;
  a.raw_start = rb.raw_start;
  a.contour = rb.contour;
  a.contour_start = rb.contour_start;
  a.counts = rb.counts;
  a.cap = rb.cap;
  a.overflow = rb.overflow;
  return a;
}

RegionPointArgs RegionArgs(const ModelSetup& st, const ModelBuffers& b, const RegionBuffers& rb,
                           const m3tb_model_params* p, int first) {
  RegionPointArgs a;
  a.zbuf = b.zbuf;
  a.R = RendererTable(st, b.bodies);
  a.r_same = st.r_same;
  a.r_occ = st.r_occ;
  a.r_fg = st.r_fg;
  a.r_bg = st.r_bg;
  a.image_size = st.S;
  a.contour = rb.contour;
  a.contour_start = rb.contour_start;
  a.counts = rb.counts;
  a.cap = rb.cap;
  a.valid = rb.valid;
  a.coords = rb.coords;
  a.normals = rb.normals;
  a.camera2body = b.camera2body + 12 * size_t(first);
  a.fu = a.fv = st.fu;
  a.ppu = a.ppv = st.pp;
  a.projection_term_a = st.projection_term_a;
  a.projection_term_b = st.projection_term_b;
  a.sphere_radius = p->sphere_radius;
  a.stride_depth_offset = p->stride_depth_offset;
  a.n_values = int(p->max_radius_depth_offset / p->stride_depth_offset + 1.0f);  // model.cpp:343
  a.n_points = p->n_points;
  a.seed = kModelSeed;
  a.points = rb.points + size_t(kRegionPointFloats) * first * p->n_points;
  a.contour_length = rb.contour_length + first;
  return a;
}

int ContourOverflow(m3tb_ctx* ctx, const RegionBuffers& rb) {
  int overflow = 0;
  CU(cudaMemcpyAsync(&overflow, rb.overflow, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (overflow)
    return Fail(ctx, M3TB_ERR_UNSUPPORTED, "the contours of a view exceed " + std::to_string(rb.cap) +
                                               " points (64 * image_size); the model is unchanged");
  return M3TB_OK;
}

}  // namespace

namespace {
// m3tb_debug_rigid_solve: one warp per system runs the rigid-body solve (SolveAndUpdateSerial) itself, on k_track's
// shared-memory layout (Shared) or k_track2's (Shared2), on the system as the kernels leave it in shared memory (sh.a
// full symmetric), with no camera to refresh pose products for.
template <class Sh>
__global__ void __launch_bounds__(32) k_debug_rigid_solve(const float* __restrict__ a, const float* __restrict__ b,
                                                          float* __restrict__ poses, float* __restrict__ theta,
                                                          int* __restrict__ updated) {
  __shared__ Sh sh;
  const int s = blockIdx.x, lane = threadIdx.x;
  for (int e = lane; e < 36; e += 32) {
    const int i = e / 6, j = e - 6 * (e / 6);
    sh.a[e] = a[36 * s + (i >= j ? 6 * i + j : 6 * j + i)];  // the lower triangle, mirrored
  }
  if (lane < 6) sh.b[lane] = b[6 * s + lane];
  if (lane < 12) sh.pose[lane] = poses[12 * s + lane];
  __syncwarp();
  const bool ok = SolveAndUpdateSerial(sh, false, false);
  __syncwarp();
  if (lane < 6) theta[6 * s + lane] = sh.x[lane];
  if (lane < 12) poses[12 * s + lane] = sh.pose[lane];
  if (lane == 0) updated[s] = ok ? 1 : 0;
}
}  // namespace

extern "C" {

void m3tb_region_params_default(m3tb_region_params* p) {
  std::memset(p, 0, sizeof(*p));
  p->n_lines_max = 200;
  p->min_continuous_distance = 3.0f;
  p->function_length = 8;
  p->distribution_length = 12;
  p->function_amplitude = 0.43f;
  p->function_slope = 0.5f;
  p->learning_rate = 1.3f;
  p->n_global_iterations = 1;
  p->n_scales = 4;
  const int s[4] = {6, 4, 2, 1};
  const float sd[4] = {15.0f, 5.0f, 3.5f, 1.5f};
  for (int i = 0; i < 4; ++i) { p->scales[i] = s[i]; p->standard_deviations[i] = sd[i]; }
  p->n_standard_deviations = 4;
  p->n_histogram_bins = 16;
  p->learning_rate_f = 0.2f;
  p->learning_rate_b = 0.2f;
  p->unconsidered_line_length = 0.5f;
  p->max_considered_line_length = 20.0f;
  p->measured_depth_offset_radius = 0.01f;
  p->measured_occlusion_radius = 0.01f;
  p->measured_occlusion_threshold = 0.03f;
  p->n_unoccluded_iterations = 10;
  p->min_n_unoccluded_lines = 0;
  p->modeled_depth_offset_radius = 0.01f;
  p->modeled_occlusion_radius = 0.01f;
  p->modeled_occlusion_threshold = 0.03f;
}

void m3tb_depth_params_default(m3tb_depth_params* p) {
  std::memset(p, 0, sizeof(*p));
  p->n_points_max = 200;
  p->stride_length = 0.005f;
  p->n_considered_distances = 3;
  const float cd[3] = {0.05f, 0.02f, 0.01f};
  const float sd[3] = {0.05f, 0.03f, 0.02f};
  for (int i = 0; i < 3; ++i) { p->considered_distances[i] = cd[i]; p->standard_deviations[i] = sd[i]; }
  p->n_standard_deviations = 3;
  p->measured_depth_offset_radius = 0.01f;
  p->measured_occlusion_radius = 0.01f;
  p->measured_occlusion_threshold = 0.03f;
  p->n_unoccluded_iterations = 10;
  p->min_n_unoccluded_points = 0;
  p->modeled_depth_offset_radius = 0.01f;
  p->modeled_occlusion_radius = 0.01f;
  p->modeled_occlusion_threshold = 0.03f;
}

void m3tb_optimizer_params_default(m3tb_optimizer_params* p) {
  p->tikhonov_parameter_rotation = 1000.0f;
  p->tikhonov_parameter_translation = 30000.0f;
}

// The device tables every context has; m3tb_create's context owns them from here on.
static int CreateTables(m3tb_ctx* ctx, bool want_timing) {
  const size_t nb = size_t(ctx->max_bodies), nc = size_t(ctx->max_cameras), nm = size_t(ctx->max_models);
  CU(cudaSetDevice(ctx->device));
  CU(ctx->d_bodies.create(nb));
  CU(ctx->d_ccams.create(nc));
  CU(ctx->d_dcams.create(nc));
  CU(ctx->d_rmodels.create(nm));
  CU(ctx->d_dmodels.create(nm));
  CU(ctx->d_poses.create(12 * nb));
  CU(ctx->d_counts.create(4 * nb));
  CU(ctx->d_gh_region.create(27 * nb));
  CU(ctx->d_gh_depth.create(27 * nb));
  CU(cudaMemset(ctx->d_poses, 0, sizeof(float) * 12 * nb));
  CU(cudaMemset(ctx->d_counts, 0, sizeof(int) * 4 * nb));
  CU(cudaMemset(ctx->d_gh_region, 0, sizeof(float) * 27 * nb));
  CU(cudaMemset(ctx->d_gh_depth, 0, sizeof(float) * 27 * nb));
  CU(ctx->d_gh_link.create(27 * nb));
  CU(cudaMemset(ctx->d_gh_link, 0, sizeof(float) * 27 * nb));
  CU(ctx->d_roi.create(2 * nb));
  CU(cudaMemset(ctx->d_roi, 0xff, sizeof(RoiRecord) * 2 * nb));  // generation -1: nothing ingested yet
  CU(ctx->d_bin_ids.create(nc));
  CU(ctx->d_tmaps.create(2 * kTileWidths));
  CU(ctx->d_ingest_bytes.create(2));
  CU(cudaMemset(ctx->d_ingest_bytes, 0, 2 * sizeof(unsigned long long)));
  if (want_timing) {
    CU(ctx->d_phase_clock.create(kPhaseSlots * nb));
    CU(cudaMemset(ctx->d_phase_clock, 0, sizeof(long long) * kPhaseSlots * nb));
  }
  return M3TB_OK;
}

int m3tb_create(int device, int max_bodies, int max_cameras, int max_models, m3tb_ctx** out) {
  if (!out || max_bodies <= 0 || max_cameras <= 0 || max_models <= 0) return M3TB_ERR_INVALID;
  *out = nullptr;
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || device < 0 || device >= n_dev) return M3TB_ERR_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return M3TB_ERR_CUDA;
  if (prop.major != 9 || prop.minor != 0) return M3TB_ERR_CUDA;  // sm_90a cubin only: no other architecture can run it
  std::unique_ptr<m3tb_ctx> ctx(new m3tb_ctx());
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  ctx->max_bodies = max_bodies;
  ctx->max_cameras = max_cameras;
  ctx->max_models = max_models;
  ctx->h_bodies.assign(max_bodies, BodyDev());
  std::memset(ctx->h_bodies.data(), 0, sizeof(BodyDev) * max_bodies);
  ctx->h_ccams.assign(max_cameras, CameraDev());
  ctx->h_dcams.assign(max_cameras, CameraDev());
  std::memset(ctx->h_ccams.data(), 0, sizeof(CameraDev) * max_cameras);
  std::memset(ctx->h_dcams.data(), 0, sizeof(CameraDev) * max_cameras);
  ctx->h_rmodels.assign(max_models, ModelDev());
  ctx->h_dmodels.assign(max_models, ModelDev());
  std::memset(ctx->h_rmodels.data(), 0, sizeof(ModelDev) * max_models);
  std::memset(ctx->h_dmodels.data(), 0, sizeof(ModelDev) * max_models);
  ctx->rmodel_alloc.resize(max_models);
  ctx->dmodel_alloc.resize(max_models);
  ctx->private_color.resize(max_cameras);
  ctx->private_depth.resize(max_cameras);
  ctx->bin_shift.assign(max_cameras, kBinsNone);
  ctx->undistort[0].resize(max_cameras);
  ctx->undistort[1].resize(max_cameras);
  ctx->h_geometry.assign(max_bodies, GeometryDev());
  std::memset(ctx->h_geometry.data(), 0, sizeof(GeometryDev) * max_bodies);
  ctx->geometry_alloc.resize(max_bodies);
  ctx->rendering_images.resize(max_bodies);
  std::array<int, RS_COUNT> detached;
  detached.fill(-1);
  ctx->attached.assign(max_bodies, detached);
  ctx->attach_uploaded.assign(max_bodies, std::array<char, RS_COUNT>{});
  ctx->tex_feat_gen.assign(max_bodies, -1);
  ctx->tex_crop.assign(max_bodies, m3tb_ctx::TexCrop{});
  ctx->orb_nmax.assign(max_bodies, -1);
  if (const char* e = std::getenv("M3TB_NO_TILES")) ctx->use_tiles = !(e[0] == '1');
  if (const char* e = std::getenv("M3TB_NO_ROI_INGEST")) ctx->roi_ingest = !(e[0] == '1');
  if (const char* e = std::getenv("M3TB_KERNEL")) ctx->use_track2 = !(e[0] == '1');
  if (const char* e = std::getenv("M3TB_TMA")) ctx->tma_mode = (e[0] >= '0' && e[0] <= '2') ? e[0] - '0' : 1;
  const char* timing_env = std::getenv("M3TB_TIMING");
  const int rc = CreateTables(ctx.get(), timing_env && timing_env[0] == '1');
  if (rc != M3TB_OK) {
    std::fprintf(stderr, "m3tb_create: %s\n", ctx->err.c_str());
    return rc;
  }
  *out = ctx.release();
  return M3TB_OK;
}

int m3tb_destroy(m3tb_ctx* ctx) {
  if (!ctx) return M3TB_ERR_INVALID;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);  // not owned: the caller's stream of m3tb_set_stream, or the default stream
  if (ctx->pf.table_stream) cudaStreamSynchronize(ctx->pf.table_stream);
  if (ctx->pf.ingest_stream) cudaStreamSynchronize(ctx->pf.ingest_stream);
  delete ctx;
  return M3TB_OK;
}

int m3tb_set_stream(m3tb_ctx* ctx, void* cuda_stream) {
  CHECK_CTX();
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->stream = static_cast<cudaStream_t>(cuda_stream);
  return M3TB_OK;
}

int m3tb_synchronize(m3tb_ctx* ctx) {
  CHECK_CTX();
  if (ctx->pf.ingest_stream) CU(cudaStreamSynchronize(ctx->pf.ingest_stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

const char* m3tb_last_error(const m3tb_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
int64_t m3tb_launch_count(const m3tb_ctx* ctx) { return ctx ? ctx->launches : 0; }
int m3tb_n_bodies(const m3tb_ctx* ctx) { return ctx ? ctx->n_bodies : 0; }

int m3tb_set_region_model(m3tb_ctx* ctx, int model_id, int n_views, int n_points, const float* orientations,
                          const float* contour_lengths, const void* points, float stride_depth_offset,
                          float max_radius_depth_offset) {
  CHECK_CTX();
  const int rc = SetModel(ctx, true, model_id, n_views, n_points, orientations, contour_lengths, points,
                          stride_depth_offset, max_radius_depth_offset);
  if (!rc && model_id < int(ctx->rmodel_generated.size())) ctx->rmodel_generated[model_id] = {};  // replaced
  return rc;
}

int m3tb_set_depth_model(m3tb_ctx* ctx, int model_id, int n_views, int n_points, const float* orientations,
                         const float* surface_areas, const void* points, float stride_depth_offset,
                         float max_radius_depth_offset) {
  CHECK_CTX();
  const int rc = SetModel(ctx, false, model_id, n_views, n_points, orientations, surface_areas, points,
                          stride_depth_offset, max_radius_depth_offset);
  if (!rc && model_id < int(ctx->dmodel_generated.size())) ctx->dmodel_generated[model_id] = {};  // replaced
  return rc;
}

int m3tb_set_color_camera(m3tb_ctx* ctx, int cam, const m3tb_intrinsics* intrinsics, const float world2camera[12]) {
  CHECK_CTX();
  return SetCamera(ctx, true, cam, intrinsics, world2camera, 0.0f);
}

int m3tb_set_depth_camera(m3tb_ctx* ctx, int cam, const m3tb_intrinsics* intrinsics, const float world2camera[12],
                          float depth_scale) {
  CHECK_CTX();
  if (!(depth_scale > 0.0f)) return Fail(ctx, M3TB_ERR_INVALID, "depth_scale must be positive");
  return SetCamera(ctx, false, cam, intrinsics, world2camera, depth_scale);
}

int m3tb_upload_color(m3tb_ctx* ctx, int cam, const uint8_t* bgr, size_t pitch) {
  CHECK_CTX();
  return Upload(ctx, true, cam, bgr, pitch, cudaMemcpyHostToDevice, PinnedAlias(ctx, bgr));
}
int m3tb_upload_depth(m3tb_ctx* ctx, int cam, const uint16_t* depth, size_t pitch) {
  CHECK_CTX();
  return Upload(ctx, false, cam, depth, pitch, cudaMemcpyHostToDevice, PinnedAlias(ctx, depth));
}
int m3tb_upload_color_device(m3tb_ctx* ctx, int cam, const void* dev_bgr, size_t pitch) {
  CHECK_CTX();
  return Upload(ctx, true, cam, dev_bgr, pitch, cudaMemcpyDeviceToDevice, nullptr);
}
int m3tb_upload_depth_device(m3tb_ctx* ctx, int cam, const void* dev_depth, size_t pitch) {
  CHECK_CTX();
  return Upload(ctx, false, cam, dev_depth, pitch, cudaMemcpyDeviceToDevice, nullptr);
}
int m3tb_upload_color_batch(m3tb_ctx* ctx, int first_cam, int count, const uint8_t* bgr, size_t frame_stride,
                            size_t pitch) {
  CHECK_CTX();
  return UploadBatch(ctx, true, first_cam, count, bgr, frame_stride, pitch);
}
int m3tb_upload_depth_batch(m3tb_ctx* ctx, int first_cam, int count, const uint16_t* depth, size_t frame_stride,
                            size_t pitch) {
  CHECK_CTX();
  return UploadBatch(ctx, false, first_cam, count, depth, frame_stride, pitch);
}

int m3tb_set_body(m3tb_ctx* ctx, int body, const m3tb_region_params* region, const m3tb_depth_params* depth,
                  const m3tb_optimizer_params* optimizer, int region_model, int depth_model, int color_camera,
                  int depth_camera) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->max_bodies) return Fail(ctx, M3TB_ERR_INVALID, "body index out of range");
  if (!region && !depth) return Fail(ctx, M3TB_ERR_INVALID, "a body needs at least one modality");
  if ((region && !(RadiusValid(region->measured_depth_offset_radius) && RadiusValid(region->measured_occlusion_radius) &&
                   RadiusValid(region->modeled_depth_offset_radius) && RadiusValid(region->modeled_occlusion_radius))) ||
      (depth && !(RadiusValid(depth->measured_depth_offset_radius) && RadiusValid(depth->measured_occlusion_radius) &&
                  RadiusValid(depth->modeled_depth_offset_radius) && RadiusValid(depth->modeled_occlusion_radius))))
    return Fail(ctx, M3TB_ERR_INVALID, "occlusion and depth-offset radii must be finite and >= 0");
  if (depth) {  // checked before anything is written, so that a refused call leaves the context as it was
    if (depth->n_considered_distances < 1 || depth->n_considered_distances > M3TB_MAX_SCHEDULE ||
        depth->n_standard_deviations < 1 || depth->n_standard_deviations > M3TB_MAX_SCHEDULE ||
        depth->n_points_max < 1 || !(depth->stride_length > 0.0f))
      return Fail(ctx, M3TB_ERR_INVALID, "bad depth schedule / n_points_max / stride_length");
    // FindCorrespondence divides the window diameter by max_n_strides_ = int(d / stride_length + 0.5f)
    // (depth_modality.cpp:651, :835): a distance below half the stride length, or NaN, gives 0 and an infinite stride,
    // and 2^31 strides or more overflow the int (the device saturates, x86 gives INT_MIN and a stride of 0)
    for (int i = 0; i < depth->n_considered_distances; ++i) {
      const float d = depth->considered_distances[i];
      const float strides = d / depth->stride_length + 0.5f;
      if (!(d > 0.0f) || !std::isfinite(d) || !(strides >= 1.0f) || !(strides < 2147483648.0f))
        return Fail(ctx, M3TB_ERR_INVALID,
                    "considered distances must be finite, at least half the stride length and under 2^31 strides");
    }
  }
  BodyDev B;
  std::memset(&B, 0, sizeof(B));
  B.first_iteration = ctx->h_bodies[body].first_iteration;
  std::memcpy(B.rend, ctx->h_bodies[body].rend, sizeof(B.rend));  // uploaded renderer images stay with the body
  // so does a texture modality (m3tb_set_texture_modality): its keyframes, renderers and parameters are its own
  B.has_texture = ctx->h_bodies[body].has_texture;
  B.texture_camera = ctx->h_bodies[body].texture_camera;
  B.tp = ctx->h_bodies[body].tp;
  m3tb_optimizer_params op;
  m3tb_optimizer_params_default(&op);
  if (optimizer) op = *optimizer;
  B.tikhonov_rotation = op.tikhonov_parameter_rotation;
  B.tikhonov_translation = op.tikhonov_parameter_translation;
  if (region) {
    if (region_model < 0 || region_model >= ctx->max_models || color_camera < 0 || color_camera >= ctx->max_cameras)
      return Fail(ctx, M3TB_ERR_INVALID, "region model / color camera id out of range");
    if (region->function_length != M3TB_FUNCTION_LENGTH || region->distribution_length != M3TB_DISTRIBUTION_LENGTH)
      return Fail(ctx, M3TB_ERR_UNSUPPORTED, "function_length / distribution_length other than 8 / 12");
    if (region->measure_occlusions && (depth_camera < 0 || depth_camera >= ctx->max_cameras))
      return Fail(ctx, M3TB_ERR_INVALID, "measure_occlusions needs a depth camera (RegionModality::MeasureOcclusions)");
    if (region->n_scales < 1 || region->n_scales > M3TB_MAX_SCHEDULE || region->n_standard_deviations < 1 ||
        region->n_standard_deviations > M3TB_MAX_SCHEDULE || region->n_lines_max < 1)
      return Fail(ctx, M3TB_ERR_INVALID, "bad region schedule / n_lines_max");
    int bs = Bitshift(region->n_histogram_bins);
    if (bs < 0) return Fail(ctx, M3TB_ERR_INVALID, "n_histogram_bins has to be 2, 4, 8, 16, 32 or 64");
    RegionParamsDev& r = B.rp;
    r.measure_occlusions = region->measure_occlusions ? 1 : 0;
    r.n_unoccluded_iterations = region->n_unoccluded_iterations;
    r.min_n_unoccluded_lines = region->min_n_unoccluded_lines;
    r.measured_depth_offset_radius = region->measured_depth_offset_radius;
    r.measured_occlusion_radius = region->measured_occlusion_radius;
    r.measured_occlusion_threshold = region->measured_occlusion_threshold;
    r.model_occlusions = region->model_occlusions ? 1 : 0;
    r.use_region_checking = region->use_region_checking ? 1 : 0;
    r.modeled_depth_offset_radius = region->modeled_depth_offset_radius;
    r.modeled_occlusion_radius = region->modeled_occlusion_radius;
    r.modeled_occlusion_threshold = region->modeled_occlusion_threshold;
    r.n_lines_max = region->n_lines_max;
    r.use_adaptive_coverage = region->use_adaptive_coverage;
    r.reference_contour_length = region->reference_contour_length;
    r.min_continuous_distance = region->min_continuous_distance;
    r.learning_rate = region->learning_rate;
    r.n_global_iterations = region->n_global_iterations;
    r.n_scales = region->n_scales;
    r.n_standard_deviations = region->n_standard_deviations;
    for (int i = 0; i < M3TB_MAX_SCHEDULE; ++i) {
      r.scales[i] = region->scales[i];
      r.standard_deviations[i] = region->standard_deviations[i];
    }
    for (int i = 0; i < r.n_scales; ++i)
      if (r.scales[i] < 1) return Fail(ctx, M3TB_ERR_INVALID, "scales must be >= 1");
    r.n_bins = region->n_histogram_bins;
    r.bitshift = bs;
    r.learning_rate_f = region->learning_rate_f;
    r.learning_rate_b = region->learning_rate_b;
    r.unconsidered_line_length = region->unconsidered_line_length;
    r.max_considered_line_length = region->max_considered_line_length;
    // PrecalculateFunctionLookup / PrecalculateDistributionVariables (region_modality.cpp:910-936): host libm,
    // exactly where the reference evaluates tanh / atanh (SetUp time, not the hot path).
    for (int i = 0; i < kFunctionLength; ++i) {
      float x = float(i) - float(kFunctionLength - 1) / 2.0f;
      if (region->function_slope == 0.0f)
        r.lookup_f[i] = 0.5f - region->function_amplitude * float((0.0f < x) - (x < 0.0f));
      else
        r.lookup_f[i] = 0.5f - region->function_amplitude * std::tanh(x / (2.0f * region->function_slope));
      r.lookup_b[i] = 1.0f - r.lookup_f[i];
    }
    float laplace = 1.0f / (2.0f * powf(atanhf(2.0f * region->function_amplitude), 2.0f));
    r.min_expected_variance = std::max(laplace, region->function_slope);
    B.has_region = 1;
    B.region_model = region_model;
    B.color_camera = color_camera;
    if (region->measure_occlusions) B.depth_camera = depth_camera;  // RegionModality::depth_camera_ptr()
    const size_t n3 = size_t(r.n_bins) * r.n_bins * r.n_bins;
    int rc = EnsureHist(ctx, n3);
    if (rc) return rc;
    // ColorHistograms::SetUpHistograms (color_histograms.cpp:161-172): uniform histograms
    std::vector<float> uni(n3, 1.0f / float(n3));
    std::vector<float2> half(n3, make_float2(0.5f, 0.5f));
    CU(cudaMemcpyAsync(ctx->d_hist_f + size_t(body) * ctx->hist_stride, uni.data(), n3 * sizeof(float),
                       cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_hist_b + size_t(body) * ctx->hist_stride, uni.data(), n3 * sizeof(float),
                       cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_lut + size_t(body) * ctx->hist_stride, half.data(), n3 * sizeof(float2),
                       cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  if (depth) {
    if (depth_model < 0 || depth_model >= ctx->max_models || depth_camera < 0 || depth_camera >= ctx->max_cameras)
      return Fail(ctx, M3TB_ERR_INVALID, "depth model / depth camera id out of range");
    DepthParamsDev& d = B.dp;
    d.measure_occlusions = depth->measure_occlusions ? 1 : 0;
    d.n_unoccluded_iterations = depth->n_unoccluded_iterations;
    d.min_n_unoccluded_points = depth->min_n_unoccluded_points;
    d.measured_depth_offset_radius = depth->measured_depth_offset_radius;
    d.measured_occlusion_radius = depth->measured_occlusion_radius;
    d.measured_occlusion_threshold = depth->measured_occlusion_threshold;
    d.model_occlusions = depth->model_occlusions ? 1 : 0;
    d.use_silhouette_checking = depth->use_silhouette_checking ? 1 : 0;
    d.modeled_depth_offset_radius = depth->modeled_depth_offset_radius;
    d.modeled_occlusion_radius = depth->modeled_occlusion_radius;
    d.modeled_occlusion_threshold = depth->modeled_occlusion_threshold;
    d.n_points_max = depth->n_points_max;
    d.use_adaptive_coverage = depth->use_adaptive_coverage;
    d.use_depth_scaling = depth->use_depth_scaling;
    d.reference_surface_area = depth->reference_surface_area;
    d.stride_length = depth->stride_length;
    d.n_considered_distances = depth->n_considered_distances;
    d.n_standard_deviations = depth->n_standard_deviations;
    for (int i = 0; i < M3TB_MAX_SCHEDULE; ++i) {
      d.considered_distances[i] = depth->considered_distances[i];
      d.standard_deviations[i] = depth->standard_deviations[i];
    }
    B.has_depth = 1;
    B.depth_model = depth_model;
    B.depth_camera = depth_camera;
  }
  B.set = 1;
  ctx->h_bodies[body] = B;
  if (!ctx->structures.empty()) {  // the implicit one-link structures follow the body table
    int prc = PullLinks(ctx);
    if (prc) return prc;
    ctx->structures_dirty = true;
  }
  ctx->n_bodies = std::max(ctx->n_bodies, body + 1);
  ctx->bodies_dirty = true;
  return M3TB_OK;
}

int m3tb_set_poses(m3tb_ctx* ctx, int first, int count, const float* body2world) {
  CHECK_CTX();
  if (first < 0 || count <= 0 || first + count > ctx->max_bodies || !body2world)
    return Fail(ctx, M3TB_ERR_INVALID, "bad pose range");
  CU(cudaMemcpyAsync(ctx->d_poses + 12 * first, body2world, sizeof(float) * 12 * count, cudaMemcpyHostToDevice,
                     ctx->stream));
  return M3TB_OK;
}

int m3tb_get_poses(m3tb_ctx* ctx, int first, int count, float* body2world) {
  CHECK_CTX();
  if (first < 0 || count <= 0 || first + count > ctx->max_bodies || !body2world)
    return Fail(ctx, M3TB_ERR_INVALID, "bad pose range");
  CU(cudaMemcpyAsync(body2world, ctx->d_poses + 12 * first, sizeof(float) * 12 * count, cudaMemcpyDeviceToHost,
                     ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

int m3tb_set_histograms(m3tb_ctx* ctx, int body, const float* histogram_f, const float* histogram_b) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->n_bodies || !ctx->h_bodies[body].has_region || !histogram_f || !histogram_b)
    return Fail(ctx, M3TB_ERR_INVALID, "body has no region modality");
  const int nb = ctx->h_bodies[body].rp.n_bins;
  const int n3 = nb * nb * nb;
  const int owner = (body < int(ctx->hist_owner.size())) ? ctx->hist_owner[body] : -1;
  for (int b = 0; b < ctx->n_bodies; ++b) {  // a shared object: every body that uses it keeps a copy
    if (b != body && (owner < 0 || ctx->hist_owner[b] != owner)) continue;
    if (!ctx->h_bodies[b].has_region || ctx->h_bodies[b].rp.n_bins != nb) continue;
    CU(cudaMemcpyAsync(ctx->d_hist_f + size_t(b) * ctx->hist_stride, histogram_f, n3 * sizeof(float),
                       cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(ctx->d_hist_b + size_t(b) * ctx->hist_stride, histogram_b, n3 * sizeof(float),
                       cudaMemcpyHostToDevice, ctx->stream));
    dim3 grid((n3 + 255) / 256, 1);
    k_lut<<<grid, 256, 0, ctx->stream>>>(ctx->d_hist_f, ctx->d_hist_b, ctx->d_lut, n3, ctx->hist_stride, b);
    CU(cudaGetLastError());
    ctx->launches++;
  }
  return M3TB_OK;
}

int m3tb_share_color_histograms(m3tb_ctx* ctx, int body, int owner_body) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->max_bodies || owner_body < -1 || owner_body >= ctx->max_bodies)
    return Fail(ctx, M3TB_ERR_INVALID, "body index out of range");
  if (ctx->hist_owner.empty()) ctx->hist_owner.assign(ctx->max_bodies, -1);
  if (owner_body < 0) {  // DoNotUseSharedColorHistograms: a body that owns a shared object cannot leave it to its members
    for (int b = 0; b < ctx->max_bodies; ++b)
      if (b != body && ctx->hist_owner[b] == body) return Fail(ctx, M3TB_ERR_INVALID, "body owns a shared object that others still use");
    ctx->hist_owner[body] = -1;
  } else {
    if (ctx->hist_owner[owner_body] >= 0 && ctx->hist_owner[owner_body] != owner_body)
      return Fail(ctx, M3TB_ERR_INVALID, "the owner uses another body's shared object itself");
    for (int b = 0; b < ctx->max_bodies; ++b)
      if (b != body && body != owner_body && ctx->hist_owner[b] == body)
        return Fail(ctx, M3TB_ERR_INVALID, "body owns a shared object that others still use");
    ctx->hist_owner[owner_body] = owner_body;
    ctx->hist_owner[body] = owner_body;
  }
  return M3TB_OK;
}

int m3tb_get_histograms(m3tb_ctx* ctx, int body, float* histogram_f, float* histogram_b) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->n_bodies || !ctx->h_bodies[body].has_region || !histogram_f || !histogram_b)
    return Fail(ctx, M3TB_ERR_INVALID, "body has no region modality");
  const int nb = ctx->h_bodies[body].rp.n_bins;
  const int n3 = nb * nb * nb;
  CU(cudaMemcpyAsync(histogram_f, ctx->d_hist_f + size_t(body) * ctx->hist_stride, n3 * sizeof(float),
                     cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(histogram_b, ctx->d_hist_b + size_t(body) * ctx->hist_stride, n3 * sizeof(float),
                     cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

int m3tb_tracking_step(m3tb_ctx* ctx, int iteration, int n_corr_iterations, int n_update_iterations) {
  CHECK_CTX();
  if (n_corr_iterations < 0 || n_update_iterations < 0) return Fail(ctx, M3TB_ERR_INVALID, "negative iteration count");
  if (HasStructures(ctx)) return StructureStep(ctx, iteration, 0, n_corr_iterations, n_update_iterations);
  const unsigned phases = PH_REGION_CORR | PH_DEPTH_CORR | PH_REGION_GH | PH_DEPTH_GH | PH_SOLVE | PH_STORE_REGION |
                          PH_STORE_DEPTH | (ctx->n_texture > 0 ? unsigned(PH_TEXTURE_GH) : 0u);
  if (ctx->n_attached == 0) return LaunchTrack(ctx, iteration, 0, n_corr_iterations, n_update_iterations, 0, phases);
  // device renderers: Tracker::CalculateCorrespondences renders before every correspondence iteration (tracker.cpp:447-456)
  for (int corr = 0; corr < n_corr_iterations; ++corr) {
    int rc = LaunchRender(ctx, kRenderAttached);
    if (!rc && corr == 0) rc = LaunchTexture(ctx, false, 1);  // texture matches of this frame (no-op without texture)
    if (!rc) rc = LaunchTrack(ctx, iteration, corr, corr + 1, n_update_iterations, 0, phases);
    if (rc) return rc;
  }
  return M3TB_OK;
}

int m3tb_corr_iteration(m3tb_ctx* ctx, int iteration, int corr_iteration, int n_update_iterations) {
  CHECK_CTX();
  if (corr_iteration < 0 || n_update_iterations < 0) return Fail(ctx, M3TB_ERR_INVALID, "negative iteration count");
  if (HasStructures(ctx)) return StructureStep(ctx, iteration, corr_iteration, corr_iteration + 1, n_update_iterations);
  if (ctx->n_attached > 0) {
    int rc = LaunchRender(ctx, kRenderAttached);
    if (!rc && corr_iteration == 0) rc = LaunchTexture(ctx, false, 1);
    if (rc) return rc;
  }
  return LaunchTrack(ctx, iteration, corr_iteration, corr_iteration + 1, n_update_iterations, 0,
                     PH_REGION_CORR | PH_DEPTH_CORR | PH_REGION_GH | PH_DEPTH_GH | PH_SOLVE | PH_STORE_REGION |
                         PH_STORE_DEPTH | (ctx->n_texture > 0 ? unsigned(PH_TEXTURE_GH) : 0u));
}

int m3tb_start_modalities(m3tb_ctx* ctx, int iteration) {
  CHECK_CTX();
  for (int b = 0; b < ctx->n_bodies; ++b) ctx->h_bodies[b].first_iteration = iteration;
  ctx->bodies_dirty = true;
  if (ctx->n_attached > 0) {  // Tracker::StartModalities renders first (tracker.cpp:430-434)
    int rc = LaunchRender(ctx, kRenderRegion);
    if (rc) return rc;
  }
  int rc = LaunchHistogram(ctx, 0, iteration);
  if (!rc) rc = LaunchTexture(ctx, true, 0);  // TextureModality::StartModality (no-op without texture)
  return rc;
}

int m3tb_calculate_results(m3tb_ctx* ctx, int iteration) {
  CHECK_CTX();
  if (ctx->n_attached > 0) {  // Tracker::CalculateResults renders first (tracker.cpp:503-506)
    int rc = LaunchRender(ctx, kRenderRegion);
    if (rc) return rc;
  }
  int rc = LaunchHistogram(ctx, 1, iteration);
  if (!rc) rc = LaunchTexture(ctx, true, 1);  // TextureModality::CalculateResults (no-op without texture)
  return rc;
}

int m3tb_region_correspondences(m3tb_ctx* ctx, int iteration, int corr_iteration) {
  CHECK_CTX();
  return LaunchTrack(ctx, iteration, corr_iteration, corr_iteration + 1, 0, 0, PH_REGION_CORR | PH_STORE_REGION);
}

static int ReadGH(m3tb_ctx* ctx, const float* d_gh, float* gradients, float* hessians) {
  if (!gradients && !hessians) return M3TB_OK;
  std::vector<float> h(size_t(27) * ctx->n_bodies);
  CU(cudaMemcpyAsync(h.data(), d_gh, h.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  for (int b = 0; b < ctx->n_bodies; ++b) {
    const float* s = h.data() + 27 * b;
    if (gradients)
      for (int i = 0; i < 6; ++i) gradients[6 * b + i] = s[i];
    if (hessians)
      for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) hessians[36 * b + 6 * i + j] = s[6 + (i >= j ? Tri(i, j) : Tri(j, i))];
  }
  return M3TB_OK;
}

int m3tb_region_gradient_hessian(m3tb_ctx* ctx, int iteration, int corr_iteration, int opt_iteration, float* gradients,
                                 float* hessians) {
  CHECK_CTX();
  int rc = LaunchTrack(ctx, iteration, corr_iteration, corr_iteration + 1, 1, opt_iteration,
                       PH_LOAD_REGION | PH_REGION_GH | PH_STORE_GH);
  if (rc) return rc;
  return ReadGH(ctx, ctx->d_gh_region, gradients, hessians);
}

int m3tb_depth_correspondences(m3tb_ctx* ctx, int iteration, int corr_iteration) {
  CHECK_CTX();
  return LaunchTrack(ctx, iteration, corr_iteration, corr_iteration + 1, 0, 0, PH_DEPTH_CORR | PH_STORE_DEPTH);
}

int m3tb_depth_gradient_hessian(m3tb_ctx* ctx, int iteration, int corr_iteration, int opt_iteration, float* gradients,
                                float* hessians) {
  CHECK_CTX();
  int rc = LaunchTrack(ctx, iteration, corr_iteration, corr_iteration + 1, 1, opt_iteration,
                       PH_LOAD_DEPTH | PH_DEPTH_GH | PH_STORE_GH);
  if (rc) return rc;
  return ReadGH(ctx, ctx->d_gh_depth, gradients, hessians);
}

int m3tb_calculate_optimization(m3tb_ctx* ctx, int iteration, int corr_iteration, int opt_iteration) {
  CHECK_CTX();
  if (HasStructures(ctx)) return LaunchStructure(ctx, 0, true);
  return LaunchTrack(ctx, iteration, corr_iteration, corr_iteration + 1, 1, opt_iteration, PH_LOAD_GH | PH_SOLVE);
}

int m3tb_debug_rigid_solve(m3tb_ctx* ctx, int solve, int n, const float* a, const float* b, float* poses, float* theta,
                           int* updated) {
  CHECK_CTX();
  if ((solve != 0 && solve != 1) || n < 0 || (n > 0 && (!a || !b || !poses || !theta || !updated)))
    return Fail(ctx, M3TB_ERR_INVALID, "bad rigid-solve arguments");
  if (n == 0) return M3TB_OK;
  DeviceBuffer<float> d_a, d_b, d_pose, d_theta;
  DeviceBuffer<int> d_upd;
  CU(d_a.create(size_t(36) * n));
  CU(d_b.create(size_t(6) * n));
  CU(d_pose.create(size_t(12) * n));
  CU(d_theta.create(size_t(6) * n));
  CU(d_upd.create(size_t(n)));
  CU(cudaMemcpyAsync(d_a, a, sizeof(float) * 36 * n, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(d_b, b, sizeof(float) * 6 * n, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(d_pose, poses, sizeof(float) * 12 * n, cudaMemcpyHostToDevice, ctx->stream));
  if (solve == 0) k_debug_rigid_solve<Shared><<<unsigned(n), 32, 0, ctx->stream>>>(d_a, d_b, d_pose, d_theta, d_upd);
  else k_debug_rigid_solve<Shared2><<<unsigned(n), 32, 0, ctx->stream>>>(d_a, d_b, d_pose, d_theta, d_upd);
  CU(cudaGetLastError());
  ctx->launches++;
  CU(cudaMemcpyAsync(poses, d_pose, sizeof(float) * 12 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(theta, d_theta, sizeof(float) * 6 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(updated, d_upd, sizeof(int) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

int m3tb_set_structure(m3tb_ctx* ctx, int structure, const m3tb_link* links, int n_links,
                       const m3tb_constraint* constraints, int n_constraints, const m3tb_optimizer_params* optimizer) {
  CHECK_CTX();
  if (structure < 0 || structure > int(ctx->structures.size()) || structure >= ctx->max_bodies)
    return Fail(ctx, M3TB_ERR_INVALID, "structure ids must be dense (0..n)");
  if (!links || n_links < 1 || n_links > kMaxLinks) return Fail(ctx, M3TB_ERR_INVALID, "a structure has 1..16 links");
  if (n_constraints < 0 || n_constraints > kMaxStructConstraints || (n_constraints > 0 && !constraints))
    return Fail(ctx, M3TB_ERR_INVALID, "a structure has at most 32 constraints");
  StructureHost h;
  int dof = 0, rows = 0;
  for (int i = 0; i < n_links; ++i) {
    const m3tb_link& in = links[i];
    if ((i == 0) != (in.parent < 0) || in.parent >= i)
      return Fail(ctx, M3TB_ERR_INVALID, "links must be listed in pre-order: link 0 is the root, parent < own index");
    if (in.body < -1 || in.body >= ctx->max_bodies) return Fail(ctx, M3TB_ERR_INVALID, "link body index out of range");
    LinkDev l;
    std::memset(&l, 0, sizeof(l));
    l.body = in.body;
    l.parent = in.parent;
    l.first_index = dof;
    for (int d = 0; d < 6; ++d) {
      l.free_directions[d] = in.free_directions[d] ? 1 : 0;
      l.dof += l.free_directions[d];
    }
    dof += l.dof;
    l.fixed_body2joint = in.fixed_body2joint_pose ? 1 : 0;
    l.level = in.parent < 0 ? 0 : h.links[in.parent].level + 1;
    std::memcpy(l.body2joint, in.body2joint, sizeof(l.body2joint));
    std::memcpy(l.joint2parent, in.joint2parent, sizeof(l.joint2parent));
    std::memcpy(l.link2world, in.link2world, sizeof(l.link2world));
    if (in.n_extra_bodies < 0 || in.n_extra_bodies > M3TB_MAX_EXTRA_BODIES || (in.n_extra_bodies > 0 && in.body < 0))
      return Fail(ctx, M3TB_ERR_INVALID, "a link has 0..3 extra bodies, and only next to a primary body");
    l.n_extra = in.n_extra_bodies;
    for (int x = 0; x < l.n_extra; ++x) {
      if (in.extra_bodies[x] < 0 || in.extra_bodies[x] >= ctx->max_bodies) return Fail(ctx, M3TB_ERR_INVALID, "extra body index out of range");
      l.extra[x] = in.extra_bodies[x];
    }
    h.links.push_back(l);
  }
  for (int c = 0; c < n_constraints; ++c) {
    const m3tb_constraint& in = constraints[c];
    if (in.link1 < 0 || in.link1 >= n_links || in.link2 < 0 || in.link2 >= n_links)
      return Fail(ctx, M3TB_ERR_INVALID, "constraint link index out of range");
    ConstraintDev k;
    std::memset(&k, 0, sizeof(k));
    k.link1 = in.link1; k.link2 = in.link2;
    k.soft = in.soft ? 1 : 0;
    for (int d = 0; d < 6; ++d) {
      k.directions[d] = in.directions[d] ? 1 : 0;
      k.n_rows += k.directions[d];
    }
    if (!k.soft) { k.first_row = rows; rows += k.n_rows; }
    std::memcpy(k.body12joint1, in.body12joint1, sizeof(k.body12joint1));
    std::memcpy(k.body22joint2, in.body22joint2, sizeof(k.body22joint2));
    k.max_distance_rotation = in.max_distance_rotation;
    k.max_distance_translation = in.max_distance_translation;
    k.sd_rotation = in.standard_deviation_rotation;
    k.sd_translation = in.standard_deviation_translation;
    if (k.soft && !(k.sd_rotation > 0.0f && k.sd_translation > 0.0f))
      return Fail(ctx, M3TB_ERR_INVALID, "soft constraint standard deviations must be positive");
    h.constraints.push_back(k);
  }
  if (dof < 1) return Fail(ctx, M3TB_ERR_INVALID, "a structure needs at least one free direction");
  if (dof > kMaxStructDof || dof + rows > kMaxSystem)
    return Fail(ctx, M3TB_ERR_UNSUPPORTED, "more than 96 degrees of freedom or 128 unknowns + constraint rows");
  m3tb_optimizer_params dflt;
  m3tb_optimizer_params_default(&dflt);
  const m3tb_optimizer_params& op = optimizer ? *optimizer : dflt;
  h.tikhonov_rotation = op.tikhonov_parameter_rotation;
  h.tikhonov_translation = op.tikhonov_parameter_translation;
  h.set = true;
  int rc = PullLinks(ctx);
  if (rc) return rc;
  h.default_links = h.links;
  if (structure == int(ctx->structures.size())) ctx->structures.push_back(h);
  else ctx->structures[structure] = h;
  ctx->structures_dirty = true;
  ctx->defaults_valid = false;  // set_joint2parent_pose / set_body2joint_pose also set the defaults (link.cpp:131-139)
  return M3TB_OK;
}

int m3tb_set_gradient_hessian(m3tb_ctx* ctx, int modality, const float* gradients, const float* hessians) {
  CHECK_CTX();
  if ((modality != 0 && modality != 1 && modality != 2) || !gradients || !hessians || ctx->n_bodies == 0)
    return Fail(ctx, M3TB_ERR_INVALID, "bad gradient / hessian arguments");
  if (modality == 2 && !ctx->d_gh_texture) return Fail(ctx, M3TB_ERR_INVALID, "no texture modality set");
  std::vector<float> h(size_t(27) * ctx->n_bodies);
  for (int b = 0; b < ctx->n_bodies; ++b) {
    for (int i = 0; i < 6; ++i) h[27 * b + i] = gradients[6 * b + i];
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j <= i; ++j) h[27 * b + 6 + Tri(i, j)] = hessians[36 * b + 6 * i + j];
  }
  CU(cudaMemcpyAsync(modality == 0 ? ctx->d_gh_region : modality == 1 ? ctx->d_gh_depth : ctx->d_gh_texture, h.data(), h.size() * sizeof(float),
                     cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

int m3tb_clear_structures(m3tb_ctx* ctx) {
  CHECK_CTX();
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->structures.clear();
  ctx->structures_dirty = true;
  ctx->defaults_valid = false;
  ctx->n_struct_launch = 0;
  return M3TB_OK;
}

int m3tb_n_structures(const m3tb_ctx* ctx) { return ctx ? int(ctx->structures.size()) : 0; }

int m3tb_reset_joint_poses(m3tb_ctx* ctx) {
  CHECK_CTX();
  if (!HasStructures(ctx)) return M3TB_OK;
  int rc = SyncStructures(ctx);
  if (rc) return rc;
  // only the joint poses are reset; link2world of body-less links is state, like Link::link2world_pose_
  LinkDev* d = ctx->d_links;
  const LinkDev* s = ctx->d_links_default;
  CU(cudaMemcpy2DAsync(reinterpret_cast<char*>(d) + offsetof(LinkDev, body2joint), sizeof(LinkDev),
                       reinterpret_cast<const char*>(s) + offsetof(LinkDev, body2joint), sizeof(LinkDev),
                       sizeof(float) * 24, ctx->n_links_total, cudaMemcpyDeviceToDevice, ctx->stream));
  return M3TB_OK;
}

int m3tb_calculate_consistent_poses(m3tb_ctx* ctx) {
  CHECK_CTX();
  if (!HasStructures(ctx)) return M3TB_OK;  // a free root link with body2joint = identity keeps its pose
  int rc = SyncTables(ctx);
  if (rc) return rc;
  return LaunchStructure(ctx, 1, false);
}

}  // extern "C"

namespace {

// Refiner::RefinePoses (refiner.cpp:76-117) for the named optimisers: Refiner::CalculateConsistentPoses, then per
// correspondence iteration StartModalities (render, ClearMemory, StartModality(0, corr), InitializeHistograms),
// CalculateCorrespondences (render, CalculateCorrespondences(0, corr)) and n_update x (CalculateGradientAndHessian,
// CalculateOptimization). The launches are the tracking step's, restricted to the refined bodies, structures and
// renderers through RefineSelection; every other body keeps its state. With `texture` (m3tb_refine_poses_orb) refined
// ORB texture bodies take part: TextureModality::StartModality is device detection (orb[body], or the defaults when
// `orb` is null) and k_texture_keyframe, and the bodies match at correspondence iteration 0; without it a refined
// texture body is refused.
int RefinePoses(m3tb_ctx* ctx, const int* bodies, int n_bodies, const int* structures, int n_structures,
                int n_corr_iterations, int n_update_iterations, bool texture, const m3tb_orb_params* orb) {
  if (n_bodies < 0 || n_structures < 0 || (n_bodies > 0 && !bodies) || (n_structures > 0 && !structures))
    return Fail(ctx, M3TB_ERR_INVALID, "bad body / structure list");
  if (n_corr_iterations < 0 || n_update_iterations < 0) return Fail(ctx, M3TB_ERR_INVALID, "negative iteration count");
  const int n_user = int(ctx->structures.size());
  std::vector<char> in_link(ctx->max_bodies, 0), body_named(ctx->max_bodies, 0), structure_named(n_user, 0);
  for (const auto& st : ctx->structures)
    for (const auto& l : st.links) {
      if (l.body >= 0 && l.body < ctx->max_bodies) in_link[l.body] = 1;
      for (int x = 0; x < l.n_extra; ++x) in_link[l.extra[x]] = 1;
    }
  for (int k = 0; k < n_bodies; ++k) {
    const int b = bodies[k];
    if (b < 0 || b >= ctx->n_bodies || !ctx->h_bodies[b].set)
      return Fail(ctx, M3TB_ERR_INVALID, "body " + std::to_string(b) + " is not set");
    if (body_named[b]) return Fail(ctx, M3TB_ERR_INVALID, "body " + std::to_string(b) + " listed twice");
    if (in_link[b])
      return Fail(ctx, M3TB_ERR_INVALID, "body " + std::to_string(b) + " belongs to a kinematic structure: name the structure");
    body_named[b] = 1;
  }
  for (int k = 0; k < n_structures; ++k) {
    const int s = structures[k];
    if (s < 0 || s >= n_user || !ctx->structures[s].set)
      return Fail(ctx, M3TB_ERR_INVALID, "structure " + std::to_string(s) + " is not set");
    if (structure_named[s]) return Fail(ctx, M3TB_ERR_INVALID, "structure " + std::to_string(s) + " listed twice");
    structure_named[s] = 1;
  }
  // the bodies whose modalities run: the named ones, then every body of the named structures
  std::vector<int> track;
  for (int k = 0; k < n_bodies; ++k) track.push_back(bodies[k]);
  for (int k = 0; k < n_structures; ++k)
    for (const auto& l : ctx->structures[structures[k]].links) {
      if (l.body < 0) continue;
      if (l.body >= ctx->n_bodies || !ctx->h_bodies[l.body].set)
        return Fail(ctx, M3TB_ERR_NOT_SET_UP, "structure references a body that is not set");
      track.push_back(l.body);
      for (int x = 0; x < l.n_extra; ++x) {
        if (l.extra[x] >= ctx->n_bodies || !ctx->h_bodies[l.extra[x]].set)
          return Fail(ctx, M3TB_ERR_NOT_SET_UP, "structure references a body that is not set");
        track.push_back(l.extra[x]);
      }
    }
  // TextureModality::StartModality detects features in a pose-dependent focus region before every correspondence
  // iteration; with detection left to the caller one call cannot serve it, so only device detection (cv::ORB) can
  RefineSelection sel;
  std::vector<m3tb_orb_params> orb_settings;  // of sel.texture_ids
  m3tb_orb_params defaults;
  m3tb_orb_params_default(&defaults);
  for (int b : track) {
    const BodyDev& B = ctx->h_bodies[b];
    if (!B.has_texture) continue;
    if (!texture)
      return Fail(ctx, M3TB_ERR_UNSUPPORTED, "body " + std::to_string(b) + " has a texture modality: it cannot be refined");
    if (B.tp.descriptor_type != M3TB_DESCRIPTOR_ORB)
      return Fail(ctx, M3TB_ERR_UNSUPPORTED, "body " + std::to_string(b) + ": " + DescriptorName(B.tp.descriptor_type) +
                                                 " features have no device detector: it cannot be refined");
    const m3tb_orb_params& p = orb ? orb[b] : defaults;
    int rc = CheckOrbDetection(ctx, b, p);
    if (!rc) rc = ValidateTextureBody(ctx, b);
    if (rc) return rc;
    sel.texture_ids.push_back(b);
    orb_settings.push_back(p);
  }
  if (track.empty()) return M3TB_OK;  // if (!optimizer_found) return true

  std::vector<int> struct_list;
  if (HasStructures(ctx)) {
    int rc = SyncStructures(ctx);
    if (rc) return rc;
    for (int k = 0; k < n_structures; ++k) struct_list.push_back(structures[k]);
    for (int k = 0; k < n_bodies; ++k)  // a rigid body is the implicit one-link structure that SyncStructures appended
      for (int si = n_user; si < ctx->n_struct_launch; ++si)
        if (ctx->h_link_bodies[ctx->h_structures[si].first_link] == bodies[k]) struct_list.push_back(si);
  }
  if (ctx->n_attached > 0) {
    int rc = SyncTables(ctx);
    if (!rc) rc = SyncRenderTables(ctx);
    if (rc) return rc;
    for (int which : {int(kRenderAttached), int(kRenderRegion)}) {
      std::vector<char> use(ctx->renderers.size(), 0);
      for (int b : track)
        for (int slot = 0; slot < RS_COUNT; ++slot) {  // the lists of SyncRenderTables
          const int r = ctx->attached[b][slot];
          if (r >= 0 && (which == kRenderAttached ? slot < RS_TEXTURE_SILHOUETTE
                                                  : slot == RS_REGION_DEPTH || slot == RS_REGION_SILHOUETTE ||
                                                        slot >= RS_TEXTURE_SILHOUETTE))
            use[r] = 1;
        }
      for (int r = 0; r < int(use.size()); ++r) {
        if (!use[r]) continue;
        const int S = ctx->renderers[r].dev.image_size;
        sel.renderer_ids[which].push_back(r);
        sel.render_smem[which] = std::max(sel.render_smem[which], size_t(S) * S * sizeof(uint32_t));
      }
    }
  }
  // shared ColorHistograms objects with a refined member: the refined members first, only they add line pixels
  std::vector<int> g_owner, g_first, g_summed, g_members;
  std::vector<char> tracked(ctx->max_bodies, 0);
  for (int b : track) tracked[b] = 1;
  for (int o = 0; o < ctx->n_bodies && o < int(ctx->hist_owner.size()); ++o) {
    if (ctx->hist_owner[o] != o) continue;
    std::vector<int> refined, rest;
    for (int b = 0; b < ctx->n_bodies; ++b)
      if (ctx->hist_owner[b] == o) (tracked[b] && ctx->h_bodies[b].has_region ? refined : rest).push_back(b);
    if (refined.empty()) continue;
    g_owner.push_back(o);
    g_first.push_back(int(g_members.size()));
    g_summed.push_back(int(refined.size()));
    g_members.insert(g_members.end(), refined.begin(), refined.end());
    g_members.insert(g_members.end(), rest.begin(), rest.end());
  }
  g_first.push_back(int(g_members.size()));

  // one device table: bodies | structures | renderers (attached) | renderers (region) | texture bodies | shared-object
  // groups
  std::vector<int> h(track);
  const size_t o_struct = h.size();
  h.insert(h.end(), struct_list.begin(), struct_list.end());
  size_t o_render[kRenderLists] = {};
  for (int which : {int(kRenderAttached), int(kRenderRegion)}) {
    o_render[which] = h.size();
    h.insert(h.end(), sel.renderer_ids[which].begin(), sel.renderer_ids[which].end());
  }
  const size_t o_texture = h.size();
  h.insert(h.end(), sel.texture_ids.begin(), sel.texture_ids.end());
  const size_t o_groups = h.size();
  if (!g_owner.empty()) {
    h.insert(h.end(), g_owner.begin(), g_owner.end());
    h.insert(h.end(), g_first.begin(), g_first.end());
    h.insert(h.end(), g_summed.begin(), g_summed.end());
    h.insert(h.end(), g_members.begin(), g_members.end());
  }
  DeviceBuffer<int> grown;
  int rc = GrowTable(ctx, ctx->d_refine, grown, h.size());
  if (rc) return rc;
  CU(cudaStreamSynchronize(ctx->stream));  // the launches of an earlier refinement may still read the old lists
  if (grown) ctx->d_refine = std::move(grown);
  CU(cudaMemcpyAsync(ctx->d_refine, h.data(), sizeof(int) * h.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));  // `h` is a temporary
  const int* d = ctx->d_refine;
  sel.bodies = d;
  sel.n_bodies = int(track.size());
  {
    std::vector<int> sorted(track);
    std::sort(sorted.begin(), sorted.end());
    for (int b : sorted) {
      if (!sel.runs.empty() && sel.runs.back().first + sel.runs.back().second == b) ++sel.runs.back().second;
      else sel.runs.push_back({b, 1});
    }
  }
  sel.structures = d + o_struct;
  sel.n_structures = int(struct_list.size());
  for (int which : {int(kRenderAttached), int(kRenderRegion)}) {
    sel.renderers[which] = d + o_render[which];
    sel.n_renderers[which] = int(sel.renderer_ids[which].size());
  }
  sel.texture = d + o_texture;
  sel.n_texture = int(sel.texture_ids.size());
  sel.hist_groups = d + o_groups;
  sel.n_hist_groups = int(g_owner.size());

  struct Scope {  // every launch helper sees the selection until this call returns
    m3tb_ctx* c;
    ~Scope() { c->refine = nullptr; }
  } scope{ctx};
  ctx->refine = &sel;
  const bool structured = !struct_list.empty();
  if (structured) {  // Refiner::CalculateConsistentPoses
    rc = LaunchStructure(ctx, 1, false);
    if (rc) return rc;
  }
  for (int b : track) ctx->h_bodies[b].first_iteration = 0;  // StartModality(0, corr)
  ctx->bodies_dirty = true;
  const unsigned corr_phases = PH_REGION_CORR | PH_DEPTH_CORR | PH_STORE_REGION | PH_STORE_DEPTH;
  const bool textured = sel.n_texture > 0;
  const unsigned tex = textured ? unsigned(PH_TEXTURE_GH) : 0u;
  for (int corr = 0; corr < n_corr_iterations; ++corr) {
    // DetectAndComputeCorrKeypoints at the pose this iteration starts from. It goes before the start renders (it reads
    // only the pose and the colour frame): a detection that fails to grow its scratch then leaves the refined bodies as
    // the completed iterations left them.
    if (textured) rc = DetectOrb(ctx, sel.texture_ids.data(), sel.n_texture, orb_settings.data());
    if (!rc && ctx->n_attached > 0) rc = LaunchRender(ctx, kRenderRegion);  // start_modality_renderer_ptrs
    if (!rc) rc = LaunchHistogram(ctx, 0, 0);
    if (!rc && textured) rc = LaunchTexture(ctx, true, 0);  // ComputeKeyframeData
    if (!rc && ctx->n_attached > 0) rc = LaunchRender(ctx, kRenderAttached);  // correspondence_renderer_ptrs
    if (!rc && textured && corr == 0) rc = LaunchTexture(ctx, false, 1);  // the texture matches (corr 0 only)
    if (rc) return rc;
    if (!structured) {
      rc = LaunchTrack(ctx, 0, corr, corr + 1, n_update_iterations, 0,
                       corr_phases | PH_REGION_GH | PH_DEPTH_GH | PH_SOLVE | tex);
      if (rc) return rc;
      continue;
    }
    if (n_update_iterations == 0) {
      rc = LaunchTrack(ctx, 0, corr, corr + 1, 0, 0, corr_phases);
      if (rc) return rc;
      continue;
    }
    for (int upd = 0; upd < n_update_iterations; ++upd) {
      rc = LaunchTrack(ctx, 0, corr, corr + 1, 1, upd,
                       (upd == 0 ? corr_phases : unsigned(PH_LOAD_REGION | PH_LOAD_DEPTH)) | PH_REGION_GH | PH_DEPTH_GH |
                           PH_STORE_LINK_GH | tex);
      if (!rc) rc = LaunchStructure(ctx, 0, false);
      if (rc) return rc;
    }
  }
  return M3TB_OK;
}

}  // namespace

extern "C" {

int m3tb_refine_poses(m3tb_ctx* ctx, const int* bodies, int n_bodies, const int* structures, int n_structures,
                      int n_corr_iterations, int n_update_iterations) {
  CHECK_CTX();
  return RefinePoses(ctx, bodies, n_bodies, structures, n_structures, n_corr_iterations, n_update_iterations, false,
                     nullptr);
}

int m3tb_refine_poses_orb(m3tb_ctx* ctx, const int* bodies, int n_bodies, const int* structures, int n_structures,
                          int n_corr_iterations, int n_update_iterations, const m3tb_orb_params* orb_params) {
  CHECK_CTX();
  return RefinePoses(ctx, bodies, n_bodies, structures, n_structures, n_corr_iterations, n_update_iterations, true,
                     orb_params);
}

int m3tb_get_link_poses(m3tb_ctx* ctx, int structure, float* body2joint, float* joint2parent, float* link2world) {
  CHECK_CTX();
  if (structure < 0 || structure >= int(ctx->structures.size())) return Fail(ctx, M3TB_ERR_INVALID, "structure index out of range");
  int rc = PullLinks(ctx);
  if (rc) return rc;
  const StructureHost& s = ctx->structures[structure];
  std::vector<float> poses;
  if (link2world) {
    poses.resize(size_t(12) * std::max(ctx->n_bodies, 1));
    CU(cudaMemcpyAsync(poses.data(), ctx->d_poses, sizeof(float) * 12 * ctx->n_bodies, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  for (size_t i = 0; i < s.links.size(); ++i) {
    const LinkDev& l = s.links[i];
    if (body2joint) std::memcpy(body2joint + 12 * i, l.body2joint, sizeof(float) * 12);
    if (joint2parent) std::memcpy(joint2parent + 12 * i, l.joint2parent, sizeof(float) * 12);
    if (link2world) std::memcpy(link2world + 12 * i, l.body >= 0 ? poses.data() + 12 * l.body : l.link2world, sizeof(float) * 12);
  }
  return M3TB_OK;
}

int m3tb_get_structure_theta(m3tb_ctx* ctx, int structure, float* theta, int capacity, int* n_out, int* updated) {
  CHECK_CTX();
  if (structure < 0 || structure >= ctx->n_struct_launch || ctx->structures_dirty)
    return Fail(ctx, M3TB_ERR_INVALID, "structure index out of range / no optimisation ran yet");
  const StructureDev& d = ctx->h_structures[structure];
  const int n = d.dof + d.n_rows;
  if (n_out) *n_out = n;
  if (theta) {
    if (capacity < n) return Fail(ctx, M3TB_ERR_INVALID, "theta buffer too small");
    const int n_copy = capacity >= kMaxSystem ? kMaxSystem : n;  // the tail holds debug stamps in M3TB_STRUCT_STAMPS builds
    CU(cudaMemcpyAsync(theta, ctx->d_theta + size_t(structure) * kMaxSystem, sizeof(float) * n_copy, cudaMemcpyDeviceToHost, ctx->stream));
  }
  int st = 0;
  CU(cudaMemcpyAsync(&st, ctx->d_struct_status + structure, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (updated) *updated = st;
  return M3TB_OK;
}

int m3tb_get_region_lines(m3tb_ctx* ctx, int body, m3tb_region_line* lines, int capacity, int* n_out) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->n_bodies || !lines || !ctx->d_rstate) return Fail(ctx, M3TB_ERR_INVALID, "bad body / no state");
  int counts[4];
  CU(cudaMemcpyAsync(counts, ctx->d_counts + 4 * body, sizeof(counts), cudaMemcpyDeviceToHost, ctx->stream));
  const int cap = ctx->line_cap;
  std::vector<float> st(size_t(RF_COUNT) * cap);
  CU(cudaMemcpyAsync(st.data(), ctx->d_rstate + size_t(body) * RF_COUNT * cap, st.size() * sizeof(float),
                     cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  int n = std::min(counts[0], capacity);
  for (int i = 0; i < n; ++i) {
    m3tb_region_line& L = lines[i];
    std::memset(&L, 0, sizeof(L));
    L.model_index = i;
    L.valid = st[RF_VALID * cap + i] != 0.0f;
    L.center_f_body[0] = st[RF_CBX * cap + i]; L.center_f_body[1] = st[RF_CBY * cap + i]; L.center_f_body[2] = st[RF_CBZ * cap + i];
    L.center_u = st[RF_CU * cap + i]; L.center_v = st[RF_CV * cap + i];
    L.normal_u = st[RF_NU * cap + i]; L.normal_v = st[RF_NV * cap + i];
    if (L.valid) {
      L.delta_r = st[RF_DR * cap + i];
      L.normal_component_to_scale = st[RF_NCTS * cap + i];
      for (int d = 0; d < kDistributionLength; ++d) L.distribution[d] = st[(RF_DIST0 + d) * cap + i];
      L.mean = st[RF_MEAN * cap + i];
      L.measured_variance = st[RF_VAR * cap + i];
    }
  }
  if (n_out) *n_out = counts[0];
  return M3TB_OK;
}

int m3tb_get_depth_points(m3tb_ctx* ctx, int body, m3tb_depth_point* points, int capacity, int* n_out) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->n_bodies || !points || !ctx->d_dstate) return Fail(ctx, M3TB_ERR_INVALID, "bad body / no state");
  int counts[4];
  CU(cudaMemcpyAsync(counts, ctx->d_counts + 4 * body, sizeof(counts), cudaMemcpyDeviceToHost, ctx->stream));
  const int cap = ctx->point_cap;
  std::vector<float> st(size_t(DF_COUNT) * cap);
  CU(cudaMemcpyAsync(st.data(), ctx->d_dstate + size_t(body) * DF_COUNT * cap, st.size() * sizeof(float),
                     cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  int n = std::min(counts[1], capacity);
  for (int i = 0; i < n; ++i) {
    m3tb_depth_point& P = points[i];
    std::memset(&P, 0, sizeof(P));
    P.model_index = i;
    P.valid = st[DF_VALID * cap + i] != 0.0f;
    P.center_f_body[0] = st[DF_CBX * cap + i]; P.center_f_body[1] = st[DF_CBY * cap + i]; P.center_f_body[2] = st[DF_CBZ * cap + i];
    P.normal_f_body[0] = st[DF_NX * cap + i]; P.normal_f_body[1] = st[DF_NY * cap + i]; P.normal_f_body[2] = st[DF_NZ * cap + i];
    if (P.valid) {
      P.correspondence_center_f_camera[0] = st[DF_YX * cap + i];
      P.correspondence_center_f_camera[1] = st[DF_YY * cap + i];
      P.correspondence_center_f_camera[2] = st[DF_YZ * cap + i];
    }
  }
  if (n_out) *n_out = counts[1];
  return M3TB_OK;
}

int m3tb_prefetch_frames(m3tb_ctx* ctx) {
  CHECK_CTX();
  if (!ctx->ingest_pending || ctx->n_bodies == 0) return M3TB_OK;
  // Only when every camera in use has a fresh pinned frame in a pool slot: the whole frame set moves to the other
  // buffer. Anything else keeps the synchronous ingest at the next consumer launch.
  for (int k = 0; k < 2; ++k) {
    const bool color = k == 0;
    const ImagePool& pool = color ? ctx->color_pool : ctx->depth_pool;
    for (int i = 0; i < ctx->max_cameras; ++i) {
      const CameraDev& c = CameraOf(ctx, color, i);
      if (!c.set || !c.image) continue;
      if (!c.host_src || !pool.base || c.image != pool.base + pool.frame_bytes * i) return M3TB_OK;
    }
  }
  // Everything this call creates is made first and moved into the context once all of it exists.
  PrefetchResources pf;
  if (!ctx->pf.ingest_stream) {
    CU(pf.ingest_stream.create());
    CU(pf.table_stream.create());
    CU(pf.ev_ingest_done.create());
    CU(pf.ev_poses_snap.create());
    CU(pf.ev_tables.create());
    for (int q = 0; q < 2; ++q) CU(pf.ev_stage[q].create());
    for (int q = 0; q < 4; ++q) CU(pf.cam_stage[q >> 1][q & 1].create(ctx->max_cameras));
    CU(pf.ccams_alt.create(ctx->max_cameras));
    CU(pf.dcams_alt.create(ctx->max_cameras));
    CU(pf.roi_alt.create(2 * size_t(ctx->max_bodies)));
    CU(cudaMemset(pf.roi_alt, 0xff, sizeof(RoiRecord) * 2 * ctx->max_bodies));
    for (int q = 0; q < 2; ++q) CU(pf.poses_snap[q].create(12 * size_t(ctx->max_bodies)));
  }
  ImagePool new_alt[2];
  for (int k = 0; k < 2; ++k) {
    const ImagePool& pool = k == 0 ? ctx->color_pool : ctx->depth_pool;
    const ImagePool& alt = k == 0 ? ctx->color_pool_alt : ctx->depth_pool_alt;
    if (pool.base && !alt.base) {
      ImagePool& n = new_alt[k];
      n.frame_bytes = pool.frame_bytes; n.pitch = pool.pitch;
      n.width = pool.width; n.height = pool.height; n.capacity = pool.capacity;
      n.bin_frame_bytes = pool.bin_frame_bytes; n.bin_pitch = pool.bin_pitch;
      CU(n.base.create(n.frame_bytes * n.capacity));
      if (pool.bins) CU(n.bins.create(n.bin_frame_bytes * n.capacity));
    }
  }
  if (pf.ingest_stream) ctx->pf = std::move(pf);
  for (int k = 0; k < 2; ++k) {
    ImagePool& pool = k == 0 ? ctx->color_pool : ctx->depth_pool;
    ImagePool& alt = k == 0 ? ctx->color_pool_alt : ctx->depth_pool_alt;
    if (new_alt[k].base) alt = std::move(new_alt[k]);
    std::swap(pool, alt);
    std::vector<CameraDev>& cams = k == 0 ? ctx->h_ccams : ctx->h_dcams;
    for (int i = 0; i < ctx->max_cameras; ++i)
      if (cams[i].set && cams[i].image) {
        cams[i].image = pool.base + pool.frame_bytes * i;
        if (k == 0 && pool.bins) cams[i].bins = pool.BinImage(i);
      }
  }
  ctx->cams_dirty = false;   // the camera tables go to the alternate device copies below, on the side stream
  int rc = SyncTables(ctx);  // bodies / models only (main stream, small)
  if (rc) return rc;
  std::swap(ctx->d_ccams, ctx->pf.ccams_alt);
  std::swap(ctx->d_dcams, ctx->pf.dcams_alt);
  std::swap(ctx->d_roi, ctx->pf.roi_alt);
  // Stream plan. The ingest stream runs the ingests back to back: anything queued on it in front of k_ingest would sit
  // between two PCIe-bound kernels (two pageable table copies, a memset and the wait for the pose snapshot would
  // lengthen every end-to-end step). So the set-up goes to a third stream, beside the ingest in flight: wait for the pose
  // snapshot of the last tracking launch (which also orders it behind every reader of the buffers swapped in above: they
  // precede that launch on the main stream), camera tables from pinned staging, counter reset; the ingest stream then
  // waits for one event that is normally long past.
  cudaStream_t is = ctx->pf.ingest_stream, ts = ctx->pf.table_stream;
  const float* poses = ctx->d_poses;
  if (ctx->poses_snap_valid) {
    CU(cudaStreamWaitEvent(ts, ctx->pf.ev_poses_snap, 0));
    poses = ctx->pf.poses_snap[ctx->snap_parity];
  } else {
    CU(cudaStreamSynchronize(ctx->stream));  // first frame: nothing in flight that could be writing the poses
  }
  ctx->stage_parity ^= 1;  // the staging of the prefetch before this one may still be in flight; the one before that
  CU(cudaEventSynchronize(ctx->pf.ev_stage[ctx->stage_parity]));  // normally is not (a host that never waits could be ahead)
  CameraDev* stage_c = ctx->pf.cam_stage[ctx->stage_parity][0];
  CameraDev* stage_d = ctx->pf.cam_stage[ctx->stage_parity][1];
  std::memcpy(stage_c, ctx->h_ccams.data(), sizeof(CameraDev) * ctx->max_cameras);
  std::memcpy(stage_d, ctx->h_dcams.data(), sizeof(CameraDev) * ctx->max_cameras);
  CU(cudaMemcpyAsync(ctx->d_ccams, stage_c, sizeof(CameraDev) * ctx->max_cameras, cudaMemcpyHostToDevice, ts));
  CU(cudaMemcpyAsync(ctx->d_dcams, stage_d, sizeof(CameraDev) * ctx->max_cameras, cudaMemcpyHostToDevice, ts));
  CU(cudaEventRecord(ctx->pf.ev_stage[ctx->stage_parity], ts));
  ctx->cams_dirty = false;
  ctx->ingest_bytes_slot ^= 1;
  CU(cudaMemsetAsync(ctx->d_ingest_bytes + ctx->ingest_bytes_slot, 0, sizeof(unsigned long long), ts));
  CU(cudaEventRecord(ctx->pf.ev_tables, ts));
  CU(cudaStreamWaitEvent(is, ctx->pf.ev_tables, 0));
  IngestArgs a;
  a.bodies = ctx->d_bodies;
  a.poses = poses;
  a.color_cams = ctx->d_ccams;
  a.depth_cams = ctx->d_dcams;
  a.region_models = ctx->d_rmodels;
  a.depth_models = ctx->d_dmodels;
  a.roi = ctx->d_roi;
  a.bytes = ctx->d_ingest_bytes + ctx->ingest_bytes_slot;
  a.n_bodies = ctx->n_bodies;
  a.body_list = nullptr;
  // Grid of the prefetch ingest: a quarter of the SMs, CTAs looping over the bodies. k_track2 takes a whole SM per body
  // (1024 threads x 64 registers), so an ingest CTA that sits on an SM keeps a body waiting for as long as the ingest
  // lasts, and whichever kernel is dispatched first wins: with one CTA per body the end-to-end step time swings widely
  // once both kernels become ready at the same moment. One CTA keeps 16 KB in flight; a few dozen keep the link busy
  // (scripts/probes/pcie_probe.cu measures it). M3TB_INGEST_CTAS overrides the grid.
  static const int forced_ctas = [] { const char* e = std::getenv("M3TB_INGEST_CTAS"); return e ? std::atoi(e) : 0; }();
  int ingest_ctas = std::max(16, ctx->sm_count / 4);
  if (forced_ctas > 0) ingest_ctas = forced_ctas;
  ingest_ctas = std::min(ingest_ctas, ctx->n_bodies);
  NoteIngestBins(ctx);
  k_ingest<<<ingest_ctas, kBlockThreads, 0, is>>>(a);
  CU(cudaGetLastError());
  CU(cudaEventRecord(ctx->pf.ev_ingest_done, is));
  ctx->launches++;
  ctx->ingest_pending = false;
  ctx->prefetched = true;
  ctx->prefetch_enabled = true;
  return M3TB_OK;
}

static int UploadRendering(m3tb_ctx* ctx, int body, int slot, const m3tb_rendering* r, int bytes_per_pixel) {
  if (body < 0 || body >= ctx->max_bodies || !r || !r->image || r->image_size <= 0 ||
      r->pitch < size_t(r->image_size) * bytes_per_pixel || !(r->scale > 0.0f))
    return Fail(ctx, M3TB_ERR_INVALID, "bad rendering arguments");
  if (ctx->attached[body][slot] >= 0)
    return Fail(ctx, M3TB_ERR_INVALID, "a device renderer is attached to this slot (m3tb_attach_renderer(..., -1) detaches it)");
  RenderingDev& d = ctx->h_bodies[body].rend[slot];
  const unsigned pitch = unsigned(Align(size_t(r->image_size) * bytes_per_pixel, 16));
  if (!d.image || d.image_size != r->image_size) {
    DeviceBuffer<uint8_t> image;
    CU(image.create(size_t(pitch) * r->image_size));
    if (d.image) CU(cudaStreamSynchronize(ctx->stream));
    ctx->rendering_images[body][slot] = std::move(image);
    d.image = ctx->rendering_images[body][slot];
    ctx->bodies_dirty = true;  // the device copy of the record must not keep the released image
  }
  CU(cudaMemcpy2DAsync(const_cast<uint8_t*>(d.image), pitch, r->image, r->pitch, size_t(r->image_size) * bytes_per_pixel,
                       r->image_size, cudaMemcpyDefault, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));  // Camera::UpdateImage-style copy semantics: the caller's image is free again
  d.image_size = r->image_size;
  d.pitch = pitch;
  d.corner_u = r->corner_u; d.corner_v = r->corner_v; d.scale = r->scale;
  d.projection_term_a = r->projection_term_a; d.projection_term_b = r->projection_term_b;
  d.id = r->id;
  d.visible = r->visible ? 1 : 0;
  ctx->bodies_dirty = true;
  return M3TB_OK;
}

int m3tb_upload_depth_rendering(m3tb_ctx* ctx, int body, int modality, const m3tb_rendering* rendering) {
  CHECK_CTX();
  if (modality != 0 && modality != 1) return Fail(ctx, M3TB_ERR_INVALID, "modality must be 0 (region) or 1 (depth)");
  return UploadRendering(ctx, body, modality == 0 ? RS_REGION_DEPTH : RS_DEPTH_DEPTH, rendering, 2);
}

int m3tb_upload_silhouette_rendering(m3tb_ctx* ctx, int body, int modality, const m3tb_rendering* rendering) {
  CHECK_CTX();
  if (modality != 0 && modality != 1) return Fail(ctx, M3TB_ERR_INVALID, "modality must be 0 (region) or 1 (depth)");
  return UploadRendering(ctx, body, modality == 0 ? RS_REGION_SILHOUETTE : RS_DEPTH_SILHOUETTE, rendering, 1);
}

int m3tb_set_body_geometry(m3tb_ctx* ctx, int body, const float* triangles, int n_triangles,
                           const float geometry2body[12], float maximum_body_diameter, int enable_culling, int body_id,
                           int region_id) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->max_bodies) return Fail(ctx, M3TB_ERR_INVALID, "body index out of range");
  if (!triangles || n_triangles < 1 || !geometry2body || !(maximum_body_diameter > 0.0f) ||
      !std::isfinite(maximum_body_diameter))
    return Fail(ctx, M3TB_ERR_INVALID, "bad geometry arguments");
  if (body_id < 0 || body_id > 255 || region_id < 0 || region_id > 255)
    return Fail(ctx, M3TB_ERR_INVALID, "body_id / region_id must be uint8 values");
  GeometryDev& G = ctx->h_geometry[body];
  DeviceBuffer<float>& soup = ctx->geometry_alloc[body];
  if (soup.size() != 9 * size_t(n_triangles)) {
    DeviceBuffer<float> s;
    CU(s.create(9 * size_t(n_triangles)));
    if (soup) CU(cudaStreamSynchronize(ctx->stream));  // a render in flight may still read the old soup
    soup = std::move(s);
    G.triangles = soup;
    G.n_triangles = n_triangles;
  }
  CU(cudaMemcpyAsync(soup, triangles, sizeof(float) * 9 * size_t(n_triangles), cudaMemcpyHostToDevice,
                     ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));  // the caller's triangles are free again
  std::memcpy(G.geometry2body, geometry2body, sizeof(G.geometry2body));
  G.radius = 0.5f * maximum_body_diameter;  // FocusedRenderer::CalculateProjectionMatrix (renderer.cpp:356)
  G.enable_culling = enable_culling ? 1 : 0;
  G.body_id = body_id;
  G.region_id = region_id;
  G.set = 1;
  ctx->render_dirty = true;
  return M3TB_OK;
}

int m3tb_set_focused_renderer(m3tb_ctx* ctx, int renderer, int camera_kind, int camera, int image_size, float z_min,
                              float z_max, int id_type, const int* geometry_bodies, int n_geometry,
                              const int* referenced_bodies, int n_referenced) {
  CHECK_CTX();
  if (renderer < 0 || renderer > int(ctx->renderers.size()) || renderer >= 4 * ctx->max_bodies)
    return Fail(ctx, M3TB_ERR_INVALID, "renderer ids must be dense (0..n) and below 4 * max_bodies");
  if (camera_kind != 0 && camera_kind != 1) return Fail(ctx, M3TB_ERR_INVALID, "camera_kind must be 0 (colour) or 1 (depth)");
  int rc = CheckCameraSet(ctx, camera_kind, camera);
  if (rc) return rc;
  if (image_size > kRenderMaxImageSize)
    return Fail(ctx, M3TB_ERR_UNSUPPORTED, "image_size above " + std::to_string(kRenderMaxImageSize) +
                                               " (the z-buffer lives in shared memory)");
  if (image_size < 1 || !(z_min > 0.0f) || !(z_max > z_min) || !std::isfinite(z_max))
    return Fail(ctx, M3TB_ERR_INVALID, "bad image_size / z_min / z_max");
  if (id_type != RID_BODY && id_type != RID_REGION) return Fail(ctx, M3TB_ERR_INVALID, "id_type must be 0 (BODY) or 1 (REGION)");
  if (!geometry_bodies || n_geometry < 1 || n_geometry > 65535 || !referenced_bodies || n_referenced < 1)
    return Fail(ctx, M3TB_ERR_INVALID, "a renderer needs geometry bodies and referenced bodies");
  rc = CheckBodyList(ctx, geometry_bodies, n_geometry);
  if (!rc) rc = CheckBodyList(ctx, referenced_bodies, n_referenced);
  if (rc) return rc;
  if (renderer < int(ctx->renderers.size()))
    for (const auto& at : ctx->attached)
      for (int r : at)
        if (r == renderer) return Fail(ctx, M3TB_ERR_INVALID, "renderer is attached to a modality: detach it first");
  const bool is_new = renderer == int(ctx->renderers.size());
  const unsigned depth_pitch = unsigned(Align(size_t(image_size) * 2, 16));
  const unsigned silhouette_pitch = unsigned(Align(size_t(image_size), 16));
  DeviceBuffer<uint16_t> depth;
  DeviceBuffer<uint8_t> silhouette;
  if (is_new || ctx->renderers[renderer].dev.image_size != image_size) {
    CU(depth.create(size_t(depth_pitch) / 2 * image_size));
    CU(silhouette.create(size_t(silhouette_pitch) * image_size));
    CU(cudaStreamSynchronize(ctx->stream));  // a render in flight may still write the old images
    CU(cudaMemsetAsync(depth, 0xff, size_t(depth_pitch) * image_size, ctx->stream));  // cleared: depth 1.0
    CU(cudaMemsetAsync(silhouette, 0, size_t(silhouette_pitch) * image_size, ctx->stream));
  }
  if (is_new) {
    ctx->renderers.emplace_back();
    std::memset(&ctx->renderers.back().dev, 0, sizeof(RendererDev));
  }
  auto& h = ctx->renderers[renderer];
  RendererDev& R = h.dev;
  if (depth) {
    h.depth = std::move(depth);
    h.silhouette = std::move(silhouette);
    R.depth = h.depth;
    R.silhouette = h.silhouette;
    R.depth_pitch = depth_pitch;
    R.silhouette_pitch = silhouette_pitch;
  }
  R.camera_kind = camera_kind;
  R.camera = camera;
  R.image_size = image_size;
  R.id_type = id_type;
  R.z_min = z_min;
  R.z_max = z_max;
  R.set = 1;
  h.geometry.assign(geometry_bodies, geometry_bodies + n_geometry);
  h.referenced.assign(referenced_bodies, referenced_bodies + n_referenced);
  h.rendered = false;
  ctx->render_dirty = true;
  return M3TB_OK;
}

// TextureModality's silhouette renderer (kind 1, IDType::BODY; it feeds the silhouette and the depth slot) and depth
// renderer (kind 0, model_occlusions), texture_modality.cpp:517-524
static int AttachTextureRenderer(m3tb_ctx* ctx, int body, int kind, int renderer) {
  BodyDev& B = ctx->h_bodies[body];
  if (!B.has_texture) return Fail(ctx, M3TB_ERR_INVALID, "body has no such modality");
  const int slots[2] = {kind == 1 ? RS_TEXTURE_SILHOUETTE : RS_TEXTURE_DEPTH, kind == 1 ? RS_TEXTURE_SILHOUETTE_DEPTH : -1};
  if (renderer != -1) {
    if (renderer < 0 || renderer >= int(ctx->renderers.size())) return Fail(ctx, M3TB_ERR_INVALID, "renderer not set");
    const auto& h = ctx->renderers[renderer];
    if (h.dev.camera_kind != 0 || h.dev.camera != B.texture_camera)
      return Fail(ctx, M3TB_ERR_INVALID, "the renderer does not render the modality's camera");
    if (std::find(h.referenced.begin(), h.referenced.end(), body) == h.referenced.end())
      return Fail(ctx, M3TB_ERR_INVALID, "the renderer does not reference the body");
    if (kind == 1 && h.dev.id_type != RID_BODY)
      return Fail(ctx, M3TB_ERR_INVALID, "the texture modality needs a silhouette renderer of id_type BODY");
  }
  for (int slot : slots) {
    if (slot < 0) continue;
    int& cur = ctx->attached[body][slot];
    RenderingDev& d = B.rend[slot];
    if (renderer == -1) {
      if (cur < 0) continue;
      std::memset(&d, 0, sizeof(d));
      cur = -1;
      ctx->n_attached--;
    } else {
      const RendererDev& R = ctx->renderers[renderer].dev;
      const bool sil = slot == RS_TEXTURE_SILHOUETTE;
      std::memset(&d, 0, sizeof(d));  // visible = 0 until the first render
      d.image = sil ? R.silhouette : reinterpret_cast<const uint8_t*>(R.depth);
      d.image_size = R.image_size;
      d.pitch = sil ? R.silhouette_pitch : R.depth_pitch;
      if (cur < 0) ctx->n_attached++;
      cur = renderer;
      ctx->attach_uploaded[body][slot] = 0;
    }
    ctx->bodies_dirty = true;
    ctx->render_dirty = true;
  }
  return M3TB_OK;
}

int m3tb_attach_renderer(m3tb_ctx* ctx, int body, int modality, int kind, int renderer) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->n_bodies || !ctx->h_bodies[body].set) return Fail(ctx, M3TB_ERR_INVALID, "body not set");
  if (modality != 0 && modality != 1 && modality != 2)
    return Fail(ctx, M3TB_ERR_INVALID, "modality must be 0 (region), 1 (depth) or 2 (texture)");
  if (kind != 0 && kind != 1) return Fail(ctx, M3TB_ERR_INVALID, "kind must be 0 (depth) or 1 (silhouette)");
  if (modality == 2) return AttachTextureRenderer(ctx, body, kind, renderer);
  BodyDev& B = ctx->h_bodies[body];
  if (!(modality == 0 ? B.has_region : B.has_depth)) return Fail(ctx, M3TB_ERR_INVALID, "body has no such modality");
  const int slot = modality == 0 ? (kind == 0 ? RS_REGION_DEPTH : RS_REGION_SILHOUETTE)
                                 : (kind == 0 ? RS_DEPTH_DEPTH : RS_DEPTH_SILHOUETTE);
  int& cur = ctx->attached[body][slot];
  if (renderer == -1) {  // DoNotModelOcclusions / DoNotUseRegionChecking / DoNotUseSilhouetteChecking
    if (cur >= 0) {
      std::memset(&B.rend[slot], 0, sizeof(RenderingDev));
      cur = -1;
      ctx->n_attached--;
      ctx->bodies_dirty = true;
      ctx->render_dirty = true;
    }
    return M3TB_OK;
  }
  if (renderer < 0 || renderer >= int(ctx->renderers.size())) return Fail(ctx, M3TB_ERR_INVALID, "renderer not set");
  const auto& h = ctx->renderers[renderer];
  const RendererDev& R = h.dev;
  // what RegionModality / DepthModality::SetUp require of the renderer (region_modality.cpp:66-86, depth_modality.cpp:56-76)
  if (R.camera_kind != modality || R.camera != (modality == 0 ? B.color_camera : B.depth_camera))
    return Fail(ctx, M3TB_ERR_INVALID, "the renderer does not render the modality's camera");
  if (std::find(h.referenced.begin(), h.referenced.end(), body) == h.referenced.end())
    return Fail(ctx, M3TB_ERR_INVALID, "the renderer does not reference the body");
  if (kind == 1 && R.id_type != (modality == 0 ? RID_REGION : RID_BODY))
    return Fail(ctx, M3TB_ERR_INVALID, modality == 0 ? "region checking needs a silhouette renderer of id_type REGION"
                                                     : "silhouette checking needs a silhouette renderer of id_type BODY");
  RenderingDev& d = B.rend[slot];
  std::memset(&d, 0, sizeof(d));  // visible = 0: the checks stay off until the first render
  d.image = kind == 1 ? R.silhouette : reinterpret_cast<const uint8_t*>(R.depth);
  d.image_size = R.image_size;
  d.pitch = kind == 1 ? R.silhouette_pitch : R.depth_pitch;
  if (cur < 0) ctx->n_attached++;
  cur = renderer;
  ctx->attach_uploaded[body][slot] = 0;
  ctx->bodies_dirty = true;
  ctx->render_dirty = true;
  return M3TB_OK;
}

int m3tb_render(m3tb_ctx* ctx) {
  CHECK_CTX();
  if (ctx->renderers.empty()) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "no device renderer set");
  return LaunchRender(ctx, kRenderAll);
}

int m3tb_get_rendering(m3tb_ctx* ctx, int renderer, void* depth_u16, void* silhouette_u8, float* corner_u, float* corner_v,
                       float* scale, float* projection_term_a, float* projection_term_b, int* visible_flags) {
  CHECK_CTX();
  if (renderer < 0 || renderer >= int(ctx->renderers.size())) return Fail(ctx, M3TB_ERR_INVALID, "renderer not set");
  const auto& h = ctx->renderers[renderer];
  if (!h.rendered) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "renderer has not rendered since it was set");
  const RendererDev& R = h.dev;
  const size_t S = size_t(R.image_size);
  if (depth_u16)
    CU(cudaMemcpy2DAsync(depth_u16, S * 2, R.depth, R.depth_pitch, S * 2, S, cudaMemcpyDeviceToHost, ctx->stream));
  if (silhouette_u8)
    CU(cudaMemcpy2DAsync(silhouette_u8, S, R.silhouette, R.silhouette_pitch, S, S, cudaMemcpyDeviceToHost, ctx->stream));
  RenderOutDev o;
  CU(cudaMemcpyAsync(&o, ctx->d_render_out + renderer, sizeof(o), cudaMemcpyDeviceToHost, ctx->stream));
  if (visible_flags)
    CU(cudaMemcpyAsync(visible_flags, ctx->d_visible + R.first_referenced, sizeof(int) * R.n_referenced,
                       cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (corner_u) *corner_u = o.corner_u;
  if (corner_v) *corner_v = o.corner_v;
  if (scale) *scale = o.scale;
  if (projection_term_a) *projection_term_a = o.projection_term_a;
  if (projection_term_b) *projection_term_b = o.projection_term_b;
  return M3TB_OK;
}

int m3tb_detach_frames(m3tb_ctx* ctx) {
  CHECK_CTX();
  if (ctx->pf.ingest_stream) CU(cudaStreamSynchronize(ctx->pf.ingest_stream));  // a prefetch may still be reading the frames
  bool any = false;
  for (int k = 0; k < 2; ++k) {
    std::vector<CameraDev>& cams = k == 0 ? ctx->h_ccams : ctx->h_dcams;
    for (CameraDev& c : cams) {
      if (!c.set || !c.image || !c.host_src) continue;
      const size_t row = size_t(c.width) * (k == 0 ? 3 : 2);
      CU(cudaMemcpy2DAsync(const_cast<uint8_t*>(c.image), c.pitch, c.host_src, c.host_pitch, row, c.height,
                           cudaMemcpyHostToDevice, ctx->stream));
      c.host_src = nullptr;  // FrameView: the whole device copy is valid from now on
      c.host_pitch = 0;
      if (k == 0) ctx->bin_shift[size_t(&c - cams.data())] = kBinsNone;
      any = true;
    }
  }
  if (any) {
    ctx->cams_dirty = true;
    ctx->ingest_pending = false;  // nothing left to fetch by rectangle
    int rc = SyncTables(ctx);
    if (rc) return rc;
  }
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

int m3tb_last_ingest_bytes(m3tb_ctx* ctx, unsigned long long* bytes) {
  CHECK_CTX();
  if (!bytes) return Fail(ctx, M3TB_ERR_INVALID, "null output");
  CU(cudaMemcpyAsync(bytes, ctx->d_ingest_bytes + ctx->ingest_bytes_slot, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

int m3tb_debug_phase_clocks(m3tb_ctx* ctx, int body, long long* out, int capacity) {
  CHECK_CTX();
  if (!ctx->d_phase_clock) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "create the context with M3TB_TIMING=1 in the environment");
  if (body < 0 || body >= ctx->max_bodies || !out) return Fail(ctx, M3TB_ERR_INVALID, "bad body");
  int n = std::min(capacity, int(kPhaseSlots));
  CU(cudaMemcpyAsync(out, ctx->d_phase_clock + size_t(body) * kPhaseSlots, sizeof(long long) * n, cudaMemcpyDeviceToHost,
                     ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

int m3tb_debug_last_launch(m3tb_ctx* ctx, m3tb_launch_info* out) {
  if (!ctx) return M3TB_ERR_INVALID;
  if (!out) return Fail(ctx, M3TB_ERR_INVALID, "null output");
  *out = ctx->last_launch;
  return M3TB_OK;
}

int m3tb_debug_bin_image(m3tb_ctx* ctx, int cam, uint16_t* out, size_t out_pitch, m3tb_bin_image_info* info) {
  CHECK_CTX();
  if (cam < 0 || cam >= ctx->max_cameras || !info) return Fail(ctx, M3TB_ERR_INVALID, "bad bin-image arguments");
  const CameraDev& c = ctx->h_ccams[cam];
  if (out && c.bins && out_pitch < size_t(c.width) * 2) return Fail(ctx, M3TB_ERR_INVALID, "pitch smaller than a row");
  if (ctx->pf.ingest_stream) CU(cudaStreamSynchronize(ctx->pf.ingest_stream));  // a prefetched ingest writes the image
  CU(cudaStreamSynchronize(ctx->stream));
  info->state = ctx->bin_shift[cam];
  info->pinned = c.host_src ? 1 : 0;
  info->has_image = c.bins ? 1 : 0;
  info->width = c.width;
  info->height = c.height;
  info->generation = c.generation;
  info->n_rois = 0;
  std::vector<RoiRecord> roi(2 * size_t(ctx->max_bodies));
  CU(cudaMemcpy(roi.data(), ctx->d_roi, sizeof(RoiRecord) * roi.size(), cudaMemcpyDeviceToHost));
  for (int b = 0; b < ctx->n_bodies; ++b) {
    const BodyDev& B = ctx->h_bodies[b];
    if (!B.set || !B.has_region || B.color_camera != cam) continue;
    if (info->rois && info->n_rois < info->roi_capacity) {
      const RoiRecord& r = roi[2 * size_t(b)];
      info->rois[info->n_rois] = m3tb_roi_record{b, r.x0, r.y0, r.x1, r.y1, r.generation};
    }
    info->n_rois++;
  }
  if (out && c.bins)
    CU(cudaMemcpy2D(out, out_pitch, c.bins, c.bin_pitch, size_t(c.width) * 2, c.height, cudaMemcpyDeviceToHost));
  return M3TB_OK;
}

int m3tb_debug_closest_view(const float* orientations, int n_views, const float* queries, int n_queries,
                            const int* prev, int* out_scan, int* out_pruned, int* out_evaluated) {
  if (!orientations || n_views <= 0 || !queries || n_queries < 0 || !out_scan || !out_pruned) return M3TB_ERR_INVALID;
  ViewClustersHost vc;
  BuildViewClusters(orientations, n_views, vc);
  for (int q = 0; q < n_queries; ++q) {
    const float* o = queries + 3 * q;
    // the reference's scan (region_model.cpp:121-128): closest_dot = -1, strict >, views_[0] otherwise
    float best = -1.0f;
    int idx = 0;
    for (int v = 0; v < n_views; ++v) {
      const float dot = o[0] * orientations[3 * v] + o[1] * orientations[3 * v + 1] + o[2] * orientations[3 * v + 2];
      if (dot > best) { best = dot; idx = v; }
    }
    out_scan[q] = idx;
    int ev = 0;
    out_pruned[q] = ClosestViewPrunedHost(vc, orientations, n_views, o, prev ? prev[q] : 0, &ev);
    if (out_evaluated) out_evaluated[q] = ev;
  }
  return M3TB_OK;
}

int m3tb_get_closest_views(m3tb_ctx* ctx, int body, int* region_view, int* depth_view) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->n_bodies) return Fail(ctx, M3TB_ERR_INVALID, "bad body");
  int counts[4];
  CU(cudaMemcpyAsync(counts, ctx->d_counts + 4 * body, sizeof(counts), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (region_view) *region_view = counts[2];
  if (depth_view) *depth_view = counts[3];
  return M3TB_OK;
}

void m3tb_model_params_default(m3tb_model_params* p) {
  if (!p) return;
  p->sphere_radius = 0.8f;  // model.h:161-167
  p->n_divides = 4;
  p->n_points = 200;
  p->max_radius_depth_offset = 0.05f;
  p->stride_depth_offset = 0.002f;
  p->use_random_seed = 0;
  p->image_size = 2000;
}

int m3tb_model_views(const m3tb_model_params* params, float* camera2body, int capacity, int* n_views) {
  if (!params || !n_views || capacity < 0 || params->n_divides < 0 || params->n_divides > kModelMaxDivides)
    return M3TB_ERR_INVALID;
  const std::vector<float> poses = GeodesicPoses(params->n_divides, params->sphere_radius);
  *n_views = int(poses.size() / 12);
  if (camera2body) std::memcpy(camera2body, poses.data(), sizeof(float) * 12 * size_t(std::min(capacity, *n_views)));
  return M3TB_OK;
}

// What both generators do after their last launch: the points (`point_floats` floats each) and per-view scalars
// (surface areas or contour lengths) come back to the host, go through the same path as m3tb_set_depth_model /
// m3tb_set_region_model (repacking, depth-offset table, cluster tables of the closest-view search), and the host copy
// is kept for m3tb_get_depth_model / m3tb_get_region_model.
static int FinishGeneratedModel(m3tb_ctx* ctx, bool region, int model_id, const ModelSetup& st,
                                const m3tb_model_params* params, const float* d_points, const float* d_view_scalars,
                                int point_floats) {
  m3tb_ctx::GeneratedModel gm;
  gm.n_views = st.n_views;
  gm.n_points = params->n_points;
  gm.stride_depth_offset = params->stride_depth_offset;
  gm.max_radius_depth_offset = params->max_radius_depth_offset;
  gm.points.resize(size_t(st.n_views) * gm.n_points * point_floats);
  gm.view_scalars.resize(st.n_views);
  CU(cudaMemcpyAsync(gm.points.data(), d_points, sizeof(float) * gm.points.size(), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(gm.view_scalars.data(), d_view_scalars, sizeof(float) * st.n_views, cudaMemcpyDeviceToHost,
                     ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  gm.orientations.resize(size_t(st.n_views) * 3);
  for (int v = 0; v < st.n_views; ++v)  // views_[i].orientation = camera2body.matrix().col(2)
    for (int r = 0; r < 3; ++r) gm.orientations[3 * size_t(v) + r] = st.camera2body[12 * size_t(v) + 4 * r + 2];
  int rc = SetModel(ctx, region, model_id, gm.n_views, gm.n_points, gm.orientations.data(), gm.view_scalars.data(),
                    gm.points.data(), params->stride_depth_offset, params->max_radius_depth_offset);
  if (rc) return rc;
  auto& generated = region ? ctx->rmodel_generated : ctx->dmodel_generated;
  if (int(generated.size()) < ctx->max_models) generated.resize(ctx->max_models);
  generated[model_id] = std::move(gm);
  return M3TB_OK;
}

// m3tb_get_depth_model / m3tb_get_region_model: the host copy FinishGeneratedModel kept
static int GetGeneratedModel(m3tb_ctx* ctx, bool region, int model_id, int* n_views, int* n_points, float* orientations,
                             float* view_scalars, void* points, float* stride_depth_offset,
                             float* max_radius_depth_offset) {
  if (!ctx) return M3TB_ERR_INVALID;
  if (model_id < 0 || model_id >= ctx->max_models) return Fail(ctx, M3TB_ERR_INVALID, "model id out of range");
  const auto& generated = region ? ctx->rmodel_generated : ctx->dmodel_generated;
  if (model_id >= int(generated.size()) || generated[model_id].n_views == 0)
    return Fail(ctx, M3TB_ERR_NOT_SET_UP, region ? "region model was not generated by m3tb_generate_region_model"
                                                 : "depth model was not generated by m3tb_generate_depth_model");
  const auto& gm = generated[model_id];
  if (n_views) *n_views = gm.n_views;
  if (n_points) *n_points = gm.n_points;
  if (orientations) std::memcpy(orientations, gm.orientations.data(), sizeof(float) * gm.orientations.size());
  if (view_scalars) std::memcpy(view_scalars, gm.view_scalars.data(), sizeof(float) * gm.view_scalars.size());
  if (points) std::memcpy(points, gm.points.data(), sizeof(float) * gm.points.size());
  if (stride_depth_offset) *stride_depth_offset = gm.stride_depth_offset;
  if (max_radius_depth_offset) *max_radius_depth_offset = gm.max_radius_depth_offset;
  return M3TB_OK;
}

int m3tb_generate_depth_model(m3tb_ctx* ctx, int model_id, int body, const int* occlusion_bodies, int n_occlusion_bodies,
                              const m3tb_model_params* params) {
  CHECK_CTX();
  if (model_id < 0 || model_id >= ctx->max_models) return Fail(ctx, M3TB_ERR_INVALID, "model id out of range");
  ModelSetup st;
  int rc = PrepareModel(ctx, body, occlusion_bodies, n_occlusion_bodies, params, st);
  if (rc) return rc;
  const int n_points = params->n_points;
  ModelBuffers b;
  rc = AllocModel(ctx, st, 0, st.n_views, n_points, b);
  if (rc) return rc;
  for (int first = 0; first < st.n_views; first += b.batch) {
    const int count = std::min(b.batch, st.n_views - first);
    rc = RenderModelViews(ctx, st, b, first, count);
    if (rc) return rc;
    k_model_points<<<unsigned(count), kModelThreads, 0, ctx->stream>>>(PointArgs(st, b, params, first));
    CU(cudaGetLastError());
    ctx->launches++;
  }
  return FinishGeneratedModel(ctx, false, model_id, st, params, b.points, b.surface_area, 36);
}

int m3tb_get_depth_model(m3tb_ctx* ctx, int model_id, int* n_views, int* n_points, float* orientations,
                         float* surface_areas, void* points, float* stride_depth_offset, float* max_radius_depth_offset) {
  return GetGeneratedModel(ctx, false, model_id, n_views, n_points, orientations, surface_areas, points,
                           stride_depth_offset, max_radius_depth_offset);
}

int m3tb_debug_render_model_view(m3tb_ctx* ctx, int body, const int* occlusion_bodies, int n_occlusion_bodies,
                                 const m3tb_model_params* params, int view, uint8_t* normal_bgra, uint16_t* depth,
                                 uint8_t* silhouette) {
  CHECK_CTX();
  ModelSetup st;
  int rc = PrepareModel(ctx, body, occlusion_bodies, n_occlusion_bodies, params, st);
  if (rc) return rc;
  if (view < 0 || view >= st.n_views) return Fail(ctx, M3TB_ERR_INVALID, "view index out of range");
  ModelBuffers b;
  rc = AllocModel(ctx, st, view, 1, 0, b);  // one view: its z-buffers and tables only
  if (!rc) rc = RenderModelViews(ctx, st, b, 0, 1);
  if (rc) return rc;
  const size_t n_pix = size_t(st.S) * st.S;
  DeviceBuffer<uint8_t> d_normal, d_sil;
  DeviceBuffer<uint16_t> d_depth;
  CU(d_normal.create(4 * n_pix));
  CU(d_depth.create(n_pix));
  CU(d_sil.create(n_pix));
  k_model_images<<<unsigned((n_pix + 255) / 256), 256, 0, ctx->stream>>>(PointArgs(st, b, params, 0), 0, d_normal,
                                                                          d_depth, d_sil);
  CU(cudaGetLastError());
  ctx->launches++;
  if (normal_bgra) CU(cudaMemcpyAsync(normal_bgra, d_normal, 4 * n_pix, cudaMemcpyDeviceToHost, ctx->stream));
  if (depth) CU(cudaMemcpyAsync(depth, d_depth, 2 * n_pix, cudaMemcpyDeviceToHost, ctx->stream));
  if (silhouette) CU(cudaMemcpyAsync(silhouette, d_sil, n_pix, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

int m3tb_generate_region_model(m3tb_ctx* ctx, int model_id, int body, const m3tb_associated_body* associated,
                               int n_associated, const m3tb_model_params* params) {
  CHECK_CTX();
  if (model_id < 0 || model_id >= ctx->max_models) return Fail(ctx, M3TB_ERR_INVALID, "model id out of range");
  ModelSetup st;
  int rc = PrepareRegionModel(ctx, body, associated, n_associated, params, st);
  if (rc) return rc;
  const int n_points = params->n_points;
  ModelBuffers b;
  rc = AllocModel(ctx, st, 0, st.n_views, 0, b, RegionViewBytes(st.S, n_points));
  if (rc) return rc;
  RegionBuffers rb;
  rc = AllocRegion(ctx, st, b.batch, st.n_views, n_points, rb);
  if (rc) return rc;
  for (int first = 0; first < st.n_views; first += b.batch) {
    const int count = std::min(b.batch, st.n_views - first);
    rc = RenderModelViews(ctx, st, b, first, count);
    if (rc) return rc;
    k_region_contours<<<unsigned(count), kModelThreads, 0, ctx->stream>>>(ContourArgs(st, b, rb));
    CU(cudaGetLastError());
    k_region_points<<<unsigned(count), kModelThreads, 0, ctx->stream>>>(RegionArgs(st, b, rb, params, first));
    CU(cudaGetLastError());
    ctx->launches += 2;
  }
  rc = ContourOverflow(ctx, rb);
  if (rc) return rc;
  return FinishGeneratedModel(ctx, true, model_id, st, params, rb.points, rb.contour_length, kRegionPointFloats);
}

int m3tb_get_region_model(m3tb_ctx* ctx, int model_id, int* n_views, int* n_points, float* orientations,
                          float* contour_lengths, void* points, float* stride_depth_offset,
                          float* max_radius_depth_offset) {
  return GetGeneratedModel(ctx, true, model_id, n_views, n_points, orientations, contour_lengths, points,
                           stride_depth_offset, max_radius_depth_offset);
}

int m3tb_debug_region_model_view(m3tb_ctx* ctx, int body, const m3tb_associated_body* associated, int n_associated,
                                 const m3tb_model_params* params, int view, uint8_t* silhouettes, int* n_silhouettes,
                                 uint16_t* depth, int32_t* contour_points, int32_t* contour_offsets, int capacity,
                                 int* n_contour_points, int* n_contours) {
  CHECK_CTX();
  ModelSetup st;
  int rc = PrepareRegionModel(ctx, body, associated, n_associated, params, st);
  if (rc) return rc;
  if (view < 0 || view >= st.n_views) return Fail(ctx, M3TB_ERR_INVALID, "view index out of range");
  if (capacity < 0) return Fail(ctx, M3TB_ERR_INVALID, "negative capacity");
  ModelBuffers b;
  rc = AllocModel(ctx, st, view, 1, 0, b);  // one view: its z-buffers and tables only
  if (!rc) rc = RenderModelViews(ctx, st, b, 0, 1);
  if (rc) return rc;
  RegionBuffers rb;
  rc = AllocRegion(ctx, st, 1, 1, 0, rb);
  if (rc) return rc;
  k_region_contours<<<1, kModelThreads, 0, ctx->stream>>>(ContourArgs(st, b, rb));
  CU(cudaGetLastError());
  const size_t n_pix = size_t(st.S) * st.S;
  DeviceBuffer<uint8_t> d_sil;
  DeviceBuffer<uint16_t> d_depth;
  CU(d_sil.create(st.n_renderers * n_pix));
  CU(d_depth.create(n_pix));
  k_region_images<<<unsigned((n_pix + 255) / 256), 256, 0, ctx->stream>>>(b.zbuf, RendererTable(st, b.bodies), st.S,
                                                                         d_sil, d_depth);
  CU(cudaGetLastError());
  ctx->launches += 2;
  rc = ContourOverflow(ctx, rb);
  if (rc) return rc;
  int counts[2];
  CU(cudaMemcpy(counts, rb.counts, sizeof(counts), cudaMemcpyDeviceToHost));
  std::vector<uint32_t> packed(counts[1]);
  std::vector<int> starts(counts[0] + 1);
  CU(cudaMemcpy(packed.data(), rb.contour, sizeof(uint32_t) * packed.size(), cudaMemcpyDeviceToHost));
  CU(cudaMemcpy(starts.data(), rb.contour_start, sizeof(int) * starts.size(), cudaMemcpyDeviceToHost));
  if (silhouettes) CU(cudaMemcpy(silhouettes, d_sil, st.n_renderers * n_pix, cudaMemcpyDeviceToHost));
  if (depth) CU(cudaMemcpy(depth, d_depth, 2 * n_pix, cudaMemcpyDeviceToHost));
  if (n_silhouettes) *n_silhouettes = st.n_renderers;
  if (n_contour_points) *n_contour_points = counts[1];
  if (n_contours) *n_contours = counts[0];
  if (contour_points)
    for (int k = 0; k < std::min(capacity, counts[1]); ++k) {
      contour_points[2 * k] = int32_t(packed[k] & 0xffffu);
      contour_points[2 * k + 1] = int32_t(packed[k] >> 16);
    }
  if (contour_offsets)
    for (int k = 0; k <= std::min(capacity, counts[0]); ++k) contour_offsets[k] = starts[k];
  return M3TB_OK;
}

// ---- camera-image renderers: what viewers and full renderers share, then viewers (NormalColorViewer /
// ---- NormalDepthViewer, normal_viewer.cpp) ------------------------------------------------------------------------

using ViewSlotHost = m3tb_ctx::ViewSlotHost;

// Images of a W x H slot of `kind`; the z-buffer is cleared (k_view_resolve clears it again after every draw)
static int MakeViewImages(m3tb_ctx* ctx, int kind, int width, int height, m3tb_ctx::ViewImages& im) {
  const size_t n = size_t(width) * height;
  CU(im.zbuf.create(n));
  if (kind == VK_FULL || kind == VK_FOCUSED) {
    CU(im.depth.create(n));
    if (kind == VK_FULL) CU(im.silhouette.create(n));
    CU(im.normal.create(4 * n));
  } else {
    CU(im.normal.create(4 * n));
    CU(im.image.create(3 * n));
  }
  CU(cudaMemsetAsync(im.zbuf, 0xff, n * sizeof(uint64_t), ctx->stream));
  return M3TB_OK;
}

static int LaunchView(m3tb_ctx* ctx, size_t n_triangles, int max_triangles, int max_pixels, const FocusArgs* focus);

// The image size of a slot: its camera's, or image_size x image_size for a focused normal renderer
static void SlotSize(m3tb_ctx* ctx, const ViewSlotHost& s, int& width, int& height) {
  const CameraDev& c = CameraOf(ctx, s.camera_kind == 0, s.camera);
  width = s.kind == VK_FOCUSED ? s.image_size : c.width;
  height = s.kind == VK_FOCUSED ? s.image_size : c.height;
}

// FullRenderer::CalculateProjectionMatrix (renderer.cpp:257-264) from the camera's intrinsics, and its world2camera
static void FullProjection(const CameraDev& c, float z_min, float z_max, ViewerDev& d) {
  d.width = c.width;
  d.height = c.height;
  d.P00 = 2.0f * c.fu / float(c.width);
  d.P02 = 2.0f * (c.ppu + 0.5f) / float(c.width) - 1.0f;
  d.P11 = 2.0f * c.fv / float(c.height);
  d.P12 = 2.0f * (c.ppv + 0.5f) / float(c.height) - 1.0f;
  d.P22 = (z_max + z_min) / (z_max - z_min);
  d.P23 = -2.0f * z_max * z_min / (z_max - z_min);
  std::memcpy(d.w2c, c.w2c, sizeof(d.w2c));
}

// Puts `slot` (kind, camera, geometry and parameters filled in, checked by the caller) into `table` at `id`, a slot
// of the table or the next free one. The images of the slot it replaces are kept while the camera has their size;
// otherwise new ones are made before anything changes.
static int InstallViewSlot(m3tb_ctx* ctx, std::vector<ViewSlotHost>& table, int id, ViewSlotHost& slot) {
  int W, H;
  SlotSize(ctx, slot, W, H);
  ViewSlotHost* old = id < int(table.size()) ? &table[id] : nullptr;
  if (!old || old->width != W || old->height != H) {
    int rc = MakeViewImages(ctx, slot.kind, W, H, slot.images);
    if (rc) return rc;
    if (old) CU(cudaStreamSynchronize(ctx->stream));  // a draw in flight may still use the old images
  } else {
    slot.images = std::move(old->images);
  }
  slot.width = W;
  slot.height = H;
  if (old) *old = std::move(slot);
  else table.push_back(std::move(slot));
  return M3TB_OK;
}

// One draw of every slot of `table` (ctx->viewers, ctx->full_renderers or ctx->focused_normal_renderers) from the
// current poses: the three k_view_* launches over tables filled here, after k_view_focus when `focus` is given
static int DrawViewSlots(m3tb_ctx* ctx, std::vector<ViewSlotHost>& table, const FocusArgs* focus = nullptr) {
  const int ns = int(table.size());
  if (ns == 0) return M3TB_OK;
  // images of slots whose camera changed size since they were made (m3tb_set_*_camera), all or nothing
  std::vector<m3tb_ctx::ViewImages> remade(ns);
  bool any_remade = false;
  for (int v = 0; v < ns; ++v) {
    const auto& h = table[v];
    int W, H;
    SlotSize(ctx, h, W, H);
    if (h.width == W && h.height == H) continue;
    int rc = MakeViewImages(ctx, h.kind, W, H, remade[v]);
    if (rc) return rc;
    any_remade = true;
  }
  if (any_remade) {
    CU(cudaStreamSynchronize(ctx->stream));  // a draw in flight may still use the images that are replaced
    for (int v = 0; v < ns; ++v) {
      if (!remade[v].zbuf) continue;
      auto& h = table[v];
      SlotSize(ctx, h, h.width, h.height);
      h.images = std::move(remade[v]);
      h.drawn = false;
    }
  }
  // the draw's tables: slots (projection, frame, images) and draws (RendererGeometry::render_data_bodies)
  std::vector<ViewerDev>& V = ctx->h_view_viewers;
  std::vector<ViewDrawDev>& D = ctx->h_view_draws;
  V.assign(ns, ViewerDev{});
  D.clear();
  size_t n_triangles = 0;
  int max_triangles = 0, max_pixels = 0;
  for (int v = 0; v < ns; ++v) {
    const auto& h = table[v];
    const CameraDev& c = CameraOf(ctx, h.camera_kind == 0, h.camera);
    ViewerDev& d = V[v];
    d.kind = h.kind;
    if (h.kind == VK_FOCUSED) {  // the projection is k_view_focus's
      d.width = d.height = h.image_size;
      std::memcpy(d.w2c, c.w2c, sizeof(d.w2c));
      d.depth = h.images.depth;
    } else if (h.kind == VK_FULL) {
      FullProjection(c, h.z_min, h.z_max, d);
      d.depth = h.images.depth;
      d.silhouette = h.images.silhouette;
    } else {
      FullProjection(c, kViewerZMin, kViewerZMax, d);  // the viewer renderer's z range
      // Camera::image(): a pinned frame's device copy is valid only inside the ROIs, the frame itself is read in place
      d.frame = c.host_src ? c.host_src : c.image;
      d.frame_pitch = c.host_src ? c.host_pitch : c.pitch;
      d.opacity = h.opacity;
      // DepthCamera::NormalizedDepthImage (camera.cpp:108-115)
      d.depth_alpha = 255.0f / ((h.max_depth - h.min_depth) / c.depth_scale);
      d.depth_beta = -(h.min_depth / c.depth_scale) * d.depth_alpha;
      d.image = h.images.image;
    }
    d.zbuf = h.images.zbuf;
    d.normal = h.images.normal;
    d.first_draw = int(D.size());
    d.n_draws = int(h.geometry.size());
    for (int g = 0; g < d.n_draws; ++g) {
      const int b = h.geometry[g];
      const GeometryDev& G = ctx->h_geometry[b];
      ViewDrawDev dd;
      dd.triangles = G.triangles;
      dd.n_triangles = G.n_triangles;
      dd.enable_culling = G.enable_culling;
      dd.viewer = v;
      dd.draw = g;
      dd.body = b;
      dd.silhouette_id = h.kind != VK_FULL ? 0 : (h.id_type == RID_REGION ? G.region_id : G.body_id);
      std::memcpy(dd.geometry2body, G.geometry2body, sizeof(dd.geometry2body));
      D.push_back(dd);
      n_triangles += size_t(G.n_triangles);
      max_triangles = std::max(max_triangles, G.n_triangles);
    }
    max_pixels = std::max(max_pixels, d.width * d.height);
  }
  int rc = LaunchView(ctx, n_triangles, max_triangles, max_pixels, focus);
  if (rc) return rc;
  for (auto& h : table) h.drawn = true;
  return M3TB_OK;
}

int m3tb_set_viewer(m3tb_ctx* ctx, int viewer, int kind, int camera, const int* geometry_bodies, int n_geometry,
                    float opacity, float min_depth, float max_depth) {
  CHECK_CTX();
  if (viewer < 0 || viewer > int(ctx->viewers.size()))
    return Fail(ctx, M3TB_ERR_INVALID, "viewer ids must be dense (0..n)");
  if (kind != VK_COLOR && kind != VK_DEPTH)
    return Fail(ctx, M3TB_ERR_INVALID, "kind must be 0 (NormalColorViewer) or 1 (NormalDepthViewer)");
  int rc = CheckCameraSet(ctx, kind, camera);
  if (rc) return rc;
  if (n_geometry < 0 || n_geometry > 65535 || (n_geometry > 0 && !geometry_bodies))
    return Fail(ctx, M3TB_ERR_INVALID, "bad geometry body list");
  rc = CheckBodyList(ctx, geometry_bodies, n_geometry);
  if (rc) return rc;
  ViewSlotHost nv;
  nv.kind = kind;
  nv.camera_kind = kind;
  nv.camera = camera;
  nv.opacity = opacity;
  nv.min_depth = min_depth;
  nv.max_depth = max_depth;
  nv.geometry.assign(geometry_bodies, geometry_bodies + n_geometry);
  return InstallViewSlot(ctx, ctx->viewers, viewer, nv);
}

int m3tb_update_viewers(m3tb_ctx* ctx) {
  CHECK_CTX();
  for (const auto& h : ctx->viewers)
    if (!CameraOf(ctx, h.camera_kind == 0, h.camera).image)
      return Fail(ctx, M3TB_ERR_NOT_SET_UP, "a viewer's camera has not received an image");
  return DrawViewSlots(ctx, ctx->viewers);
}

// The three k_view_* launches over the tables in ctx->h_view_viewers / h_view_draws (viewers, full renderers or focused
// normal renderers), after k_view_focus when `focus` is given
static int LaunchView(m3tb_ctx* ctx, size_t n_triangles, int max_triangles, int max_pixels, const FocusArgs* focus) {
  const std::vector<ViewerDev>& V = ctx->h_view_viewers;
  const std::vector<ViewDrawDev>& D = ctx->h_view_draws;
  const int nv = int(V.size());
  const int n_draws = int(D.size());
  const size_t fan_cap = 2 * n_triangles;
  if (fan_cap > size_t(INT32_MAX)) return Fail(ctx, M3TB_ERR_INVALID, "too many triangles for one update");
  // device tables, all or nothing
  DeviceBuffer<ViewerDev> viewers;
  DeviceBuffer<ViewDrawDev> draws;
  DeviceBuffer<float> rot;
  DeviceBuffer<ViewFanDev> fans;
  DeviceBuffer<uint64_t> fan_tile;
  DeviceBuffer<unsigned long long> counter;
  int rc = GrowTable(ctx, ctx->d_view_viewers, viewers, size_t(nv));
  if (!rc) rc = GrowTable(ctx, ctx->d_view_draws, draws, std::max<size_t>(n_draws, 1));
  if (!rc) rc = GrowTable(ctx, ctx->d_view_rot, rot, 9 * std::max<size_t>(n_draws, 1));
  if (!rc) rc = GrowTable(ctx, ctx->d_view_fans, fans, std::max<size_t>(fan_cap, 1));
  if (!rc) rc = GrowTable(ctx, ctx->d_view_fan_tile, fan_tile, std::max<size_t>(fan_cap, 1));
  if (rc) return rc;
  if (!ctx->d_view_counter) {
    CU(counter.create(1));
    CU(cudaMemsetAsync(counter, 0, sizeof(unsigned long long), ctx->stream));
  }
  if (viewers || draws || rot || fans || fan_tile || counter) {
    CU(cudaStreamSynchronize(ctx->stream));  // an update in flight may still read the tables that are replaced
    if (viewers) ctx->d_view_viewers = std::move(viewers);
    if (draws) ctx->d_view_draws = std::move(draws);
    if (rot) ctx->d_view_rot = std::move(rot);
    if (fans) ctx->d_view_fans = std::move(fans);
    if (fan_tile) ctx->d_view_fan_tile = std::move(fan_tile);
    if (counter) ctx->d_view_counter = std::move(counter);
  }
  CU(cudaMemcpyAsync(ctx->d_view_viewers, V.data(), sizeof(ViewerDev) * nv, cudaMemcpyHostToDevice, ctx->stream));
  if (n_draws)
    CU(cudaMemcpyAsync(ctx->d_view_draws, D.data(), sizeof(ViewDrawDev) * n_draws, cudaMemcpyHostToDevice, ctx->stream));
  ViewArgs a;
  a.viewers = ctx->d_view_viewers;
  a.n_viewers = nv;
  a.draws = ctx->d_view_draws;
  a.n_draws = n_draws;
  a.poses = ctx->d_poses;
  a.rot = ctx->d_view_rot;
  a.fans = ctx->d_view_fans;
  a.fan_tile = ctx->d_view_fan_tile;
  a.fan_cap = int(fan_cap);
  a.counter = ctx->d_view_counter;
  if (focus) {
    FocusArgs f = *focus;
    f.viewers = ctx->d_view_viewers;
    f.draws = ctx->d_view_draws;
    k_view_focus<<<unsigned((f.n_focus + kViewThreads - 1) / kViewThreads), kViewThreads, 0, ctx->stream>>>(f);
    CU(cudaGetLastError());
    ctx->launches++;
  }
  // the three launches always run (a grid dimension of 0 is not launchable, so empty ones get one idle block)
  const dim3 setup_grid(unsigned(std::max(1, (max_triangles + kViewThreads - 1) / kViewThreads)),
                        unsigned(std::max(1, n_draws)));
  k_view_setup<<<setup_grid, kViewThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  k_view_raster<<<unsigned(ctx->sm_count * (2048 / kViewThreads)), kViewThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  k_view_resolve<<<dim3(unsigned((max_pixels + kViewThreads - 1) / kViewThreads), unsigned(nv)), kViewThreads, 0,
                   ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches += 3;
  return M3TB_OK;
}

int m3tb_get_viewer_image(m3tb_ctx* ctx, int viewer, uint8_t* bgr, size_t pitch, uint8_t* normal_bgra,
                          size_t normal_pitch) {
  CHECK_CTX();
  if (viewer < 0 || viewer >= int(ctx->viewers.size())) return Fail(ctx, M3TB_ERR_INVALID, "viewer not set");
  const auto& h = ctx->viewers[viewer];
  if (!h.drawn) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "viewer has not been updated since it was set");
  const size_t W = size_t(h.width), H = size_t(h.height);
  if ((bgr && pitch < 3 * W) || (normal_bgra && normal_pitch < 4 * W))
    return Fail(ctx, M3TB_ERR_INVALID, "pitch smaller than a row");
  if (bgr) CU(cudaMemcpy2DAsync(bgr, pitch, h.images.image, 3 * W, 3 * W, H, cudaMemcpyDeviceToHost, ctx->stream));
  if (normal_bgra)
    CU(cudaMemcpy2DAsync(normal_bgra, normal_pitch, h.images.normal, 4 * W, 4 * W, H, cudaMemcpyDeviceToHost,
                         ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

// ---- full renderers (FullBasicDepthRenderer / FullSilhouetteRenderer / FullNormalRenderer, renderer.cpp) -----------

int m3tb_set_full_renderer(m3tb_ctx* ctx, int renderer, int camera_kind, int camera, float z_min, float z_max,
                           int id_type, const int* geometry_bodies, int n_geometry) {
  CHECK_CTX();
  if (renderer < 0 || renderer > int(ctx->full_renderers.size()))
    return Fail(ctx, M3TB_ERR_INVALID, "full renderer ids must be dense (0..n)");
  if (camera_kind != 0 && camera_kind != 1) return Fail(ctx, M3TB_ERR_INVALID, "camera_kind must be 0 (colour) or 1 (depth)");
  int rc = CheckCameraSet(ctx, camera_kind, camera);
  if (rc) return rc;
  if (!(z_min > 0.0f) || !(z_max > z_min) || !std::isfinite(z_max))
    return Fail(ctx, M3TB_ERR_INVALID, "bad z_min / z_max");
  if (id_type != RID_BODY && id_type != RID_REGION) return Fail(ctx, M3TB_ERR_INVALID, "id_type must be 0 (BODY) or 1 (REGION)");
  if (n_geometry < 0 || n_geometry > 65535 || (n_geometry > 0 && !geometry_bodies))
    return Fail(ctx, M3TB_ERR_INVALID, "bad geometry body list");
  rc = CheckBodyList(ctx, geometry_bodies, n_geometry);
  if (rc) return rc;
  ViewSlotHost nr;
  nr.kind = VK_FULL;
  nr.camera_kind = camera_kind;
  nr.camera = camera;
  nr.id_type = id_type;
  nr.z_min = z_min;
  nr.z_max = z_max;
  nr.geometry.assign(geometry_bodies, geometry_bodies + n_geometry);
  return InstallViewSlot(ctx, ctx->full_renderers, renderer, nr);
}

int m3tb_render_full(m3tb_ctx* ctx) {
  CHECK_CTX();
  return DrawViewSlots(ctx, ctx->full_renderers);
}

// true when `p` is device memory (a write to it needs no synchronisation with the host)
static bool IsDevicePointer(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();  // an unknown pointer is host memory
    return false;
  }
  return at.type == cudaMemoryTypeDevice;
}

int m3tb_get_full_rendering(m3tb_ctx* ctx, int renderer, void* depth_u16, size_t depth_pitch, void* silhouette_u8,
                            size_t silhouette_pitch, void* normal_bgra, size_t normal_pitch, float* projection_term_a,
                            float* projection_term_b) {
  CHECK_CTX();
  if (renderer < 0 || renderer >= int(ctx->full_renderers.size()))
    return Fail(ctx, M3TB_ERR_INVALID, "full renderer not set");
  const auto& h = ctx->full_renderers[renderer];
  const CameraDev& c = CameraOf(ctx, h.camera_kind == 0, h.camera);
  if (!h.drawn || h.width != c.width || h.height != c.height)
    return Fail(ctx, M3TB_ERR_NOT_SET_UP, "full renderer has not rendered since it was set or its camera changed size");
  const size_t W = size_t(h.width), H = size_t(h.height);
  if ((depth_u16 && depth_pitch < 2 * W) || (silhouette_u8 && silhouette_pitch < W) ||
      (normal_bgra && normal_pitch < 4 * W))
    return Fail(ctx, M3TB_ERR_INVALID, "pitch smaller than a row");
  bool to_host = false;
  if (depth_u16) {
    CU(cudaMemcpy2DAsync(depth_u16, depth_pitch, h.images.depth, 2 * W, 2 * W, H, cudaMemcpyDefault, ctx->stream));
    to_host = to_host || !IsDevicePointer(depth_u16);
  }
  if (silhouette_u8) {
    CU(cudaMemcpy2DAsync(silhouette_u8, silhouette_pitch, h.images.silhouette, W, W, H, cudaMemcpyDefault, ctx->stream));
    to_host = to_host || !IsDevicePointer(silhouette_u8);
  }
  if (normal_bgra) {
    CU(cudaMemcpy2DAsync(normal_bgra, normal_pitch, h.images.normal, 4 * W, 4 * W, H, cudaMemcpyDefault, ctx->stream));
    to_host = to_host || !IsDevicePointer(normal_bgra);
  }
  // FullDepthRenderer's projection terms (renderer.cpp:476-477): depth = a / (b - depth_image_value)
  if (projection_term_a) *projection_term_a = h.z_max * h.z_min * float(USHRT_MAX) / (h.z_max - h.z_min);
  if (projection_term_b) *projection_term_b = h.z_max * float(USHRT_MAX) / (h.z_max - h.z_min);
  if (to_host) CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

// ---- focused normal renderers (FocusedNormalRenderer, normal_renderer.cpp:295-423) ---------------------------------

int m3tb_set_focused_normal_renderer(m3tb_ctx* ctx, int renderer, int camera_kind, int camera, int image_size,
                                     float z_min, float z_max, const int* geometry_bodies, int n_geometry,
                                     const int* referenced_bodies, int n_referenced) {
  CHECK_CTX();
  if (renderer < 0 || renderer > int(ctx->focused_normal_renderers.size()))
    return Fail(ctx, M3TB_ERR_INVALID, "focused normal renderer ids must be dense (0..n)");
  if (camera_kind != 0 && camera_kind != 1) return Fail(ctx, M3TB_ERR_INVALID, "camera_kind must be 0 (colour) or 1 (depth)");
  int rc = CheckCameraSet(ctx, camera_kind, camera);
  if (rc) return rc;
  if (image_size > kFocusedNormalMaxImageSize)
    return Fail(ctx, M3TB_ERR_UNSUPPORTED, "image_size above " + std::to_string(kFocusedNormalMaxImageSize));
  if (image_size < 1 || !(z_min > 0.0f) || !(z_max > z_min) || !std::isfinite(z_max))
    return Fail(ctx, M3TB_ERR_INVALID, "bad image_size / z_min / z_max");
  if (!geometry_bodies || n_geometry < 1 || n_geometry > 65535 || !referenced_bodies || n_referenced < 1)
    return Fail(ctx, M3TB_ERR_INVALID, "a renderer needs geometry bodies and referenced bodies");
  rc = CheckBodyList(ctx, geometry_bodies, n_geometry);
  if (!rc) rc = CheckBodyList(ctx, referenced_bodies, n_referenced);
  if (rc) return rc;
  ViewSlotHost nr;
  nr.kind = VK_FOCUSED;
  nr.camera_kind = camera_kind;
  nr.camera = camera;
  nr.image_size = image_size;
  nr.z_min = z_min;
  nr.z_max = z_max;
  nr.geometry.assign(geometry_bodies, geometry_bodies + n_geometry);
  nr.referenced.assign(referenced_bodies, referenced_bodies + n_referenced);
  return InstallViewSlot(ctx, ctx->focused_normal_renderers, renderer, nr);
}

int m3tb_render_focused_normals(m3tb_ctx* ctx) {
  CHECK_CTX();
  auto& table = ctx->focused_normal_renderers;
  const int n = int(table.size());
  if (n == 0) return M3TB_OK;
  // k_view_focus's tables: one FocusDev per renderer, the referenced bodies and their radii
  std::vector<FocusDev>& F = ctx->h_focus;
  std::vector<int>& ref = ctx->h_focus_referenced;
  std::vector<float>& radius = ctx->h_focus_radius;
  F.assign(n, FocusDev{});
  ref.clear();
  radius.clear();
  for (int v = 0; v < n; ++v) {
    const auto& h = table[v];
    FocusDev& f = F[v];
    f.cam = CameraOf(ctx, h.camera_kind == 0, h.camera);
    f.image_size = h.image_size;
    f.z_min = h.z_min;
    f.z_max = h.z_max;
    f.viewer = v;
    f.first_referenced = int(ref.size());
    f.n_referenced = int(h.referenced.size());
    for (int b : h.referenced) {
      ref.push_back(b);
      radius.push_back(ctx->h_geometry[b].radius);
    }
  }
  // grown tables stay local until the render has been launched, so that a failure leaves the context as it was
  DeviceBuffer<FocusDev> focus;
  DeviceBuffer<int> referenced, visible;
  DeviceBuffer<float> radii;
  DeviceBuffer<RenderOutDev> out;
  int rc = GrowTable(ctx, ctx->d_focus, focus, size_t(n));
  if (!rc) rc = GrowTable(ctx, ctx->d_focus_referenced, referenced, ref.size());
  if (!rc) rc = GrowTable(ctx, ctx->d_focus_radius, radii, ref.size());
  if (!rc) rc = GrowTable(ctx, ctx->d_focus_visible, visible, ref.size());
  if (!rc) rc = GrowTable(ctx, ctx->d_focus_out, out, size_t(n));
  if (rc) return rc;
  FocusDev* d_focus = focus ? focus.get() : ctx->d_focus.get();
  int* d_referenced = referenced ? referenced.get() : ctx->d_focus_referenced.get();
  float* d_radius = radii ? radii.get() : ctx->d_focus_radius.get();
  CU(cudaMemcpyAsync(d_focus, F.data(), sizeof(FocusDev) * n, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(d_referenced, ref.data(), sizeof(int) * ref.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(d_radius, radius.data(), sizeof(float) * radius.size(), cudaMemcpyHostToDevice, ctx->stream));
  FocusArgs fa = {};
  fa.focus = d_focus;
  fa.n_focus = n;
  fa.referenced = d_referenced;
  fa.radius = d_radius;
  fa.poses = ctx->d_poses;
  fa.visible = visible ? visible.get() : ctx->d_focus_visible.get();
  fa.out = out ? out.get() : ctx->d_focus_out.get();
  const int64_t launches = ctx->launches;
  rc = DrawViewSlots(ctx, table, &fa);
  if (rc) {
    // k_view_focus ran but a later launch failed: the flags and focus in the tables no longer match the images
    if (ctx->launches != launches)
      for (auto& h : table) h.drawn = false;
    return rc;
  }
  // the replaced tables are released after the device-wide synchronisation of cudaFree (a render in flight may still
  // use them)
  if (focus) ctx->d_focus = std::move(focus);
  if (referenced) ctx->d_focus_referenced = std::move(referenced);
  if (radii) ctx->d_focus_radius = std::move(radii);
  if (visible) ctx->d_focus_visible = std::move(visible);
  if (out) ctx->d_focus_out = std::move(out);
  for (int v = 0; v < n; ++v) table[v].first_referenced = F[v].first_referenced;
  return M3TB_OK;
}

int m3tb_get_focused_normal_rendering(m3tb_ctx* ctx, int renderer, void* depth_u16, void* normal_bgra, float* corner_u,
                                      float* corner_v, float* scale, float* projection_term_a,
                                      float* projection_term_b, int* visible_flags) {
  CHECK_CTX();
  if (renderer < 0 || renderer >= int(ctx->focused_normal_renderers.size()))
    return Fail(ctx, M3TB_ERR_INVALID, "focused normal renderer not set");
  const auto& h = ctx->focused_normal_renderers[renderer];
  if (!h.drawn) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "focused normal renderer has not rendered since it was set");
  const size_t S = size_t(h.image_size);
  bool to_host = false;
  if (depth_u16) {
    CU(cudaMemcpyAsync(depth_u16, h.images.depth, 2 * S * S, cudaMemcpyDefault, ctx->stream));
    to_host = to_host || !IsDevicePointer(depth_u16);
  }
  if (normal_bgra) {
    CU(cudaMemcpyAsync(normal_bgra, h.images.normal, 4 * S * S, cudaMemcpyDefault, ctx->stream));
    to_host = to_host || !IsDevicePointer(normal_bgra);
  }
  RenderOutDev o;
  const bool want_focus = corner_u || corner_v || scale || projection_term_a || projection_term_b;
  if (want_focus)
    CU(cudaMemcpyAsync(&o, ctx->d_focus_out + renderer, sizeof(o), cudaMemcpyDeviceToHost, ctx->stream));
  if (visible_flags)
    CU(cudaMemcpyAsync(visible_flags, ctx->d_focus_visible + h.first_referenced, sizeof(int) * h.referenced.size(),
                       cudaMemcpyDeviceToHost, ctx->stream));
  if (to_host || want_focus || visible_flags) CU(cudaStreamSynchronize(ctx->stream));
  if (corner_u) *corner_u = o.corner_u;
  if (corner_v) *corner_v = o.corner_v;
  if (scale) *scale = o.scale;
  if (projection_term_a) *projection_term_a = o.projection_term_a;
  if (projection_term_b) *projection_term_b = o.projection_term_b;
  return M3TB_OK;
}

// ---- NormalizedDepthImage (DepthCamera, camera.cpp:108-115; FullDepthRenderer, renderer.cpp:407-427) ---------------

int m3tb_get_normalized_depth_image(m3tb_ctx* ctx, int source, int id, float min_depth, float max_depth, void* dst,
                                    size_t pitch) {
  CHECK_CTX();
  if ((source != M3TB_NORMALIZED_DEPTH_CAMERA && source != M3TB_NORMALIZED_DEPTH_FULL_RENDERER) || !dst)
    return Fail(ctx, M3TB_ERR_INVALID, "bad normalized depth image arguments");
  if (!(max_depth > min_depth)) return Fail(ctx, M3TB_ERR_INVALID, "max_depth must exceed min_depth");
  NormalizedDepthArgs a = {};
  if (source == M3TB_NORMALIZED_DEPTH_CAMERA) {
    if (id < 0 || id >= ctx->max_cameras || !ctx->h_dcams[id].set)
      return Fail(ctx, M3TB_ERR_INVALID, "depth camera not set");
    const CameraDev& c = ctx->h_dcams[id];
    if (!c.image) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "depth camera has no image");
    if (ctx->prefetched) CU(cudaStreamWaitEvent(ctx->stream, ctx->pf.ev_ingest_done, 0));
    // Camera::image(): a pinned frame's device copy is valid only inside the ROIs, the frame itself is read in place
    a.src = c.host_src ? c.host_src : c.image;
    a.src_pitch = c.host_src ? c.host_pitch : c.pitch;
    a.width = c.width;
    a.height = c.height;
    a.alpha = 255.0f / ((max_depth - min_depth) / c.depth_scale);
    a.beta = -(min_depth / c.depth_scale) * a.alpha;
  } else {
    if (id < 0 || id >= int(ctx->full_renderers.size())) return Fail(ctx, M3TB_ERR_INVALID, "full renderer not set");
    const auto& h = ctx->full_renderers[id];
    const CameraDev& c = CameraOf(ctx, h.camera_kind == 0, h.camera);
    if (!h.drawn || h.width != c.width || h.height != c.height)
      return Fail(ctx, M3TB_ERR_NOT_SET_UP, "full renderer has not rendered since it was set or its camera changed size");
    a.src = reinterpret_cast<const uint8_t*>(static_cast<const uint16_t*>(h.images.depth));
    a.src_pitch = unsigned(2 * h.width);
    a.width = h.width;
    a.height = h.height;
    a.renderer = 1;
    a.a = h.z_max * h.z_min * float(USHRT_MAX) / (h.z_max - h.z_min);  // renderer.cpp:476-477
    a.b = h.z_max * float(USHRT_MAX) / (h.z_max - h.z_min);
    a.min_depth = min_depth;
    a.delta = max_depth - min_depth;
    a.scale = 255.0f / a.delta;
  }
  const size_t W = size_t(a.width), H = size_t(a.height);
  if (pitch < W) return Fail(ctx, M3TB_ERR_INVALID, "pitch smaller than a row");
  const bool to_host = !IsDevicePointer(dst);
  if (to_host) {  // the kernel writes into device scratch, which is then copied
    DeviceBuffer<uint8_t> grown;
    int rc = GrowTable(ctx, ctx->d_normalized_depth, grown, W * H);
    if (rc) return rc;
    if (grown) {
      CU(cudaStreamSynchronize(ctx->stream));  // a copy in flight may still read the scratch that is replaced
      ctx->d_normalized_depth = std::move(grown);
    }
    a.dst = ctx->d_normalized_depth;
    a.dst_pitch = W;
  } else {
    a.dst = static_cast<uint8_t*>(dst);
    a.dst_pitch = pitch;
  }
  k_normalized_depth<<<unsigned((W * H + kViewThreads - 1) / kViewThreads), kViewThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  if (to_host) {
    CU(cudaMemcpy2DAsync(dst, pitch, a.dst, W, W, H, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  return M3TB_OK;
}

int m3tb_set_camera_undistortion(m3tb_ctx* ctx, int camera_kind, int cam, const int16_t* map_xy, size_t map_pitch,
                                 int channels, int32_t depth_value_offset) {
  CHECK_CTX();
  if ((camera_kind != 0 && camera_kind != 1) || cam < 0 || cam >= ctx->max_cameras)
    return Fail(ctx, M3TB_ERR_INVALID, "bad camera kind / index");
  const bool color = camera_kind == 0;
  const CameraDev& c = CameraOf(ctx, color, cam);
  if (!c.set) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "set the camera before its undistortion");
  auto& slot = ctx->undistort[camera_kind][cam];
  if (!map_xy) {
    slot = {};
    return M3TB_OK;
  }
  if (color ? (channels != 3 && channels != 4) : channels != 1)
    return Fail(ctx, M3TB_ERR_INVALID, "channels must be 3 or 4 (colour) or 1 (depth)");
  if (depth_value_offset < SHRT_MIN || depth_value_offset > SHRT_MAX || (color && depth_value_offset != 0))
    return Fail(ctx, M3TB_ERR_INVALID, "the depth value offset is a short, and 0 for colour cameras");
  const size_t row = 4 * size_t(c.width);
  if (map_pitch < row) return Fail(ctx, M3TB_ERR_INVALID, "map pitch smaller than a row");
  m3tb_ctx::UndistortHost h;
  h.map_pitch = unsigned(Align(row, 16));
  h.channels = channels;
  h.offset = depth_value_offset;
  CU(h.map.create(size_t(h.map_pitch / 2) * c.height));
  CU(cudaMemcpy2DAsync(h.map, h.map_pitch, map_xy, map_pitch, row, c.height, cudaMemcpyDefault, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));  // the caller's map may be released on return
  slot = std::move(h);
  return M3TB_OK;
}

int m3tb_get_camera_image(m3tb_ctx* ctx, int camera_kind, int cam, void* dst, size_t pitch) {
  CHECK_CTX();
  if ((camera_kind != 0 && camera_kind != 1) || cam < 0 || cam >= ctx->max_cameras || !dst)
    return Fail(ctx, M3TB_ERR_INVALID, "bad camera image arguments");
  const CameraDev& c = CameraOf(ctx, camera_kind == 0, cam);
  if (!c.set || !c.image) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "camera not set / no image uploaded");
  const size_t row = size_t(c.width) * (camera_kind == 0 ? 3 : 2);
  if (pitch < row) return Fail(ctx, M3TB_ERR_INVALID, "pitch smaller than a row");
  if (ctx->prefetched) CU(cudaStreamWaitEvent(ctx->stream, ctx->pf.ev_ingest_done, 0));
  // a pinned frame's device copy is valid only inside the fetched rectangles: the frame itself is read
  const uint8_t* src = c.host_src ? c.host_src : c.image;
  const size_t src_pitch = c.host_src ? c.host_pitch : c.pitch;
  CU(cudaMemcpy2DAsync(dst, pitch, src, src_pitch, row, c.height, cudaMemcpyDefault, ctx->stream));
  if (!IsDevicePointer(dst)) CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

// ---- texture modality (TextureModality, texture_modality.cpp) --------------------------------------------------------
void m3tb_texture_params_default(m3tb_texture_params* p) {
  if (!p) return;
  std::memset(p, 0, sizeof(*p));
  p->descriptor_type = M3TB_DESCRIPTOR_ORB;
  p->focused_image_size = 200;
  p->descriptor_distance_threshold = 0.7f;
  p->tukey_norm_constant = 20.0f;
  p->n_standard_deviations = 2;
  p->standard_deviations[0] = 15.0f;
  p->standard_deviations[1] = 5.0f;
  p->max_keyframe_rotation_difference = 10.0f * 3.14159265358979323846f / 180.0f;  // kPi, common.h
  p->max_keyframe_age = 100;
  p->n_keyframes = 1;
  p->measured_occlusion_radius = 0.01f;
  p->measured_occlusion_threshold = 0.03f;
  p->modeled_occlusion_radius = 0.01f;
  p->modeled_occlusion_threshold = 0.03f;
  p->n_features_max = kTexMaxFeatures;
}

}  // extern "C"

namespace {

// One capacity-sized texture table: `rows` rows of per_feature * cap elements. make() creates its replacement at
// capacity `cap` (when it is wanted and missing, or the tables grow), copy() moves each row of the table it replaces to
// the front of its new row, replace() swaps it in.
template <typename T>
struct TexTable {
  DeviceBuffer<T>& cur;
  size_t rows, per_feature;
  DeviceBuffer<T> out;
  cudaError_t make(bool want, bool grow, int cap) {
    return want && (grow || !cur) ? out.create(rows * per_feature * size_t(cap)) : cudaSuccess;
  }
  cudaError_t copy(int old_cap, int cap, cudaStream_t stream) {
    if (!out || !cur) return cudaSuccess;
    const size_t w_old = sizeof(T) * per_feature * size_t(old_cap), w_new = sizeof(T) * per_feature * size_t(cap);
    return cudaMemcpy2DAsync(out, w_new, cur, w_old, w_old, rows, cudaMemcpyDeviceToDevice, stream);
  }
  void replace() {
    if (out) cur = std::move(out);
  }
};

// The texture tables for max_bodies at `cap` features per body (m3tb_set_texture_modality): the base tables, with knn
// the kNN match table, with wide also the wide descriptor tables (and the match table). Whatever is missing is made,
// and when `cap` exceeds the capacity of the existing tables every capacity-sized table is remade at `cap` with its
// contents kept; all of it in one all-or-nothing step. A context whose bodies keep kTexMaxFeatures never grows.
int EnsureTextureTables(m3tb_ctx* ctx, bool wide, bool knn, int cap) {
  const size_t nb = size_t(ctx->max_bodies), K = kTexMaxKeyframes;
  const bool base = !ctx->d_tex_xy;
  cap = std::max(cap, base ? kTexMaxFeatures : ctx->tex_cap);
  const bool grow = !base && cap > ctx->tex_cap;
  wide = wide || ctx->d_tex_fdesc;
  knn = knn || wide || ctx->d_tex_knn;
  if (!base && !grow && (!wide || ctx->d_tex_fdesc) && (!knn || ctx->d_tex_knn)) return M3TB_OK;
  TexTable<float> fdesc{ctx->d_tex_fdesc, nb, kTexMaxFloatDesc};
  TexTable<float> kf_fdesc{ctx->d_tex_kf_fdesc, nb * K, kTexMaxFloatDesc};
  TexTable<int> knn_t{ctx->d_tex_knn, nb * K, 1};
  TexTable<float2> xy{ctx->d_tex_xy, nb, 1};
  TexTable<uint32_t> desc{ctx->d_tex_desc, nb, kTexDescWords};
  TexTable<uint32_t> kf_desc{ctx->d_tex_kf_desc, nb * K, kTexDescWords};
  TexTable<float> kf_points{ctx->d_tex_kf_points, nb * K * 3, 1};
  TexTable<float> points{ctx->d_tex_points, nb * TF_COUNT, K};
  CU(fdesc.make(wide, grow, cap));
  CU(kf_fdesc.make(wide, grow, cap));
  CU(knn_t.make(knn, grow, cap));
  CU(xy.make(true, grow, cap));
  CU(desc.make(true, grow, cap));
  CU(kf_desc.make(true, grow, cap));
  DeviceBuffer<int> nfeat, kf_n, counts;
  DeviceBuffer<float> pose, gh;
  DeviceBuffer<TexKeyframeState> state;
  if (base) {
    CU(nfeat.create(nb));
    CU(kf_n.create(nb * K));
    CU(counts.create(nb));
  }
  CU(kf_points.make(true, grow, cap));
  CU(points.make(true, grow, cap));
  if (base) {
    CU(pose.create(nb * 12));
    CU(gh.create(nb * 27));
    CU(state.create(nb));
    CU(cudaMemsetAsync(nfeat, 0, nb * sizeof(int), ctx->stream));
    CU(cudaMemsetAsync(kf_n, 0, nb * K * sizeof(int), ctx->stream));
    CU(cudaMemsetAsync(counts, 0, nb * sizeof(int), ctx->stream));
    CU(cudaMemsetAsync(pose, 0, nb * 12 * sizeof(float), ctx->stream));
    CU(cudaMemsetAsync(gh, 0, nb * 27 * sizeof(float), ctx->stream));
    CU(cudaMemsetAsync(state, 0, nb * sizeof(TexKeyframeState), ctx->stream));
  }
  // every table exists: the ones that are remade keep their rows
  const int old_cap = ctx->tex_cap;
  CU(fdesc.copy(old_cap, cap, ctx->stream));
  CU(kf_fdesc.copy(old_cap, cap, ctx->stream));
  CU(knn_t.copy(old_cap, cap, ctx->stream));
  CU(xy.copy(old_cap, cap, ctx->stream));
  CU(desc.copy(old_cap, cap, ctx->stream));
  CU(kf_desc.copy(old_cap, cap, ctx->stream));
  CU(kf_points.copy(old_cap, cap, ctx->stream));
  CU(points.copy(old_cap, cap, ctx->stream));
  if (grow) CU(cudaStreamSynchronize(ctx->stream));  // the copies read the tables released below
  fdesc.replace();
  kf_fdesc.replace();
  knn_t.replace();
  xy.replace();
  desc.replace();
  kf_desc.replace();
  kf_points.replace();
  points.replace();
  if (base) {
    ctx->d_tex_nfeat = std::move(nfeat);
    ctx->d_tex_kf_n = std::move(kf_n);
    ctx->d_tex_counts = std::move(counts);
    ctx->d_tex_pose = std::move(pose);
    ctx->d_gh_texture = std::move(gh);
    ctx->d_tex_kf_state = std::move(state);
  }
  ctx->tex_cap = cap;
  return M3TB_OK;
}

// m3tb_set_body assigned the body a depth camera (its depth modality's, or its region modality's for measured occlusions)
bool HasDepthCamera(const BodyDev& B) { return B.has_depth || (B.has_region && B.rp.measure_occlusions); }

// TextureModality::SetUp's conditions for body b (a set body with a texture modality)
int ValidateTextureBody(m3tb_ctx* ctx, int b) {
  const BodyDev& B = ctx->h_bodies[b];
  if (ctx->attached[b][RS_TEXTURE_SILHOUETTE] < 0)
    return Fail(ctx, M3TB_ERR_NOT_SET_UP, "texture modality of body " + std::to_string(b) + ": no silhouette renderer attached");
  if (B.tp.model_occlusions && ctx->attached[b][RS_TEXTURE_DEPTH] < 0)
    return Fail(ctx, M3TB_ERR_NOT_SET_UP, "texture modality: model_occlusions needs a depth renderer attached");
  if (B.tp.measure_occlusions) {
    if (!HasDepthCamera(B)) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "texture measure_occlusions: the body has no depth camera");
    const CameraDev& d = ctx->h_dcams[B.depth_camera];
    if (!d.set || !d.image) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "texture measure_occlusions: depth camera not set / no image uploaded");
  }
  return M3TB_OK;
}

// TextureModality::SetUp's conditions, checked before every texture launch ("Set up ... first"): of every texture body,
// or of the refined ones while a refinement runs
int ValidateTexture(m3tb_ctx* ctx) {
  if (const RefineSelection* sel = ctx->refine) {
    for (int b : sel->texture_ids) {
      int rc = ValidateTextureBody(ctx, b);
      if (rc) return rc;
    }
    return M3TB_OK;
  }
  for (int b = 0; b < ctx->n_bodies; ++b) {
    const BodyDev& B = ctx->h_bodies[b];
    if (!B.set || !B.has_texture) continue;
    int rc = ValidateTextureBody(ctx, b);
    if (rc) return rc;
  }
  return M3TB_OK;
}

// Features belong to the colour frame they were uploaded for: a body whose camera has received a newer frame since
// has none (the reference's detection on that frame found nothing to work with). A refinement touches only its bodies.
int SyncTextureFeatures(m3tb_ctx* ctx) {
  const RefineSelection* sel = ctx->refine;
  const int n = sel ? sel->n_texture : ctx->n_bodies;
  for (int k = 0; k < n; ++k) {
    const int b = sel ? sel->texture_ids[k] : k;
    const BodyDev& B = ctx->h_bodies[b];
    if (!B.has_texture) continue;
    const int gen = ctx->h_ccams[B.texture_camera].generation;
    if (ctx->tex_feat_gen[b] != gen) {
      CU(cudaMemsetAsync(ctx->d_tex_nfeat + b, 0, sizeof(int), ctx->stream));
      ctx->tex_feat_gen[b] = gen;
    }
  }
  return M3TB_OK;
}

// k_texture_keyframe (keyframe = true) or k_texture_match over every body, or over the refined texture bodies while a
// refinement runs; mode as TextureArgs::mode. Matching (mode 1) first runs k_texture_knn_l2 when an L2 body has keyframe
// descriptors to match, and k_texture_knn_hamming once for every TexHammingKnn body.
int LaunchTexture(m3tb_ctx* ctx, bool keyframe, int mode) {
  const RefineSelection* sel = ctx->refine;
  if (ctx->n_texture == 0 || (sel && sel->n_texture == 0)) return M3TB_OK;
  int rc = ValidateTexture(ctx);
  if (!rc) rc = SyncTables(ctx);
  if (!rc) rc = SyncTextureFeatures(ctx);
  if (rc) return rc;
  TextureArgs a;
  a.bodies = ctx->d_bodies;
  a.poses = ctx->d_poses;
  a.tex_pose = ctx->d_tex_pose;
  a.color_cams = ctx->d_ccams;
  a.depth_cams = ctx->d_dcams;
  a.feat_xy = ctx->d_tex_xy;
  a.feat_desc = ctx->d_tex_desc;
  a.feat_n = ctx->d_tex_nfeat;
  a.kf_points = ctx->d_tex_kf_points;
  a.kf_desc = ctx->d_tex_kf_desc;
  a.feat_fdesc = ctx->d_tex_fdesc;
  a.kf_fdesc = ctx->d_tex_kf_fdesc;
  a.knn = ctx->d_tex_knn;
  a.kf_n = ctx->d_tex_kf_n;
  a.kf_state = ctx->d_tex_kf_state;
  a.points = ctx->d_tex_points;
  a.counts = ctx->d_tex_counts;
  a.mode = mode;
  a.cap = ctx->tex_cap;
  a.list = sel ? sel->texture : nullptr;
  const int n_launch = sel ? sel->n_texture : ctx->n_bodies;
  // the widest row, longest deque and largest n_features_max of the L2 bodies and of the Hamming bodies matched by kNN
  int l2_length = 0, l2_keyframes = 0, l2_features = 0, ham_words = 0, ham_keyframes = 0, ham_features = 0;
  for (int k = 0; k < n_launch; ++k) {
    const BodyDev& B = ctx->h_bodies[sel ? sel->texture_ids[k] : k];
    if (!B.set || !B.has_texture) continue;
    if (!TexHamming(B.tp.descriptor_type)) {
      l2_length = std::max(l2_length, TexRowWords(B.tp));
      l2_keyframes = std::max(l2_keyframes, B.tp.n_keyframes);
      l2_features = std::max(l2_features, B.tp.n_features_max);
    } else if (TexHammingKnn(B.tp)) {
      ham_words = std::max(ham_words, TexRowWords(B.tp));
      ham_keyframes = std::max(ham_keyframes, B.tp.n_keyframes);
      ham_features = std::max(ham_features, B.tp.n_features_max);
    }
  }
  if (!keyframe && mode == 1 && l2_length > 0) {  // a body without a length has no features, hence no keyframe points
    CU(cudaFuncSetAttribute(k_texture_knn_l2, cudaFuncAttributeMaxDynamicSharedMemorySize, KnnSharedBytes(l2_length)));
    const dim3 grid(kKnnSplits * l2_keyframes * KnnTilesPerKeyframe(l2_features), n_launch);
    k_texture_knn_l2<<<grid, kKnnThreads, KnnSharedBytes(l2_length), ctx->stream>>>(a);
    CU(cudaGetLastError());
    ctx->launches++;
  }
  if (!keyframe && mode == 1 && ham_features > 0) {
    const dim3 grid(kKnnSplits * ham_keyframes * KnnTilesPerKeyframe(ham_features), n_launch);
    k_texture_knn_hamming<<<grid, kKnnThreads, KnnSharedBytes(ham_words), ctx->stream>>>(a);
    CU(cudaGetLastError());
    ctx->launches++;
  }
  if (keyframe) k_texture_keyframe<<<n_launch, kTexThreads, 0, ctx->stream>>>(a);
  else k_texture_match<<<n_launch, kTexThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  return M3TB_OK;
}

// CalculateScaleAndRegionOfInterest (texture_modality.cpp:890-931) with PrecalculatePoseVariables' body2camera, from
// body b's body2world `pose`: false (roi and scale 0) when the reference returns false or b has no texture modality
bool TextureFocus(const m3tb_ctx* ctx, int b, const float* pose, int32_t* roi, float* scale) {
  const BodyDev& B = ctx->h_bodies[b];
  roi[0] = roi[1] = roi[2] = roi[3] = 0;
  *scale = 0.0f;
  if (!B.set || !B.has_texture) return false;
  const CameraDev& c = ctx->h_ccams[B.texture_camera];
  float b2c[12];
  PoseMul(c.w2c, pose, b2c);
  const float r = ctx->h_geometry[b].radius;  // 0.5f * maximum_body_diameter
  const float x = b2c[3], y = b2c[7], z = b2c[11];
  if (z < r * 1.5f) return false;
  const float abs_x = std::abs(x), abs_y = std::abs(y);
  const float x2 = x * x, y2 = y * y, z2 = z * z, r2 = r * r, rz = r * z;
  const float z2_r2 = z2 - r2, z3_zr2 = z2_r2 * z;
  const float r_u = c.fu * (abs_x * r2 + rz * std::sqrt(z2_r2 + x2)) / z3_zr2;
  const float r_v = c.fv * (abs_y * r2 + rz * std::sqrt(z2_r2 + y2)) / z3_zr2;
  const float center_u = x * c.fu / z + c.ppu, center_v = y * c.fv / z + c.ppv;
  int u_min = int(center_u - r_u - float(kTexRoiMargin) + 0.5f);
  int u_max = int(center_u + r_u + float(kTexRoiMargin) + 0.5f);
  int v_min = int(center_v - r_v - float(kTexRoiMargin) + 0.5f);
  int v_max = int(center_v + r_v + float(kTexRoiMargin) + 0.5f);
  u_min = std::max(u_min, 0);
  u_max = std::min(u_max, c.width - 1);
  v_min = std::max(v_min, 0);
  v_max = std::min(v_max, c.height - 1);
  if (u_min >= u_max || v_min >= v_max) return false;
  roi[0] = u_min;
  roi[1] = v_min;
  roi[2] = u_max - u_min;
  roi[3] = v_max - v_min;
  *scale = float(B.tp.focused_image_size) / std::max(2.0f * r_u, 2.0f * r_v);
  return true;
}

int CheckTextureBody(m3tb_ctx* ctx, int body) {
  if (body < 0 || body >= ctx->n_bodies || !ctx->h_bodies[body].set || !ctx->h_bodies[body].has_texture)
    return Fail(ctx, M3TB_ERR_INVALID, "body has no texture modality");
  return M3TB_OK;
}

// The focused crop of texture body b at `pose`, as m3tb_texture_crop and m3tb_texture_detect_orb both make it: roi and
// scale always (zero without a focus), and when the body has a focus with a non-empty output, the output size and the
// source frame (returns true). The destination is the caller's.
bool FocusCropJob(const m3tb_ctx* ctx, int b, const float* pose, TexCropJob* j) {
  std::memset(j, 0, sizeof(*j));
  int32_t r[4];
  float s;
  bool ok = TextureFocus(ctx, b, pose, r, &s);
  // cv::resize's dsize for Size(): saturate_cast<int>(roi.w * double(scale)), rounded half to even
  const int w = ok ? int(std::nearbyint(double(r[2]) * double(s))) : 0;
  const int h = ok ? int(std::nearbyint(double(r[3]) * double(s))) : 0;
  ok = ok && w >= 1 && h >= 1;  // cv::resize refuses an empty output
  j->roi_x = r[0]; j->roi_y = r[1]; j->roi_w = r[2]; j->roi_h = r[3];
  j->scale = s;
  if (!ok) return false;
  const CameraDev& c = ctx->h_ccams[ctx->h_bodies[b].texture_camera];
  j->src = c.host_src ? c.host_src : c.image;  // a pinned frame is read in place: its device copy holds only ROIs
  j->src_pitch = c.host_src ? c.host_pitch : c.pitch;
  j->out_w = w;
  j->out_h = h;
  return true;
}

// Body b has no device detection any more (its texture modality was set or removed): no read-back, a count of 0
int ForgetDetection(m3tb_ctx* ctx, int b) {
  ctx->orb_nmax[b] = -1;
  if (ctx->d_orb_found) CU(cudaMemsetAsync(ctx->d_orb_found + b, 0, sizeof(int), ctx->stream));
  return M3TB_OK;
}

// Records body b's crop (of its camera's current frame) for m3tb_upload_texture_features_device; none without a focus
void RecordCrop(m3tb_ctx* ctx, int b, const TexCropJob& j) {
  m3tb_ctx::TexCrop& t = ctx->tex_crop[b];
  t.roi_x = j.roi_x;
  t.roi_y = j.roi_y;
  t.scale = j.scale;
  t.gen = j.out_w > 0 ? ctx->h_ccams[ctx->h_bodies[b].texture_camera].generation : -1;
}

}  // namespace

extern "C" {

int m3tb_set_texture_modality(m3tb_ctx* ctx, int body, const m3tb_texture_params* params, int color_camera) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->n_bodies || !ctx->h_bodies[body].set) return Fail(ctx, M3TB_ERR_INVALID, "body not set");
  BodyDev& B = ctx->h_bodies[body];
  if (!params) {  // the body no longer has a texture modality; its renderer slots are detached
    if (!B.has_texture) return M3TB_OK;
    CU(cudaStreamSynchronize(ctx->stream));
    for (int slot = RS_TEXTURE_SILHOUETTE; slot < RS_COUNT; ++slot)
      if (ctx->attached[body][slot] >= 0) {
        std::memset(&B.rend[slot], 0, sizeof(RenderingDev));
        ctx->attached[body][slot] = -1;
        ctx->n_attached--;
        ctx->render_dirty = true;
      }
    if (ctx->d_tex_nonfinite) CU(cudaMemsetAsync(ctx->d_tex_nonfinite + body, 0, sizeof(int), ctx->stream));
    int rc = ForgetDetection(ctx, body);
    if (rc) return rc;
    ctx->tex_crop[body].gen = -1;
    B.has_texture = 0;
    ctx->n_texture--;
    ctx->bodies_dirty = true;
    return M3TB_OK;
  }
  const m3tb_texture_params& p = *params;
  if (p.descriptor_type != M3TB_DESCRIPTOR_ORB && p.descriptor_type != M3TB_DESCRIPTOR_BRISK &&
      p.descriptor_type != M3TB_DESCRIPTOR_FREAK && p.descriptor_type != M3TB_DESCRIPTOR_SIFT &&
      p.descriptor_type != M3TB_DESCRIPTOR_DAISY)
    return Fail(ctx, M3TB_ERR_UNSUPPORTED,
                "only DescriptorType::ORB, BRISK, FREAK (NORM_HAMMING), SIFT and DAISY (NORM_L2) are implemented");
  // m3tb_upload_texture_features and m3tb_get_texture_keyframes take no row width: the body's type sets it. A body's
  // modality therefore moves between the 64-byte types and the others only through its removal (NULL params), so that
  // the same calls on the same body never read or write the caller's buffers at a width they were not sized for.
  const auto binary64 = [](int type) { return TexHamming(type) && TexWideRows(type); };
  if (B.has_texture && binary64(B.tp.descriptor_type) != binary64(p.descriptor_type))
    return Fail(ctx, M3TB_ERR_UNSUPPORTED, std::string("the body's texture modality is ") +
                                               DescriptorName(B.tp.descriptor_type) + ": remove it before setting " +
                                               DescriptorName(p.descriptor_type));
  if (p.n_keyframes > kTexMaxKeyframes) return Fail(ctx, M3TB_ERR_UNSUPPORTED, "n_keyframes above 8");
  if (p.n_features_max > kTexFeatureLimit) return Fail(ctx, M3TB_ERR_UNSUPPORTED, "n_features_max above 4096");
  if (p.n_features_max < kTexMaxFeatures) return Fail(ctx, M3TB_ERR_INVALID, "n_features_max below 512");
  if (color_camera < 0 || color_camera >= ctx->max_cameras || !ctx->h_ccams[color_camera].set)
    return Fail(ctx, M3TB_ERR_INVALID, "color camera not set");
  if (p.n_keyframes < 1 || p.focused_image_size < 1 || p.n_standard_deviations < 1 ||
      p.n_standard_deviations > M3TB_MAX_SCHEDULE || !(p.tukey_norm_constant > 0.0f) || !std::isfinite(p.tukey_norm_constant) ||
      !std::isfinite(p.descriptor_distance_threshold) || p.max_keyframe_age < 0)
    return Fail(ctx, M3TB_ERR_INVALID, "bad texture parameters");
  if (!RadiusValid(p.measured_occlusion_radius) || !RadiusValid(p.modeled_occlusion_radius))
    return Fail(ctx, M3TB_ERR_INVALID, "occlusion radii must be finite and >= 0");
  for (int k = 0; k < p.n_standard_deviations; ++k)
    if (!(p.standard_deviations[k] > 0.0f) || !std::isfinite(p.standard_deviations[k]))
      return Fail(ctx, M3TB_ERR_INVALID, "standard deviations must be positive");
  if (p.measure_occlusions && !(HasDepthCamera(B) && ctx->h_dcams[B.depth_camera].set))
    return Fail(ctx, M3TB_ERR_INVALID, "measure_occlusions needs the body's depth camera");
  if (!ctx->h_geometry[body].set)
    return Fail(ctx, M3TB_ERR_INVALID, "the texture modality needs the body's geometry (m3tb_set_body_geometry)");
  int rc = EnsureTextureTables(ctx, TexWideRows(p.descriptor_type), p.n_features_max > kTexMaxFeatures, p.n_features_max);
  if (rc) return rc;
  CU(cudaStreamSynchronize(ctx->stream));  // a launch in flight may still read this body's keyframes
  CU(cudaMemsetAsync(ctx->d_tex_kf_state + body, 0, sizeof(TexKeyframeState), ctx->stream));
  CU(cudaMemsetAsync(ctx->d_tex_counts + body, 0, sizeof(int), ctx->stream));
  CU(cudaMemsetAsync(ctx->d_tex_nfeat + body, 0, sizeof(int), ctx->stream));
  if (ctx->d_tex_nonfinite) CU(cudaMemsetAsync(ctx->d_tex_nonfinite + body, 0, sizeof(int), ctx->stream));
  TextureParamsDev& t = B.tp;
  t.focused_image_size = p.focused_image_size;
  t.descriptor_distance_threshold = p.descriptor_distance_threshold;
  t.tukey_norm_constant = p.tukey_norm_constant;
  t.n_standard_deviations = p.n_standard_deviations;
  for (int k = 0; k < kMaxSchedule; ++k) t.standard_deviations[k] = k < p.n_standard_deviations ? p.standard_deviations[k] : 0.0f;
  t.max_keyframe_rotation_difference = p.max_keyframe_rotation_difference;
  t.max_keyframe_age = p.max_keyframe_age;
  t.n_keyframes = p.n_keyframes;
  t.measure_occlusions = p.measure_occlusions ? 1 : 0;
  t.measured_occlusion_radius = p.measured_occlusion_radius;
  t.measured_occlusion_threshold = p.measured_occlusion_threshold;
  t.model_occlusions = p.model_occlusions ? 1 : 0;
  t.modeled_occlusion_radius = p.modeled_occlusion_radius;
  t.modeled_occlusion_threshold = p.modeled_occlusion_threshold;
  t.descriptor_type = p.descriptor_type;
  t.descriptor_length = 0;  // SIFT / DAISY: the next upload fixes it
  t.n_features_max = p.n_features_max;
  if (B.has_texture && B.texture_camera != color_camera)  // renderers of the old camera no longer fit
    for (int slot = RS_TEXTURE_SILHOUETTE; slot < RS_COUNT; ++slot)
      if (ctx->attached[body][slot] >= 0) {
        std::memset(&B.rend[slot], 0, sizeof(RenderingDev));
        ctx->attached[body][slot] = -1;
        ctx->n_attached--;
        ctx->render_dirty = true;
      }
  if (!B.has_texture) ctx->n_texture++;
  B.has_texture = 1;
  B.texture_camera = color_camera;
  ctx->tex_feat_gen[body] = -1;
  ctx->tex_crop[body].gen = -1;
  ctx->bodies_dirty = true;
  return ForgetDetection(ctx, body);
}

int m3tb_get_texture_focus(m3tb_ctx* ctx, int first, int count, int32_t* roi, float* scale, int32_t* valid) {
  CHECK_CTX();
  if (first < 0 || count < 0 || first + count > ctx->n_bodies || (count > 0 && (!roi || !scale || !valid)))
    return Fail(ctx, M3TB_ERR_INVALID, "bad body range / null output");
  std::vector<float> poses(size_t(12) * count);
  if (count > 0) {
    CU(cudaMemcpyAsync(poses.data(), ctx->d_poses + 12 * first, poses.size() * sizeof(float), cudaMemcpyDeviceToHost,
                       ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  for (int k = 0; k < count; ++k)
    valid[k] = TextureFocus(ctx, first + k, poses.data() + 12 * k, roi + 4 * k, scale + k) ? 1 : 0;
  return M3TB_OK;
}

}  // extern "C"

namespace {

// m3tb_upload_texture_features (l2 false: binary rows of the body's width) and m3tb_upload_texture_float_features
// (l2 true: rows of `length` floats)
int UploadTextureFeatures(m3tb_ctx* ctx, int body, const float* keypoints_xy, const void* descriptors, bool l2, int n,
                          int length, int roi_x, int roi_y, float scale) {
  int rc = CheckTextureBody(ctx, body);
  if (rc) return rc;
  if (n > ctx->h_bodies[body].tp.n_features_max)
    return Fail(ctx, M3TB_ERR_UNSUPPORTED, "more than the body's n_features_max features");
  if (n < 0 || (n > 0 && (!keypoints_xy || !descriptors)) || !(scale > 0.0f) || !std::isfinite(scale))
    return Fail(ctx, M3TB_ERR_INVALID, "bad feature arguments");
  TextureParamsDev& tp = ctx->h_bodies[body].tp;
  const float* float_descriptors = static_cast<const float*>(descriptors);
  if (l2 == TexHamming(tp.descriptor_type))
    return Fail(ctx, M3TB_ERR_INVALID, l2 ? "ORB, BRISK and FREAK descriptors are uploaded as binary rows"
                                          : "SIFT / DAISY descriptors are uploaded as floats");
  if (l2) {
    if (tp.descriptor_type == M3TB_DESCRIPTOR_SIFT ? length != 128 : (length < 1 || length > kTexMaxFloatDesc))
      return Fail(ctx, M3TB_ERR_INVALID, "descriptor length: 128 for SIFT, 1 .. 256 for DAISY");
    if (tp.descriptor_length != 0 && length != tp.descriptor_length)
      return Fail(ctx, M3TB_ERR_INVALID, "descriptor length differs from the first upload's");
    for (size_t k = 0; k < size_t(n) * length; ++k)
      if (!std::isfinite(float_descriptors[k])) return Fail(ctx, M3TB_ERR_INVALID, "non-finite descriptor");
  }
  // DetectAndComputeCorrKeypoints adds the focus offset (texture_modality.cpp:884-887)
  std::vector<float2> xy(size_t(std::max(n, 1)));
  for (int i = 0; i < n; ++i) {
    xy[i].x = float(roi_x) + keypoints_xy[2 * i] / scale;
    xy[i].y = float(roi_y) + keypoints_xy[2 * i + 1] / scale;
  }
  if (n > 0) {
    const size_t cap = size_t(ctx->tex_cap);
    CU(cudaMemcpyAsync(ctx->d_tex_xy + size_t(body) * cap, xy.data(), sizeof(float2) * n, cudaMemcpyHostToDevice,
                       ctx->stream));
    // a row is `length` floats or the binary width of the body's type, copied bit for bit
    const size_t row = l2 ? sizeof(float) * length : sizeof(uint32_t) * TexRowWords(tp);
    if (TexWideRows(tp.descriptor_type))
      CU(cudaMemcpy2DAsync(ctx->d_tex_fdesc + size_t(body) * cap * kTexMaxFloatDesc, sizeof(float) * kTexMaxFloatDesc,
                           descriptors, row, row, n, cudaMemcpyHostToDevice, ctx->stream));
    else
      CU(cudaMemcpyAsync(ctx->d_tex_desc + size_t(body) * cap * kTexDescWords, descriptors, size_t(32) * n,
                         cudaMemcpyHostToDevice, ctx->stream));
  }
  CU(cudaMemcpyAsync(ctx->d_tex_nfeat + body, &n, sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));  // xy and n are on this stack frame
  ctx->tex_feat_gen[body] = ctx->h_ccams[ctx->h_bodies[body].texture_camera].generation;
  if (l2 && tp.descriptor_length == 0) {
    tp.descriptor_length = length;
    ctx->bodies_dirty = true;
  }
  return M3TB_OK;
}

}  // namespace

extern "C" {

int m3tb_upload_texture_features(m3tb_ctx* ctx, int body, const float* keypoints_xy, const uint8_t* descriptors, int n,
                                 int roi_x, int roi_y, float scale) {
  CHECK_CTX();
  return UploadTextureFeatures(ctx, body, keypoints_xy, descriptors, false, n, 0, roi_x, roi_y, scale);
}

int m3tb_upload_texture_float_features(m3tb_ctx* ctx, int body, const float* keypoints_xy, const float* descriptors,
                                       int n, int length, int roi_x, int roi_y, float scale) {
  CHECK_CTX();
  return UploadTextureFeatures(ctx, body, keypoints_xy, descriptors, true, n, length, roi_x, roi_y, scale);
}

int m3tb_texture_crop(m3tb_ctx* ctx, const int* bodies, int count, uint8_t* out, size_t pitch, size_t body_stride,
                      int capacity_width, int capacity_height, int32_t* roi, float* scale, int32_t* size, int32_t* valid) {
  CHECK_CTX();
  if (count < 0 || (count > 0 && (!bodies || !out)) || capacity_width < 1 || capacity_height < 1 ||
      pitch < size_t(capacity_width) || (count > 1 && body_stride < pitch * size_t(capacity_height)))
    return Fail(ctx, M3TB_ERR_INVALID, "bad crop arguments");
  std::vector<char> listed(ctx->n_bodies, 0);
  for (int k = 0; k < count; ++k) {
    int rc = CheckTextureBody(ctx, bodies[k]);
    if (rc) return rc;
    if (listed[bodies[k]]++) return Fail(ctx, M3TB_ERR_INVALID, "body listed twice");
    const CameraDev& c = ctx->h_ccams[ctx->h_bodies[bodies[k]].texture_camera];
    if (!c.image) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "texture crop: no colour frame uploaded");
  }
  if (count == 0) return M3TB_OK;
  std::vector<float> poses(size_t(12) * ctx->n_bodies);
  CU(cudaMemcpyAsync(poses.data(), ctx->d_poses, poses.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  std::vector<TexCropJob> jobs;
  std::vector<int> job_body;
  bool too_large = false;
  for (int k = 0; k < count; ++k) {
    const int b = bodies[k];
    TexCropJob j;
    const bool ok = FocusCropJob(ctx, b, poses.data() + 12 * b, &j);
    too_large = too_large || (ok && (j.out_w > capacity_width || j.out_h > capacity_height));
    if (roi) { roi[4 * k] = j.roi_x; roi[4 * k + 1] = j.roi_y; roi[4 * k + 2] = j.roi_w; roi[4 * k + 3] = j.roi_h; }
    if (scale) scale[k] = j.scale;
    if (size) { size[2 * k] = j.out_w; size[2 * k + 1] = j.out_h; }
    if (valid) valid[k] = ok ? 1 : 0;
    if (!ok) continue;
    j.dst = out + body_stride * size_t(k);
    jobs.push_back(j);
    job_body.push_back(b);
  }
  if (too_large) return Fail(ctx, M3TB_ERR_INVALID, "a crop is larger than the capacity (see size)");
  for (int k = 0; k < count; ++k) ctx->tex_crop[bodies[k]].gen = -1;
  for (size_t k = 0; k < jobs.size(); ++k) RecordCrop(ctx, job_body[k], jobs[k]);
  for (size_t first = 0; first < jobs.size(); first += kTexJobs) {
    TexCropArgs a;
    a.n_jobs = int(std::min<size_t>(kTexJobs, jobs.size() - first));
    a.dst_pitch = pitch;
    size_t threads = 0;
    for (int k = 0; k < a.n_jobs; ++k) {
      a.jobs[k] = jobs[first + k];
      threads = std::max(threads, size_t((a.jobs[k].out_w + kTexCropPixels - 1) / kTexCropPixels) * a.jobs[k].out_h);
    }
    const unsigned blocks = unsigned((threads + kTexCropThreads - 1) / kTexCropThreads);
    k_texture_crop<<<dim3(blocks, unsigned(a.n_jobs)), kTexCropThreads, 0, ctx->stream>>>(a);
    CU(cudaGetLastError());
    ctx->launches++;
  }
  return M3TB_OK;
}

int m3tb_upload_texture_features_device(m3tb_ctx* ctx, const int* bodies, const m3tb_device_features* features,
                                        int count) {
  CHECK_CTX();
  if (count < 0 || (count > 0 && (!bodies || !features))) return Fail(ctx, M3TB_ERR_INVALID, "bad feature arguments");
  std::vector<char> listed(ctx->n_bodies, 0);
  for (int k = 0; k < count; ++k) {  // every refusal before anything is launched
    const int b = bodies[k];
    const m3tb_device_features& f = features[k];
    int rc = CheckTextureBody(ctx, b);
    if (rc) return rc;
    if (listed[b]++) return Fail(ctx, M3TB_ERR_INVALID, "body listed twice");
    if (f.n > ctx->h_bodies[b].tp.n_features_max)
      return Fail(ctx, M3TB_ERR_UNSUPPORTED, "more than the body's n_features_max features");
    if (f.n < 0 || (f.n > 0 && (!f.x || !f.y || !f.descriptors || f.xy_stride < 1)))
      return Fail(ctx, M3TB_ERR_INVALID, "bad feature arguments");
    const TextureParamsDev& tp = ctx->h_bodies[b].tp;
    const bool l2 = f.length != 0;
    if (l2 == TexHamming(tp.descriptor_type))
      return Fail(ctx, M3TB_ERR_INVALID, l2 ? "ORB, BRISK and FREAK descriptors are binary rows (length 0)"
                                            : "SIFT / DAISY descriptors are uploaded as floats");
    if (l2) {
      if (tp.descriptor_type == M3TB_DESCRIPTOR_SIFT ? f.length != 128 : (f.length < 1 || f.length > kTexMaxFloatDesc))
        return Fail(ctx, M3TB_ERR_INVALID, "descriptor length: 128 for SIFT, 1 .. 256 for DAISY");
      if (tp.descriptor_length != 0 && f.length != tp.descriptor_length)
        return Fail(ctx, M3TB_ERR_INVALID, "descriptor length differs from the first upload's");
    }
    const size_t row = l2 ? sizeof(float) * size_t(f.length) : sizeof(uint32_t) * TexRowWords(tp);
    if (f.n > 1 && f.descriptor_pitch < row) return Fail(ctx, M3TB_ERR_INVALID, "descriptor pitch smaller than a row");
    if (l2 && ((reinterpret_cast<uintptr_t>(f.descriptors) | f.descriptor_pitch) & 3))
      return Fail(ctx, M3TB_ERR_INVALID, "float descriptors not aligned to 4 bytes");
    // the features belong to the body's last crop, which must be of the camera's current frame
    if (ctx->tex_crop[b].gen != ctx->h_ccams[ctx->h_bodies[b].texture_camera].generation)
      return Fail(ctx, M3TB_ERR_INVALID, "no crop of the body's current frame (m3tb_texture_crop)");
  }
  if (count == 0) return M3TB_OK;
  if (!ctx->d_tex_nonfinite) {
    DeviceBuffer<int> flags;
    CU(flags.create(size_t(ctx->max_bodies)));
    CU(cudaMemsetAsync(flags, 0, sizeof(int) * size_t(ctx->max_bodies), ctx->stream));
    ctx->d_tex_nonfinite = std::move(flags);
  }
  for (int first = 0; first < count; first += kTexJobs) {
    TexFeatArgs a;
    a.n_jobs = std::min(kTexJobs, count - first);
    a.feat_xy = ctx->d_tex_xy;
    a.feat_desc = ctx->d_tex_desc;
    a.feat_fdesc = ctx->d_tex_fdesc;
    a.feat_n = ctx->d_tex_nfeat;
    a.nonfinite = ctx->d_tex_nonfinite;
    a.cap = ctx->tex_cap;
    for (int k = 0; k < a.n_jobs; ++k) {
      const m3tb_device_features& f = features[first + k];
      const m3tb_ctx::TexCrop& c = ctx->tex_crop[bodies[first + k]];
      TexFeatJob& j = a.jobs[k];
      j.x = f.x;
      j.y = f.y;
      j.desc = static_cast<const uint8_t*>(f.descriptors);
      j.desc_pitch = f.descriptor_pitch;
      j.body = bodies[first + k];
      j.n = f.n;
      j.xy_stride = f.xy_stride;
      j.length = f.length;
      j.roi_x = c.roi_x;
      j.roi_y = c.roi_y;
      j.scale = c.scale;
      const TextureParamsDev& tp = ctx->h_bodies[j.body].tp;
      j.words = TexRowWords(tp);
      j.wide = TexWideRows(tp.descriptor_type) ? 1 : 0;
      j.pad[0] = j.pad[1] = j.pad[2] = 0;
    }
    k_texture_features<<<a.n_jobs, kTexThreads, 0, ctx->stream>>>(a);
    CU(cudaGetLastError());
    ctx->launches++;
  }
  for (int k = 0; k < count; ++k) {
    const int b = bodies[k];
    ctx->tex_feat_gen[b] = ctx->tex_crop[b].gen;
    TextureParamsDev& tp = ctx->h_bodies[b].tp;
    if (features[k].length != 0 && tp.descriptor_length == 0) {
      tp.descriptor_length = features[k].length;
      ctx->bodies_dirty = true;
    }
  }
  return M3TB_OK;
}

int m3tb_get_texture_feature_flags(m3tb_ctx* ctx, int first, int count, int32_t* nonfinite) {
  CHECK_CTX();
  if (first < 0 || count < 0 || first + count > ctx->n_bodies || (count > 0 && !nonfinite))
    return Fail(ctx, M3TB_ERR_INVALID, "bad body range / null output");
  if (count == 0) return M3TB_OK;
  if (!ctx->d_tex_nonfinite) {
    std::memset(nonfinite, 0, sizeof(int32_t) * size_t(count));
    return M3TB_OK;
  }
  CU(cudaMemcpyAsync(nonfinite, ctx->d_tex_nonfinite + first, sizeof(int32_t) * size_t(count), cudaMemcpyDeviceToHost,
                     ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

void m3tb_orb_params_default(m3tb_orb_params* p) {
  if (!p) return;
  p->n_features = 300;  // texture_modality.h:410-412
  p->scale_factor = 1.2f;
  p->n_levels = 3;
}

}  // extern "C"

namespace {

// One body's ORB job from its crop size and settings (orb.cpp: getScale, the level sizes and nfeaturesPerLevel),
// in the float arithmetic of cv::ORB
TexOrbJob OrbJob(int body, int w, int h, const m3tb_orb_params& p) {
  TexOrbJob j;
  std::memset(&j, 0, sizeof(j));
  j.body = body;
  j.n_levels = p.n_levels;
  const double sf = double(p.scale_factor);
  bool empty_level = false;
  for (int l = 0; l < p.n_levels; ++l) {
    const float s = float(std::pow(sf, double(l)));
    const float inv = 1.0f / s;
    j.layer_scale[l] = s;
    j.w[l] = w > 0 ? int(std::nearbyint(float(w) * inv)) : 0;
    j.h[l] = h > 0 ? int(std::nearbyint(float(h) * inv)) : 0;
    empty_level = empty_level || j.w[l] < 1 || j.h[l] < 1;
  }
  // cv::ORB builds the whole pyramid before it detects, and cv::resize throws on a level of size 0: detect returns
  // nothing for such a crop, keypoints of the earlier levels included. w[0] = 0 gives the body no keypoints.
  if (empty_level) j.w[0] = 0;
  const float factor = float(1.0 / sf);
  float desired = float(p.n_features) * (1.0f - factor) / (1.0f - float(std::pow(double(factor), double(p.n_levels))));
  int sum = 0;
  for (int l = 0; l < p.n_levels - 1; ++l) {
    j.per_level[l] = int(std::nearbyint(desired));
    sum += j.per_level[l];
    desired *= factor;
  }
  j.per_level[p.n_levels - 1] = std::max(p.n_features - sum, 0);
  return j;
}

// The refusals of device detection for ORB texture body b with settings p, apart from the body checks
int CheckOrbDetection(m3tb_ctx* ctx, int b, const m3tb_orb_params& p) {
  if (p.n_features < 1 || !std::isfinite(p.scale_factor) || !(p.scale_factor > 1.0f) || p.n_levels < 1)
    return Fail(ctx, M3TB_ERR_INVALID, "ORB settings: n_features >= 1, finite scale_factor > 1, n_levels >= 1");
  if (p.n_levels > kOrbMaxLevels) return Fail(ctx, M3TB_ERR_UNSUPPORTED, "ORB n_levels above 8");
  if (p.n_features > kOrbFeatureLimit) return Fail(ctx, M3TB_ERR_UNSUPPORTED, "ORB n_features above 2^24");
  if (!ctx->h_ccams[ctx->h_bodies[b].texture_camera].image)
    return Fail(ctx, M3TB_ERR_NOT_SET_UP, "texture detection: no colour frame uploaded");
  return M3TB_OK;
}

// cv::ORB on the focused crops of `count` checked ORB texture bodies at their current poses, with settings params[k]
// for bodies[k] (m3tb_texture_detect_orb, and m3tb_refine_poses_orb before every correspondence iteration). Reads the
// poses back (one host synchronisation) to size the crops; the scratch and parity tables grow all or nothing before
// anything is committed, so a failed allocation returns M3TB_ERR_CUDA with every body as it was.
int DetectOrb(m3tb_ctx* ctx, const int* bodies, int count, const m3tb_orb_params* params) {
  if (count == 0) return M3TB_OK;
  std::vector<float> poses(size_t(12) * ctx->n_bodies);
  CU(cudaMemcpyAsync(poses.data(), ctx->d_poses, poses.size() * sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  // the focus and crop of every body, as m3tb_texture_crop makes them
  std::vector<TexCropJob> crops(count);
  std::vector<TexOrbJob> jobs(count);
  int width = 1, height = 1;
  for (int k = 0; k < count; ++k) {
    const int b = bodies[k];
    const bool ok = FocusCropJob(ctx, b, poses.data() + 12 * b, &crops[k]);
    width = std::max(width, crops[k].out_w);
    height = std::max(height, crops[k].out_h);
    jobs[k] = OrbJob(b, crops[k].out_w, crops[k].out_h, params[k]);
    jobs[k].n_features_max = ctx->h_bodies[b].tp.n_features_max;
    jobs[k].roi_x = crops[k].roi_x;
    jobs[k].roi_y = crops[k].roi_y;
    jobs[k].scale = ok ? crops[k].scale : 1.0f;
  }
  const int pitch = (width + 15) / 16 * 16;
  const size_t job_bytes = (size_t(pitch) * size_t(height) * kOrbScratchBytesPerPixel + 255) / 256 * 256;
  const size_t scratch_bytes = job_bytes * size_t(std::min(count, kTexJobs));
  // scratch and parity tables, each grown all or nothing before anything is committed
  DeviceBuffer<uint8_t> scratch;
  if (ctx->d_orb_scratch.size() < scratch_bytes) CU(scratch.create(scratch_bytes));
  const bool tables = ctx->orb_cap != ctx->tex_cap || !ctx->d_orb_found;
  DeviceBuffer<float2> t_xy;
  DeviceBuffer<float> t_angle, t_response;
  DeviceBuffer<int> t_octave, t_found;
  DeviceBuffer<uint32_t> t_desc;
  if (tables) {
    const size_t slots = size_t(ctx->max_bodies) * size_t(ctx->tex_cap);
    CU(t_xy.create(slots));
    CU(t_angle.create(slots));
    CU(t_response.create(slots));
    CU(t_octave.create(slots));
    CU(t_desc.create(slots * kTexDescWords));
    if (!ctx->d_orb_found) CU(t_found.create(size_t(ctx->max_bodies)));
  }
  if (scratch) ctx->d_orb_scratch = std::move(scratch);
  if (tables) {
    // new tables at the current feature capacity: every other body's last detection is forgotten
    ctx->d_orb_xy = std::move(t_xy);
    ctx->d_orb_angle = std::move(t_angle);
    ctx->d_orb_response = std::move(t_response);
    ctx->d_orb_octave = std::move(t_octave);
    ctx->d_orb_desc = std::move(t_desc);
    if (t_found) ctx->d_orb_found = std::move(t_found);
    ctx->orb_cap = ctx->tex_cap;
    std::fill(ctx->orb_nmax.begin(), ctx->orb_nmax.end(), -1);
    CU(cudaMemsetAsync(ctx->d_orb_found, 0, sizeof(int) * size_t(ctx->max_bodies), ctx->stream));
  }
  for (int k = 0; k < count; ++k) {
    const int b = bodies[k];
    RecordCrop(ctx, b, crops[k]);
    ctx->tex_feat_gen[b] = ctx->h_ccams[ctx->h_bodies[b].texture_camera].generation;  // none without a focus
    ctx->orb_nmax[b] = jobs[k].n_features_max;
  }
  for (int first = 0; first < count; first += kTexJobs) {
    const int n = std::min(kTexJobs, count - first);
    TexCropArgs ca;
    ca.n_jobs = 0;
    ca.dst_pitch = size_t(pitch);
    size_t threads = 0;
    for (int k = 0; k < n; ++k) {
      if (crops[first + k].out_w == 0) continue;
      TexCropJob cj = crops[first + k];
      cj.dst = ctx->d_orb_scratch + job_bytes * size_t(k);
      ca.jobs[ca.n_jobs++] = cj;
      threads = std::max(threads, size_t((cj.out_w + kTexCropPixels - 1) / kTexCropPixels) * cj.out_h);
    }
    if (ca.n_jobs > 0) {
      const unsigned blocks = unsigned((threads + kTexCropThreads - 1) / kTexCropThreads);
      k_texture_crop<<<dim3(blocks, unsigned(ca.n_jobs)), kTexCropThreads, 0, ctx->stream>>>(ca);
      CU(cudaGetLastError());
      ctx->launches++;
    }
    TexOrbArgs oa;
    for (int k = 0; k < n; ++k) oa.jobs[k] = jobs[first + k];
    oa.scratch = ctx->d_orb_scratch;
    oa.job_bytes = job_bytes;
    oa.pitch = pitch;
    oa.height = height;
    oa.feat_xy = ctx->d_tex_xy;
    oa.feat_desc = ctx->d_tex_desc;
    oa.feat_n = ctx->d_tex_nfeat;
    oa.orb_xy = ctx->d_orb_xy;
    oa.orb_angle = ctx->d_orb_angle;
    oa.orb_response = ctx->d_orb_response;
    oa.orb_octave = ctx->d_orb_octave;
    oa.orb_desc = ctx->d_orb_desc;
    oa.found = ctx->d_orb_found;
    oa.cap = ctx->tex_cap;
    oa.orb_cap = ctx->orb_cap;
    k_texture_orb<<<n, kOrbThreads, 0, ctx->stream>>>(oa);
    CU(cudaGetLastError());
    ctx->launches++;
  }
  return M3TB_OK;
}

}  // namespace

extern "C" {

int m3tb_texture_detect_orb(m3tb_ctx* ctx, const int* bodies, int count, const m3tb_orb_params* params) {
  CHECK_CTX();
  if (count < 0 || (count > 0 && !bodies)) return Fail(ctx, M3TB_ERR_INVALID, "bad detection arguments");
  m3tb_orb_params defaults;
  m3tb_orb_params_default(&defaults);
  std::vector<char> listed(ctx->n_bodies, 0);
  std::vector<m3tb_orb_params> settings(count);
  for (int k = 0; k < count; ++k) {  // every refusal before anything is allocated or launched
    const int b = bodies[k];
    int rc = CheckTextureBody(ctx, b);
    if (rc) return rc;
    if (listed[b]++) return Fail(ctx, M3TB_ERR_INVALID, "body listed twice");
    if (ctx->h_bodies[b].tp.descriptor_type != M3TB_DESCRIPTOR_ORB)
      return Fail(ctx, M3TB_ERR_INVALID, "device detection is cv::ORB: the body's descriptor type is not ORB");
    settings[k] = params ? params[k] : defaults;
    rc = CheckOrbDetection(ctx, b, settings[k]);
    if (rc) return rc;
  }
  return DetectOrb(ctx, bodies, count, settings.data());
}

int m3tb_get_texture_detections(m3tb_ctx* ctx, int first, int count, int32_t* n_found) {
  CHECK_CTX();
  if (first < 0 || count < 0 || first + count > ctx->n_bodies || (count > 0 && !n_found))
    return Fail(ctx, M3TB_ERR_INVALID, "bad body range / null output");
  if (count == 0) return M3TB_OK;
  if (!ctx->d_orb_found) {
    std::memset(n_found, 0, sizeof(int32_t) * size_t(count));
    return M3TB_OK;
  }
  CU(cudaMemcpyAsync(n_found, ctx->d_orb_found + first, sizeof(int32_t) * size_t(count), cudaMemcpyDeviceToHost,
                     ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return M3TB_OK;
}

int m3tb_get_texture_orb_keypoints(m3tb_ctx* ctx, int body, float* xy, float* angle, float* response, int32_t* octave,
                                   uint8_t* descriptors, int capacity, int* n_out) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->n_bodies || capacity < 0 || !n_out) return Fail(ctx, M3TB_ERR_INVALID, "bad read-back arguments");
  *n_out = 0;
  if (!ctx->d_orb_found || ctx->orb_nmax[body] < 0) return M3TB_OK;
  int found = 0;
  CU(cudaMemcpyAsync(&found, ctx->d_orb_found + body, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const int n = std::min(found <= ctx->orb_nmax[body] ? found : 0, capacity);
  const size_t at = size_t(body) * size_t(ctx->orb_cap);
  if (n > 0) {
    if (xy) CU(cudaMemcpyAsync(xy, ctx->d_orb_xy + at, sizeof(float2) * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (angle) CU(cudaMemcpyAsync(angle, ctx->d_orb_angle + at, sizeof(float) * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (response)
      CU(cudaMemcpyAsync(response, ctx->d_orb_response + at, sizeof(float) * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (octave) CU(cudaMemcpyAsync(octave, ctx->d_orb_octave + at, sizeof(int) * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (descriptors)
      CU(cudaMemcpyAsync(descriptors, ctx->d_orb_desc + at * kTexDescWords, size_t(32) * n, cudaMemcpyDeviceToHost,
                         ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  *n_out = n;
  return M3TB_OK;
}

int m3tb_texture_correspondences(m3tb_ctx* ctx, int iteration, int corr_iteration) {
  CHECK_CTX();
  (void)iteration;
  if (corr_iteration < 0) return Fail(ctx, M3TB_ERR_INVALID, "negative iteration count");
  if (ctx->n_texture == 0) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "no texture modality set");
  return LaunchTexture(ctx, false, corr_iteration == 0 ? 1 : 0);
}

int m3tb_texture_gradient_hessian(m3tb_ctx* ctx, int iteration, int corr_iteration, int opt_iteration, float* gradients,
                                  float* hessians) {
  CHECK_CTX();
  if (ctx->n_texture == 0) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "no texture modality set");
  int rc = ValidateTexture(ctx);
  if (!rc) rc = LaunchTrack(ctx, iteration, corr_iteration, corr_iteration + 1, 1, opt_iteration, PH_TEXTURE_GH | PH_STORE_GH);
  if (rc) return rc;
  return ReadGH(ctx, ctx->d_gh_texture, gradients, hessians);
}

int m3tb_get_texture_points(m3tb_ctx* ctx, int body, m3tb_texture_point* points, int capacity, int* n_out) {
  CHECK_CTX();
  int rc = CheckTextureBody(ctx, body);
  if (rc) return rc;
  if (capacity < 0 || (capacity > 0 && !points)) return Fail(ctx, M3TB_ERR_INVALID, "bad output");
  int n = 0;
  CU(cudaMemcpyAsync(&n, ctx->d_tex_counts + body, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if (n_out) *n_out = n;
  const int m = std::min(n, capacity);
  if (m <= 0) return M3TB_OK;
  std::vector<float> f(size_t(TF_COUNT) * m);
  const size_t point_cap = size_t(kTexMaxKeyframes) * ctx->tex_cap;
  const float* src = ctx->d_tex_points + size_t(body) * TF_COUNT * point_cap;
  CU(cudaMemcpy2DAsync(f.data(), sizeof(float) * m, src, sizeof(float) * point_cap, sizeof(float) * m, TF_COUNT,
                       cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < m; ++i) {
    m3tb_texture_point& p = points[i];
    p.center_f_body[0] = f[TF_CBX * m + i];
    p.center_f_body[1] = f[TF_CBY * m + i];
    p.center_f_body[2] = f[TF_CBZ * m + i];
    p.correspondence_center[0] = f[TF_CU * m + i];
    p.correspondence_center[1] = f[TF_CV * m + i];
    p.center[0] = f[TF_PU * m + i];
    p.center[1] = f[TF_PV * m + i];
  }
  return M3TB_OK;
}

int m3tb_get_texture_keyframes(m3tb_ctx* ctx, int body, int* n_keyframes, int* sizes, float* points, uint8_t* descriptors,
                               int capacity, int* age, float* orientation) {
  CHECK_CTX();
  int rc = CheckTextureBody(ctx, body);
  if (rc) return rc;
  if (capacity < 0) return Fail(ctx, M3TB_ERR_INVALID, "bad capacity");
  TexKeyframeState st;
  const TextureParamsDev& tp = ctx->h_bodies[body].tp;
  // a descriptor is `width` bytes in rows of `stride` words (m3t_b200_texture.cuh)
  const size_t stride = TexRowStride(tp), width = sizeof(uint32_t) * TexRowWords(tp);
  const size_t cap = size_t(ctx->tex_cap);
  std::vector<int> kn(kTexMaxKeyframes);
  const uint32_t* kd_src = TexWideRows(tp.descriptor_type) ? reinterpret_cast<const uint32_t*>(ctx->d_tex_kf_fdesc.get())
                                                           : ctx->d_tex_kf_desc.get();
  CU(cudaMemcpyAsync(&st, ctx->d_tex_kf_state + body, sizeof(st), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(kn.data(), ctx->d_tex_kf_n + body * kTexMaxKeyframes, sizeof(int) * kn.size(), cudaMemcpyDeviceToHost,
                     ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  // the rows of the deque's keyframes only: a keyframe slot holds up to cap points
  std::vector<float> kp(size_t(kTexMaxKeyframes) * 3 * cap);
  std::vector<uint32_t> kd(size_t(kTexMaxKeyframes) * cap * stride);
  for (int k = 0; k < st.size; ++k) {
    const int slot = (st.head + k) % kTexMaxKeyframes;
    if (kn[slot] <= 0) continue;
    const size_t kf = size_t(body) * kTexMaxKeyframes + slot;
    CU(cudaMemcpy2DAsync(kp.data() + size_t(slot) * 3 * cap, sizeof(float) * cap, ctx->d_tex_kf_points + kf * 3 * cap,
                         sizeof(float) * cap, sizeof(float) * kn[slot], 3, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(kd.data() + size_t(slot) * cap * stride, kd_src + kf * cap * stride,
                       sizeof(uint32_t) * kn[slot] * stride, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CU(cudaStreamSynchronize(ctx->stream));
  if (n_keyframes) *n_keyframes = st.size;
  if (age) *age = st.age;
  if (orientation) std::memcpy(orientation, st.orientation, sizeof(float) * 3);
  int written = 0;
  for (int k = 0; k < st.size; ++k) {
    const int slot = (st.head + k) % kTexMaxKeyframes;
    if (sizes) sizes[k] = kn[slot];
    for (int i = 0; i < kn[slot] && written < capacity; ++i, ++written) {
      if (points)
        for (int c = 0; c < 3; ++c) points[3 * written + c] = kp[(size_t(slot) * 3 + c) * cap + i];
      if (descriptors) std::memcpy(descriptors + width * written, kd.data() + (size_t(slot) * cap + i) * stride, width);
    }
  }
  return M3TB_OK;
}

int m3tb_debug_resources(int fail_after, long long* live) {
  if (fail_after >= 0) g_fail_after.store(fail_after);
  if (live) *live = g_live_resources.load();
  return M3TB_OK;
}

// ---- pose scoring ------------------------------------------------------------------------------------------------

static std::vector<EvalBodyDev>& EvalBodies(m3tb_ctx* ctx) {
  if (ctx->h_eval_bodies.empty()) {
    EvalBodyDev none = {};
    none.model = -1;
    ctx->h_eval_bodies.assign(size_t(ctx->max_bodies), none);
  }
  return ctx->h_eval_bodies;
}

// Uploads the model and body tables when they changed; on failure they keep what they held and stay dirty.
static int SyncEvalTables(m3tb_ctx* ctx) {
  if (!ctx->eval_dirty) return M3TB_OK;
  std::vector<EvalModelDev> models(ctx->eval_models.size());
  for (size_t i = 0; i < models.size(); ++i) {
    const auto& h = ctx->eval_models[i];
    models[i] = {h.full, h.reduced, h.n_full, h.n_reduced};
  }
  const auto& bodies = EvalBodies(ctx);
  DeviceBuffer<EvalModelDev> gm;
  DeviceBuffer<EvalBodyDev> gb;
  int rc = GrowTable(ctx, ctx->d_eval_models, gm, models.size());
  if (!rc) rc = GrowTable(ctx, ctx->d_eval_bodies, gb, bodies.size());
  if (rc) return rc;
  if (gm || gb) CU(cudaStreamSynchronize(ctx->stream));  // a scoring launch in flight may still read the old tables
  if (gm) ctx->d_eval_models = std::move(gm);
  if (gb) ctx->d_eval_bodies = std::move(gb);
  CU(cudaMemcpyAsync(ctx->d_eval_models, models.data(), sizeof(EvalModelDev) * models.size(), cudaMemcpyHostToDevice,
                     ctx->stream));
  CU(cudaMemcpyAsync(ctx->d_eval_bodies, bodies.data(), sizeof(EvalBodyDev) * bodies.size(), cudaMemcpyHostToDevice,
                     ctx->stream));
  ctx->eval_dirty = false;
  return M3TB_OK;
}

// Grows the per-call scratch tables, all or nothing.
static int GrowScoreScratch(m3tb_ctx* ctx, size_t n_ids, size_t n_gt, size_t n_partial, size_t n_out, size_t n_curves,
                            size_t n_diameter) {
  DeviceBuffer<int> ids;
  DeviceBuffer<float> gt, partial, curves;
  DeviceBuffer<m3tb_pose_score> out;
  DeviceBuffer<unsigned> diameter;
  int rc = GrowTable(ctx, ctx->d_score_ids, ids, n_ids);
  if (!rc) rc = GrowTable(ctx, ctx->d_score_gt, gt, n_gt);
  if (!rc) rc = GrowTable(ctx, ctx->d_score_partial, partial, n_partial);
  if (!rc) rc = GrowTable(ctx, ctx->d_score_out, out, n_out);
  if (!rc) rc = GrowTable(ctx, ctx->d_score_curves, curves, n_curves);
  if (!rc) rc = GrowTable(ctx, ctx->d_diameter, diameter, n_diameter);
  if (rc) return rc;
  if (ids || gt || partial || out || curves || diameter) CU(cudaStreamSynchronize(ctx->stream));
  if (ids) ctx->d_score_ids = std::move(ids);
  if (gt) ctx->d_score_gt = std::move(gt);
  if (partial) ctx->d_score_partial = std::move(partial);
  if (out) ctx->d_score_out = std::move(out);
  if (curves) ctx->d_score_curves = std::move(curves);
  if (diameter) ctx->d_diameter = std::move(diameter);
  return M3TB_OK;
}

// Slices of the full set so that small batches still fill the device: (n_chunks, chunk) for `ctas` blocks per slice.
static void ScoreSlices(const m3tb_ctx* ctx, long long ctas, int max_full, int* n_chunks, int* chunk) {
  const int tiles = (max_full + kScoreTile - 1) / kScoreTile;
  long long want = (2LL * ctx->sm_count + ctas - 1) / ctas;
  const int c = int(std::max(1LL, std::min<long long>(want, tiles)));
  const int tiles_per_chunk = (tiles + c - 1) / c;
  *chunk = tiles_per_chunk * kScoreTile;
  *n_chunks = (tiles + tiles_per_chunk - 1) / tiles_per_chunk;
}

void m3tb_score_params_default(m3tb_score_params* p) {
  if (!p) return;
  p->threshold_max = 0.1f;    // ycb_evaluator.h:46
  p->curve_scale = 1.0f;
  p->auc_scale = 1.0f;
  p->translation_error_threshold = 0.05f;  // rbot_evaluator.h:192-193, kPi of common.h
  p->rotation_error_threshold = 5.0f * 3.1415926535897f / 180.0f;
}

int m3tb_set_evaluation_model(m3tb_ctx* ctx, int model, const float* vertices, int n_vertices, int n_vertices_evaluation) {
  CHECK_CTX();
  if (model < 0 || model >= ctx->max_models || model > int(ctx->eval_models.size()))
    return Fail(ctx, M3TB_ERR_INVALID, "evaluation model ids are dense (0..n) and below max_models");
  if (!vertices || n_vertices < 1) return Fail(ctx, M3TB_ERR_INVALID, "an evaluation model needs vertices");
  std::vector<float4> full(static_cast<size_t>(n_vertices));
  for (int i = 0; i < n_vertices; ++i) {
    const float* v = vertices + 3 * size_t(i);
    if (!std::isfinite(v[0]) || !std::isfinite(v[1]) || !std::isfinite(v[2]))
      return Fail(ctx, M3TB_ERR_INVALID, "evaluation vertex " + std::to_string(i) + " is not finite");
    full[i] = make_float4(v[0], v[1], v[2], 0.0f);
  }
  // GenderateReducedVertices (ycb_evaluator.cpp:1222-1248)
  std::vector<float4> reduced;
  if (n_vertices_evaluation <= 0 || n_vertices_evaluation >= n_vertices) {
    reduced = full;
  } else {
    std::mt19937 generator{7};
    reduced.resize(size_t(n_vertices_evaluation));
    for (auto& v : reduced) v = full[int(generator() % n_vertices)];
  }
  m3tb_ctx::EvalModelHost h;
  CU(h.full.create(full.size()));
  CU(h.reduced.create(reduced.size()));
  h.n_full = int(full.size());
  h.n_reduced = int(reduced.size());
  CU(cudaMemcpyAsync(h.full, full.data(), sizeof(float4) * full.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(h.reduced, reduced.data(), sizeof(float4) * reduced.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));  // the staging vectors end with this call
  if (model == int(ctx->eval_models.size())) ctx->eval_models.push_back(std::move(h));
  else ctx->eval_models[model] = std::move(h);
  ctx->eval_dirty = true;
  return M3TB_OK;
}

int m3tb_set_body_evaluation_model(m3tb_ctx* ctx, int body, int model, const float geometry2body[12]) {
  CHECK_CTX();
  if (body < 0 || body >= ctx->max_bodies) return Fail(ctx, M3TB_ERR_INVALID, "body index out of range");
  if (model < 0 || model >= int(ctx->eval_models.size())) return Fail(ctx, M3TB_ERR_INVALID, "evaluation model not set");
  EvalBodyDev e = {};
  e.model = model;
  e.has_geometry2body = geometry2body ? 1 : 0;
  if (geometry2body) std::memcpy(e.geometry2body, geometry2body, sizeof(e.geometry2body));
  EvalBodies(ctx)[body] = e;
  ctx->eval_dirty = true;
  return M3TB_OK;
}

int m3tb_get_evaluation_vertices(m3tb_ctx* ctx, int model, float* vertices, int capacity, int* n_vertices) {
  CHECK_CTX();
  if (model < 0 || model >= int(ctx->eval_models.size())) return Fail(ctx, M3TB_ERR_INVALID, "evaluation model not set");
  if (capacity < 0 || (capacity > 0 && !vertices)) return Fail(ctx, M3TB_ERR_INVALID, "bad capacity");
  const auto& h = ctx->eval_models[model];
  if (n_vertices) *n_vertices = h.n_reduced;
  const int n = std::min(capacity, h.n_reduced);
  if (n == 0) return M3TB_OK;
  std::vector<float4> v(static_cast<size_t>(n));
  CU(cudaMemcpyAsync(v.data(), h.reduced, sizeof(float4) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < n; ++i) {
    vertices[3 * i + 0] = v[i].x;
    vertices[3 * i + 1] = v[i].y;
    vertices[3 * i + 2] = v[i].z;
  }
  return M3TB_OK;
}

int m3tb_score_poses(m3tb_ctx* ctx, const int* bodies, int n, const float* gt_body2world, int gt_on_device,
                     const m3tb_score_params* params, m3tb_pose_score* out, float* add_curve, float* adds_curve,
                     int out_on_device) {
  CHECK_CTX();
  if (!bodies || n < 1 || !gt_body2world || !params || !out || (!add_curve) != (!adds_curve))
    return Fail(ctx, M3TB_ERR_INVALID, "bad scoring arguments");
  if (!(params->threshold_max > 0.0f) || !std::isfinite(params->threshold_max) || !(params->curve_scale > 0.0f) ||
      !std::isfinite(params->curve_scale))
    return Fail(ctx, M3TB_ERR_INVALID, "threshold_max and curve_scale must be finite and positive");
  const auto& eb = EvalBodies(ctx);
  int max_full = 0, max_reduced = 0;
  for (int q = 0; q < n; ++q) {
    const int b = bodies[q];
    if (b < 0 || b >= ctx->max_bodies) return Fail(ctx, M3TB_ERR_INVALID, "body index out of range");
    if (eb[b].model < 0) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "body " + std::to_string(b) + " has no evaluation model");
    const auto& m = ctx->eval_models[eb[b].model];
    max_full = std::max(max_full, m.n_full);
    max_reduced = std::max(max_reduced, m.n_reduced);
  }
  const int blocks = (max_reduced + kScoreBlock - 1) / kScoreBlock;
  int n_chunks = 1, chunk = 0;
  ScoreSlices(ctx, (long long)n * blocks, max_full, &n_chunks, &chunk);
  const bool curves = add_curve != nullptr;
  const size_t nq = size_t(n);
  int rc = GrowScoreScratch(ctx, nq, gt_on_device ? 0 : 12 * nq, nq * size_t(n_chunks) * size_t(max_reduced),
                            out_on_device ? 0 : nq, (out_on_device || !curves) ? 0 : 2 * M3TB_N_CURVE_VALUES * nq, 0);
  if (!rc) rc = SyncEvalTables(ctx);
  if (rc) return rc;
  ScoreArgs a = {};
  a.models = ctx->d_eval_models;
  a.eval_bodies = ctx->d_eval_bodies;
  a.poses = ctx->d_poses;
  a.bodies = ctx->d_score_ids;
  a.n = n;
  a.n_chunks = n_chunks;
  a.chunk = chunk;
  a.max_reduced = max_reduced;
  a.partial = ctx->d_score_partial;
  a.threshold_max = params->threshold_max;
  a.curve_scale = params->curve_scale;
  a.auc_scale = params->auc_scale;
  a.translation_threshold = params->translation_error_threshold;
  a.rotation_threshold = params->rotation_error_threshold;
  CU(cudaMemcpyAsync(ctx->d_score_ids, bodies, sizeof(int) * nq, cudaMemcpyHostToDevice, ctx->stream));
  if (gt_on_device) {
    a.gt = gt_body2world;
  } else {
    CU(cudaMemcpyAsync(ctx->d_score_gt, gt_body2world, sizeof(float) * 12 * nq, cudaMemcpyHostToDevice, ctx->stream));
    a.gt = ctx->d_score_gt;
  }
  if (out_on_device) {
    a.out = out;
    a.add_curve = add_curve;
    a.adds_curve = adds_curve;
  } else {
    a.out = ctx->d_score_out;
    if (curves) {
      a.add_curve = ctx->d_score_curves;
      a.adds_curve = ctx->d_score_curves + M3TB_N_CURVE_VALUES * nq;
    }
  }
  k_score<<<dim3(unsigned(n), unsigned(n_chunks), unsigned(blocks)), kScoreThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  k_score_finish<<<unsigned(n), kScoreThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  if (!out_on_device) {
    CU(cudaMemcpyAsync(out, a.out, sizeof(m3tb_pose_score) * nq, cudaMemcpyDeviceToHost, ctx->stream));
    if (curves) {
      CU(cudaMemcpyAsync(add_curve, a.add_curve, sizeof(float) * M3TB_N_CURVE_VALUES * nq, cudaMemcpyDeviceToHost,
                         ctx->stream));
      CU(cudaMemcpyAsync(adds_curve, a.adds_curve, sizeof(float) * M3TB_N_CURVE_VALUES * nq, cudaMemcpyDeviceToHost,
                         ctx->stream));
    }
    CU(cudaStreamSynchronize(ctx->stream));
  }
  return M3TB_OK;
}

int m3tb_calculate_diameters(m3tb_ctx* ctx, const int* models, int n, float* out) {
  CHECK_CTX();
  if (!models || n < 1 || !out) return Fail(ctx, M3TB_ERR_INVALID, "bad diameter arguments");
  int max_full = 0;
  for (int q = 0; q < n; ++q) {
    if (models[q] < 0 || models[q] >= int(ctx->eval_models.size()))
      return Fail(ctx, M3TB_ERR_INVALID, "evaluation model not set");
    max_full = std::max(max_full, ctx->eval_models[models[q]].n_full);
  }
  const int blocks = (max_full + kScoreBlock - 1) / kScoreBlock;
  int n_chunks = 1, chunk = 0;
  ScoreSlices(ctx, (long long)n * blocks, max_full, &n_chunks, &chunk);
  int rc = GrowScoreScratch(ctx, size_t(n), 0, 0, 0, 0, size_t(n));
  if (!rc) rc = SyncEvalTables(ctx);
  if (rc) return rc;
  DiameterArgs a = {};
  a.models = ctx->d_eval_models;
  a.model_ids = ctx->d_score_ids;
  a.n_chunks = n_chunks;
  a.chunk = chunk;
  a.max_sq = ctx->d_diameter;
  CU(cudaMemcpyAsync(ctx->d_score_ids, models, sizeof(int) * size_t(n), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemsetAsync(a.max_sq, 0, sizeof(unsigned) * size_t(n), ctx->stream));
  k_diameter<<<dim3(unsigned(n), unsigned(n_chunks), unsigned(blocks)), kScoreThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  std::vector<unsigned> bits(static_cast<size_t>(n));
  CU(cudaMemcpyAsync(bits.data(), a.max_sq, sizeof(unsigned) * size_t(n), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  for (int q = 0; q < n; ++q) {
    float sq;
    std::memcpy(&sq, &bits[q], sizeof(sq));
    out[q] = std::sqrt(sq);
  }
  return M3TB_OK;
}

}  // extern "C"
