// m3t_b200.cu — host side of libm3t_b200.so: context, device memory, launches; implements include/m3t_b200.h.
// No CPU fallback anywhere: if CUDA is unusable every compute entry point returns M3TB_ERR_CUDA.
#include "m3t_b200.h"

#include <cudaTypedefs.h>  // PFN_cuTensorMapEncodeTiled

#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "m3t_b200_structures.cuh"
#include "m3t_b200_kernels.cuh"
#include "m3t_b200_views.cuh"

#include "m3t_b200_track_variants.h"
#include "m3t_b200_track2.cuh"

namespace m3tb {
extern template __global__ void k_track2<512, true>(const __grid_constant__ TrackArgs);
extern template __global__ void k_track2<512, false>(const __grid_constant__ TrackArgs);
extern template __global__ void k_track2<1024, true>(const __grid_constant__ TrackArgs);
extern template __global__ void k_track2<1024, false>(const __grid_constant__ TrackArgs);
// the fused kernel's variants are compiled in m3t_b200_track_<g>.cu
#define M3TB_DECLARE(T_, K_, L_, O_, C_) extern template __global__ void k_track<T_, K_, L_, O_, C_>(const __grid_constant__ TrackArgs);
M3TB_TRACK_ALL(M3TB_DECLARE)
#undef M3TB_DECLARE
}  // namespace m3tb

using namespace m3tb;

namespace {

struct ImagePool {
  uint8_t* base = nullptr;
  size_t frame_bytes = 0;
  unsigned pitch = 0;
  int width = 0, height = 0, capacity = 0;
  // colour pools: the bin-index images (u16 per pixel), same slot order
  uint16_t* bins = nullptr;
  size_t bin_frame_bytes = 0;
  unsigned bin_pitch = 0;
};

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
  float4* orientations = nullptr;
  float* view_scalars = nullptr;
  float4* points = nullptr;
  float* depth_offsets = nullptr;
  float4* cluster_info = nullptr;
  float4* sorted_views = nullptr;
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
  std::vector<uint8_t*> private_color, private_depth;  // images that do not fit the pools
  bool bodies_dirty = true, cams_dirty = true, models_dirty = true;

  BodyDev* d_bodies = nullptr;
  CameraDev *d_ccams = nullptr, *d_dcams = nullptr;
  ModelDev *d_rmodels = nullptr, *d_dmodels = nullptr;
  float* d_poses = nullptr;
  ImagePool color_pool, depth_pool;

  float *d_hist_f = nullptr, *d_hist_b = nullptr, *d_mem_f = nullptr, *d_mem_b = nullptr;
  float2* d_lut = nullptr;
  size_t hist_stride = 0;

  float *d_rstate = nullptr, *d_dstate = nullptr;
  int line_cap = 0, point_cap = 0;
  int* d_counts = nullptr;
  float *d_gh_region = nullptr, *d_gh_depth = nullptr;
  size_t max_dyn_smem = 0;
  RoiRecord* d_roi = nullptr;             // [max_bodies][2]
  unsigned long long* d_ingest_bytes = nullptr;  // [2]: one counter per ingest launch in flight
  int ingest_bytes_slot = 0;              // the counter of the last ingest launch
  int sm_count = 132;
  bool ingest_pending = false;            // a pinned frame was handed over since the last k_ingest launch
  // frame prefetch (m3tb_prefetch_frames): second set of image pools / camera tables / ROI records, side stream
  ImagePool color_pool_alt, depth_pool_alt;
  CameraDev *d_ccams_alt = nullptr, *d_dcams_alt = nullptr;
  RoiRecord* d_roi_alt = nullptr;
  float* d_poses_snap[2] = {nullptr, nullptr};  // poses at the start of the last two tracking launches; [snap_parity] is
  int snap_parity = 0;                    //   what the next prefetch projects with, the other one may still be read by the ingest in flight
  cudaStream_t ingest_stream = nullptr;
  cudaStream_t table_stream = nullptr;    // camera tables + counter reset of a prefetch: beside the ingest in flight, not behind it
  CameraDev* h_cam_stage[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // pinned staging [parity][colour | depth]
  int stage_parity = 0;
  cudaEvent_t ev_ingest_done = nullptr, ev_poses_snap = nullptr, ev_tables = nullptr;
  cudaEvent_t ev_stage[2] = {nullptr, nullptr};  // the table copies out of h_cam_stage[parity] have run
  bool prefetch_enabled = false;          // set by the first m3tb_prefetch_frames
  bool prefetched = false;                // the next consumer launch has to wait for ev_ingest_done
  bool poses_snap_valid = false;
  bool roi_ingest = true;                 // M3TB_NO_ROI_INGEST=1 forces full-frame copies
  long long* d_phase_clock = nullptr;  // allocated when M3TB_TIMING=1
  bool use_tiles = true;  // stage ROI tiles in shared memory (M3TB_NO_TILES=1 in the environment disables it)
  bool use_track2 = true; // second-generation fused kernel where it applies (M3TB_KERNEL=1 forces k_track)
  std::vector<char> bin_stale;            // per colour camera: the bin-index image does not match the frame copy
  int bin_bitshift = -1;                  // what the bin-index images were built with
  int* d_bin_ids = nullptr;               // staging for k_bin
  std::vector<uint8_t*> rendering_allocs; // device copies of the renderer images (m3tb_upload_*_rendering)
  std::vector<PoolMaps> pool_maps;        // tensor maps of the pools seen so far (current / alternate x bins / depth)
  int tma_mode = 1;                       // M3TB_TMA: 0 legacy staging, 1 tensor maps in the kernel parameters, 2 in global memory
  CUtensorMap* d_tmaps = nullptr;         // tma_mode 2: [2][kTileWidths]
  const void* d_tmaps_bases[2] = {nullptr, nullptr};  // the pools d_tmaps currently describes

  // kinematic structures (empty: every body is its own rigid-body optimiser inside k_track)
  // shared ColorHistograms objects (m3tb_share_color_histograms): per body the owner of the object it uses, -1 = its own
  std::vector<int> hist_owner;
  std::vector<int> hist_table_uploaded;  // what d_hist_owner / d_hist_groups hold
  int n_hist_groups = 0;
  int* d_hist_owner = nullptr;     // [max_bodies]
  int* d_hist_groups = nullptr;    // group_owner[n] | group_first[n + 1] | members[...]
  int hist_groups_capacity = 0;
  std::vector<StructureHost> structures;
  bool structures_dirty = false;
  int n_struct_launch = 0;                 // user structures + one implicit structure per unreferenced body
  std::vector<int> struct_first_link;      // per launched structure
  std::vector<int> h_link_bodies;          // body index of every launched link
  bool use_clusters = false;               // M3TB_CLUSTER=1: cluster-fused structure path (see DESIGN.md: measured slower)
  std::vector<StructureDev> h_structures;
  StructureDev* d_structures = nullptr;
  LinkDev* d_links = nullptr;
  LinkDev* d_links_default = nullptr;      // Link::default_body2joint_pose_ / default_joint2parent_pose_
  int n_links_total = 0;
  bool defaults_valid = false;
  std::vector<LinkDev> h_links_default;
  ConstraintDev* d_constraints = nullptr;
  int cap_structures = 0, cap_links = 0, cap_constraints = 0;
  float* d_gh_link = nullptr;
  float* d_theta = nullptr;
  int* d_struct_status = nullptr;
  size_t struct_smem = 0;
};

namespace {

int Fail(m3tb_ctx* ctx, int code, const std::string& msg) {
  if (ctx) ctx->err = msg;
  return code;
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

int EnsureHist(m3tb_ctx* ctx, size_t stride) {
  if (stride <= ctx->hist_stride) return M3TB_OK;
  const size_t nb = size_t(ctx->max_bodies);
  float* nf[4] = {nullptr, nullptr, nullptr, nullptr};
  float2* nl = nullptr;
  for (int k = 0; k < 4; ++k) {
    CU(cudaMalloc(&nf[k], nb * stride * sizeof(float)));
    CU(cudaMemsetAsync(nf[k], 0, nb * stride * sizeof(float), ctx->stream));
  }
  CU(cudaMalloc(&nl, nb * stride * sizeof(float2)));
  CU(cudaMemsetAsync(nl, 0, nb * stride * sizeof(float2), ctx->stream));
  float* old[4] = {ctx->d_hist_f, ctx->d_hist_b, ctx->d_mem_f, ctx->d_mem_b};
  if (ctx->hist_stride) {
    for (int k = 0; k < 4; ++k)
      CU(cudaMemcpy2DAsync(nf[k], stride * sizeof(float), old[k], ctx->hist_stride * sizeof(float),
                           ctx->hist_stride * sizeof(float), nb, cudaMemcpyDeviceToDevice, ctx->stream));
    CU(cudaMemcpy2DAsync(nl, stride * sizeof(float2), ctx->d_lut, ctx->hist_stride * sizeof(float2),
                         ctx->hist_stride * sizeof(float2), nb, cudaMemcpyDeviceToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < 4; ++k) cudaFree(old[k]);
    cudaFree(ctx->d_lut);
  }
  ctx->d_hist_f = nf[0]; ctx->d_hist_b = nf[1]; ctx->d_mem_f = nf[2]; ctx->d_mem_b = nf[3];
  ctx->d_lut = nl;
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
  if (lc > ctx->line_cap || !ctx->d_rstate) {
    if (ctx->d_rstate) cudaFree(ctx->d_rstate);
    CU(cudaMalloc(&ctx->d_rstate, size_t(ctx->max_bodies) * RF_COUNT * lc * sizeof(float)));
    CU(cudaMemsetAsync(ctx->d_rstate, 0, size_t(ctx->max_bodies) * RF_COUNT * lc * sizeof(float), ctx->stream));
    // the stored correspondences are gone: a load-state call before the next CalculateCorrespondences sees 0 lines
    if (ctx->d_counts) CU(cudaMemsetAsync(ctx->d_counts, 0, sizeof(int) * 4 * ctx->max_bodies, ctx->stream));
    ctx->line_cap = lc;
  }
  if (pc > ctx->point_cap || !ctx->d_dstate) {
    if (ctx->d_dstate) cudaFree(ctx->d_dstate);
    CU(cudaMalloc(&ctx->d_dstate, size_t(ctx->max_bodies) * DF_COUNT * pc * sizeof(float)));
    CU(cudaMemsetAsync(ctx->d_dstate, 0, size_t(ctx->max_bodies) * DF_COUNT * pc * sizeof(float), ctx->stream));
    if (ctx->d_counts) CU(cudaMemsetAsync(ctx->d_counts, 0, sizeof(int) * 4 * ctx->max_bodies, ctx->stream));
    ctx->point_cap = pc;
  }
  return M3TB_OK;
}

int SyncTables(m3tb_ctx* ctx) {
  if (ctx->bodies_dirty) {
    CU(cudaMemcpyAsync(ctx->d_bodies, ctx->h_bodies.data(), sizeof(BodyDev) * ctx->max_bodies, cudaMemcpyHostToDevice,
                       ctx->stream));
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
      if (B.rp.measure_occlusions) {  // RegionModality::SetUp / PrecalculateModelVariables (region_modality.cpp:965-977)
        const CameraDev& d = ctx->h_dcams[B.depth_camera];
        if (!d.set || !d.image) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "measure_occlusions: depth camera not set / no image uploaded");
        if (B.rp.measured_depth_offset_radius > ctx->h_rmodels[B.region_model].max_radius_depth_offset)
          return Fail(ctx, M3TB_ERR_INVALID, "Measured depth offset radius too large");
      }
      if (B.rp.model_occlusions &&  // region_modality.cpp:979-991
          B.rp.modeled_depth_offset_radius > ctx->h_rmodels[B.region_model].max_radius_depth_offset)
        return Fail(ctx, M3TB_ERR_INVALID, "Modeled depth offset radius too large");
    }
    if (B.has_depth) {
      if (!ctx->h_dmodels[B.depth_model].set) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "depth model not set");
      const CameraDev& c = ctx->h_dcams[B.depth_camera];
      if (!c.set || !c.image) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "depth camera not set / no image uploaded");
    }
  }
  return M3TB_OK;
}

// Frame ingest for pinned host frames: fetch every body's ROI (k_ingest) before the first consumer of the new frame.
int LaunchIngestIfPending(m3tb_ctx* ctx) {
  if (ctx->prefetched) {  // the frames were prefetched on the side stream: order the consumers behind that ingest
    CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_ingest_done, 0));
    ctx->prefetched = false;
  }
  if (!ctx->ingest_pending) return M3TB_OK;
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
  a.n_bodies = ctx->n_bodies;
  CU(cudaMemsetAsync(a.bytes, 0, sizeof(unsigned long long), ctx->stream));
  k_ingest<<<ctx->n_bodies, kBlockThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  ctx->ingest_pending = false;
  return M3TB_OK;
}

int SyncStructures(m3tb_ctx* ctx);

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
// full (k_bin) and fills the tensor maps of `a`.
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
    // frames that arrived by full copy: (re)build their bin-index images
    if (ctx->bin_bitshift != bitshift) {
      for (int i = 0; i < ctx->max_cameras; ++i)
        if (!ctx->h_ccams[i].host_src) ctx->bin_stale[i] = 1;
      ctx->bin_bitshift = bitshift;
    }
    std::vector<int> ids;
    for (int i = 0; i < ctx->max_cameras; ++i) {
      const CameraDev& c = ctx->h_ccams[i];
      if (c.set && c.image && c.bins && !c.host_src && ctx->bin_stale[i]) ids.push_back(i);
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
      for (int i : ids) ctx->bin_stale[i] = 0;
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

// cluster > 0: one thread-block cluster of `cluster` CTAs per kinematic structure (PH_CLUSTER_SOLVE)
int LaunchTrack(m3tb_ctx* ctx, int iteration, int corr_begin, int corr_end, int n_update, int opt_base,
                unsigned phases, int cluster = 0) {
  int rc = ValidateBodies(ctx);
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
    CU(cudaMemcpyAsync(ctx->d_poses_snap[ctx->snap_parity], ctx->d_poses, sizeof(float) * 12 * ctx->n_bodies,
                       cudaMemcpyDeviceToDevice, ctx->stream));
    CU(cudaEventRecord(ctx->ev_poses_snap, ctx->stream));
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
  a.iteration = iteration;
  a.corr_begin = corr_begin;
  a.corr_end = corr_end;
  a.n_update = n_update;
  a.opt_base = opt_base;
  a.phases = phases;
  a.phase_clock = ctx->d_phase_clock;
  a.roi = ctx->d_roi;
  a.structures = ctx->d_structures;
  a.links = ctx->d_links;
  a.constraints = ctx->d_constraints;
  a.theta_out = ctx->d_theta;
  a.struct_status = ctx->d_struct_status;
  a.struct_offset = 0u;
  // thread <-> line mapping: T threads per body, K lines and K points per thread (state in registers)
  const int items = std::max(ctx->line_cap, ctx->point_cap);
  bool lut_smem = true;  // normalised LUT staged in shared memory when every region body has <= 16 bins (32 KB)
  for (int b = 0; b < ctx->n_bodies; ++b)
    if (ctx->h_bodies[b].has_region && ctx->h_bodies[b].rp.n_bins > 16) lut_smem = false;
  // dynamic shared memory: [normalised LUT 32 KB (16 bins)] [colour bin-index tile] [depth tile]
  const size_t lut_bytes = lut_smem ? size_t(16 * 16 * 16) * sizeof(float2) : 0;
  // with cluster-fused structures the solver workspace sits at the end of the dynamic shared memory
  const size_t struct_bytes = cluster > 0 ? Align(ctx->struct_smem, 128) : 0;
  bool bins_fit_u16 = true;  // the colour tile holds 16-bit bin indices: 64 bins (18 bits) go without tiles
  for (int b = 0; b < ctx->n_bodies; ++b)
    if (ctx->h_bodies[b].has_region && ctx->h_bodies[b].rp.n_bins > 32) bins_fit_u16 = false;
  const bool tiles = ctx->use_tiles && cluster == 0 && bins_fit_u16;
  const size_t dyn = tiles ? size_t(kDynSmemBytes) : lut_bytes + struct_bytes;
  a.tile_bytes = tiles ? int(dyn - lut_bytes - struct_bytes) : 0;
  a.struct_offset = unsigned(dyn - struct_bytes);
  bool occ = false;  // measured occlusion handling anywhere: the kernel variant that carries the depth-window scans
  for (int b = 0; b < ctx->n_bodies; ++b) {
    const BodyDev& B = ctx->h_bodies[b];
    occ = occ || (B.has_region && B.rp.measure_occlusions) || (B.has_depth && B.dp.measure_occlusions);
    // the renderer-image checks live in the same kernel variants
    occ = occ || (B.has_region && (B.rp.model_occlusions || B.rp.use_region_checking)) ||
          (B.has_depth && (B.dp.model_occlusions || B.dp.use_silhouette_checking));
  }
  // ---- k_track2: rigid bodies, <= 512 items per modality, no measured occlusion handling, correspondence / fused phases,
  //      one function lookup for the whole batch (m3t_b200_track2.cuh) --------------------------------------------------
  {
    const unsigned k2_phases = PH_REGION_CORR | PH_DEPTH_CORR | PH_REGION_GH | PH_DEPTH_GH | PH_SOLVE | PH_STORE_REGION |
                               PH_STORE_DEPTH;
    bool ok = ctx->use_track2 && cluster == 0 && !occ && items <= kGroup && (phases & ~k2_phases) == 0 &&
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
      return M3TB_OK;
    }
  }
#define M3TB_LAUNCH1(T_, K_, L_, O_)                                                                                   \
  do {                                                                                                                 \
    CU(cudaFuncSetAttribute(k_track<T_, K_, L_, O_, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(dyn)));   \
    k_track<T_, K_, L_, O_, false><<<ctx->n_bodies, T_, dyn, ctx->stream>>>(a);                                        \
  } while (0)
#define M3TB_LAUNCH_CLUSTER(T_, K_, L_)                                                                                \
  do {                                                                                                                 \
    CU(cudaFuncSetAttribute(k_track<T_, K_, L_, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(dyn))); \
    cudaLaunchConfig_t cfg = {};                                                                                       \
    cfg.gridDim = dim3(unsigned(ctx->n_bodies));                                                                       \
    cfg.blockDim = dim3(T_);                                                                                           \
    cfg.dynamicSmemBytes = dyn;                                                                                        \
    cfg.stream = ctx->stream;                                                                                          \
    cudaLaunchAttribute attr;                                                                                          \
    attr.id = cudaLaunchAttributeClusterDimension;                                                                     \
    attr.val.clusterDim.x = unsigned(cluster);                                                                         \
    attr.val.clusterDim.y = 1;                                                                                         \
    attr.val.clusterDim.z = 1;                                                                                         \
    cfg.attrs = &attr;                                                                                                 \
    cfg.numAttrs = 1;                                                                                                  \
    if (ctx->d_phase_clock) {                                                                                          \
      int n_clusters = -1;                                                                                             \
      cudaOccupancyMaxActiveClusters(&n_clusters, k_track<T_, K_, L_, false, true>, &cfg);                             \
      std::fprintf(stderr, "m3tb: cluster launch %d x %d CTAs, dyn smem %zu, max active clusters %d\n",                \
                   ctx->n_bodies / cluster, cluster, size_t(dyn), n_clusters);                                         \
    }                                                                                                                  \
    CU(cudaLaunchKernelEx(&cfg, k_track<T_, K_, L_, false, true>, a));                                                 \
  } while (0)
#define M3TB_LAUNCH(T_, K_)                                       \
  do {                                                            \
    if (lut_smem && !occ) M3TB_LAUNCH1(T_, K_, true, false);      \
    else if (lut_smem) M3TB_LAUNCH1(T_, K_, true, true);          \
    else if (!occ) M3TB_LAUNCH1(T_, K_, false, false);            \
    else M3TB_LAUNCH1(T_, K_, false, true);                       \
  } while (0)
  if (cluster > 0) {
    // cluster-fused structures: 256-thread CTAs without ROI tiles, so that two CTAs share an SM and every cluster of
    // a 32-chain shard is resident at once (with 220 KB tiles at most 16 clusters of 8 fit on the 132 SMs)
    if (items <= 256) { if (lut_smem) M3TB_LAUNCH_CLUSTER(256, 1, true); else M3TB_LAUNCH_CLUSTER(256, 1, false); }
    else if (items <= 512) { if (lut_smem) M3TB_LAUNCH_CLUSTER(256, 2, true); else M3TB_LAUNCH_CLUSTER(256, 2, false); }
    else return Fail(ctx, M3TB_ERR_UNSUPPORTED, "cluster-fused structures: n_lines_max / n_points_max above 512");
  } else if (items <= 256) M3TB_LAUNCH(256, 1);
  else if (items <= 512) M3TB_LAUNCH(512, 1);
  else if (items <= 1024) M3TB_LAUNCH(512, 2);
  else if (items <= 2048) M3TB_LAUNCH(512, 4);
  else return Fail(ctx, M3TB_ERR_UNSUPPORTED, "n_lines_max / n_points_max above 2048");
#undef M3TB_LAUNCH
#undef M3TB_LAUNCH1
#undef M3TB_LAUNCH_CLUSTER
  CU(cudaGetLastError());
  ctx->launches++;
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
  ctx->struct_first_link.clear();
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
    ctx->struct_first_link.push_back(d.first_link);
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
  if (ns > ctx->cap_structures) {
    cudaFree(ctx->d_structures); cudaFree(ctx->d_theta); cudaFree(ctx->d_struct_status);
    CU(cudaMalloc(&ctx->d_structures, sizeof(StructureDev) * ns));
    CU(cudaMalloc(&ctx->d_theta, sizeof(float) * kMaxSystem * ns));
    CU(cudaMalloc(&ctx->d_struct_status, sizeof(int) * ns));
    ctx->cap_structures = ns;
  }
  if (nl > ctx->cap_links) {
    cudaFree(ctx->d_links); cudaFree(ctx->d_links_default);
    CU(cudaMalloc(&ctx->d_links, sizeof(LinkDev) * nl));
    CU(cudaMalloc(&ctx->d_links_default, sizeof(LinkDev) * nl));
    ctx->cap_links = nl;
  }
  if (nc > ctx->cap_constraints) {
    cudaFree(ctx->d_constraints);
    CU(cudaMalloc(&ctx->d_constraints, sizeof(ConstraintDev) * nc));
    ctx->cap_constraints = nc;
  }
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
  a.gh_link = from_modalities ? nullptr : ctx->d_gh_link;
  a.gh_region = ctx->d_gh_region;
  a.gh_depth = ctx->d_gh_depth;
  a.mode = mode;
  a.theta_out = ctx->d_theta;
  a.status = ctx->d_struct_status;
  if (ctx->struct_smem > 48 * 1024)
    CU(cudaFuncSetAttribute(k_structure, cudaFuncAttributeMaxDynamicSharedMemorySize, int(ctx->struct_smem)));
  k_structure<<<ctx->n_struct_launch, kStructThreads, ctx->struct_smem, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  return M3TB_OK;
}

// Can every structure run as one thread-block cluster inside k_track? All structures have the same number of links
// (2..8, the portable cluster size), every link carries a body, and structure s, link l is body s * n_links + l, so
// that CTA rank = link index. Anything else takes the general multi-launch path below.
int ClusterLinks(m3tb_ctx* ctx) {
  if (!ctx->use_clusters || ctx->n_struct_launch == 0) return 0;
  const int nl = ctx->h_structures[0].n_links;
  if (nl < 2 || nl > 8 || ctx->n_struct_launch * nl != ctx->n_bodies) return 0;
  for (int si = 0; si < ctx->n_struct_launch; ++si) {
    const StructureDev& d = ctx->h_structures[si];
    if (d.n_links != nl) return 0;
    for (int l = 0; l < nl; ++l)
      if (ctx->h_link_bodies[d.first_link + l] != si * nl + l) return 0;
    if (si < int(ctx->structures.size()))
      for (const auto& lk : ctx->structures[si].links)
        if (lk.n_extra > 0) return 0;
  }
  for (int b = 0; b < ctx->n_bodies; ++b) {
    const BodyDev& B = ctx->h_bodies[b];
    if ((B.has_region && B.rp.measure_occlusions) || (B.has_depth && B.dp.measure_occlusions)) return 0;
    if ((B.has_region && B.rp.n_lines_max > 512) || (B.has_depth && B.dp.n_points_max > 512)) return 0;
  }
  return nl;
}

// Tracker::ExecuteTrackingStep's loop nest (tracker.cpp:344-361) when the optimisers are kinematic structures: the
// per-body work stays in k_track (correspondences, gradient / Hessian -> gh_link), every
// Optimizer::CalculateOptimization is one k_structure launch over all structures.
int StructureStep(m3tb_ctx* ctx, int iteration, int corr_begin, int corr_end, int n_update) {
  int rc0 = SyncStructures(ctx);
  if (rc0) return rc0;
  if (const int nl = ClusterLinks(ctx)) {
    // fused: the whole corr x update loop nest in ONE launch, one cluster per structure, CalculateOptimization over
    // distributed shared memory
    if (n_update > 0)
      return LaunchTrack(ctx, iteration, corr_begin, corr_end, n_update, 0,
                         PH_REGION_CORR | PH_DEPTH_CORR | PH_REGION_GH | PH_DEPTH_GH | PH_CLUSTER_SOLVE | PH_STORE_REGION |
                             PH_STORE_DEPTH,
                         nl);
  }
  for (int corr = corr_begin; corr < corr_end; ++corr) {
    if (n_update == 0) {
      int rc = LaunchTrack(ctx, iteration, corr, corr + 1, 0, 0, PH_REGION_CORR | PH_DEPTH_CORR | PH_STORE_REGION | PH_STORE_DEPTH);
      if (rc) return rc;
      continue;
    }
    int rc = LaunchTrack(ctx, iteration, corr, corr + 1, 1, 0,
                         PH_REGION_CORR | PH_DEPTH_CORR | PH_REGION_GH | PH_DEPTH_GH | PH_STORE_LINK_GH | PH_STORE_REGION |
                             PH_STORE_DEPTH);
    if (rc) return rc;
    rc = LaunchStructure(ctx, 0, false);
    if (rc) return rc;
    for (int upd = 1; upd < n_update; ++upd) {
      rc = LaunchTrack(ctx, iteration, corr, corr + 1, 1, upd,
                       PH_LOAD_REGION | PH_LOAD_DEPTH | PH_REGION_GH | PH_DEPTH_GH | PH_STORE_LINK_GH);
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
    if (!ctx->d_hist_owner) CU(cudaMalloc(&ctx->d_hist_owner, sizeof(int) * ctx->max_bodies));
    if (int(table.size()) > ctx->hist_groups_capacity) {
      CU(cudaStreamSynchronize(ctx->stream));
      cudaFree(ctx->d_hist_groups);
      ctx->d_hist_groups = nullptr;
      CU(cudaMalloc(&ctx->d_hist_groups, sizeof(int) * table.size()));
      ctx->hist_groups_capacity = int(table.size());
    }
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
  k_histogram<<<ctx->n_bodies, kBlockThreads, 0, ctx->stream>>>(a);
  CU(cudaGetLastError());
  ctx->launches++;
  if (any_shared) {
    SharedHistArgs s;
    s.bodies = ctx->d_bodies;
    s.hist_f = ctx->d_hist_f; s.hist_b = ctx->d_hist_b; s.mem_f = ctx->d_mem_f; s.mem_b = ctx->d_mem_b; s.lut = ctx->d_lut;
    s.stride = ctx->hist_stride;
    s.mode = mode;
    s.group_owner = ctx->d_hist_groups;
    s.group_first = ctx->d_hist_groups + ctx->n_hist_groups;
    s.members = ctx->d_hist_groups + 2 * ctx->n_hist_groups + 1;
    k_histogram_shared<<<ctx->n_hist_groups, kBlockThreads, 0, ctx->stream>>>(s);
    CU(cudaGetLastError());
    ctx->launches++;
  }
  return M3TB_OK;
}

int SetModel(m3tb_ctx* ctx, bool region, int model_id, int n_views, int n_points, const float* orientations,
             const float* scalars, const void* points, float stride_depth_offset, float max_radius_depth_offset) {
  if (model_id < 0 || model_id >= ctx->max_models || n_views <= 0 || n_points <= 0 || !orientations || !points)
    return Fail(ctx, M3TB_ERR_INVALID, "bad model arguments");
  std::vector<ModelAlloc>& allocs = region ? ctx->rmodel_alloc : ctx->dmodel_alloc;
  ModelAlloc& al = allocs[model_id];
  if (al.orientations) {
    cudaFree(al.orientations); cudaFree(al.view_scalars); cudaFree(al.points); cudaFree(al.depth_offsets);
    cudaFree(al.cluster_info); cudaFree(al.sorted_views);
    al = ModelAlloc();
  }
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
  CU(cudaMalloc(&al.orientations, sizeof(float4) * n_views));
  CU(cudaMalloc(&al.view_scalars, sizeof(float) * n_views));
  CU(cudaMalloc(&al.points, sizeof(float) * packed.size()));
  CU(cudaMalloc(&al.depth_offsets, sizeof(float) * offsets.size()));
  CU(cudaMemcpyAsync(al.depth_offsets, offsets.data(), sizeof(float) * offsets.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(al.orientations, ori4.data(), sizeof(float4) * n_views, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(al.view_scalars, sc.data(), sizeof(float) * n_views, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(al.points, packed.data(), sizeof(float) * packed.size(), cudaMemcpyHostToDevice, ctx->stream));
  // cluster tables of the pruned closest-view search (one-time, host)
  ViewClustersHost vc;
  BuildViewClusters(orientations, n_views, vc);
  CU(cudaMalloc(&al.cluster_info, sizeof(float) * std::max<size_t>(vc.info.size(), 8)));
  CU(cudaMalloc(&al.sorted_views, sizeof(float) * vc.sorted.size()));
  CU(cudaMemcpyAsync(al.cluster_info, vc.info.data(), sizeof(float) * vc.info.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(al.sorted_views, vc.sorted.data(), sizeof(float) * vc.sorted.size(), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));  // staging vectors go out of scope
  ModelDev& m = (region ? ctx->h_rmodels : ctx->h_dmodels)[model_id];
  m.n_views = n_views;
  m.n_points = n_points;
  m.orientations4 = al.orientations;
  m.view_scalars = al.view_scalars;
  m.points = al.points;
  m.max_view_scalar = max_scalar;
  m.radius = std::sqrt(radius2);
  m.depth_offsets = al.depth_offsets;
  m.stride_depth_offset = stride_depth_offset;
  m.max_radius_depth_offset = max_radius_depth_offset;
  m.cluster_info = al.cluster_info;
  m.sorted_views = al.sorted_views;
  m.n_clusters = vc.n_clusters;
  m.set = 1;
  ctx->models_dirty = true;
  return M3TB_OK;
}

int SetCamera(m3tb_ctx* ctx, bool color, int cam, const m3tb_intrinsics* in, const float* w2c, float depth_scale) {
  if (cam < 0 || cam >= ctx->max_cameras || !in || !w2c || in->width <= 0 || in->height <= 0)
    return Fail(ctx, M3TB_ERR_INVALID, "bad camera arguments");
  CameraDev& c = (color ? ctx->h_ccams : ctx->h_dcams)[cam];
  const bool dims_changed = c.set && (c.width != in->width || c.height != in->height);
  c.fu = in->fu; c.fv = in->fv; c.ppu = in->ppu; c.ppv = in->ppv;
  c.width = in->width; c.height = in->height;
  std::memcpy(c.w2c, w2c, sizeof(float) * 12);
  c.depth_scale = depth_scale;
  if (dims_changed) c.image = nullptr;
  c.set = 1;
  ctx->cams_dirty = true;
  return M3TB_OK;
}

// Device storage of camera `cam`'s frame: a slot of the shared pool when the dimensions match the
// pool's (so that a batch of frames is one contiguous copy), a private allocation otherwise.
int EnsureImage(m3tb_ctx* ctx, bool color, int cam) {
  CameraDev& c = (color ? ctx->h_ccams : ctx->h_dcams)[cam];
  if (!c.set) return Fail(ctx, M3TB_ERR_NOT_SET_UP, "set the camera before uploading images");
  if (c.image) return M3TB_OK;
  ImagePool& pool = color ? ctx->color_pool : ctx->depth_pool;
  const unsigned pitch = unsigned(Align(size_t(c.width) * (color ? 3 : 2), 16));
  if (!pool.base) {
    pool.width = c.width; pool.height = c.height; pool.pitch = pitch;
    pool.frame_bytes = size_t(pitch) * c.height;
    pool.capacity = ctx->max_cameras;
    CU(cudaMalloc(&pool.base, pool.frame_bytes * pool.capacity));
    if (color && (c.width & 3) == 0) {
      pool.bin_pitch = unsigned(Align(size_t(c.width) * 2, 16));
      pool.bin_frame_bytes = size_t(pool.bin_pitch) * c.height;
      CU(cudaMalloc(&pool.bins, pool.bin_frame_bytes * pool.capacity));
    }
  }
  if (pool.width == c.width && pool.height == c.height) {
    c.image = pool.base + pool.frame_bytes * cam;
    c.pitch = pool.pitch;
    if (color && pool.bins) {
      c.bins = reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(pool.bins) + pool.bin_frame_bytes * cam);
      c.bin_pitch = pool.bin_pitch;
    }
  } else {
    c.bins = nullptr;
    c.bin_pitch = 0;
    uint8_t*& priv = (color ? ctx->private_color : ctx->private_depth)[cam];
    if (priv) cudaFree(priv);
    CU(cudaMalloc(&priv, size_t(pitch) * c.height));
    c.image = priv;
    c.pitch = pitch;
  }
  ctx->cams_dirty = true;
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
int Upload(m3tb_ctx* ctx, bool color, int cam, const void* src, size_t pitch, cudaMemcpyKind kind,
           const uint8_t* pinned_alias) {
  if (cam < 0 || cam >= ctx->max_cameras || !src) return Fail(ctx, M3TB_ERR_INVALID, "bad upload arguments");
  int rc = EnsureImage(ctx, color, cam);
  if (rc) return rc;
  CameraDev& c = (color ? ctx->h_ccams : ctx->h_dcams)[cam];
  const size_t row = size_t(c.width) * (color ? 3 : 2);
  if (pitch < row) return Fail(ctx, M3TB_ERR_INVALID, "pitch smaller than a row");
  c.generation = (c.generation + 1) & 0x3fffffff;
  ctx->cams_dirty = true;
  if (pinned_alias) {
    c.host_src = pinned_alias;
    c.host_pitch = unsigned(pitch);
    ctx->ingest_pending = true;
    if (color) ctx->bin_stale[cam] = 0;  // k_ingest writes the bin indices of every rectangle it fetches
    return M3TB_OK;
  }
  c.host_src = nullptr;
  c.host_pitch = 0;
  if (color) ctx->bin_stale[cam] = 1;
  CU(cudaMemcpy2DAsync(const_cast<uint8_t*>(c.image), c.pitch, src, pitch, row, c.height, kind, ctx->stream));
  return M3TB_OK;
}

int UploadBatch(m3tb_ctx* ctx, bool color, int first, int count, const void* src, size_t frame_stride, size_t pitch) {
  if (first < 0 || count <= 0 || first + count > ctx->max_cameras || !src)
    return Fail(ctx, M3TB_ERR_INVALID, "bad batch upload arguments");
  ImagePool& pool = color ? ctx->color_pool : ctx->depth_pool;
  bool pooled = true;
  for (int k = 0; k < count; ++k) {
    int rc = EnsureImage(ctx, color, first + k);
    if (rc) return rc;
    const CameraDev& c = (color ? ctx->h_ccams : ctx->h_dcams)[first + k];
    pooled = pooled && pool.base && c.image == pool.base + pool.frame_bytes * (first + k);
  }
  const uint8_t* s = static_cast<const uint8_t*>(src);
  if (const uint8_t* alias = PinnedAlias(ctx, src)) {
    for (int k = 0; k < count; ++k) {
      int rc = Upload(ctx, color, first + k, s + frame_stride * k, pitch, cudaMemcpyHostToDevice, alias + frame_stride * k);
      if (rc) return rc;
    }
    return M3TB_OK;
  }
  for (int k = 0; k < count; ++k) {
    CameraDev& c = (color ? ctx->h_ccams : ctx->h_dcams)[first + k];
    c.host_src = nullptr; c.host_pitch = 0; c.generation = (c.generation + 1) & 0x3fffffff;
    if (color) ctx->bin_stale[first + k] = 1;
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

int m3tb_create(int device, int max_bodies, int max_cameras, int max_models, m3tb_ctx** out) {
  if (!out || max_bodies <= 0 || max_cameras <= 0 || max_models <= 0) return M3TB_ERR_INVALID;
  *out = nullptr;
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || device < 0 || device >= n_dev) return M3TB_ERR_CUDA;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return M3TB_ERR_CUDA;
  if (prop.major != 9 || prop.minor != 0) return M3TB_ERR_CUDA;  // sm_90a cubin only: no other architecture can run it
  m3tb_ctx* ctx = new m3tb_ctx();
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
  ctx->rmodel_alloc.assign(max_models, ModelAlloc());
  ctx->dmodel_alloc.assign(max_models, ModelAlloc());
  ctx->private_color.assign(max_cameras, nullptr);
  ctx->private_depth.assign(max_cameras, nullptr);
  ctx->bin_stale.assign(max_cameras, 1);
  if (const char* e = std::getenv("M3TB_NO_TILES")) ctx->use_tiles = !(e[0] == '1');
  if (const char* e = std::getenv("M3TB_NO_ROI_INGEST")) ctx->roi_ingest = !(e[0] == '1');
  if (const char* e = std::getenv("M3TB_CLUSTER")) ctx->use_clusters = e[0] == '1';
  if (const char* e = std::getenv("M3TB_KERNEL")) ctx->use_track2 = !(e[0] == '1');
  if (const char* e = std::getenv("M3TB_TMA")) ctx->tma_mode = (e[0] >= '0' && e[0] <= '2') ? e[0] - '0' : 1;
  const char* timing_env = std::getenv("M3TB_TIMING");
  const bool want_timing = timing_env && timing_env[0] == '1';
  auto alloc = [&]() -> int {
    CU(cudaSetDevice(device));
    CU(cudaMalloc(&ctx->d_bodies, sizeof(BodyDev) * max_bodies));
    CU(cudaMalloc(&ctx->d_ccams, sizeof(CameraDev) * max_cameras));
    CU(cudaMalloc(&ctx->d_dcams, sizeof(CameraDev) * max_cameras));
    CU(cudaMalloc(&ctx->d_rmodels, sizeof(ModelDev) * max_models));
    CU(cudaMalloc(&ctx->d_dmodels, sizeof(ModelDev) * max_models));
    CU(cudaMalloc(&ctx->d_poses, sizeof(float) * 12 * max_bodies));
    CU(cudaMalloc(&ctx->d_counts, sizeof(int) * 4 * max_bodies));
    CU(cudaMalloc(&ctx->d_gh_region, sizeof(float) * 27 * max_bodies));
    CU(cudaMalloc(&ctx->d_gh_depth, sizeof(float) * 27 * max_bodies));
    CU(cudaMemset(ctx->d_poses, 0, sizeof(float) * 12 * max_bodies));
    CU(cudaMemset(ctx->d_counts, 0, sizeof(int) * 4 * max_bodies));
    CU(cudaMemset(ctx->d_gh_region, 0, sizeof(float) * 27 * max_bodies));
    CU(cudaMemset(ctx->d_gh_depth, 0, sizeof(float) * 27 * max_bodies));
    CU(cudaMalloc(&ctx->d_gh_link, sizeof(float) * 27 * max_bodies));
    CU(cudaMemset(ctx->d_gh_link, 0, sizeof(float) * 27 * max_bodies));
    CU(cudaMalloc(&ctx->d_roi, sizeof(RoiRecord) * 2 * max_bodies));
    CU(cudaMemset(ctx->d_roi, 0xff, sizeof(RoiRecord) * 2 * max_bodies));  // generation -1: nothing ingested yet
    CU(cudaMalloc(&ctx->d_bin_ids, sizeof(int) * max_cameras));
    CU(cudaMalloc(&ctx->d_tmaps, sizeof(CUtensorMap) * 2 * kTileWidths));
    CU(cudaMalloc(&ctx->d_ingest_bytes, 2 * sizeof(unsigned long long)));
    CU(cudaMemset(ctx->d_ingest_bytes, 0, 2 * sizeof(unsigned long long)));
    if (want_timing) {
      CU(cudaMalloc(&ctx->d_phase_clock, sizeof(long long) * kPhaseSlots * max_bodies));
      CU(cudaMemset(ctx->d_phase_clock, 0, sizeof(long long) * kPhaseSlots * max_bodies));
    }
    return M3TB_OK;
  };
  int rc = alloc();
  if (rc != M3TB_OK) {
    std::fprintf(stderr, "m3tb_create: %s\n", ctx->err.c_str());
    m3tb_destroy(ctx);
    return rc;
  }
  *out = ctx;
  return M3TB_OK;
}

int m3tb_destroy(m3tb_ctx* ctx) {
  if (!ctx) return M3TB_ERR_INVALID;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  for (auto* al : {&ctx->rmodel_alloc, &ctx->dmodel_alloc})
    for (auto& a : *al) {
      cudaFree(a.orientations); cudaFree(a.view_scalars); cudaFree(a.points); cudaFree(a.depth_offsets);
      cudaFree(a.cluster_info); cudaFree(a.sorted_views);
    }
  for (auto p : ctx->rendering_allocs) cudaFree(p);
  for (auto p : ctx->private_color) cudaFree(p);
  for (auto p : ctx->private_depth) cudaFree(p);
  cudaFree(ctx->color_pool.base); cudaFree(ctx->depth_pool.base);
  cudaFree(ctx->color_pool.bins); cudaFree(ctx->color_pool_alt.bins); cudaFree(ctx->d_bin_ids); cudaFree(ctx->d_tmaps);
  cudaFree(ctx->d_bodies); cudaFree(ctx->d_ccams); cudaFree(ctx->d_dcams); cudaFree(ctx->d_rmodels);
  cudaFree(ctx->d_dmodels); cudaFree(ctx->d_poses); cudaFree(ctx->d_counts); cudaFree(ctx->d_gh_region);
  cudaFree(ctx->d_gh_depth); cudaFree(ctx->d_hist_f); cudaFree(ctx->d_hist_b); cudaFree(ctx->d_mem_f);
  cudaFree(ctx->d_mem_b); cudaFree(ctx->d_lut); cudaFree(ctx->d_rstate); cudaFree(ctx->d_dstate);
  cudaFree(ctx->d_phase_clock); cudaFree(ctx->d_roi); cudaFree(ctx->d_ingest_bytes);
  cudaFree(ctx->color_pool_alt.base); cudaFree(ctx->depth_pool_alt.base); cudaFree(ctx->d_ccams_alt);
  cudaFree(ctx->d_dcams_alt); cudaFree(ctx->d_roi_alt); cudaFree(ctx->d_poses_snap[0]); cudaFree(ctx->d_poses_snap[1]);
  if (ctx->table_stream) { cudaStreamSynchronize(ctx->table_stream); cudaStreamDestroy(ctx->table_stream); }
  if (ctx->ingest_stream) { cudaStreamSynchronize(ctx->ingest_stream); cudaStreamDestroy(ctx->ingest_stream); }
  for (int q = 0; q < 4; ++q) cudaFreeHost(ctx->h_cam_stage[q >> 1][q & 1]);
  if (ctx->ev_ingest_done) cudaEventDestroy(ctx->ev_ingest_done);
  if (ctx->ev_poses_snap) cudaEventDestroy(ctx->ev_poses_snap);
  if (ctx->ev_tables) cudaEventDestroy(ctx->ev_tables);
  for (int q = 0; q < 2; ++q) if (ctx->ev_stage[q]) cudaEventDestroy(ctx->ev_stage[q]);
  cudaFree(ctx->d_structures); cudaFree(ctx->d_links); cudaFree(ctx->d_links_default); cudaFree(ctx->d_constraints);
  cudaFree(ctx->d_gh_link);
  cudaFree(ctx->d_theta); cudaFree(ctx->d_struct_status); cudaFree(ctx->d_hist_owner); cudaFree(ctx->d_hist_groups);
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
  if (ctx->ingest_stream) CU(cudaStreamSynchronize(ctx->ingest_stream));
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
  return SetModel(ctx, true, model_id, n_views, n_points, orientations, contour_lengths, points, stride_depth_offset,
                  max_radius_depth_offset);
}

int m3tb_set_depth_model(m3tb_ctx* ctx, int model_id, int n_views, int n_points, const float* orientations,
                         const float* surface_areas, const void* points, float stride_depth_offset,
                         float max_radius_depth_offset) {
  CHECK_CTX();
  return SetModel(ctx, false, model_id, n_views, n_points, orientations, surface_areas, points, stride_depth_offset,
                  max_radius_depth_offset);
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
  BodyDev B;
  std::memset(&B, 0, sizeof(B));
  B.first_iteration = ctx->h_bodies[body].first_iteration;
  std::memcpy(B.rend, ctx->h_bodies[body].rend, sizeof(B.rend));  // uploaded renderer images stay with the body
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
    if (depth->n_considered_distances < 1 || depth->n_considered_distances > M3TB_MAX_SCHEDULE ||
        depth->n_standard_deviations < 1 || depth->n_standard_deviations > M3TB_MAX_SCHEDULE ||
        depth->n_points_max < 1 || !(depth->stride_length > 0.0f))
      return Fail(ctx, M3TB_ERR_INVALID, "bad depth schedule / n_points_max / stride_length");
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
  return LaunchTrack(ctx, iteration, 0, n_corr_iterations, n_update_iterations, 0,
                     PH_REGION_CORR | PH_DEPTH_CORR | PH_REGION_GH | PH_DEPTH_GH | PH_SOLVE | PH_STORE_REGION |
                         PH_STORE_DEPTH);
}

int m3tb_corr_iteration(m3tb_ctx* ctx, int iteration, int corr_iteration, int n_update_iterations) {
  CHECK_CTX();
  if (corr_iteration < 0 || n_update_iterations < 0) return Fail(ctx, M3TB_ERR_INVALID, "negative iteration count");
  if (HasStructures(ctx)) return StructureStep(ctx, iteration, corr_iteration, corr_iteration + 1, n_update_iterations);
  return LaunchTrack(ctx, iteration, corr_iteration, corr_iteration + 1, n_update_iterations, 0,
                     PH_REGION_CORR | PH_DEPTH_CORR | PH_REGION_GH | PH_DEPTH_GH | PH_SOLVE | PH_STORE_REGION |
                         PH_STORE_DEPTH);
}

int m3tb_start_modalities(m3tb_ctx* ctx, int iteration) {
  CHECK_CTX();
  for (int b = 0; b < ctx->n_bodies; ++b) ctx->h_bodies[b].first_iteration = iteration;
  ctx->bodies_dirty = true;
  return LaunchHistogram(ctx, 0, iteration);
}

int m3tb_calculate_results(m3tb_ctx* ctx, int iteration) {
  CHECK_CTX();
  return LaunchHistogram(ctx, 1, iteration);
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
  if ((modality != 0 && modality != 1) || !gradients || !hessians || ctx->n_bodies == 0)
    return Fail(ctx, M3TB_ERR_INVALID, "bad gradient / hessian arguments");
  std::vector<float> h(size_t(27) * ctx->n_bodies);
  for (int b = 0; b < ctx->n_bodies; ++b) {
    for (int i = 0; i < 6; ++i) h[27 * b + i] = gradients[6 * b + i];
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j <= i; ++j) h[27 * b + 6 + Tri(i, j)] = hessians[36 * b + 6 * i + j];
  }
  CU(cudaMemcpyAsync(modality == 0 ? ctx->d_gh_region : ctx->d_gh_depth, h.data(), h.size() * sizeof(float),
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
      const CameraDev& c = (color ? ctx->h_ccams : ctx->h_dcams)[i];
      if (!c.set || !c.image) continue;
      if (!c.host_src || !pool.base || c.image != pool.base + pool.frame_bytes * i) return M3TB_OK;
    }
  }
  if (!ctx->ingest_stream) {
    CU(cudaStreamCreateWithFlags(&ctx->ingest_stream, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&ctx->table_stream, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&ctx->ev_ingest_done, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&ctx->ev_poses_snap, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&ctx->ev_tables, cudaEventDisableTiming));
    for (int q = 0; q < 2; ++q) CU(cudaEventCreateWithFlags(&ctx->ev_stage[q], cudaEventDisableTiming));
    for (int q = 0; q < 4; ++q) CU(cudaMallocHost(&ctx->h_cam_stage[q >> 1][q & 1], sizeof(CameraDev) * ctx->max_cameras));
    CU(cudaMalloc(&ctx->d_ccams_alt, sizeof(CameraDev) * ctx->max_cameras));
    CU(cudaMalloc(&ctx->d_dcams_alt, sizeof(CameraDev) * ctx->max_cameras));
    CU(cudaMalloc(&ctx->d_roi_alt, sizeof(RoiRecord) * 2 * ctx->max_bodies));
    CU(cudaMemset(ctx->d_roi_alt, 0xff, sizeof(RoiRecord) * 2 * ctx->max_bodies));
    for (int q = 0; q < 2; ++q) CU(cudaMalloc(&ctx->d_poses_snap[q], sizeof(float) * 12 * ctx->max_bodies));
  }
  for (int k = 0; k < 2; ++k) {
    ImagePool& pool = k == 0 ? ctx->color_pool : ctx->depth_pool;
    ImagePool& alt = k == 0 ? ctx->color_pool_alt : ctx->depth_pool_alt;
    if (pool.base && !alt.base) {
      alt = pool;
      alt.base = nullptr;
      alt.bins = nullptr;
      CU(cudaMalloc(&alt.base, alt.frame_bytes * alt.capacity));
      if (pool.bins) CU(cudaMalloc(&alt.bins, alt.bin_frame_bytes * alt.capacity));
    }
    std::swap(pool, alt);
    std::vector<CameraDev>& cams = k == 0 ? ctx->h_ccams : ctx->h_dcams;
    for (int i = 0; i < ctx->max_cameras; ++i)
      if (cams[i].set && cams[i].image) {
        cams[i].image = pool.base + pool.frame_bytes * i;
        if (k == 0 && pool.bins)
          cams[i].bins = reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(pool.bins) + pool.bin_frame_bytes * i);
      }
  }
  ctx->cams_dirty = false;   // the camera tables go to the alternate device copies below, on the side stream
  int rc = SyncTables(ctx);  // bodies / models only (main stream, small)
  if (rc) return rc;
  std::swap(ctx->d_ccams, ctx->d_ccams_alt);
  std::swap(ctx->d_dcams, ctx->d_dcams_alt);
  std::swap(ctx->d_roi, ctx->d_roi_alt);
  // Stream plan. The ingest stream runs the ingests back to back: anything queued on it in front of k_ingest would sit
  // between two PCIe-bound kernels (two pageable table copies, a memset and the wait for the pose snapshot would
  // lengthen every end-to-end step). So the set-up goes to a third stream, beside the ingest in flight: wait for the pose
  // snapshot of the last tracking launch (which also orders it behind every reader of the buffers swapped in above: they
  // precede that launch on the main stream), camera tables from pinned staging, counter reset; the ingest stream then
  // waits for one event that is normally long past.
  cudaStream_t is = ctx->ingest_stream, ts = ctx->table_stream;
  const float* poses = ctx->d_poses;
  if (ctx->poses_snap_valid) {
    CU(cudaStreamWaitEvent(ts, ctx->ev_poses_snap, 0));
    poses = ctx->d_poses_snap[ctx->snap_parity];
  } else {
    CU(cudaStreamSynchronize(ctx->stream));  // first frame: nothing in flight that could be writing the poses
  }
  ctx->stage_parity ^= 1;  // the staging of the prefetch before this one may still be in flight; the one before that
  CU(cudaEventSynchronize(ctx->ev_stage[ctx->stage_parity]));  // normally is not (a host that never waits could be ahead)
  CameraDev* stage_c = ctx->h_cam_stage[ctx->stage_parity][0];
  CameraDev* stage_d = ctx->h_cam_stage[ctx->stage_parity][1];
  std::memcpy(stage_c, ctx->h_ccams.data(), sizeof(CameraDev) * ctx->max_cameras);
  std::memcpy(stage_d, ctx->h_dcams.data(), sizeof(CameraDev) * ctx->max_cameras);
  CU(cudaMemcpyAsync(ctx->d_ccams, stage_c, sizeof(CameraDev) * ctx->max_cameras, cudaMemcpyHostToDevice, ts));
  CU(cudaMemcpyAsync(ctx->d_dcams, stage_d, sizeof(CameraDev) * ctx->max_cameras, cudaMemcpyHostToDevice, ts));
  CU(cudaEventRecord(ctx->ev_stage[ctx->stage_parity], ts));
  ctx->cams_dirty = false;
  ctx->ingest_bytes_slot ^= 1;
  CU(cudaMemsetAsync(ctx->d_ingest_bytes + ctx->ingest_bytes_slot, 0, sizeof(unsigned long long), ts));
  CU(cudaEventRecord(ctx->ev_tables, ts));
  CU(cudaStreamWaitEvent(is, ctx->ev_tables, 0));
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
  // Grid of the prefetch ingest: a quarter of the SMs, CTAs looping over the bodies. k_track2 takes a whole SM per body
  // (1024 threads x 64 registers), so an ingest CTA that sits on an SM keeps a body waiting for as long as the ingest
  // lasts, and whichever kernel is dispatched first wins: with one CTA per body the end-to-end step time swings widely
  // once both kernels become ready at the same moment. One CTA keeps 16 KB in flight; a few dozen keep the link busy
  // (scripts/probes/pcie_probe.cu measures it). M3TB_INGEST_CTAS overrides the grid.
  static const int forced_ctas = [] { const char* e = std::getenv("M3TB_INGEST_CTAS"); return e ? std::atoi(e) : 0; }();
  int ingest_ctas = std::max(16, ctx->sm_count / 4);
  if (forced_ctas > 0) ingest_ctas = forced_ctas;
  ingest_ctas = std::min(ingest_ctas, ctx->n_bodies);
  k_ingest<<<ingest_ctas, kBlockThreads, 0, is>>>(a);
  CU(cudaGetLastError());
  CU(cudaEventRecord(ctx->ev_ingest_done, is));
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
  RenderingDev& d = ctx->h_bodies[body].rend[slot];
  const unsigned pitch = unsigned(Align(size_t(r->image_size) * bytes_per_pixel, 16));
  if (!d.image || d.image_size != r->image_size) {
    if (d.image) {
      CU(cudaStreamSynchronize(ctx->stream));
      uint8_t* old = const_cast<uint8_t*>(d.image);
      for (auto& q : ctx->rendering_allocs)
        if (q == old) q = nullptr;
      cudaFree(old);
      d.image = nullptr;
    }
    uint8_t* p = nullptr;
    CU(cudaMalloc(&p, size_t(pitch) * r->image_size));
    ctx->rendering_allocs.push_back(p);
    d.image = p;
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

int m3tb_detach_frames(m3tb_ctx* ctx) {
  CHECK_CTX();
  if (ctx->ingest_stream) CU(cudaStreamSynchronize(ctx->ingest_stream));  // a prefetch may still be reading the frames
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
      if (k == 0) ctx->bin_stale[size_t(&c - cams.data())] = 1;
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

}  // extern "C"
