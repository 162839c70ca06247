// m3t_b200_texture.cu — k_texture_keyframe, k_texture_knn_l2 / _hamming and k_texture_match (TextureModality,
// texture_modality.cpp). k_texture_keyframe / k_texture_match: one CTA of kTexThreads threads per body;
// the kNN kernels: clusters over a body's queries (m3t_b200_texture.cuh). Bodies without a texture modality return
// at once.
#include <cfloat>
#include <climits>

#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include "m3t_b200_texture.cuh"

namespace m3tb {

namespace {

// Exclusive prefix of `keep` over the CTA in thread order; returns the thread's offset, *total the CTA's count.
__device__ __forceinline__ int BlockCompact(bool keep, int* s_warp, int* total) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned ballot = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) s_warp[warp] = __popc(ballot);
  __syncthreads();
  int before = 0, sum = 0;
  for (int w = 0; w < kTexThreads / 32; ++w) {
    if (w < warp) before += s_warp[w];
    sum += s_warp[w];
  }
  __syncthreads();  // s_warp is reused by the next call
  *total = sum;
  return before + __popc(ballot & ((1u << lane) - 1u));
}

__device__ __forceinline__ const uint8_t* Row(const RenderingDev& r, int v) { return r.image + size_t(v) * r.pitch; }

// TextureModality::IsPointUnoccludedMeasured (texture_modality.cpp:1035-1085)
__device__ bool UnoccludedMeasured(const CameraDev& d, const float* b2d, const TextureParamsDev& tp, float bx, float by,
                                   float bz) {
  const float x = b2d[0] * bx + b2d[1] * by + b2d[2] * bz + b2d[3];
  const float y = b2d[4] * bx + b2d[5] * by + b2d[6] * bz + b2d[7];
  const float z = b2d[8] * bx + b2d[9] * by + b2d[10] * bz + b2d[11];
  const float center_u = x * d.fu / z + d.ppu, center_v = y * d.fv / z + d.ppv;
  const float meter_to_pixel = d.fu / z;
  const float diameter = 2.0f * tp.measured_occlusion_radius * meter_to_pixel;
  if (!ScanDiameterValid(diameter)) return true;
  const int stride = int(diameter / float(kMaxNOcclusionStrides) + 1.0f);
  const int n_strides = int(diameter / float(stride) + 0.5f);
  const int rounded_diameter = n_strides * stride;
  const float rounded_radius = 0.5f * float(rounded_diameter);
  int u_min = int(center_u - rounded_radius + 0.5f), v_min = int(center_v - rounded_radius + 0.5f);
  int u_max = u_min + rounded_diameter, v_max = v_min + rounded_diameter;
  u_min = max(u_min, 0);
  v_min = max(v_min, 0);
  u_max = min(u_max, d.width - 1);
  v_max = min(v_max, d.height - 1);
  // ushort(x) of the reference: truncation to int, then reduction modulo 2^16, as in WindowUnoccluded. A threshold
  // above z + depth_scale wraps the bound to about 65 k, so almost any valid depth pixel in the window occludes
  const unsigned min_depth = unsigned(int((z - tp.measured_occlusion_threshold) / d.depth_scale)) & 0xffffu;
  // a camera that refers to a pinned frame is read from it: its device copy is valid only inside the tracking ROIs
  const uint8_t* img = d.host_src ? d.host_src : d.image;
  const unsigned pitch = d.host_src ? d.host_pitch : d.pitch;
  for (int v = v_min; v <= v_max; v += stride) {
    const uint16_t* row = reinterpret_cast<const uint16_t*>(img + size_t(v) * pitch);
    for (int u = u_min; u <= u_max; u += stride) {
      const unsigned depth = row[u];
      if (depth > 0u && depth < min_depth) return false;
    }
  }
  return true;
}

// TextureModality::IsPointUnoccludedModeled (texture_modality.cpp:1087-1127)
__device__ bool UnoccludedModeled(const CameraDev& c, const RenderingDev& r, const float* b2c, const TextureParamsDev& tp,
                                  float bx, float by, float bz) {
  const float x = b2c[0] * bx + b2c[1] * by + b2c[2] * bz + b2c[3];
  const float y = b2c[4] * bx + b2c[5] * by + b2c[6] * bz + b2c[7];
  const float z = b2c[8] * bx + b2c[9] * by + b2c[10] * bz + b2c[11];
  const float meter_to_pixel = (c.fu / z) * r.scale;
  const float diameter = 2.0f * tp.modeled_occlusion_radius * meter_to_pixel;
  if (!ScanDiameterValid(diameter)) return true;
  const int stride = int(diameter / float(kMaxNOcclusionStrides) + 1.0f);
  const int n_strides = int(diameter / float(stride) + 0.5f);
  const int rounded_diameter = n_strides * stride;
  const float rounded_radius = 0.5f * float(rounded_diameter);
  const float center_u = x * c.fu / z + c.ppu, center_v = y * c.fv / z + c.ppv;
  const float fcu = (center_u - r.corner_u) * r.scale, fcv = (center_v - r.corner_v) * r.scale;
  int u_min = int(fcu - rounded_radius + 0.5f), v_min = int(fcv - rounded_radius + 0.5f);
  int u_max = u_min + rounded_diameter, v_max = v_min + rounded_diameter;
  u_min = max(u_min, 0);
  v_min = max(v_min, 0);
  u_max = min(u_max, r.image_size - 1);
  v_max = min(v_max, r.image_size - 1);
  unsigned short min_value = 65535;
  for (int v = v_min; v <= v_max; v += stride) {
    const uint16_t* row = reinterpret_cast<const uint16_t*>(Row(r, v));
    for (int u = u_min; u <= u_max; u += stride) min_value = min(min_value, row[u]);
  }
  const float min_depth = r.projection_term_a / (r.projection_term_b - float(min_value));
  return min_depth > z - tp.modeled_occlusion_threshold;
}

// R^T normalize(t) of a body2camera pose (orientation_last_keyframe_, texture_modality.cpp:1016-1018); like Eigen's
// normalized(), a zero translation stays zero
__device__ void Orientation(const float* b2c, float* o) {
  const float n2 = b2c[3] * b2c[3] + b2c[7] * b2c[7] + b2c[11] * b2c[11];
  float tx = b2c[3], ty = b2c[7], tz = b2c[11];
  if (n2 > 0.0f) {
    const float n = sqrtf(n2);
    tx = tx / n; ty = ty / n; tz = tz / n;
  }
  for (int i = 0; i < 3; ++i) o[i] = b2c[i] * tx + b2c[4 + i] * ty + b2c[8 + i] * tz;
}

}  // namespace

// StartModality (mode 0: PrecalculatePoseVariables from the current pose, then ComputeKeyframeData) and CalculateResults
// (mode 1: the rotation / age rule with the pose of the last gradient pass, texture_modality.cpp:456-472).
__global__ void __launch_bounds__(kTexThreads) k_texture_keyframe(const __grid_constant__ TextureArgs a) {
  const int b = a.list ? a.list[blockIdx.x] : int(blockIdx.x), tid = threadIdx.x;
  const BodyDev& body = a.bodies[b];
  if (!body.set || !body.has_texture) return;
  __shared__ float b2c[12], c2b[12], b2d[12];
  __shared__ int s_fire, s_visible, s_slot;
  __shared__ int s_warp[kTexThreads / 32];
  const CameraDev& cam = a.color_cams[body.texture_camera];
  const TextureParamsDev& tp = body.tp;
  TexKeyframeState* st = a.kf_state + b;
  if (tid == 0) {
    float pose[12];
    for (int k = 0; k < 12; ++k) pose[k] = a.mode == 0 ? a.poses[12 * b + k] : a.tex_pose[12 * b + k];
    if (a.mode == 0)
      for (int k = 0; k < 12; ++k) a.tex_pose[12 * b + k] = pose[k];
    PoseMul(cam.w2c, pose, b2c);
    PoseInverse(b2c, c2b);
    if (tp.measure_occlusions) PoseMul(a.depth_cams[body.depth_camera].w2c, pose, b2d);
    int fire = 1;
    if (a.mode == 1) {
      float o[3];
      Orientation(b2c, o);
      const float rotation_difference = acosf(o[0] * st->orientation[0] + o[1] * st->orientation[1] + o[2] * st->orientation[2]);
      st->age += 1;
      fire = rotation_difference > tp.max_keyframe_rotation_difference || st->age > tp.max_keyframe_age;
    }
    int visible = 0;
    if (fire) {
      if (st->size >= tp.n_keyframes) {  // pop_front, before the visibility test
        st->head = (st->head + 1) % kTexMaxKeyframes;
        st->size -= 1;
      }
      const RenderingDev& sil = body.rend[RS_TEXTURE_SILHOUETTE];
      visible = sil.image != nullptr && sil.visible;
    }
    s_fire = fire;
    s_visible = visible;
    s_slot = (st->head + st->size) % kTexMaxKeyframes;
  }
  __syncthreads();
  if (!s_fire || !s_visible) return;
  const RenderingDev& sil = body.rend[RS_TEXTURE_SILHOUETTE];
  const RenderingDev& sdep = body.rend[RS_TEXTURE_SILHOUETTE_DEPTH];
  const RenderingDev& mdep = body.rend[RS_TEXTURE_DEPTH];
  const bool modeled = tp.model_occlusions && mdep.image != nullptr && mdep.visible;
  const int n = a.feat_n[b];
  const size_t cap = size_t(a.cap);
  const float2* xy = a.feat_xy + size_t(b) * cap;
  // a descriptor is TexRowWords 32-bit words, copied as words (binary or float alike) in rows of TexRowStride
  const bool wide = TexWideRows(tp.descriptor_type);
  const int words = TexRowWords(tp), stride = int(TexRowStride(tp));
  const uint32_t* desc = wide ? reinterpret_cast<const uint32_t*>(a.feat_fdesc) : a.feat_desc;
  desc += size_t(b) * cap * stride;
  const int slot = s_slot;
  float* kp = a.kf_points + (size_t(b) * kTexMaxKeyframes + slot) * 3 * cap;
  uint32_t* kd = wide ? reinterpret_cast<uint32_t*>(a.kf_fdesc) : a.kf_desc;
  kd += (size_t(b) * kTexMaxKeyframes + slot) * cap * stride;
  int written = 0;
  for (int i0 = 0; i0 < n; i0 += kTexThreads) {
    const int i = i0 + tid;
    bool keep = false;
    float px = 0.0f, py = 0.0f, pz = 0.0f;
    if (i < n) {  // Reconstruct3DPoint (texture_modality.cpp:987-1023) + IsPointValid
      const float2 c = xy[i];
      const int us = int((c.x - sil.corner_u) * sil.scale + 0.5f), vs = int((c.y - sil.corner_v) * sil.scale + 0.5f);
      const int s1 = sil.image_size - 1;
      if (us >= 0 && us <= s1 && vs >= 0 && vs <= s1 && Row(sil, vs)[us] == uint8_t(sil.id)) {
        const unsigned short value = reinterpret_cast<const uint16_t*>(Row(sdep, vs))[us];
        const float depth = sdep.projection_term_a / (sdep.projection_term_b - float(value));
        const float cx = depth * (c.x - cam.ppu) / cam.fu, cy = depth * (c.y - cam.ppv) / cam.fv, cz = depth;
        px = c2b[0] * cx + c2b[1] * cy + c2b[2] * cz + c2b[3];
        py = c2b[4] * cx + c2b[5] * cy + c2b[6] * cz + c2b[7];
        pz = c2b[8] * cx + c2b[9] * cy + c2b[10] * cz + c2b[11];
        keep = true;
        if (tp.measure_occlusions) keep = UnoccludedMeasured(a.depth_cams[body.depth_camera], b2d, tp, px, py, pz);
        if (keep && modeled) keep = UnoccludedModeled(cam, mdep, b2c, tp, px, py, pz);
      }
    }
    int total;
    const int pos = written + BlockCompact(keep, s_warp, &total);
    if (keep) {
      kp[0 * cap + pos] = px;
      kp[1 * cap + pos] = py;
      kp[2 * cap + pos] = pz;
      for (int w = 0; w < words; ++w) kd[size_t(pos) * stride + w] = desc[size_t(i) * stride + w];
    }
    written += total;
  }
  if (tid == 0) {
    a.kf_n[b * kTexMaxKeyframes + slot] = written;
    st->size += 1;
    Orientation(b2c, st->orientation);
    st->age = 0;
  }
}

namespace {

// A top-2 list under (distance, train index) order, best first; empty entries are (FLT_MAX, INT_MAX), which every
// candidate that can enter (a finite distance below FLT_MAX) precedes.
struct Top2 {
  float d0, d1;
  int i0, i1;
};

__device__ __forceinline__ bool Precedes(float da, int ia, float db, int ib) { return da < db || (da == db && ia < ib); }

// cv::batchDistance's K = 2 insertion for candidates in increasing train index: a distance enters only if strictly
// below the second (so NaN and inf never enter), and ties keep the earlier index
__device__ __forceinline__ void Insert(Top2& t, float d, int j) {
  if (d < t.d1) {
    if (d < t.d0) { t.d1 = t.d0; t.i1 = t.i0; t.d0 = d; t.i0 = j; }
    else { t.d1 = d; t.i1 = j; }
  }
}

// The two first of the union of two lists with distinct indices: what the insertion gives over both index ranges
__device__ __forceinline__ Top2 Merge(const Top2& a, const Top2& b) {
  Top2 r;
  if (Precedes(b.d0, b.i0, a.d0, a.i0)) {
    r.d0 = b.d0; r.i0 = b.i0;
    if (Precedes(b.d1, b.i1, a.d0, a.i0)) { r.d1 = b.d1; r.i1 = b.i1; }
    else { r.d1 = a.d0; r.i1 = a.i0; }
  } else {
    r.d0 = a.d0; r.i0 = a.i0;
    if (Precedes(b.d0, b.i0, a.d1, a.i1)) { r.d1 = b.d0; r.i1 = b.i0; }
    else { r.d1 = a.d1; r.i1 = a.i1; }
  }
  return r;
}

// rows [0, n) of a table of 32-bit words in rows of src_stride into shared rows of `stride` words: the first `length`
// words, zero up to the next multiple of 4 and in rows [n, rows)
__device__ __forceinline__ void StageRows(const uint32_t* src, size_t src_stride, int n, int rows, int length, int stride,
                                          uint32_t* dst) {
  const int d4 = (length + 3) / 4;
  for (int e = threadIdx.x; e < rows * d4; e += kKnnThreads) {
    const int r = e / d4, c = e - r * d4;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r < n) {
      v = *reinterpret_cast<const uint4*>(src + r * src_stride + 4 * c);
      const int k = 4 * c;
      if (k + 1 >= length) v.y = 0u;
      if (k + 2 >= length) v.z = 0u;
      if (k + 3 >= length) v.w = 0u;
    }
    *reinterpret_cast<uint4*>(dst + r * stride + 4 * c) = v;
  }
}

// The distance sums of one (query, train) pair over four 32-bit words: L2, float descriptors: squared differences
// in descriptor order; Hamming, binary descriptors: bits that differ
template <bool kHamming>
__device__ __forceinline__ void KnnAccumulate(const uint4& q, const uint4& t, float& acc) {
  if constexpr (kHamming) {
    acc += float(__popc(q.x ^ t.x) + __popc(q.y ^ t.y) + __popc(q.z ^ t.z) + __popc(q.w ^ t.w));
  } else {
    float d = __uint_as_float(q.x) - __uint_as_float(t.x);
    acc = fmaf(d, d, acc);
    d = __uint_as_float(q.y) - __uint_as_float(t.y);
    acc = fmaf(d, d, acc);
    d = __uint_as_float(q.z) - __uint_as_float(t.z);
    acc = fmaf(d, d, acc);
    d = __uint_as_float(q.w) - __uint_as_float(t.w);
    acc = fmaf(d, d, acc);
  }
}

// One cluster's tile of k_texture_knn_l2 / k_texture_knn_hamming: kKnnQueries queries of one keyframe against the
// frame's train set. Each thread holds a 4 x 4 block of (query, train) sums, queries ty + 16 i and train rows tx + 16 j
// of the CTA's slice of a chunk, and a running top-2 list per query over its train rows in increasing index: the
// insertion of cv::batchDistance. The lists of the 16 lanes sharing a query and then of the cluster's CTAs are merged
// under (distance, train index) order, which is what that insertion gives over the union. kWords: the body's
// TexRowWords as a constant of the inner loop (the caller has checked it), 0 for a width known at run time only.
template <bool kHamming, int kWords>
__device__ __forceinline__ void KnnTile(const TextureArgs& a, int b) {
  namespace cg = cooperative_groups;
  const int tid = threadIdx.x;
  const BodyDev& body = a.bodies[b];
  // every return before the first cluster barrier depends on (body, tile) alone: a cluster leaves or stays whole
  if (!body.set || !body.has_texture || (kHamming ? !TexHammingKnn(body.tp) : TexHamming(body.tp.descriptor_type)))
    return;
  const int rank = blockIdx.x % kKnnSplits, tile = blockIdx.x / kKnnSplits;
  const int tiles = KnnTilesPerKeyframe(body.tp.n_features_max);
  const int k = tile / tiles, q0 = tile % tiles * kKnnQueries;
  const TexKeyframeState st = a.kf_state[b];
  if (k >= st.size) return;
  const int slot = (st.head + k) % kTexMaxKeyframes;
  const int nq = min(kKnnQueries, a.kf_n[b * kTexMaxKeyframes + slot] - q0);
  if (nq <= 0) return;
  // rows of `length` words, `src_stride` words apart in the tables
  const int length = kWords ? kWords : TexRowWords(body.tp), stride = KnnStride(length);
  const size_t src_stride = TexRowStride(body.tp), cap = size_t(a.cap);
  const bool wide = TexWideRows(body.tp.descriptor_type);
  const uint32_t* kf_rows = wide ? reinterpret_cast<const uint32_t*>(a.kf_fdesc) : a.kf_desc;
  const uint32_t* feat_rows = wide ? reinterpret_cast<const uint32_t*>(a.feat_fdesc) : a.feat_desc;
  const int n_train = a.feat_n[b];
  extern __shared__ uint4 s_dyn[];
  uint32_t* s_q = reinterpret_cast<uint32_t*>(s_dyn);
  uint32_t* s_t = s_q + kKnnQueries * stride;
  __shared__ Top2 s_part[kKnnQueries];
  StageRows(kf_rows + ((size_t(b) * kTexMaxKeyframes + slot) * cap + q0) * src_stride, src_stride, nq, kKnnQueries,
            length, stride, s_q);
  const int ty = tid / 16, tx = tid % 16, s4 = stride / 4, d4 = (length + 3) / 4;
  const uint4* q4 = reinterpret_cast<const uint4*>(s_q);
  const uint4* t4 = reinterpret_cast<const uint4*>(s_t);
  Top2 top[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) top[i] = Top2{FLT_MAX, FLT_MAX, INT_MAX, INT_MAX};
  for (int c0 = 0; c0 < n_train; c0 += kKnnChunk) {
    const int t0 = c0 + rank * kKnnTrain, nt = max(0, min(kKnnTrain, n_train - t0));
    if (c0 > 0) __syncthreads();  // every thread is done with the previous chunk's rows
    StageRows(feat_rows + (size_t(b) * cap + t0) * src_stride, src_stride, nt, kKnnTrain, length, stride, s_t);
    __syncthreads();
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
    for (int c = 0; c < d4; ++c) {
      uint4 qv[4], tv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) qv[i] = q4[(ty + 16 * i) * s4 + c];
#pragma unroll
      for (int j = 0; j < 4; ++j) tv[j] = t4[(tx + 16 * j) * s4 + c];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) KnnAccumulate<kHamming>(qv[i], tv[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (tx + 16 * j < nt) Insert(top[i], kHamming ? acc[i][j] : sqrtf(acc[i][j]), t0 + tx + 16 * j);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    Top2 t = top[i];
    // the 16 lanes of a half-warp share ty: merge their lists
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) {
      Top2 o;
      o.d0 = __shfl_xor_sync(0xffffffffu, t.d0, off);
      o.d1 = __shfl_xor_sync(0xffffffffu, t.d1, off);
      o.i0 = __shfl_xor_sync(0xffffffffu, t.i0, off);
      o.i1 = __shfl_xor_sync(0xffffffffu, t.i1, off);
      t = Merge(t, o);
    }
    if (tx == 0) s_part[ty + 16 * i] = t;
  }
  cg::cluster_group cluster = cg::this_cluster();
  cluster.sync();
  if (rank == 0 && tid < nq) {
    Top2 t = s_part[tid];
    for (int r = 1; r < kKnnSplits; ++r) t = Merge(t, cluster.map_shared_rank(s_part, r)[tid]);
    // knn_match[0].distance / knn_match[1].distance >= threshold drops the match; 0 / 0 is NaN and keeps it
    const bool keep = t.i1 != INT_MAX && !(t.d0 / t.d1 >= body.tp.descriptor_distance_threshold);
    a.knn[(size_t(b) * kTexMaxKeyframes + slot) * cap + q0 + tid] = keep ? t.i0 : -1;
  }
  cluster.sync();  // the partial lists of ranks 1.. stay in place until rank 0 has read them
}

}  // namespace

// cv::BFMatcher(NORM_L2).knnMatch(keyframe descriptors, frame descriptors, k = 2) and the ratio test of
// CalculateCorrespondences for every L2 body at correspondence iteration 0. distance = sqrt of the float sum of
// squared float differences, summed in descriptor order. For SIFT's whole-number descriptors every partial sum is an
// integer below 2^24, so any order gives OpenCV's distance bit for bit (DESIGN.md section 3).
__global__ void __cluster_dims__(kKnnSplits, 1, 1) __launch_bounds__(kKnnThreads)
    k_texture_knn_l2(const __grid_constant__ TextureArgs a) {
  KnnTile<false, 0>(a, a.list ? a.list[blockIdx.y] : int(blockIdx.y));
}

// cv::BFMatcher(NORM_HAMMING).knnMatch(k = 2) and the ratio test for every TexHammingKnn body (ORB above
// kTexMaxFeatures, BRISK, FREAK), at correspondence iteration 0. Distances are bit counts, exact as floats. The row
// width is the CTA's body's, the same for the whole cluster (grid y), and a constant of each inner loop. Three CTAs
// per SM, as before 16-word rows: unbounded, their unrolled loop takes 127 registers, and every body of the launch,
// ORB's included, would run at two.
__global__ void __cluster_dims__(kKnnSplits, 1, 1) __launch_bounds__(kKnnThreads, 3)
    k_texture_knn_hamming(const __grid_constant__ TextureArgs a) {
  const int b = a.list ? a.list[blockIdx.y] : int(blockIdx.y);
  if (TexRowWords(a.bodies[b].tp) == kTexBinary64Words) KnnTile<true, kTexBinary64Words>(a, b);
  else KnnTile<true, kTexDescWords>(a, b);
}

// CalculateCorrespondences (texture_modality.cpp:322-386): with mode 1 (correspondence iteration 0) every keyframe's
// descriptors (queries) are matched against the frame's (train set) by brute-force kNN, k = 2, and the matches that pass
// the ratio test become the data points, keyframe by keyframe in query order. ORB bodies up to kTexMaxFeatures are
// matched here (Hamming, the train set in shared memory); k_texture_knn_l2 / _hamming have matched the others, BRISK
// and FREAK bodies always, just before. Every call then projects the data points with the current pose (data_point.center) and records that pose.
__global__ void __launch_bounds__(kTexThreads) k_texture_match(const __grid_constant__ TextureArgs a) {
  const int b = a.list ? a.list[blockIdx.x] : int(blockIdx.x), tid = threadIdx.x;
  const BodyDev& body = a.bodies[b];
  if (!body.set || !body.has_texture) return;
  __shared__ uint4 s_train[kTexMaxFeatures * 2];
  __shared__ int s_warp[kTexThreads / 32];
  const size_t cap = size_t(a.cap), point_cap = kTexMaxKeyframes * cap;
  float* pts = a.points + size_t(b) * TF_COUNT * point_cap;
  const CameraDev& cam = a.color_cams[body.texture_camera];
  if (a.mode == 1) {
    const int n_train = a.feat_n[b];
    const bool knn_matched = !TexHamming(body.tp.descriptor_type) || TexHammingKnn(body.tp);
    const uint4* train = reinterpret_cast<const uint4*>(a.feat_desc + size_t(b) * cap * kTexDescWords);
    if (!knn_matched)
      for (int k = tid; k < 2 * n_train; k += kTexThreads) s_train[k] = train[k];
    __syncthreads();
    const float2* xy = a.feat_xy + size_t(b) * cap;
    const TexKeyframeState st = a.kf_state[b];
    const float thr = body.tp.descriptor_distance_threshold;
    int written = 0;
    for (int k = 0; k < st.size; ++k) {
      const int slot = (st.head + k) % kTexMaxKeyframes;
      const int nq = a.kf_n[b * kTexMaxKeyframes + slot];
      const size_t kf = size_t(b) * kTexMaxKeyframes + slot;
      const float* kp = a.kf_points + kf * 3 * cap;
      const uint4* kd = reinterpret_cast<const uint4*>(a.kf_desc + kf * cap * kTexDescWords);
      const int* knn = knn_matched ? a.knn + kf * cap : nullptr;
      for (int q0 = 0; q0 < nq; q0 += kTexThreads) {
        const int q = q0 + tid;
        bool keep = false;
        int i0 = -1;
        if (q < nq && knn) {
          i0 = knn[q];
          keep = i0 >= 0;
        } else if (q < nq && n_train >= 2) {
          const uint4 qa = kd[2 * q], qb = kd[2 * q + 1];
          // cv::batchDistance's K = 2 insertion: strictly smaller distances enter, ties keep the earlier train index
          int d0 = INT_MAX, d1 = INT_MAX, i1 = -1;
          for (int j = 0; j < n_train; ++j) {
            const uint4 ta = s_train[2 * j], tb = s_train[2 * j + 1];
            const int d = __popc(qa.x ^ ta.x) + __popc(qa.y ^ ta.y) + __popc(qa.z ^ ta.z) + __popc(qa.w ^ ta.w) +
                          __popc(qb.x ^ tb.x) + __popc(qb.y ^ tb.y) + __popc(qb.z ^ tb.z) + __popc(qb.w ^ tb.w);
            if (d < d1) {
              if (d < d0) { d1 = d0; i1 = i0; d0 = d; i0 = j; }
              else { d1 = d; i1 = j; }
            }
          }
          // knn_match[0].distance / knn_match[1].distance >= threshold drops the match; 0 / 0 is NaN and keeps it
          keep = i1 >= 0 && !(float(d0) / float(d1) >= thr);
        }
        int total;
        const int pos = written + BlockCompact(keep, s_warp, &total);
        if (keep) {
          pts[TF_CBX * point_cap + pos] = kp[0 * cap + q];
          pts[TF_CBY * point_cap + pos] = kp[1 * cap + q];
          pts[TF_CBZ * point_cap + pos] = kp[2 * cap + q];
          const float2 c = xy[i0];
          pts[TF_CU * point_cap + pos] = c.x;
          pts[TF_CV * point_cap + pos] = c.y;
        }
        written += total;
      }
    }
    if (tid == 0) a.counts[b] = written;
    __syncthreads();
  }
  __shared__ float b2c[12];
  if (tid < 12) a.tex_pose[12 * b + tid] = a.poses[12 * b + tid];
  if (tid == 0) PoseMul(cam.w2c, a.poses + 12 * b, b2c);
  __syncthreads();
  const int n = a.counts[b];
  for (int i = tid; i < n; i += kTexThreads) {
    const float bx = pts[TF_CBX * point_cap + i], by = pts[TF_CBY * point_cap + i], bz = pts[TF_CBZ * point_cap + i];
    const float x = b2c[0] * bx + b2c[1] * by + b2c[2] * bz + b2c[3];
    const float y = b2c[4] * bx + b2c[5] * by + b2c[6] * bz + b2c[7];
    const float z = b2c[8] * bx + b2c[9] * by + b2c[10] * bz + b2c[11];
    pts[TF_PU * point_cap + i] = x * cam.fu / z + cam.ppu;
    pts[TF_PV * point_cap + i] = y * cam.fv / z + cam.ppv;
  }
}

namespace {

// cvtColor(BGR2GRAY) on 8-bit pixels: equal to OpenCV's result on all 2^24 triples
// (tests/texture_crop_reference.py)
__device__ __forceinline__ int Grey(const uint8_t* p) {
  return (3735 * int(p[0]) + 19235 * int(p[1]) + 9798 * int(p[2]) + 16384) >> 15;
}

// cv::resize's INTER_LINEAR coefficient of output position d (resize.cpp): the two source positions and their weights
// in 1/2048. Columns pin a position before the first or at the last source pixel to it with weights (2048, 0); rows
// keep their weights and only clamp the two source rows. The build compiles without FMA contraction, so
// (d + 0.5) * inv - 0.5 rounds twice in double, as on the host.
struct Tap {
  int s0, s1, w0, w1;
};
__device__ __forceinline__ Tap LinearTap(int d, double inv, int n, bool column) {
  float f = float((double(d) + 0.5) * inv - 0.5);
  int s = int(floorf(f));
  f -= float(s);
  if (column && s < 0) { s = 0; f = 0.0f; }
  if (column && s >= n - 1) { s = n - 1; f = 0.0f; }
  Tap t;
  t.w0 = __float2int_rn((1.0f - f) * 2048.0f);
  t.w1 = __float2int_rn(f * 2048.0f);
  t.s0 = min(max(s, 0), n - 1);
  t.s1 = min(max(s + 1, 0), n - 1);
  return t;
}

__device__ __forceinline__ int GreyAt(const TexCropJob& j, int x, int y) {
  return Grey(j.src + size_t(j.roi_y + y) * j.src_pitch + size_t(j.roi_x + x) * 3u);
}

// One output pixel (tests/texture_crop_reference.py states every case)
__device__ __forceinline__ uint8_t CropPixel(const TexCropJob& j, int dx, int dy, double inv, bool area, bool copy) {
  if (copy) return uint8_t(GreyAt(j, dx, dy));
  if (area) {  // cv::resize's fast INTER_AREA path at exactly 2x
    const int x0 = 2 * dx, y0 = 2 * dy;
    const bool full_row = 2 * (dy + 1) <= j.roi_h;
    if (full_row && x0 + 1 < j.roi_w)
      return uint8_t((GreyAt(j, x0, y0) + GreyAt(j, x0 + 1, y0) + GreyAt(j, x0, y0 + 1) + GreyAt(j, x0 + 1, y0 + 1) + 2) >> 2);
    int sum = 0, count = 0;
    for (int y = y0; y < min(y0 + 2, j.roi_h); ++y)
      for (int x = x0; x < min(x0 + 2, j.roi_w); ++x) {
        sum += GreyAt(j, x, y);
        ++count;
      }
    return uint8_t(min(__float2int_rn(float(sum) / float(count)), 255));
  }
  const Tap tx = LinearTap(dx, inv, j.roi_w, true), ty = LinearTap(dy, inv, j.roi_h, false);
  const int h0 = GreyAt(j, tx.s0, ty.s0) * tx.w0 + GreyAt(j, tx.s1, ty.s0) * tx.w1;
  const int h1 = GreyAt(j, tx.s0, ty.s1) * tx.w0 + GreyAt(j, tx.s1, ty.s1) * tx.w1;
  // OpenCV's vectorised vertical pass: 16-bit high products of the weights and the sums shifted by 4
  const int v = (((ty.w0 * min(h0 >> 4, 32767)) >> 16) + ((ty.w1 * min(h1 >> 4, 32767)) >> 16) + 2) >> 2;
  return uint8_t(min(max(v, 0), 255));
}

}  // namespace

// Each thread writes kTexCropPixels consecutive pixels of one output row of job blockIdx.y.
__global__ void __launch_bounds__(kTexCropThreads) k_texture_crop(const __grid_constant__ TexCropArgs a) {
  const TexCropJob& j = a.jobs[blockIdx.y];
  const int groups = (j.out_w + kTexCropPixels - 1) / kTexCropPixels;
  const int t = blockIdx.x * kTexCropThreads + threadIdx.x;
  if (t >= groups * j.out_h) return;
  const int dy = t / groups, dx0 = (t - dy * groups) * kTexCropPixels;
  const bool copy = j.out_w == j.roi_w && j.out_h == j.roi_h;
  const bool area = !copy && j.scale == 0.5f;
  const double inv = 1.0 / double(j.scale);
  uint8_t* row = j.dst + size_t(dy) * a.dst_pitch;
#pragma unroll
  for (int k = 0; k < kTexCropPixels; ++k)
    if (dx0 + k < j.out_w) row[dx0 + k] = CropPixel(j, dx0 + k, dy, inv, area, copy);
}

// The host upload's conversion (UploadTextureFeatures): keypoint roi + pt / scale, descriptors into the frame tables.
// Float descriptors are checked here: a body with a non-finite value gets no features and its flag is raised. Binary
// rows are copied byte by byte, never read as floats.
__global__ void __launch_bounds__(kTexThreads) k_texture_features(const __grid_constant__ TexFeatArgs a) {
  const TexFeatJob& j = a.jobs[blockIdx.x];
  const int tid = threadIdx.x, b = j.body;
  const size_t cap = size_t(a.cap);
  float2* xy = a.feat_xy + size_t(b) * cap;
  for (int i = tid; i < j.n; i += kTexThreads) {
    const float x = j.x[size_t(i) * j.xy_stride], y = j.y[size_t(i) * j.xy_stride];
    xy[i] = make_float2(float(j.roi_x) + x / j.scale, float(j.roi_y) + y / j.scale);
  }
  int bad = 0;
  if (j.length == 0) {
    const size_t stride = j.wide ? kTexMaxFloatDesc : kTexDescWords;
    uint8_t* dst = reinterpret_cast<uint8_t*>((j.wide ? reinterpret_cast<uint32_t*>(a.feat_fdesc) : a.feat_desc) +
                                              size_t(b) * cap * stride);
    const int width = 4 * j.words;
    for (int e = tid; e < j.n * width; e += kTexThreads) {  // byte by byte: the caller's rows need no alignment
      const int i = e / width, c = e - i * width;
      dst[size_t(i) * 4 * stride + c] = j.desc[size_t(i) * j.desc_pitch + c];
    }
  } else {
    float* dst = a.feat_fdesc + size_t(b) * cap * kTexMaxFloatDesc;
    for (int e = tid; e < j.n * j.length; e += kTexThreads) {
      const int i = e / j.length, c = e - i * j.length;
      const float v = reinterpret_cast<const float*>(j.desc + size_t(i) * j.desc_pitch)[c];
      bad |= !isfinite(v);
      dst[size_t(i) * kTexMaxFloatDesc + c] = v;
    }
  }
  bad = __syncthreads_or(bad);
  if (tid == 0) {
    a.feat_n[b] = bad ? 0 : j.n;
    a.nonfinite[b] = bad;
  }
}

}  // namespace m3tb
