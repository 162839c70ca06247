// m3t_b200_texture.cuh — TextureModality on the device (texture_modality.cpp): keyframe reconstruction from the device
// silhouette renderer, brute-force kNN matching (Hamming for ORB's 32-byte descriptors, L2 for SIFT / DAISY float
// descriptors), and the Tukey-weighted reprojection gradient / Hessian that k_track adds to a body's link. Feature
// detection stays with the caller, or for ORB bodies runs in k_texture_orb (m3t_b200_orb.cu); the keypoints in image
// coordinates and the descriptors are all the matching kernels read of the colour frame.
#pragma once

#include "m3t_b200_device.cuh"

namespace m3tb {

// Frame features per body: n_features_max, kTexMaxFeatures (the default) .. kTexFeatureLimit. The tables of a context
// hold TextureArgs::cap features per body, the largest n_features_max any of its texture bodies has asked for.
// k_texture_match stages an ORB body's train set in shared memory up to kTexMaxFeatures; ORB bodies above it and every
// L2 body are matched by the cluster kNN kernels below.
constexpr int kTexMaxFeatures = 512;
constexpr int kTexFeatureLimit = 4096;
constexpr int kTexMaxKeyframes = 8;    // n_keyframes
constexpr int kTexDescWords = 8;       // 32-byte ORB descriptors
constexpr int kTexMaxFloatDesc = 256;  // float descriptor cap and the stride of the float tables (SIFT 128, DAISY 104)
constexpr int kTexThreads = 256;
constexpr int kTexRoiMargin = 10;      // kRegionOfInterestMargin, texture_modality.h:132

// per-data-point fields (SoA, [field][point]): center_f_body, correspondence_center, center
enum TextureField { TF_CBX = 0, TF_CBY, TF_CBZ, TF_CU, TF_CV, TF_PU, TF_PV, TF_COUNT };

// The keyframe deque of one body (points_keyframes_ / descriptors_keyframes_ as a ring of kTexMaxKeyframes slots)
struct TexKeyframeState {
  int size, head, age, pad;
  float orientation[3];  // orientation_last_keyframe_
  float pad1;
};

struct TextureArgs {
  const BodyDev* bodies;
  const float* poses;           // body2world [n_bodies][12]
  float* tex_pose;              // [n_bodies][12]: the pose of the texture modality's last PrecalculatePoseVariables
  const CameraDev* color_cams;
  const CameraDev* depth_cams;
  const float2* feat_xy;        // [n_bodies][cap] keypoints_ in image coordinates
  const uint32_t* feat_desc;    // [n_bodies][cap][8]
  const float* feat_fdesc;      // [n_bodies][cap][kTexMaxFloatDesc] (L2 bodies; null without any)
  const int* feat_n;            // [n_bodies]
  float* kf_points;             // [n_bodies][kTexMaxKeyframes][3][cap]
  uint32_t* kf_desc;            // [n_bodies][kTexMaxKeyframes][cap][8]
  float* kf_fdesc;              // [n_bodies][kTexMaxKeyframes][cap][kTexMaxFloatDesc] (L2 bodies)
  int* knn;                     // [n_bodies][kTexMaxKeyframes][cap] k_texture_knn_l2 / _hamming: the train index of
                                // a query's best match that passes the ratio test, -1 otherwise (by keyframe slot)
  int* kf_n;                    // [n_bodies][kTexMaxKeyframes]
  TexKeyframeState* kf_state;   // [n_bodies]
  float* points;                // [n_bodies][TF_COUNT][kTexMaxKeyframes * cap]
  int* counts;                  // [n_bodies]
  int mode;                     // k_texture_keyframe: 0 StartModality, 1 CalculateResults; k_texture_match: 1 = match
  int cap;                      // features per body of every table above (kTexMaxFeatures .. kTexFeatureLimit)
};

// k_texture_match reads an ORB body's matches from knn (k_texture_knn_hamming) instead of scanning its train set
__host__ __device__ __forceinline__ bool TexHammingKnn(const TextureParamsDev& tp) {
  return !tp.l2 && tp.n_features_max > kTexMaxFeatures;
}

__global__ void k_texture_keyframe(const __grid_constant__ TextureArgs a);
__global__ void k_texture_match(const __grid_constant__ TextureArgs a);

// k_texture_knn_l2 (SIFT / DAISY bodies) and k_texture_knn_hamming (ORB bodies above kTexMaxFeatures): a cluster of
// kKnnSplits CTAs per tile of kKnnQueries queries of one keyframe. The train set is walked in chunks of kKnnChunk rows;
// CTA r of the cluster scans rows [c * kKnnChunk + r * kKnnTrain, ... + kKnnTrain) of every chunk c and rank 0 merges
// the partial top-2 lists. Grid: (kKnnSplits * keyframes * KnnTilesPerKeyframe(features), n_bodies), with the longest
// deque and the largest n_features_max of the bodies the kernel matches; dynamic shared memory KnnSharedBytes(row
// length in 32-bit words: the longest descriptor of the context's L2 bodies, kTexDescWords for Hamming).
constexpr int kKnnQueries = 64, kKnnTrain = 64, kKnnThreads = 256;
constexpr int kKnnSplits = 8;                       // the portable cluster size
constexpr int kKnnChunk = kKnnSplits * kKnnTrain;   // 512 train rows per chunk
__host__ __device__ constexpr int KnnTilesPerKeyframe(int features) { return (features + kKnnQueries - 1) / kKnnQueries; }
// shared rows are padded to a stride of 4 (mod 8) words, so the 8 16-byte reads of a quarter-warp hit distinct banks
__host__ __device__ constexpr int KnnStride(int length) { return (length + 7) / 8 * 8 + 4; }
__host__ __device__ constexpr int KnnSharedBytes(int length) {
  return int(sizeof(float)) * (kKnnQueries + kKnnTrain) * KnnStride(length);
}
__global__ void k_texture_knn_l2(const __grid_constant__ TextureArgs a);
__global__ void k_texture_knn_hamming(const __grid_constant__ TextureArgs a);

// k_texture_crop / k_texture_features: up to kTexJobs bodies per launch; the jobs travel in the kernel parameters
constexpr int kTexJobs = 128;
constexpr int kTexCropThreads = 256;
constexpr int kTexCropPixels = 4;  // output pixels per thread (one row, consecutive columns)

// One body's focused grey image (DetectAndComputeCorrKeypoints, texture_modality.cpp:862-868):
// resize(cvtColor(image, BGR2GRAY)(roi), Size(), scale, scale, INTER_LINEAR) into out_w x out_h bytes at dst.
struct TexCropJob {
  const uint8_t* src;  // BGR8 frame: the camera's device copy, or its pinned frame read in place
  uint8_t* dst;        // rows dst_pitch apart (TexCropArgs)
  unsigned src_pitch;
  int roi_x, roi_y, roi_w, roi_h;
  int out_w, out_h;
  float scale;
};

struct TexCropArgs {
  TexCropJob jobs[kTexJobs];
  size_t dst_pitch;
  int n_jobs;
};

// grid: (ceil(max over jobs of ceil(out_w / kTexCropPixels) * out_h / kTexCropThreads), n_jobs)
__global__ void k_texture_crop(const __grid_constant__ TexCropArgs a);

// One body's features from device memory, converted as the host upload converts them.
struct TexFeatJob {
  const float* x;        // keypoint i at x[i * xy_stride], y[i * xy_stride] (crop coordinates)
  const float* y;
  const uint8_t* desc;   // descriptor row i at desc + i * desc_pitch: 32 bytes (ORB) or `length` floats
  size_t desc_pitch;
  int body, n, xy_stride, length;  // length 0: ORB
  int roi_x, roi_y;
  float scale;
  int pad;
};

struct TexFeatArgs {
  TexFeatJob jobs[kTexJobs];
  float2* feat_xy;       // TextureArgs' frame-feature tables, `cap` features per body
  uint32_t* feat_desc;
  float* feat_fdesc;
  int* feat_n;
  int* nonfinite;        // [n_bodies] 1: the body's last device upload held a non-finite descriptor value
  int n_jobs;
  int cap;
};

// one CTA of kTexThreads per job
__global__ void k_texture_features(const __grid_constant__ TexFeatArgs a);

// k_texture_orb: cv::ORB detect + compute on the crops k_texture_crop wrote into the scratch, one CTA per job.
constexpr int kOrbThreads = 512;
constexpr int kOrbMaxLevels = 8;
constexpr int kOrbFeatureLimit = 1 << 24;  // n_features: the per-level counts stay exact in float and 2 n in int
// scratch bytes per job: two ping-pong levels, the blurred level and the FAST scores (1 byte per pixel each), and the
// candidate positions, keys and Harris responses (4 bytes per pixel each)
constexpr int kOrbScratchBytesPerPixel = 4 + 3 * 4;

struct TexOrbJob {
  int body;
  int n_levels;
  int n_features_max;            // the body's capacity: more keypoints than this and it gets none
  int roi_x, roi_y;
  float scale;                   // crop scale: image keypoint = roi + pt / scale
  int w[kOrbMaxLevels], h[kOrbMaxLevels];  // level sizes (w[0] = 0: no focus or an empty level, no features)
  int per_level[kOrbMaxLevels];  // nfeaturesPerLevel
  float layer_scale[kOrbMaxLevels];
};

struct TexOrbArgs {
  TexOrbJob jobs[kTexJobs];
  uint8_t* scratch;              // job k at scratch + k * job_bytes; its level-0 crop there with rows `pitch` apart
  size_t job_bytes;
  int pitch, height;             // the largest crop of the launch
  float2* feat_xy;               // TextureArgs' frame-feature tables, `cap` features per body
  uint32_t* feat_desc;
  int* feat_n;
  float2* orb_xy;                // parity tables [n_bodies][orb_cap]: crop (level-0) keypoint, angle, response, octave
  float* orb_angle;
  float* orb_response;
  int* orb_octave;
  uint32_t* orb_desc;            // [n_bodies][orb_cap][8]
  int* found;                    // [n_bodies] keypoints cv::ORB keeps, before the n_features_max check
  int cap;                       // of the frame-feature tables
  int orb_cap;                   // of the parity tables (the same; kept apart as the tables are made apart)
};

__global__ void k_texture_orb(const __grid_constant__ TexOrbArgs a);

// TextureModality::TukeyNorm (texture_modality.cpp:1231-1237)
__host__ __device__ __forceinline__ float TexTukeyNorm(float error, float c) {
  if (fabsf(error) <= c) return powf(c, 2.0f) / 6.0f * (1.0f - powf(1.0f - powf(error / c, 2.0f), 3.0f));
  return powf(c, 2.0f) / 6.0f;
}

// TextureModality::CalculateGradientAndHessian (texture_modality.cpp:397-444) over the data points i = first, first +
// stride, ... of one body (fields point_cap floats apart), added to acc (g[6], H lower [21], the reference's signs). Also
// refreshes data_point.center.
__device__ __forceinline__ void TextureGradient(const CameraDev& cam, const float* pose, const TextureParamsDev& tp,
                                                int corr, float* pts, int point_cap, int n, int first, int stride,
                                                float* acc) {
  float b2c[12];
  PoseMul(cam.w2c, pose, b2c);
  const float sd = LastValid(tp.standard_deviations, tp.n_standard_deviations, corr);
  const float variance = powf(sd, 2.0f);
  for (int i = first; i < n; i += stride) {
    const float bx = pts[TF_CBX * point_cap + i], by = pts[TF_CBY * point_cap + i], bz = pts[TF_CBZ * point_cap + i];
    const float x = b2c[0] * bx + b2c[1] * by + b2c[2] * bz + b2c[3];
    const float y = b2c[4] * bx + b2c[5] * by + b2c[6] * bz + b2c[7];
    const float z = b2c[8] * bx + b2c[9] * by + b2c[10] * bz + b2c[11];
    const float cu = x * cam.fu / z + cam.ppu, cv = y * cam.fv / z + cam.ppv;
    pts[TF_PU * point_cap + i] = cu;
    pts[TF_PV * point_cap + i] = cv;
    const float z2 = z * z;
    const float d0 = cu - pts[TF_CU * point_cap + i], d1 = cv - pts[TF_CV * point_cap + i];
    const float squared_error = d0 * d0 + d1 * d1;
    const float error = sqrtf(squared_error);
    float weight = 1.0f / variance;
    if (error > 1.17549435e-38f) weight = (TexTukeyNorm(error, tp.tukey_norm_constant) / squared_error) / variance;
    // dx_dX (2x3) * body2camera rotation -> dx_dtranslation; rotation part = center_f_body x row
    const float a00 = cam.fu / z, a02 = -x * cam.fu / z2, a11 = cam.fv / z, a12 = -y * cam.fv / z2;
    float t0[3], t1[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      t0[c] = a00 * b2c[c] + a02 * b2c[8 + c];
      t1[c] = a11 * b2c[4 + c] + a12 * b2c[8 + c];
    }
    const float J0[6] = {by * t0[2] - bz * t0[1], bz * t0[0] - bx * t0[2], bx * t0[1] - by * t0[0], t0[0], t0[1], t0[2]};
    const float J1[6] = {by * t1[2] - bz * t1[1], bz * t1[0] - bx * t1[2], bx * t1[1] - by * t1[0], t1[0], t1[1], t1[2]};
    const float wd0 = weight * d0, wd1 = weight * d1;
#pragma unroll
    for (int k = 0; k < 6; ++k) acc[k] -= wd0 * J0[k] + wd1 * J1[k];
#pragma unroll
    for (int r = 0; r < 6; ++r) {
      const float w0 = weight * J0[r], w1 = weight * J1[r];
#pragma unroll
      for (int c = 0; c <= r; ++c) acc[6 + r * (r + 1) / 2 + c] -= w0 * J0[c] + w1 * J1[c];
    }
  }
}

}  // namespace m3tb
