// m3t_b200_undistort.cu — k_undistort (the per-pixel gather of cv::remap INTER_NEAREST / BORDER_CONSTANT through a
// CV_16SC2 map) and the host construction of that map (m3tb_undistortion_map).
#include <climits>
#include <cmath>

#include "m3t_b200.h"
#include "m3t_b200_undistort.cuh"

namespace m3tb {

// One thread: kUndistortPixels consecutive output pixels of one row. Reads one 16-B map group, gathers the raw pixels
// (0 outside the raw frame: BORDER_CONSTANT) and writes the group with full-width stores.
__global__ void __launch_bounds__(kUndistortThreads) k_undistort(const __grid_constant__ UndistortArgs a) {
  const UndistortJob& J = a.jobs[blockIdx.y];
  const int groups = (J.width + kUndistortPixels - 1) / kUndistortPixels;
  const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = int(t / unsigned(groups));
  if (row >= J.height) return;
  const int g = int(t - unsigned(row) * unsigned(groups));
  const int x0 = g * kUndistortPixels;
  const int n = min(kUndistortPixels, J.width - x0);
  const int4 m = __ldg(reinterpret_cast<const int4*>(reinterpret_cast<const uint8_t*>(J.map) +
                                                     size_t(row) * J.map_pitch) + g);
  const int words[kUndistortPixels] = {m.x, m.y, m.z, m.w};
  int sx[kUndistortPixels], sy[kUndistortPixels];
  bool inside[kUndistortPixels];
#pragma unroll
  for (int k = 0; k < kUndistortPixels; ++k) {
    sx[k] = int(int16_t(words[k] & 0xffff));  // little-endian (x, y) pair
    sy[k] = words[k] >> 16;                  // arithmetic shift: the signed y
    inside[k] = k < n && unsigned(sx[k]) < unsigned(J.width) && unsigned(sy[k]) < unsigned(J.height);
  }
  uint8_t* dst_row = J.dst + size_t(row) * J.dst_pitch;
  if (J.channels == 1) {
    // cv::remap, then image_ += short(offset) with saturation (azure_kinect_camera.cpp:338-341)
    unsigned v[kUndistortPixels];
#pragma unroll
    for (int k = 0; k < kUndistortPixels; ++k) {
      int raw = 0;
      if (inside[k])
        raw = __ldg(reinterpret_cast<const uint16_t*>(J.src + size_t(sy[k]) * J.src_pitch) + sx[k]);
      v[k] = unsigned(min(max(raw + J.offset, 0), 65535));
    }
    uint16_t* d = reinterpret_cast<uint16_t*>(dst_row) + x0;
    if (n == kUndistortPixels) {
      *reinterpret_cast<uint2*>(d) = make_uint2(v[0] | (v[1] << 16), v[2] | (v[3] << 16));  // 8-B aligned: x0 % 4 == 0
    } else {
      for (int k = 0; k < n; ++k) d[k] = uint16_t(v[k]);
    }
    return;
  }
  // colour: B, G, R of each raw pixel (COLOR_RGBA2RGB drops byte 3 of a BGRA32 pixel and keeps the order)
  const bool words4 = J.channels == 4 && ((reinterpret_cast<uintptr_t>(J.src) | J.src_pitch) & 3u) == 0;
  unsigned px[kUndistortPixels];
#pragma unroll
  for (int k = 0; k < kUndistortPixels; ++k) {
    px[k] = 0;
    if (inside[k]) {
      const uint8_t* p = J.src + size_t(sy[k]) * J.src_pitch + size_t(sx[k]) * J.channels;
      if (words4) {
        px[k] = __ldg(reinterpret_cast<const unsigned*>(p)) & 0xffffffu;
      } else {
        px[k] = unsigned(__ldg(p)) | (unsigned(__ldg(p + 1)) << 8) | (unsigned(__ldg(p + 2)) << 16);
      }
    }
  }
  uint8_t* d = dst_row + size_t(x0) * 3;
  if (n == kUndistortPixels) {  // 12 B at a multiple of 12 from a 16-B aligned row: three aligned words
    unsigned* w = reinterpret_cast<unsigned*>(d);
    w[0] = px[0] | (px[1] << 24);
    w[1] = (px[1] >> 8) | (px[2] << 16);
    w[2] = (px[2] >> 16) | (px[3] << 8);
  } else {
    for (int k = 0; k < n; ++k) {
      d[3 * k] = uint8_t(px[k]);
      d[3 * k + 1] = uint8_t(px[k] >> 8);
      d[3 * k + 2] = uint8_t(px[k] >> 16);
    }
  }
}

namespace {

// cvRound(float) as the x86 conversion performs it (round half to even; NaN and values outside int give INT_MIN),
// then saturate_cast<short>: what convertMaps(CV_16SC2, nninterpolation = true) stores.
int16_t RoundToShort(float f) {
  int i = INT_MIN;
  if (f >= -2147483648.0f && f < 2147483648.0f) i = int(std::nearbyint(f));
  return int16_t(i < SHRT_MIN ? SHRT_MIN : i > SHRT_MAX ? SHRT_MAX : i);
}

}  // namespace

// initUndistortRectifyMap (OpenCV undistort.dispatch.cpp / undistort.simd.hpp) in float64, one rounding per operation
// in the order OpenCV evaluates it (x86-64 host code has no fused multiply-add, so nothing is contracted):
//  - iR = newCameraMatrix^-1 by the 3x3 cofactor formula Mat::inv(DECOMP_LU) uses for 3x3 matrices;
//  - the homogeneous ray of pixel (j, i) is (i*ir[1] + ir[2] + j*ir[0], ...), the rational / tangential model applied;
//  - the float32 map value is (float)(fx * xd + cx); convertMaps then rounds it to int16.
// Checked against cv2 4.13 by tests/test_undistortion_map.py.
void UndistortionMap(const double camera[4], const double k[8], const double new_camera[4], int width, int height,
                     int16_t* map_xy, size_t map_pitch) {
  const double S[3][3] = {{new_camera[0], 0.0, new_camera[2]}, {0.0, new_camera[1], new_camera[3]}, {0.0, 0.0, 1.0}};
  double d = S[0][0] * (S[1][1] * S[2][2] - S[2][1] * S[1][2]) - S[0][1] * (S[1][0] * S[2][2] - S[2][0] * S[1][2]) +
             S[0][2] * (S[1][0] * S[2][1] - S[2][0] * S[1][1]);
  d = 1.0 / d;
  const double ir[9] = {(S[1][1] * S[2][2] - S[1][2] * S[2][1]) * d, (S[0][2] * S[2][1] - S[0][1] * S[2][2]) * d,
                        (S[0][1] * S[1][2] - S[0][2] * S[1][1]) * d, (S[1][2] * S[2][0] - S[1][0] * S[2][2]) * d,
                        (S[0][0] * S[2][2] - S[0][2] * S[2][0]) * d, (S[0][2] * S[1][0] - S[0][0] * S[1][2]) * d,
                        (S[1][0] * S[2][1] - S[1][1] * S[2][0]) * d, (S[0][1] * S[2][0] - S[0][0] * S[2][1]) * d,
                        (S[0][0] * S[1][1] - S[0][1] * S[1][0]) * d};
  const double fx = camera[0], fy = camera[1], u0 = camera[2], v0 = camera[3];
  const double k1 = k[0], k2 = k[1], p1 = k[2], p2 = k[3], k3 = k[4], k4 = k[5], k5 = k[6], k6 = k[7];
  for (int i = 0; i < height; ++i) {
    int16_t* out = reinterpret_cast<int16_t*>(reinterpret_cast<uint8_t*>(map_xy) + size_t(i) * map_pitch);
    const double _x = i * ir[1] + ir[2], _y = i * ir[4] + ir[5], _w = i * ir[7] + ir[8];
    for (int j = 0; j < width; ++j) {
      const double w = 1.0 / (_w + j * ir[6]);
      const double x = (_x + j * ir[0]) * w, y = (_y + j * ir[3]) * w;
      const double x2 = x * x, y2 = y * y;
      const double r2 = x2 + y2, _2xy = 2 * x * y;
      const double kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1 + ((k6 * r2 + k5) * r2 + k4) * r2);
      const double xd = x * kr + p1 * _2xy + p2 * (r2 + 2 * x2);
      const double yd = y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy;
      out[2 * j] = RoundToShort(float(fx * xd + u0));
      out[2 * j + 1] = RoundToShort(float(fy * yd + v0));
    }
  }
}

}  // namespace m3tb

extern "C" int m3tb_undistortion_map(const m3tb_intrinsics* raw, const float distortion[8],
                                     const m3tb_intrinsics* rectified, int16_t* map_xy, size_t map_pitch) {
  if (!raw || !distortion || !rectified || !map_xy) return M3TB_ERR_INVALID;
  if (raw->width != rectified->width || raw->height != rectified->height || raw->width <= 0 || raw->height <= 0)
    return M3TB_ERR_INVALID;
  if (map_pitch < 4 * size_t(raw->width)) return M3TB_ERR_INVALID;
  for (const m3tb_intrinsics* c : {raw, rectified}) {
    if (!std::isfinite(c->fu) || !std::isfinite(c->fv) || !std::isfinite(c->ppu) || !std::isfinite(c->ppv))
      return M3TB_ERR_INVALID;
    if (!(c->fu > 0.0f) || !(c->fv > 0.0f) || c->ppu < 0.0f || c->ppv < 0.0f) return M3TB_ERR_INVALID;
  }
  double k[8];
  for (int i = 0; i < 8; ++i) {
    if (!std::isfinite(distortion[i])) return M3TB_ERR_INVALID;
    k[i] = distortion[i];
  }
  // cv::Mat1f camera matrices, converted to double inside initUndistortRectifyMap
  const double camera[4] = {raw->fu, raw->fv, raw->ppu, raw->ppv};
  const double new_camera[4] = {rectified->fu, rectified->fv, rectified->ppu, rectified->ppv};
  m3tb::UndistortionMap(camera, k, new_camera, raw->width, raw->height, map_xy, map_pitch);
  return M3TB_OK;
}
