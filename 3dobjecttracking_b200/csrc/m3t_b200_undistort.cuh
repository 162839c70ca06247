// m3t_b200_undistort.cuh — undistortion of raw camera frames as they are uploaded (AzureKinectColorCamera /
// AzureKinectDepthCamera::UpdateImage, azure_kinect_camera.cpp:175-195, 321-345): cv::remap with INTER_NEAREST and
// BORDER_CONSTANT through a CV_16SC2 map, the colour frame's fourth byte dropped (COLOR_RGBA2RGB on BGRA32), the depth
// offset added with saturation. DESIGN.md §3 "k_undistort" states what is computed.
#pragma once

#include <cstddef>
#include <cstdint>

namespace m3tb {

constexpr int kUndistortThreads = 256;
constexpr int kUndistortPixels = 4;    // consecutive output pixels per thread: 16 B of map in
constexpr int kUndistortMaxJobs = 64;  // frames per launch (the jobs travel in the kernel parameters)

// One frame to rectify.
struct UndistortJob {
  const int16_t* map;     // [height][width] (x, y) int16 pairs, rows map_pitch bytes apart (a multiple of 16)
  const uint8_t* src;     // raw frame: `channels` bytes per colour pixel, or u16 depth
  uint8_t* dst;           // rectified frame: BGR8 or u16, rows dst_pitch bytes apart (a multiple of 16)
  unsigned map_pitch, src_pitch, dst_pitch;  // bytes
  int width, height;      // of the raw and of the rectified frame
  int channels;           // 3 or 4: colour; 1: depth
  int offset;             // depth only: added to every pixel, the result clamped to 0 .. 65535
};

struct UndistortArgs {
  UndistortJob jobs[kUndistortMaxJobs];
  int n_jobs;
};

// grid: (ceil(max over jobs of ceil(width / 4) * height / kUndistortThreads), n_jobs)
__global__ void k_undistort(const __grid_constant__ UndistortArgs a);

// Host restatement of initUndistortRectifyMap(CV_32FC1) + convertMaps(CV_16SC2, nninterpolation = true) with R = I
// (the body of m3tb_undistortion_map; arguments already checked). `camera` / `new_camera`: fx, fy, cx, cy.
void UndistortionMap(const double camera[4], const double coefficients[8], const double new_camera[4], int width,
                     int height, int16_t* map_xy, size_t map_pitch);

}  // namespace m3tb
