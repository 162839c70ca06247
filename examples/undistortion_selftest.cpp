// undistortion_selftest.cpp — the C++ mirror's AzureKinectColorCamera / AzureKinectDepthCamera without the SDK.
// Host checks (no device needed): the intrinsics rule of GetIntrinsicsAndDistortionMap, the depth value offset
// short(depth_offset / depth_scale), the refusals of m3tb_undistortion_map and of SetUp / UpdateImage. With a device it
// also rectifies one synthetic BGRA and one depth frame and writes the raw and the rectified frames to <out_dir>
// (color_raw.bin, color_image.bin, depth_raw.bin, depth_image.bin). Prints one JSON line; exit status 0 when every
// host check passed (and, with a device, every device step succeeded).
//
//   undistortion_selftest <out_dir>
#include <cmath>
#include <cstdio>
#include <fstream>
#include <iostream>
#include <limits>
#include <memory>
#include <string>
#include <vector>

#include "m3t_b200/m3t_b200.hpp"

using namespace m3t_b200;

template <typename T>
static bool WriteRaw(const std::string& path, const std::vector<T>& v) {
  std::ofstream f(path, std::ios::binary);
  f.write(reinterpret_cast<const char*>(v.data()), std::streamsize(v.size() * sizeof(T)));
  return bool(f);
}

static void PrintCalibration(const char* key, const AzureKinectCalibration& c, const Intrinsics& in, int offset) {
  std::printf("\"%s\": {\"width\": %d, \"height\": %d, \"fx\": %.9g, \"fy\": %.9g, \"cx\": %.9g, \"cy\": %.9g, "
              "\"fu\": %.9g, \"fv\": %.9g, \"coefficients\": [%.9g, %.9g, %.9g, %.9g, %.9g, %.9g, %.9g, %.9g], "
              "\"depth_value_offset\": %d}",
              key, c.width, c.height, double(c.fx), double(c.fy), double(c.cx), double(c.cy), double(in.fu),
              double(in.fv), double(c.k1), double(c.k2), double(c.p1), double(c.p2), double(c.k3), double(c.k4),
              double(c.k5), double(c.k6), offset);
}

int main(int argc, char** argv) {
  if (argc != 2) {
    std::cerr << "usage: undistortion_selftest <out_dir>" << std::endl;
    return 2;
  }
  const std::string out_dir = argv[1];
  int failed = 0;
  auto expect = [&](bool ok, const char* what) {
    if (!ok) {
      std::cerr << "FAILED: " << what << std::endl;
      ++failed;
    }
  };

  AzureKinectCalibration color;
  color.fx = 303.1f; color.fy = 302.9f; color.cx = 158.7f; color.cy = 91.4f;
  color.k1 = 0.52f; color.k2 = -2.61f; color.k3 = 1.45f; color.k4 = 0.40f; color.k5 = -2.43f; color.k6 = 1.38f;
  color.p1 = 6e-4f; color.p2 = -3e-4f;
  color.width = 320; color.height = 180;
  AzureKinectCalibration depth;
  depth.fx = 126.1f; depth.fy = 126.0f; depth.cx = 79.6f; depth.cy = 84.2f;
  depth.k1 = 3.12f; depth.k2 = 1.88f; depth.k3 = 0.09f; depth.k4 = 3.45f; depth.k5 = 2.85f; depth.k6 = 0.48f;
  depth.p1 = 4e-5f; depth.p2 = -1e-5f;
  depth.width = 160; depth.height = 144;

  // ---- host checks ----
  {  // GetIntrinsicsAndDistortionMap: fu / fv scaled in float, ppu / ppv and the size kept
    Intrinsics in{};
    std::vector<int16_t> map;
    expect(AzureKinectIntrinsicsAndDistortionMap(color, 1.05f, &in, &map), "intrinsics and map");
    expect(in.fu == color.fx * 1.05f && in.fv == color.fy * 1.05f && in.ppu == color.cx && in.ppv == color.cy &&
               in.width == color.width && in.height == color.height,
           "intrinsics rule");
    expect(map.size() == size_t(color.width) * color.height * 2, "map size");
    // all-zero coefficients at image_scale 1: the exact identity
    AzureKinectCalibration plain = color;
    plain.k1 = plain.k2 = plain.k3 = plain.k4 = plain.k5 = plain.k6 = plain.p1 = plain.p2 = 0.0f;
    expect(AzureKinectIntrinsicsAndDistortionMap(plain, 1.0f, &in, &map), "identity map");
    bool identity = true;
    for (int v = 0; v < plain.height; ++v)
      for (int u = 0; u < plain.width; ++u)
        identity = identity && map[2 * (size_t(v) * plain.width + u)] == u &&
                   map[2 * (size_t(v) * plain.width + u) + 1] == v;
    expect(identity, "zero coefficients give the identity");
  }
  {  // refusals of m3tb_undistortion_map
    const Intrinsics good{100.0f, 100.0f, 50.0f, 40.0f, 100, 80};
    const float k[8] = {0.1f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    std::vector<int16_t> map(100 * 80 * 2);
    Intrinsics other = good;
    other.width = 99;
    expect(m3tb_undistortion_map(&good, k, &other, map.data(), 400) == M3TB_ERR_INVALID, "size mismatch refused");
    other = good;
    other.fu = std::numeric_limits<float>::quiet_NaN();
    expect(m3tb_undistortion_map(&good, k, &other, map.data(), 400) == M3TB_ERR_INVALID, "NaN intrinsics refused");
    other = good;
    other.fv = 0.0f;
    expect(m3tb_undistortion_map(&other, k, &good, map.data(), 400) == M3TB_ERR_INVALID, "zero focal length refused");
    float bad_k[8] = {0.1f, 0.0f, 0.0f, 0.0f, 0.0f, INFINITY, 0.0f, 0.0f};
    expect(m3tb_undistortion_map(&good, bad_k, &good, map.data(), 400) == M3TB_ERR_INVALID, "inf coefficient refused");
    expect(m3tb_undistortion_map(&good, k, &good, map.data(), 399) == M3TB_ERR_INVALID, "small pitch refused");
    expect(m3tb_undistortion_map(&good, k, &good, nullptr, 400) == M3TB_ERR_INVALID, "null map refused");
    expect(m3tb_undistortion_map(&good, k, &good, map.data(), 400) == M3TB_OK, "valid arguments accepted");
  }

  // ---- cameras ----
  auto batch = std::make_shared<Batch>(0, 1, 1, 1);
  const bool device = batch->ok();
  AzureKinectColorCamera color_camera("azure_kinect_color", batch, color, 1.05f);
  AzureKinectDepthCamera depth_camera("azure_kinect_depth", batch, depth, 1.0f, -0.0375f, 0.001f);
  AzureKinectDepthCamera far_camera("azure_kinect_depth_far", batch, depth, 1.0f, 40.0f, 0.001f);
  {  // short(depth_offset / depth_scale), truncated; outside the range of short refused
    int offset = 0;
    expect(depth_camera.depth_value_offset(&offset) && offset == int(short(-0.0375f / 0.001f)), "depth value offset");
    expect(!far_camera.depth_value_offset(&offset) && !far_camera.SetUp(), "depth offset outside short refused");
  }
  std::vector<uint8_t> color_raw(size_t(color.width) * color.height * 4);
  std::vector<uint16_t> depth_raw(size_t(depth.width) * depth.height);
  for (size_t i = 0; i < color_raw.size(); ++i) color_raw[i] = uint8_t((i * 2654435761u) >> 13);
  for (size_t i = 0; i < depth_raw.size(); ++i) depth_raw[i] = uint16_t(i % 97 == 0 ? 0 : 400 + (i * 40503u) % 3000);
  expect(!color_camera.UpdateImage(color_raw.data(), size_t(color.width) * 4), "UpdateImage before SetUp fails");

  bool device_ok = true;
  if (device) {
    device_ok = color_camera.SetUp() && depth_camera.SetUp() &&
                color_camera.UpdateImage(color_raw.data(), size_t(color.width) * 4) &&
                depth_camera.UpdateImage(reinterpret_cast<const uint8_t*>(depth_raw.data()), size_t(depth.width) * 2);
    std::vector<uint8_t> color_image(size_t(color.width) * color.height * 3);
    std::vector<uint16_t> depth_image(size_t(depth.width) * depth.height);
    device_ok = device_ok &&
                m3tb_get_camera_image(batch->ctx(), 0, color_camera.index(), color_image.data(),
                                      size_t(color.width) * 3) == M3TB_OK &&
                m3tb_get_camera_image(batch->ctx(), 1, depth_camera.index(), depth_image.data(),
                                      size_t(depth.width) * 2) == M3TB_OK;
    device_ok = device_ok && WriteRaw(out_dir + "/color_raw.bin", color_raw) &&
                WriteRaw(out_dir + "/color_image.bin", color_image) && WriteRaw(out_dir + "/depth_raw.bin", depth_raw) &&
                WriteRaw(out_dir + "/depth_image.bin", depth_image);
  }
  int offset = 0;
  depth_camera.depth_value_offset(&offset);
  std::printf("{\"host_checks_failed\": %d, \"device\": %d, \"device_ok\": %d, ", failed, int(device), int(device_ok));
  Intrinsics ci{}, di{};
  std::vector<int16_t> scratch;
  AzureKinectIntrinsicsAndDistortionMap(color, color_camera.image_scale(), &ci, &scratch);
  AzureKinectIntrinsicsAndDistortionMap(depth, depth_camera.image_scale(), &di, &scratch);
  PrintCalibration("color", color, ci, 0);
  std::printf(", ");
  PrintCalibration("depth", depth, di, offset);
  std::printf("}\n");
  return failed == 0 && device_ok ? 0 : 1;
}
