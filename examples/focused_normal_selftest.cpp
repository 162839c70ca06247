// focused_normal_selftest.cpp — the C++ mirror's FocusedNormalRenderer, FullDepthRenderer::NormalizedDepthImage,
// DepthCamera::NormalizedDepthImage and the image viewers (ImageColorViewer / ImageDepthViewer, updated by
// Tracker::UpdateViewers next to a NormalColorViewer) on one scene, with the reference's structural rules
// (StartRendering before SetUp fails, a fetch before a render fails, SetUp without referenced bodies fails). Writes the
// images and prints one JSON line with the focus, the visible flags, NormalImageValue / NormalVector at the requested
// camera pixels and NormalVector of the requested byte values (floats with 9 significant digits, so float32 values
// round-trip).
//
//   focused_normal_selftest <spec>
//   spec: n_bodies, then per body "<triangles.f32> geometry2body[12] diameter culling body_id region_id
//         body2world[12]"; "fu fv ppu ppv width height" of the colour camera; its world2camera[12]; the same two lines
//         of the depth camera and its depth_scale; "<colour frame.u8 (BGR)> <depth frame.u16>";
//         "image_size z_min z_max"; n_referenced, then the referenced body indices; "min_depth max_depth" of the
//         normalised depth images; n_points, then "x y" per colour-camera pixel; n_values, then "b g r a" per byte
//         value; the output directory
#include <cstdio>
#include <fstream>
#include <iostream>
#include <memory>
#include <string>
#include <vector>

#include "m3t_b200/m3t_b200.hpp"

using namespace m3t_b200;

static bool ReadPose(std::istream& in, Transform3fA& p) {
  for (float& v : p.m) in >> v;
  return bool(in);
}

template <typename T>
static std::vector<T> ReadRaw(const std::string& path) {
  std::ifstream f(path, std::ios::binary | std::ios::ate);
  std::vector<T> v(size_t(f.tellg()) / sizeof(T));
  f.seekg(0);
  f.read(reinterpret_cast<char*>(v.data()), std::streamsize(v.size() * sizeof(T)));
  return v;
}

template <typename T>
static bool WriteRaw(const std::string& path, const std::vector<T>& v) {
  std::ofstream f(path, std::ios::binary);
  f.write(reinterpret_cast<const char*>(v.data()), std::streamsize(v.size() * sizeof(T)));
  return bool(f);
}

static void PrintVector(const std::array<float, 3>& n) {
  std::printf("[%.9g, %.9g, %.9g]", double(n[0]), double(n[1]), double(n[2]));
}

int main(int argc, char** argv) {
  if (argc != 2) {
    std::cerr << "usage: focused_normal_selftest <spec>" << std::endl;
    return 2;
  }
  std::ifstream spec(argv[1]);
  int n_bodies = 0;
  spec >> n_bodies;
  auto batch = std::make_shared<Batch>(0, n_bodies, 1, 1);
  if (!batch->ok()) return 3;
  auto geometry = std::make_shared<RendererGeometry>("renderer_geometry", batch);
  std::vector<std::shared_ptr<Body>> bodies;
  std::vector<Transform3fA> poses;
  for (int b = 0; b < n_bodies; ++b) {
    std::string tri_path;
    Transform3fA g2b, pose;
    float diameter;
    int culling, body_id, region_id;
    spec >> tri_path;
    ReadPose(spec, g2b);
    spec >> diameter >> culling >> body_id >> region_id;
    ReadPose(spec, pose);
    auto body = std::make_shared<Body>("body" + std::to_string(b), batch);
    body->set_geometry_triangles(ReadRaw<float>(tri_path));
    body->set_geometry2body_pose(g2b);
    body->set_maximum_body_diameter(diameter);
    body->set_geometry_enable_culling(culling != 0);
    body->set_body_id(uint8_t(body_id));
    body->set_region_id(uint8_t(region_id));
    bodies.push_back(body);
    poses.push_back(pose);
  }
  Intrinsics color_intr{}, depth_intr{};
  Transform3fA color_w2c, depth_w2c;
  float depth_scale;
  spec >> color_intr.fu >> color_intr.fv >> color_intr.ppu >> color_intr.ppv >> color_intr.width >> color_intr.height;
  ReadPose(spec, color_w2c);
  spec >> depth_intr.fu >> depth_intr.fv >> depth_intr.ppu >> depth_intr.ppv >> depth_intr.width >> depth_intr.height;
  ReadPose(spec, depth_w2c);
  spec >> depth_scale;
  std::string color_path, depth_path;
  spec >> color_path >> depth_path;
  int image_size, n_referenced;
  float z_min, z_max, min_depth, max_depth;
  spec >> image_size >> z_min >> z_max >> n_referenced;
  std::vector<int> referenced(n_referenced);
  for (int& r : referenced) spec >> r;
  spec >> min_depth >> max_depth;
  int n_points, n_values;
  spec >> n_points;
  std::vector<Point2i> points(n_points);
  for (auto& p : points) spec >> p.x >> p.y;
  spec >> n_values;
  std::vector<Vec4b> values(n_values);
  for (auto& v : values)
    for (auto& c : v) {
      int x;
      spec >> x;
      c = uint8_t(x);
    }
  std::string out_dir;
  spec >> out_dir;
  if (!spec) return 4;

  auto color_camera = std::make_shared<ColorCamera>("color_camera", batch, color_intr, color_w2c);
  auto depth_camera = std::make_shared<DepthCamera>("depth_camera", batch, depth_intr, depth_w2c, depth_scale);
  FocusedNormalRenderer renderer("focused_normal_renderer", batch, geometry, color_camera, image_size, z_min, z_max);
  FullBasicDepthRenderer full_renderer("full_renderer", batch, geometry, color_camera, z_min, z_max);
  // structural rules before anything is set up
  const bool start_before_setup_fails = !renderer.StartRendering();
  const bool fetch_before_setup_fails = !renderer.FetchNormalImage() && !renderer.FetchDepthImage();
  if (!color_camera->SetUp() || !depth_camera->SetUp()) return 5;
  for (int b = 0; b < n_bodies; ++b) {
    if (!geometry->AddBody(bodies[b])) return 6;
    if (!bodies[b]->set_body2world_pose(poses[b])) return 6;
  }
  geometry->SetUp();
  const bool setup_without_referenced_fails = !renderer.SetUp();
  for (int r : referenced)
    if (!renderer.AddReferencedBody(bodies[r])) return 7;
  if (!renderer.SetUp() || !full_renderer.SetUp()) return 7;
  const bool fetch_before_render_fails = !renderer.FetchNormalImage() && !renderer.FetchDepthImage();
  if (!renderer.StartRendering() || !renderer.FetchNormalImage() || !renderer.FetchDepthImage()) return 8;
  if (!full_renderer.StartRendering()) return 8;

  // the frames, the image viewers and a normal viewer, updated together by the tracker
  const std::vector<uint8_t> color_frame = ReadRaw<uint8_t>(color_path);
  const std::vector<uint16_t> depth_frame = ReadRaw<uint16_t>(depth_path);
  if (!color_camera->UpdateImage(color_frame.data(), size_t(color_intr.width) * 3) ||
      !depth_camera->UpdateImage(depth_frame.data(), size_t(depth_intr.width) * 2))
    return 9;
  auto image_color_viewer = std::make_shared<ImageColorViewer>("image_color_viewer", color_camera);
  auto image_depth_viewer = std::make_shared<ImageDepthViewer>("image_depth_viewer", depth_camera, min_depth, max_depth);
  auto normal_viewer = std::make_shared<NormalColorViewer>("normal_viewer", batch, color_camera, geometry);
  const bool update_before_setup_fails = !image_depth_viewer->UpdateViewer(0);
  Tracker tracker("tracker", batch);
  if (!tracker.AddViewer(image_color_viewer) || !tracker.AddViewer(image_depth_viewer) ||
      !tracker.AddViewer(normal_viewer))
    return 10;
  if (!tracker.SetUp() || !tracker.UpdateViewers(0)) return 10;

  const std::vector<uint8_t> camera_normalized = depth_camera->NormalizedDepthImage(min_depth, max_depth);
  const std::vector<uint8_t> full_normalized = full_renderer.NormalizedDepthImage(min_depth, max_depth);
  if (camera_normalized.empty() || full_normalized.empty()) return 11;
  if (!WriteRaw(out_dir + "/focused_depth.u16", renderer.focused_depth_image()) ||
      !WriteRaw(out_dir + "/focused_normal.u8", renderer.focused_normal_image()) ||
      !WriteRaw(out_dir + "/camera_normalized.u8", camera_normalized) ||
      !WriteRaw(out_dir + "/full_normalized.u8", full_normalized) ||
      !WriteRaw(out_dir + "/image_color_viewer.u8", image_color_viewer->image()) ||
      !WriteRaw(out_dir + "/image_depth_viewer.u8", image_depth_viewer->image()) ||
      !WriteRaw(out_dir + "/normal_viewer.u8", normal_viewer->image()))
    return 12;

  std::printf("{\"ok\": 1, \"start_before_setup_fails\": %d, \"fetch_before_setup_fails\": %d, "
              "\"setup_without_referenced_fails\": %d, \"fetch_before_render_fails\": %d, "
              "\"update_before_setup_fails\": %d, \"focus\": [%.9g, %.9g, %.9g, %.9g, %.9g], \"visible\": [",
              int(start_before_setup_fails), int(fetch_before_setup_fails), int(setup_without_referenced_fails),
              int(fetch_before_render_fails), int(update_before_setup_fails), double(renderer.corner_u()),
              double(renderer.corner_v()), double(renderer.scale()), double(renderer.projection_term_a()),
              double(renderer.projection_term_b()));
  for (int k = 0; k < n_bodies; ++k)
    std::printf("%s%d", k ? ", " : "", int(renderer.IsBodyVisible(bodies[k]->name())));
  std::printf("], \"points\": [");
  for (int k = 0; k < n_points; ++k) {
    const Vec4b v = renderer.NormalImageValue(points[k]);
    std::printf("%s{\"value\": [%d, %d, %d, %d], \"normal\": ", k ? ", " : "", v[0], v[1], v[2], v[3]);
    PrintVector(renderer.NormalVector(points[k]));
    std::printf("}");
  }
  std::printf("], \"values\": [");
  for (int k = 0; k < n_values; ++k) {
    std::printf("%s", k ? ", " : "");
    PrintVector(renderer.NormalVector(values[k]));
  }
  std::printf("]}\n");
  return 0;
}
