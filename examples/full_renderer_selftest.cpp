// full_renderer_selftest.cpp — the C++ mirror's FullBasicDepthRenderer, FullSilhouetteRenderer and FullNormalRenderer
// on one scene, with the reference's structural rules (renderer_test.cpp: StartRendering before SetUp fails, a fetch
// before a render fails). Writes the three images and prints one JSON line with Depth / DepthImageValue / PointVector /
// SilhouetteValue at the requested pixels (floats with 9 significant digits, so float32 values round-trip).
//
//   full_renderer_selftest <spec>
//   spec: n_bodies, then per body "<triangles.f32> geometry2body[12] diameter culling body_id region_id
//         body2world[12]"; "fu fv ppu ppv width height"; world2camera[12]; "z_min z_max id_type(0 body, 1 region)";
//         n_points, then "x y" per point; the output directory (depth.u16, silhouette.u8, normal.u8 are written there)
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
static bool WriteRaw(const std::string& path, const std::vector<T>& v) {
  std::ofstream f(path, std::ios::binary);
  f.write(reinterpret_cast<const char*>(v.data()), std::streamsize(v.size() * sizeof(T)));
  return bool(f);
}

int main(int argc, char** argv) {
  if (argc != 2) {
    std::cerr << "usage: full_renderer_selftest <spec>" << std::endl;
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
    std::ifstream tf(tri_path, std::ios::binary | std::ios::ate);
    std::vector<float> tri(size_t(tf.tellg()) / sizeof(float));
    tf.seekg(0);
    tf.read(reinterpret_cast<char*>(tri.data()), std::streamsize(tri.size() * sizeof(float)));
    auto body = std::make_shared<Body>("body" + std::to_string(b), batch);
    body->set_geometry_triangles(tri);
    body->set_geometry2body_pose(g2b);
    body->set_maximum_body_diameter(diameter);
    body->set_geometry_enable_culling(culling != 0);
    body->set_body_id(uint8_t(body_id));
    body->set_region_id(uint8_t(region_id));
    bodies.push_back(body);
    poses.push_back(pose);
  }
  Intrinsics intr{};
  spec >> intr.fu >> intr.fv >> intr.ppu >> intr.ppv >> intr.width >> intr.height;
  Transform3fA w2c;
  ReadPose(spec, w2c);
  float z_min, z_max;
  int id_type;
  spec >> z_min >> z_max >> id_type;
  int n_points;
  spec >> n_points;
  std::vector<Point2i> points(n_points);
  for (auto& p : points) spec >> p.x >> p.y;
  std::string out_dir;
  spec >> out_dir;
  if (!spec) return 4;

  auto camera = std::make_shared<ColorCamera>("camera", batch, intr, w2c);
  FullBasicDepthRenderer depth_renderer("depth_renderer", batch, geometry, camera, z_min, z_max);
  FullSilhouetteRenderer silhouette_renderer("silhouette_renderer", batch, geometry, camera, IDType(id_type), z_min,
                                             z_max);
  FullNormalRenderer normal_renderer("normal_renderer", batch, geometry, camera, z_min, z_max);
  // structural rules before anything is set up (renderer_test.cpp: TestWithoutSetUp)
  const bool start_before_setup_fails = !depth_renderer.StartRendering();
  const bool fetch_before_setup_fails = !silhouette_renderer.FetchSilhouetteImage() &&
                                        !silhouette_renderer.FetchDepthImage();
  const bool setup_without_camera_fails = !depth_renderer.SetUp();  // the camera is not set up yet
  if (!camera->SetUp()) return 5;
  for (int b = 0; b < n_bodies; ++b) {
    if (!geometry->AddBody(bodies[b])) return 6;
    if (!bodies[b]->set_body2world_pose(poses[b])) return 6;
  }
  const bool setup_without_geometry_setup_fails = !depth_renderer.SetUp();  // RendererGeometry::SetUp not called
  geometry->SetUp();
  if (!depth_renderer.SetUp() || !silhouette_renderer.SetUp() || !normal_renderer.SetUp()) return 7;
  // renderer_test.cpp: TestWithoutRendering
  const bool fetch_before_render_fails = !silhouette_renderer.FetchSilhouetteImage() &&
                                         !depth_renderer.FetchDepthImage() && !normal_renderer.FetchNormalImage();
  if (!depth_renderer.StartRendering() || !silhouette_renderer.StartRendering() || !normal_renderer.StartRendering())
    return 8;
  if (!depth_renderer.FetchDepthImage() || !silhouette_renderer.FetchSilhouetteImage() ||
      !normal_renderer.FetchNormalImage())
    return 9;
  if (!WriteRaw(out_dir + "/depth.u16", depth_renderer.depth_image()) ||
      !WriteRaw(out_dir + "/silhouette.u8", silhouette_renderer.silhouette_image()) ||
      !WriteRaw(out_dir + "/normal.u8", normal_renderer.normal_image()))
    return 10;
  std::printf("{\"ok\": 1, \"start_before_setup_fails\": %d, \"fetch_before_setup_fails\": %d, "
              "\"setup_without_camera_fails\": %d, \"setup_without_geometry_setup_fails\": %d, "
              "\"fetch_before_render_fails\": %d, \"projection_terms\": [%.9g, %.9g], \"points\": [",
              int(start_before_setup_fails), int(fetch_before_setup_fails), int(setup_without_camera_fails),
              int(setup_without_geometry_setup_fails), int(fetch_before_render_fails),
              double(depth_renderer.projection_term_a()), double(depth_renderer.projection_term_b()));
  for (int k = 0; k < n_points; ++k) {
    const Point2i& p = points[k];
    const uint16_t value = depth_renderer.DepthImageValue(p);
    const auto v = depth_renderer.PointVector(p);
    std::printf("%s{\"value\": %d, \"depth_of_value\": %.9g, \"depth\": %.9g, \"point\": [%.9g, %.9g, %.9g], "
                "\"silhouette\": %d}",
                k ? ", " : "", int(value), double(depth_renderer.Depth(value)), double(depth_renderer.Depth(p)),
                double(v[0]), double(v[1]), double(v[2]), int(silhouette_renderer.SilhouetteValue(p)));
  }
  std::printf("]}\n");
  return 0;
}
