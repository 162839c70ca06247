// region_model_save_selftest.cpp — RegionModel::AddAssociatedBody / GenerateModel / SaveModel of the C++ mirror,
// driven by a spec file so that a test can compare the written .bin with 3dobjecttracking_b200/model_io.py's writer
// byte for byte.
//
// spec (whitespace separated):
//   mode out_path                       mode: "save" (views from an existing .bin) | "generate" (on the device)
//   sphere_radius n_divides n_points max_radius_depth_offset stride_depth_offset image_size
//   n_bodies                            the body, then its associated bodies in insertion order
//   n_bodies x: geometry_path unit_in_meter counterclockwise enable_culling maximum_body_diameter geometry2body[12]
//               movable same_region     (ignored for the body)
//               triangle_file           raw float32 [n][3][3] soup, or "-" (not needed to save)
//   save only: model_path view_block_offset n_views
// Prints one JSON line {"ok": 0 | 1}.
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <memory>
#include <string>
#include <vector>

#include "m3t_b200/m3t_b200.hpp"

using namespace m3t_b200;

int main(int argc, char** argv) {
  if (argc != 2) {
    std::fprintf(stderr, "usage: %s SPEC\n", argv[0]);
    return 2;
  }
  std::ifstream spec(argv[1]);
  std::string mode, out;
  float sphere_radius, max_radius, stride;
  int n_divides, n_points, image_size, n_bodies;
  spec >> mode >> out >> sphere_radius >> n_divides >> n_points >> max_radius >> stride >> image_size >> n_bodies;
  auto batch = std::make_shared<Batch>(0, n_bodies, 1, 1);  // without a device only "save" can work
  std::vector<std::shared_ptr<Body>> bodies;
  std::vector<int> movable(n_bodies), same_region(n_bodies);
  for (int k = 0; k < n_bodies; ++k) {
    std::string path, tri_file;
    float unit, diameter;
    int ccw, cull;
    Transform3fA g2b;
    spec >> path >> unit >> ccw >> cull >> diameter;
    for (int i = 0; i < 12; ++i) spec >> g2b.m[i];
    spec >> movable[k] >> same_region[k] >> tri_file;
    auto body = std::make_shared<Body>("body" + std::to_string(k), batch);
    body->set_geometry_path(path);
    body->set_geometry_unit_in_meter(unit);
    body->set_geometry_counterclockwise(ccw != 0);
    body->set_geometry_enable_culling(cull != 0);
    body->set_maximum_body_diameter(diameter);
    body->set_geometry2body_pose(g2b);
    if (tri_file != "-") {
      std::ifstream f(tri_file, std::ios::binary);
      std::vector<char> raw((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
      std::vector<float> tri(raw.size() / sizeof(float));
      std::memcpy(tri.data(), raw.data(), tri.size() * sizeof(float));
      body->set_geometry_triangles(tri);
    }
    bodies.push_back(body);
  }
  RegionModel model("region_model", batch, bodies[0]);
  model.set_sphere_radius(sphere_radius);
  model.set_n_divides(n_divides);
  model.set_n_points(n_points);
  model.set_max_radius_depth_offset(max_radius);
  model.set_stride_depth_offset(stride);
  model.set_image_size(image_size);
  bool ok = true;
  for (int k = 1; k < n_bodies; ++k) ok = ok && model.AddAssociatedBody(bodies[k], movable[k] != 0, same_region[k] != 0);
  if (n_bodies > 1) ok = ok && !model.AddAssociatedBody(bodies[1], true, true);  // a second time is refused
  if (mode == "save") {
    std::string model_path;
    size_t offset;
    int n_views;
    spec >> model_path >> offset >> n_views;
    ok = ok && model.LoadViews(model_path, offset, n_views, n_points);
  } else {
    ok = ok && model.GenerateModel() && model.set_up();
  }
  ok = ok && model.SaveModel(out);
  std::printf("{\"ok\": %d}\n", ok ? 1 : 0);
  return ok ? 0 : 1;
}
