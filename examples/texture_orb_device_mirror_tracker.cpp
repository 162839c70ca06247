// texture_orb_device_mirror_tracker.cpp — the scene of texture_device_mirror_tracker.cpp (one rigid body and a 3-link
// chain, region, depth and texture modalities on every body, a noisy rendered frame per body) tracked with the C++
// mirror's device detection: TextureModality::DetectFeatures runs cv::ORB on every body's focused crop
// (m3tb_texture_detect_orb). On the start frame body 0 detects alone (DetectFeatures()) and the chain in one call; on
// the tracked frame all four bodies go in one DetectFeatures(modalities) call. A second scene takes the same features
// through the C ABI read-back (m3tb_get_texture_orb_keypoints) and the host SetFeatures; both take one
// Tracker::ExecuteTrackingStep. Prints JSON for tests/test_gpu_texture_orb.py.
//
//   usage: texture_orb_device_mirror_tracker [seed=1] [orb_n_features=300]
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <memory>
#include <string>
#include <vector>

#include "m3t_b200/m3t_b200.hpp"
#include "m3t_synth.h"

using namespace m3t_b200;

namespace {

constexpr int kBodies = 4;  // body 0 rigid, bodies 1..3 the chain
constexpr int kChainRoot = 1;

Transform3fA Mul(const Transform3fA& a, const Transform3fA& b) {
  Transform3fA r;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) r(i, j) = a(i, 0) * b(0, j) + a(i, 1) * b(1, j) + a(i, 2) * b(2, j);
    r(i, 3) = a(i, 0) * b(0, 3) + a(i, 1) * b(1, 3) + a(i, 2) * b(2, 3) + a(i, 3);
  }
  return r;
}
Transform3fA InverseRigid(const Transform3fA& a) {
  Transform3fA r;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r(i, j) = a(j, i);
  for (int i = 0; i < 3; ++i) r(i, 3) = -(r(i, 0) * a(0, 3) + r(i, 1) * a(1, 3) + r(i, 2) * a(2, 3));
  return r;
}
Transform3fA JointPose(float tx, float angle_x_deg) {  // Tx(tx) * Rx(angle)
  Transform3fA r;
  const float a = angle_x_deg * 3.14159265358979f / 180.0f;
  r(1, 1) = std::cos(a); r(1, 2) = -std::sin(a);
  r(2, 1) = std::sin(a); r(2, 2) = std::cos(a);
  r(0, 3) = tx;
  return r;
}

const float kPrism[6][3] = {{-0.038305f, 0.0f, -0.006f}, {-0.038305f, 0.0f, 0.006f}, {0.019152f, -0.033231f, -0.006f},
                            {0.019152f, -0.033231f, 0.006f}, {0.019152f, 0.033231f, -0.006f}, {0.019152f, 0.033231f, 0.006f}};

// the reference's triangle prism (data/_body/triangle.obj, geometry2body applied), counter-clockwise seen from outside
std::vector<float> PrismTriangles(float* diameter) {
  const int f[8][3] = {{0, 2, 3}, {2, 4, 3}, {3, 5, 1}, {4, 0, 1}, {0, 4, 2}, {1, 0, 3}, {4, 5, 3}, {5, 4, 1}};
  std::vector<float> out;
  for (auto& t : f) {
    const float* a = kPrism[t[0]];
    const float* b = kPrism[t[1]];
    const float* c = kPrism[t[2]];
    const float e1[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, e2[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
    const float n[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
    const bool outward = n[0] * (a[0] + b[0] + c[0]) + n[1] * (a[1] + b[1] + c[1]) + n[2] * (a[2] + b[2] + c[2]) > 0.0f;
    for (const float* p : {a, outward ? b : c, outward ? c : b}) out.insert(out.end(), p, p + 3);
  }
  float r = 0.0f;
  for (auto& p : kPrism) r = std::max(r, std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]));
  *diameter = 2.0f * r;
  return out;
}

struct Scene {
  std::shared_ptr<Batch> batch;
  std::vector<std::shared_ptr<Body>> bodies;
  std::vector<std::shared_ptr<TextureModality>> textures;
  std::vector<std::shared_ptr<Optimizer>> optimizers;
  std::shared_ptr<Tracker> tracker;
};

// the host path: the device scene's last detection of each body, read back through the C ABI, handed to the host
// scene's SetFeatures in the crop of its own (equal) focus
bool CopyDetections(Scene& from, Scene& to) {
  for (size_t b = 0; b < from.textures.size(); ++b) {
    std::vector<float> xy(2 * 4096);
    std::vector<uint8_t> desc(32 * 4096);
    int n = 0;
    if (m3tb_get_texture_orb_keypoints(from.batch->ctx(), int(b), xy.data(), nullptr, nullptr, nullptr, desc.data(), 4096,
                                       &n) != M3TB_OK)
      return false;
    xy.resize(2 * size_t(n));
    desc.resize(32 * size_t(n));
    std::array<int32_t, 4> roi{};
    float scale = 0.0f;
    if (!to.textures[b]->CalculateFocus(&roi, &scale)) return false;
    if (!to.textures[b]->SetFeatures(xy, desc, roi, scale)) return false;
  }
  return true;
}

void PrintPoses(const char* key, const std::vector<Transform3fA>& poses) {
  std::printf("\"%s\": [", key);
  for (size_t b = 0; b < poses.size(); ++b) {
    std::printf("%s[", b ? ", " : "");
    for (int k = 0; k < 12; ++k) std::printf("%s%.9g", k ? ", " : "", poses[b].m[k]);
    std::printf("]");
  }
  std::printf("]");
}

std::vector<Transform3fA> Poses(Scene& s) {
  std::vector<Transform3fA> out;
  for (auto& b : s.bodies) out.push_back(b->body2world_pose());
  return out;
}

}  // namespace

int main(int argc, char** argv) {
  const uint64_t seed = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 1;
  const int orb_n_features = argc > 2 ? std::atoi(argv[2]) : 300;
  const int n_lines = 200, n_points = 200, n_divides = 2;
  float prism_diameter = 0.0f;
  const std::vector<float> prism = PrismTriangles(&prism_diameter);

  const int nv = m3ts_n_views(n_divides);
  std::vector<float> r_ori(3 * nv), r_len(nv), d_ori(3 * nv), d_area(nv);
  std::vector<float> r_pts(size_t(nv) * n_lines * 38), d_pts(size_t(nv) * n_points * 36);
  m3ts_generate_region_model(n_divides, n_lines, 0.8f, seed, r_ori.data(), r_len.data(), r_pts.data());
  m3ts_generate_depth_model(n_divides, n_points, 0.8f, seed, d_ori.data(), d_area.data(), d_pts.data());

  Intrinsics ci{614.0f, 614.5f, 321.3f, 238.9f, 640, 480};
  Intrinsics di{385.7f, 385.9f, 322.1f, 241.6f, 640, 480};
  m3ts_intrinsics sci{ci.fu, ci.fv, ci.ppu, ci.ppv, ci.width, ci.height}, sdi{di.fu, di.fv, di.ppu, di.ppv, di.width, di.height};
  Transform3fA color_w2c;  // identity
  Transform3fA depth_w2c;
  depth_w2c(0, 3) = -0.015f;
  depth_w2c(1, 3) = 0.001f;

  // ground truth, frames (strong per-pixel noise, so FAST finds corners on and around every body), start poses
  const size_t cpitch = 1920, dpitch = 1280;
  std::vector<std::vector<uint8_t>> color(kBodies, std::vector<uint8_t>(cpitch * 480));
  std::vector<std::vector<uint16_t>> depth(kBodies, std::vector<uint16_t>(640 * 480));
  std::vector<Transform3fA> gt(kBodies), start_root(kBodies);
  std::vector<float> q_start(kBodies);
  const uint8_t fg[3] = {40, 80, 200}, bg[3] = {120, 120, 120};
  for (int b = 0; b < kBodies; ++b) {
    const float q_gt = 10.0f * std::sin(1.3f * float(b));
    q_start[b] = q_gt + 2.5f * std::cos(2.1f * float(b));
    if (b <= kChainRoot) {
      const bool chain = b == kChainRoot;
      Transform3fA gt_b2c;
      m3ts_ground_truth_pose(seed, b, &sci, chain ? 200.0f : 132.0f, chain ? 0.6f : 0.5f, chain ? 0.8f : 0.7f, gt_b2c.data());
      gt[b] = Mul(InverseRigid(color_w2c), gt_b2c);
      m3ts_perturb_pose(seed, b, 3.0f, 0.005f, gt[b].data(), start_root[b].data());
    } else {
      gt[b] = Mul(gt[b - 1], JointPose(0.01f, q_gt));
    }
    m3ts_render_color(&sci, Mul(color_w2c, gt[b]).data(), seed * 1000003 + b, fg, bg, 45.0f, color[b].data(), cpitch);
    m3ts_render_depth(&sdi, Mul(depth_w2c, gt[b]).data(), seed * 1000003 + b, 1.0f, 0.001f, 0.01f, 0.001f, depth[b].data(), dpitch);
  }

  std::vector<Transform3fA> start;
  std::vector<std::shared_ptr<ColorCamera>> cameras;
  auto build = [&](Scene& s) -> bool {
    s.batch = std::make_shared<Batch>(0, kBodies, kBodies, 1);
    if (!s.batch->ok()) return false;
    auto region_model = std::make_shared<RegionModel>("triangle_region_model", s.batch);
    region_model->SetViews(nv, n_lines, r_ori.data(), r_len.data(), r_pts.data());
    auto depth_model = std::make_shared<DepthModel>("triangle_depth_model", s.batch);
    depth_model->SetViews(nv, n_points, d_ori.data(), d_area.data(), d_pts.data());
    if (!region_model->SetUp() || !depth_model->SetUp()) return false;
    s.tracker = std::make_shared<Tracker>("tracker", s.batch, 5, 2);
    std::shared_ptr<Link> previous;
    for (int b = 0; b < kBodies; ++b) {
      auto body = std::make_shared<Body>("triangle_" + std::to_string(b), s.batch);
      body->set_geometry_triangles(prism);
      body->set_maximum_body_diameter(prism_diameter);
      body->set_body_id(uint8_t(b + 1));
      body->set_region_id(7);
      auto geometry = std::make_shared<RendererGeometry>("geometry_" + std::to_string(b), s.batch);
      if (!geometry->AddBody(body) || !geometry->SetUp()) return false;
      auto cc = std::make_shared<ColorCamera>("color_camera_" + std::to_string(b), s.batch, ci, color_w2c);
      auto dc = std::make_shared<DepthCamera>("depth_camera_" + std::to_string(b), s.batch, di, depth_w2c, 0.001f);
      if (!cc->SetUp() || !dc->SetUp()) return false;
      auto silhouette = std::make_shared<FocusedSilhouetteRenderer>("silhouette_" + std::to_string(b), s.batch, geometry, cc);
      if (!silhouette->AddReferencedBody(body) || !silhouette->SetUp()) return false;
      auto rm = std::make_shared<RegionModality>("region_modality_" + std::to_string(b), s.batch, body, cc, region_model);
      rm->set_n_lines_max(n_lines);
      auto dm = std::make_shared<DepthModality>("depth_modality_" + std::to_string(b), s.batch, body, dc, depth_model);
      dm->set_n_points_max(n_points);
      auto tm = std::make_shared<TextureModality>("texture_modality_" + std::to_string(b), s.batch, body, cc, silhouette);
      tm->set_orb_n_features(orb_n_features);
      tm->set_n_features_max(2048);
      auto link = std::make_shared<Link>("link_" + std::to_string(b), body);
      link->AddModality(rm);
      link->AddModality(dm);
      link->AddModality(tm);
      if (b < kChainRoot) {
        s.optimizers.push_back(std::make_shared<Optimizer>("rigid", s.batch, link));
        s.tracker->AddOptimizer(s.optimizers.back());
      } else if (b == kChainRoot) {
        s.optimizers.push_back(std::make_shared<Optimizer>("chain", s.batch, link, 100.0f, 1000.0f));
      } else {
        link->set_joint2parent_pose(JointPose(0.01f, q_start[b]));
        link->set_free_directions({true, false, false, false, false, false});
        previous->AddChildLink(link);
      }
      previous = link;
      s.bodies.push_back(body);
      s.textures.push_back(tm);
      if (!cc->UpdateImage(color[b].data(), cpitch) || !dc->UpdateImage(depth[b].data(), dpitch)) return false;
    }
    s.tracker->AddOptimizer(s.optimizers.back());  // the chain's tree is complete
    if (!s.tracker->SetUp()) return false;
    for (int b = 0; b <= kChainRoot; ++b)  // a detector sets the roots' poses; the other links follow from the joints
      if (!s.bodies[b]->set_body2world_pose(start_root[b])) return false;
    if (!s.optimizers.back()->CalculateConsistentPoses()) return false;
    start = Poses(s);
    return true;
  };

  Scene device, host;
  if (!build(device) || !build(host)) {
    std::cerr << "setup failed" << std::endl;
    return 2;
  }
  // the start frame: body 0 alone, the chain in one call
  std::vector<std::shared_ptr<TextureModality>> chain(device.textures.begin() + 1, device.textures.end());
  if (!device.textures[0]->DetectFeatures() || !TextureModality::DetectFeatures(chain)) return 3;
  std::vector<int> found_start;
  for (auto& t : device.textures) found_start.push_back(t->detections());
  if (!CopyDetections(device, host)) return 3;
  if (!device.tracker->StartModalities(0) || !host.tracker->StartModalities(0)) return 4;
  // the tracked frame: a new copy of each frame, all bodies in one call
  for (Scene* s : {&device, &host})
    for (int b = 0; b < kBodies; ++b)
      if (!s->textures[b]->color_camera_ptr()->UpdateImage(color[b].data(), cpitch)) return 5;
  if (!TextureModality::DetectFeatures(device.textures)) return 5;
  if (!CopyDetections(device, host)) return 5;
  if (!device.tracker->ExecuteTrackingStep(0) || !host.tracker->ExecuteTrackingStep(0)) return 6;

  auto points = [&](Scene& s) {
    std::printf("[");
    for (int b = 0; b < kBodies; ++b) {
      std::vector<m3tb_texture_point> pts(8 * 2048);
      int n = 0;
      m3tb_get_texture_points(s.batch->ctx(), b, pts.data(), int(pts.size()), &n);
      std::printf("%s%d", b ? ", " : "", n);
    }
    std::printf("]");
  };
  std::printf("{\"n_bodies\": %d, \"orb_n_features\": %d, \"found_start\": [", kBodies, device.textures[0]->orb_n_features());
  for (int b = 0; b < kBodies; ++b) std::printf("%s%d", b ? ", " : "", found_start[b]);
  std::printf("], \"found\": [");
  for (int b = 0; b < kBodies; ++b) std::printf("%s%d", b ? ", " : "", device.textures[b]->detections());
  std::printf("], \"texture_points_device\": ");
  points(device);
  std::printf(", \"texture_points_host\": ");
  points(host);
  std::printf(", ");
  PrintPoses("gt", gt);
  std::printf(", ");
  PrintPoses("start", start);
  std::printf(", ");
  PrintPoses("device", Poses(device));
  std::printf(", ");
  PrintPoses("host", Poses(host));
  std::printf("}\n");
  return 0;
}
