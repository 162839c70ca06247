// texture_mirror_tracker.cpp — drives the C++ mirror's TextureModality on a seeded synthetic scene: one rigid body and
// one 3-link chain (root with 6 DoF, revolute-x children at Tx(0.01)), every body with region, depth and texture
// modalities on its own RGB-D pair and its own focused silhouette renderer. The features a detector would find are
// generated here from a seed: points on the prism's mid-plane with random 32-byte descriptors (orb), 64-byte
// descriptors (brisk, matched through k_texture_knn_hamming at every n_features_max) or 128 whole-number floats in
// 0 .. 255, as cv::SIFT writes them (sift), seen at the start pose for StartModality and at the
// ground-truth pose for the tracked frame. The scene is tracked once through Tracker::ExecuteTrackingStep and once
// through ExecuteTrackingStepObjectWise; both pose sets are printed as JSON for tests/test_gpu_texture_mirror.py and
// tests/test_gpu_texture_l2.py. Above 512 features per body (up to 4096) every texture modality raises its
// n_features_max to n_features, so the frame's features are matched in full (k_texture_knn_hamming for orb).
//
//   usage: texture_mirror_tracker [seed=1] [n_features=300] [orb|sift|brisk]
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <memory>
#include <random>
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

constexpr int kSiftLength = 128;

// a body's texture: n points on the prism's triangular mid-plane (body frame) and their descriptors
struct Texture {
  std::vector<float> points;  // [n][3]
  std::vector<uint8_t> descriptors;  // [n][32] (orb) or [n][64] (brisk)
  std::vector<float> float_descriptors;  // [n][kSiftLength] (sift)
};
Texture MakeTexture(uint64_t seed, int body, int n, bool sift, int binary_bytes) {
  std::mt19937 rng(uint32_t(seed * 7919u + uint64_t(body)));
  std::uniform_real_distribution<float> u(0.0f, 1.0f);
  std::uniform_int_distribution<int> byte(0, 255);
  Texture t;
  for (int i = 0; i < n; ++i) {
    float a = u(rng), b = u(rng);
    if (a + b > 1.0f) { a = 1.0f - a; b = 1.0f - b; }
    for (int k = 0; k < 2; ++k)  // vertices 0, 2, 4 span the triangle
      t.points.push_back(kPrism[0][k] + a * (kPrism[2][k] - kPrism[0][k]) + b * (kPrism[4][k] - kPrism[0][k]));
    t.points.push_back(0.0f);
    if (sift)
      for (int k = 0; k < kSiftLength; ++k) t.float_descriptors.push_back(float(byte(rng)));
    else
      for (int k = 0; k < binary_bytes; ++k) t.descriptors.push_back(uint8_t(byte(rng)));
  }
  return t;
}

struct Scene {
  std::shared_ptr<Batch> batch;
  std::vector<std::shared_ptr<Body>> bodies;
  std::vector<std::shared_ptr<TextureModality>> textures;
  std::vector<std::shared_ptr<Optimizer>> optimizers;
  std::shared_ptr<Tracker> tracker;
};

// the detection hook: the texture's points seen at body2camera, in the crop of the modality's focus region
bool UploadFeatures(TextureModality& m, const Texture& t, const Transform3fA& body2camera, const Intrinsics& ci) {
  std::array<int32_t, 4> roi{};
  float scale = 0.0f;
  if (!m.CalculateFocus(&roi, &scale)) return false;
  std::vector<float> xy;
  for (size_t i = 0; i < t.points.size() / 3; ++i) {
    const float* p = &t.points[3 * i];
    const float x = body2camera(0, 0) * p[0] + body2camera(0, 1) * p[1] + body2camera(0, 2) * p[2] + body2camera(0, 3);
    const float y = body2camera(1, 0) * p[0] + body2camera(1, 1) * p[1] + body2camera(1, 2) * p[2] + body2camera(1, 3);
    const float z = body2camera(2, 0) * p[0] + body2camera(2, 1) * p[1] + body2camera(2, 2) * p[2] + body2camera(2, 3);
    xy.push_back((x * ci.fu / z + ci.ppu - float(roi[0])) * scale);
    xy.push_back((y * ci.fv / z + ci.ppv - float(roi[1])) * scale);
  }
  if (!t.float_descriptors.empty()) return m.SetFeatures(xy, t.float_descriptors, kSiftLength, roi, scale);
  return m.SetFeatures(xy, t.descriptors, roi, scale);
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
  const int n_features = argc > 2 ? std::atoi(argv[2]) : 300;
  const bool sift = argc > 3 && std::string(argv[3]) == "sift";
  const bool brisk = argc > 3 && std::string(argv[3]) == "brisk";
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

  // ground truth, frames, start poses of the rigid body and the chain's root, textures
  const size_t cpitch = 1920, dpitch = 1280;
  std::vector<std::vector<uint8_t>> color(kBodies, std::vector<uint8_t>(cpitch * 480));
  std::vector<std::vector<uint16_t>> depth(kBodies, std::vector<uint16_t>(640 * 480));
  std::vector<Transform3fA> gt(kBodies), start_root(kBodies);
  std::vector<float> q_start(kBodies);
  std::vector<Texture> textures;
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
    m3ts_render_color(&sci, Mul(color_w2c, gt[b]).data(), seed * 1000003 + b, fg, bg, 10.0f, color[b].data(), cpitch);
    m3ts_render_depth(&sdi, Mul(depth_w2c, gt[b]).data(), seed * 1000003 + b, 1.0f, 0.001f, 0.01f, 0.001f, depth[b].data(), dpitch);
    textures.push_back(MakeTexture(seed, b, n_features, sift, brisk ? 64 : 32));
  }

  std::vector<Transform3fA> start;
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
      // one renderer geometry per body: every body has its own RGB-D pair
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
      if (sift) tm->set_descriptor_type(TextureModality::DescriptorType::SIFT);
      if (brisk) tm->set_descriptor_type(TextureModality::DescriptorType::BRISK);
      tm->set_n_features_max(std::max(n_features, tm->n_features_max()));
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
    // the start frame's features (seen at the start pose), then the tracked frame's (seen at the ground truth)
    for (int b = 0; b < kBodies; ++b)
      if (!UploadFeatures(*s.textures[b], textures[b], Mul(color_w2c, start[b]), ci)) return false;
    if (!s.tracker->StartModalities(0)) return false;
    for (int b = 0; b < kBodies; ++b)
      if (!UploadFeatures(*s.textures[b], textures[b], Mul(color_w2c, gt[b]), ci)) return false;
    return true;
  };

  Scene fused, object_wise;
  if (!build(fused) || !build(object_wise)) {
    std::cerr << "setup failed" << std::endl;
    return 2;
  }
  if (!fused.tracker->ExecuteTrackingStep(0)) return 3;
  if (!object_wise.tracker->ExecuteTrackingStepObjectWise(0)) return 4;
  std::printf("{\"descriptor\": \"%s\", \"n_bodies\": %d, \"n_features_max\": %d, \"texture_points\": [",
              sift ? "sift" : brisk ? "brisk" : "orb", kBodies, fused.textures[0]->n_features_max());
  for (int b = 0; b < kBodies; ++b) {
    std::vector<m3tb_texture_point> pts(512);
    int n = 0;
    if (m3tb_get_texture_points(fused.batch->ctx(), b, pts.data(), int(pts.size()), &n) != M3TB_OK) return 5;
    std::printf("%s%d", b ? ", " : "", n);
  }
  std::printf("], \"launches_fused\": %lld, ", (long long)m3tb_launch_count(fused.batch->ctx()));
  PrintPoses("gt", gt);
  std::printf(", ");
  PrintPoses("start", start);
  std::printf(", ");
  PrintPoses("fused", Poses(fused));
  std::printf(", ");
  PrintPoses("object_wise", Poses(object_wise));
  std::printf("}\n");
  return 0;
}
