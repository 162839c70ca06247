// run_synthetic_tracker.cpp — drives the m3t_b200 C++ mirror (Body / Camera / Model / Modality / Link / Optimizer /
// Tracker, 3dobjecttracking_b200/host/m3t_b200/m3t_b200.hpp) on a seeded synthetic scene, the way an M3T application
// drives m3t::Tracker: once through the fused fast path (Tracker::ExecuteTrackingStep -> one launch) and once object by
// object through the Modality / Optimizer methods; prints both pose sets as JSON for tests/test_gpu_host_mirror.py.
//
//   usage: run_synthetic_tracker [n_bodies=3] [n_lines=200] [n_points=200] [n_divides=2] [seed=1] [links_per_structure=1]
//                                [renderers=0] [viewer_dir]
// With viewer_dir a NormalColorViewer and a NormalDepthViewer on camera 0 draw every body; after the tracking step
// Tracker::UpdateViewers renders them and the overlays are written as viewer_dir/color_viewer.ppm and depth_viewer.ppm
// (binary PPM); the same viewers through the plain C ABI must give the same bytes ("viewers_equal_c_abi").
// With renderers = 1 every body's modalities model occlusions and check regions / silhouettes with device renderers
// (one FocusedSilhouetteRenderer per camera over all bodies of one RendererGeometry), and the same scene is also run
// through the plain C ABI ("c_abi" poses), which the fused Tracker path must reproduce bit for bit.
// With links_per_structure > 1 the bodies are grouped into serial kinematic chains (root link with 6 DoF, every further
// link a revolute-x child at Tx(0.01) of the previous one, as in the reference's examples/optimization_time.cpp) that
// are tracked by one Optimizer each; the children's start poses come from Optimizer::CalculateConsistentPoses.
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

// the reference's triangle prism (data/_body/triangle.obj, geometry2body applied), counter-clockwise seen from outside
std::vector<float> PrismTriangles(float* diameter) {
  const float v[6][3] = {{-0.038305f, 0.0f, -0.006f}, {-0.038305f, 0.0f, 0.006f}, {0.019152f, -0.033231f, -0.006f},
                         {0.019152f, -0.033231f, 0.006f}, {0.019152f, 0.033231f, -0.006f}, {0.019152f, 0.033231f, 0.006f}};
  const int f[8][3] = {{0, 2, 3}, {2, 4, 3}, {3, 5, 1}, {4, 0, 1}, {0, 4, 2}, {1, 0, 3}, {4, 5, 3}, {5, 4, 1}};
  std::vector<float> out;
  for (auto& t : f) {
    const float* a = v[t[0]];
    const float* b = v[t[1]];
    const float* c = v[t[2]];
    const float e1[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, e2[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
    const float n[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
    const bool outward = n[0] * (a[0] + b[0] + c[0]) + n[1] * (a[1] + b[1] + c[1]) + n[2] * (a[2] + b[2] + c[2]) > 0.0f;
    for (const float* p : {a, outward ? b : c, outward ? c : b}) out.insert(out.end(), p, p + 3);
  }
  float r = 0.0f;
  for (auto& p : v) r = std::max(r, std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]));
  *diameter = 2.0f * r;
  return out;
}

struct Scene {
  std::shared_ptr<Batch> batch;
  std::vector<std::shared_ptr<FocusedSilhouetteRenderer>> renderers;
  std::vector<std::shared_ptr<Body>> bodies;
  std::vector<std::shared_ptr<ColorCamera>> color_cameras;
  std::vector<std::shared_ptr<DepthCamera>> depth_cameras;
  std::vector<std::shared_ptr<Optimizer>> optimizers;
  std::shared_ptr<Tracker> tracker;
  std::shared_ptr<NormalColorViewer> color_viewer;
  std::shared_ptr<NormalDepthViewer> depth_viewer;
};

// binary PPM (P6) of a BGR8 image, the viewer image a display would show
bool WritePpm(const std::string& path, const std::vector<uint8_t>& bgr, int width, int height) {
  std::FILE* f = std::fopen(path.c_str(), "wb");
  if (!f) return false;
  std::fprintf(f, "P6\n%d %d\n255\n", width, height);
  std::vector<uint8_t> rgb(bgr.size());
  for (size_t k = 0; k + 2 < bgr.size(); k += 3) {
    rgb[k] = bgr[k + 2];
    rgb[k + 1] = bgr[k + 1];
    rgb[k + 2] = bgr[k];
  }
  const bool ok = std::fwrite(rgb.data(), 1, rgb.size(), f) == rgb.size();
  return std::fclose(f) == 0 && ok;
}

void PrintPoses(const char* key, Scene& s) {
  std::printf("\"%s\": [", key);
  for (size_t b = 0; b < s.bodies.size(); ++b) {
    const Transform3fA& p = s.bodies[b]->body2world_pose();
    std::printf("%s[", b ? ", " : "");
    for (int k = 0; k < 12; ++k) std::printf("%s%.9g", k ? ", " : "", p.m[k]);
    std::printf("]");
  }
  std::printf("]");
}

}  // namespace

int main(int argc, char** argv) {
  const int n_bodies = argc > 1 ? std::atoi(argv[1]) : 3;
  const int n_lines = argc > 2 ? std::atoi(argv[2]) : 200;
  const int n_points = argc > 3 ? std::atoi(argv[3]) : 200;
  const int n_divides = argc > 4 ? std::atoi(argv[4]) : 2;
  const uint64_t seed = argc > 5 ? std::strtoull(argv[5], nullptr, 10) : 1;
  const int chain = argc > 6 ? std::max(1, std::atoi(argv[6])) : 1;
  const bool with_renderers = argc > 7 && std::atoi(argv[7]) != 0;
  // viewer mode: a NormalColorViewer and a NormalDepthViewer on camera 0 draw every body; after the tracking step the
  // two overlays are written as binary PPM files into this directory
  const std::string viewer_dir = argc > 8 ? argv[8] : "";
  const bool with_viewers = !viewer_dir.empty();
  float prism_diameter = 0.0f;
  const std::vector<float> prism = PrismTriangles(&prism_diameter);
  if (n_bodies % chain != 0) {
    std::cerr << "n_bodies must be a multiple of links_per_structure" << std::endl;
    return 1;
  }

  // analytic sparse viewpoint models of the triangle prism, in the reference's DataPoint layout
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

  // frames + poses
  const size_t cpitch = 1920, dpitch = 1280;
  std::vector<std::vector<uint8_t>> color(n_bodies, std::vector<uint8_t>(cpitch * 480));
  std::vector<std::vector<uint16_t>> depth(n_bodies, std::vector<uint16_t>(640 * 480));
  std::vector<Transform3fA> start(n_bodies);
  const uint8_t fg[3] = {40, 80, 200}, bg[3] = {120, 120, 120};
  std::vector<float> q_gt(n_bodies), q_start(n_bodies);
  Transform3fA gt_prev;
  for (int b = 0; b < n_bodies; ++b) {
    Transform3fA gt_b2w;
    q_gt[b] = 10.0f * std::sin(1.3f * float(b));
    q_start[b] = q_gt[b] + 2.5f * std::cos(2.1f * float(b));
    if (b % chain == 0) {
      Transform3fA gt_b2c;
      m3ts_ground_truth_pose(seed, b, &sci, chain > 1 ? 200.0f : 132.0f, chain > 1 ? 0.6f : 0.5f, chain > 1 ? 0.8f : 0.7f,
                             gt_b2c.data());
      gt_b2w = Mul(InverseRigid(color_w2c), gt_b2c);
      m3ts_perturb_pose(seed, b, 3.0f, 0.005f, gt_b2w.data(), start[b].data());
    } else {
      gt_b2w = Mul(gt_prev, JointPose(0.01f, q_gt[b]));
      start[b] = Mul(start[b - 1], JointPose(0.01f, q_start[b]));  // reporting only: the device derives it itself
    }
    gt_prev = gt_b2w;
    m3ts_render_color(&sci, Mul(color_w2c, gt_b2w).data(), seed * 1000003 + b, fg, bg, 10.0f, color[b].data(), cpitch);
    m3ts_render_depth(&sdi, Mul(depth_w2c, gt_b2w).data(), seed * 1000003 + b, 1.0f, 0.001f, 0.01f, 0.001f, depth[b].data(), dpitch);
  }

  auto build = [&](Scene& s) -> bool {
    s.batch = std::make_shared<Batch>(0, n_bodies, n_bodies, 1);
    if (!s.batch->ok()) return false;
    auto region_model = std::make_shared<RegionModel>("triangle_region_model", s.batch);
    region_model->SetViews(nv, n_lines, r_ori.data(), r_len.data(), r_pts.data());
    auto depth_model = std::make_shared<DepthModel>("triangle_depth_model", s.batch);
    depth_model->SetViews(nv, n_points, d_ori.data(), d_area.data(), d_pts.data());
    if (!region_model->SetUp() || !depth_model->SetUp()) return false;
    s.tracker = std::make_shared<Tracker>("tracker", s.batch, 7, 2);
    std::vector<std::shared_ptr<Link>> links;  // links of the chain being assembled
    auto geometry = std::make_shared<RendererGeometry>("renderer_geometry", s.batch);
    std::vector<std::shared_ptr<Body>> all_bodies;
    for (int b = 0; b < n_bodies; ++b) {
      all_bodies.push_back(std::make_shared<Body>("triangle_" + std::to_string(b), s.batch));
      all_bodies.back()->set_geometry_triangles(prism);
      all_bodies.back()->set_maximum_body_diameter(prism_diameter);
      all_bodies.back()->set_body_id(uint8_t(b + 1));
      all_bodies.back()->set_region_id(7);
      if ((with_renderers || with_viewers) && !geometry->AddBody(all_bodies.back())) return false;
    }
    if (!geometry->SetUp()) return false;
    for (int b = 0; b < n_bodies; ++b) {
      auto body = all_bodies[b];
      auto cc = std::make_shared<ColorCamera>("color_camera_" + std::to_string(b), s.batch, ci, color_w2c);
      auto dc = std::make_shared<DepthCamera>("depth_camera_" + std::to_string(b), s.batch, di, depth_w2c, 0.001f);
      if (!cc->SetUp() || !dc->SetUp()) return false;
      auto rm = std::make_shared<RegionModality>("region_modality_" + std::to_string(b), s.batch, body, cc, region_model);
      rm->set_n_lines_max(n_lines);
      auto dm = std::make_shared<DepthModality>("depth_modality_" + std::to_string(b), s.batch, body, dc, depth_model);
      dm->set_n_points_max(n_points);
      if (with_renderers) {
        auto cr = std::make_shared<FocusedSilhouetteRenderer>("color_renderer_" + std::to_string(b), s.batch, geometry, cc,
                                                              IDType::REGION);
        auto dr = std::make_shared<FocusedSilhouetteRenderer>("depth_renderer_" + std::to_string(b), s.batch, geometry, dc,
                                                              IDType::BODY);
        if (!cr->AddReferencedBody(body) || !dr->AddReferencedBody(body) || !cr->SetUp() || !dr->SetUp()) return false;
        rm->ModelOcclusions(cr);
        rm->UseRegionChecking(cr);
        rm->set_n_unoccluded_iterations(0);
        dm->ModelOcclusions(dr);
        dm->UseSilhouetteChecking(dr);
        dm->set_n_unoccluded_iterations(0);
        s.renderers.push_back(cr);
        s.renderers.push_back(dr);
      }
      auto link = std::make_shared<Link>("link_" + std::to_string(b), body);
      link->AddModality(rm);
      link->AddModality(dm);
      if (b % chain == 0) {
        links.clear();
        s.optimizers.push_back(std::make_shared<Optimizer>("optimizer_" + std::to_string(b / chain), s.batch, link,
                                                           chain > 1 ? 100.0f : 1000.0f, chain > 1 ? 1000.0f : 30000.0f));
      } else {
        link->set_joint2parent_pose(JointPose(0.01f, q_start[b]));
        link->set_free_directions({true, false, false, false, false, false});
        links.back()->AddChildLink(link);
      }
      links.push_back(link);
      if (b % chain == chain - 1) s.tracker->AddOptimizer(s.optimizers.back());  // the tree is complete
      s.bodies.push_back(body);
      s.color_cameras.push_back(cc);
      s.depth_cameras.push_back(dc);
    }
    if (with_viewers) {
      s.color_viewer = std::make_shared<NormalColorViewer>("color_viewer", s.batch, s.color_cameras[0], geometry);
      s.depth_viewer = std::make_shared<NormalDepthViewer>("depth_viewer", s.batch, s.depth_cameras[0], geometry, 0.0f, 1.0f);
      s.color_viewer->set_opacity(0.6f);
      if (!s.tracker->AddViewer(s.color_viewer) || !s.tracker->AddViewer(s.depth_viewer)) return false;
    }
    if (!s.tracker->SetUp()) return false;
    for (int b = 0; b < n_bodies; ++b) {
      if (!s.color_cameras[b]->UpdateImage(color[b].data(), cpitch)) return false;
      if (!s.depth_cameras[b]->UpdateImage(depth[b].data(), dpitch)) return false;
      // a detector sets the root link's pose; the other links follow from the joints
      if (b % chain == 0 && !s.bodies[b]->set_body2world_pose(start[b])) return false;
    }
    if (chain > 1)
      for (auto& o : s.optimizers)
        if (!o->CalculateConsistentPoses()) return false;
    return s.tracker->StartModalities(0);
  };

  Scene fused, object_wise;
  if (!build(fused) || !build(object_wise)) {
    std::cerr << "setup failed" << std::endl;
    return 2;
  }
  // the same renderer scene through the plain C ABI (rigid bodies only)
  std::vector<float> c_abi(size_t(12) * n_bodies, 0.0f);
  if (with_renderers && chain == 1) {
    m3tb_ctx* raw = nullptr;
    bool ok = m3tb_create(0, n_bodies, n_bodies, 1, &raw) == M3TB_OK;
    m3tb_region_params rp;
    m3tb_depth_params dp;
    m3tb_region_params_default(&rp);
    m3tb_depth_params_default(&dp);
    rp.n_lines_max = n_lines;
    dp.n_points_max = n_points;
    rp.model_occlusions = rp.use_region_checking = 1;
    dp.model_occlusions = dp.use_silhouette_checking = 1;
    rp.n_unoccluded_iterations = dp.n_unoccluded_iterations = 0;
    const m3tb_optimizer_params op{1000.0f, 30000.0f};
    ok = ok && m3tb_set_region_model(raw, 0, nv, n_lines, r_ori.data(), r_len.data(), r_pts.data(), 0.002f, 0.05f) == 0 &&
         m3tb_set_depth_model(raw, 0, nv, n_points, d_ori.data(), d_area.data(), d_pts.data(), 0.002f, 0.05f) == 0;
    std::vector<int> all(n_bodies);
    for (int b = 0; b < n_bodies; ++b) all[b] = b;
    const Transform3fA identity;
    for (int b = 0; b < n_bodies && ok; ++b)
      ok = m3tb_set_color_camera(raw, b, &ci, color_w2c.data()) == 0 &&
           m3tb_set_depth_camera(raw, b, &di, depth_w2c.data(), 0.001f) == 0 &&
           m3tb_upload_color(raw, b, color[b].data(), cpitch) == 0 && m3tb_upload_depth(raw, b, depth[b].data(), dpitch) == 0 &&
           m3tb_set_body(raw, b, &rp, &dp, &op, 0, 0, b, b) == 0 && m3tb_set_poses(raw, b, 1, start[b].data()) == 0 &&
           m3tb_set_body_geometry(raw, b, prism.data(), int(prism.size() / 9), identity.data(), prism_diameter, 1, b + 1, 7) == 0;
    for (int b = 0; b < n_bodies && ok; ++b)
      ok = m3tb_set_focused_renderer(raw, 2 * b, 0, b, 200, 0.02f, 10.0f, 1, all.data(), n_bodies, &b, 1) == 0 &&
           m3tb_set_focused_renderer(raw, 2 * b + 1, 1, b, 200, 0.02f, 10.0f, 0, all.data(), n_bodies, &b, 1) == 0;
    for (int b = 0; b < n_bodies && ok; ++b)
      for (int m = 0; m < 2 && ok; ++m)
        for (int k = 0; k < 2 && ok; ++k) ok = m3tb_attach_renderer(raw, b, m, k, 2 * b + m) == 0;
    ok = ok && m3tb_start_modalities(raw, 0) == 0 && m3tb_tracking_step(raw, 0, 7, 2) == 0 &&
         m3tb_calculate_results(raw, 0) == 0 && m3tb_get_poses(raw, 0, n_bodies, c_abi.data()) == 0;
    if (!ok) {
      std::cerr << "C ABI run failed: " << (raw ? m3tb_last_error(raw) : "no context") << std::endl;
      return 6;
    }
    m3tb_destroy(raw);
  }
  // an unset-up tracker must refuse to run, like the reference (tracker.cpp:224-228)
  Tracker not_set_up("not_set_up", fused.batch);
  const bool refused = !not_set_up.ExecuteTrackingStep(0);

  if (!fused.tracker->ExecuteTrackingStep(0)) return 3;
  bool viewers_equal = true;
  if (with_viewers) {  // the overlays of the tracked poses, and the same viewers through the plain C ABI
    if (!fused.tracker->UpdateViewers(0)) return 7;
    const std::vector<uint8_t>& cimg = fused.color_viewer->image();
    const std::vector<uint8_t>& dimg = fused.depth_viewer->image();
    if (!WritePpm(viewer_dir + "/color_viewer.ppm", cimg, ci.width, ci.height) ||
        !WritePpm(viewer_dir + "/depth_viewer.ppm", dimg, di.width, di.height))
      return 8;
    std::vector<float> poses(size_t(12) * n_bodies);
    m3tb_ctx* raw = nullptr;
    bool ok = m3tb_create(0, n_bodies, 1, 1, &raw) == M3TB_OK &&
              m3tb_get_poses(fused.batch->ctx(), 0, n_bodies, poses.data()) == 0 &&
              m3tb_set_poses(raw, 0, n_bodies, poses.data()) == 0 &&
              m3tb_set_color_camera(raw, 0, &ci, color_w2c.data()) == 0 &&
              m3tb_set_depth_camera(raw, 0, &di, depth_w2c.data(), 0.001f) == 0 &&
              m3tb_upload_color(raw, 0, color[0].data(), cpitch) == 0 && m3tb_upload_depth(raw, 0, depth[0].data(), dpitch) == 0;
    const Transform3fA identity;
    std::vector<int> all(n_bodies);
    for (int b = 0; b < n_bodies && ok; ++b) {
      all[b] = b;
      ok = m3tb_set_body_geometry(raw, b, prism.data(), int(prism.size() / 9), identity.data(), prism_diameter, 1, b + 1, 7) == 0;
    }
    std::vector<uint8_t> c2(cimg.size()), d2(dimg.size());
    ok = ok && m3tb_set_viewer(raw, 0, 0, 0, all.data(), n_bodies, 0.6f, 0.0f, 1.0f) == 0 &&
         m3tb_set_viewer(raw, 1, 1, 0, all.data(), n_bodies, 0.5f, 0.0f, 1.0f) == 0 && m3tb_update_viewers(raw) == 0 &&
         m3tb_get_viewer_image(raw, 0, c2.data(), size_t(ci.width) * 3, nullptr, 0) == 0 &&
         m3tb_get_viewer_image(raw, 1, d2.data(), size_t(di.width) * 3, nullptr, 0) == 0;
    if (!ok) {
      std::cerr << "C ABI viewer run failed: " << (raw ? m3tb_last_error(raw) : "no context") << std::endl;
      return 9;
    }
    m3tb_destroy(raw);
    viewers_equal = c2 == cimg && d2 == dimg;
  }
  if (!object_wise.tracker->ExecuteTrackingStepObjectWise(0)) return 4;
  bool joints_ok = true;
  if (chain > 1) {  // the children still hang on their parents at Tx(0.01), rotated about x only
    for (auto& o : fused.optimizers) {
      if (!o->FetchLinkPoses()) return 5;
      for (auto& l : o->ReferencedLinks()) {
        if (l == o->root_link_ptr()) continue;
        const Transform3fA& j = l->joint2parent_pose();
        joints_ok = joints_ok && std::fabs(j(0, 3) - 0.01f) < 1e-6f && std::fabs(j(1, 3)) < 1e-6f && std::fabs(j(2, 3)) < 1e-6f &&
                    std::fabs(j(0, 0) - 1.0f) < 1e-5f && std::fabs(j(0, 1)) < 1e-5f && std::fabs(j(0, 2)) < 1e-5f;
      }
    }
  }
  std::printf("{\"links_per_structure\": %d, \"joints_ok\": %s, ", chain, joints_ok ? "true" : "false");
  std::printf("\"n_bodies\": %d, \"refused_without_setup\": %s, \"launches_fused\": %lld, \"launches_object_wise\": %lld, ",
              n_bodies, refused ? "true" : "false", (long long)m3tb_launch_count(fused.batch->ctx()),
              (long long)m3tb_launch_count(object_wise.batch->ctx()));
  if (with_viewers) std::printf("\"viewers_equal_c_abi\": %s, ", viewers_equal ? "true" : "false");
  if (with_renderers) {
    bool visible = true;
    for (int b = 0; b < n_bodies; ++b)
      visible = visible && fused.renderers[2 * b]->IsBodyVisible(fused.bodies[b]->name()) &&
                fused.renderers[2 * b + 1]->IsBodyVisible(fused.bodies[b]->name());
    std::printf("\"renderers_visible\": %s, \"c_abi\": [", visible ? "true" : "false");
    for (int b = 0; b < n_bodies; ++b) {
      std::printf("%s[", b ? ", " : "");
      for (int k = 0; k < 12; ++k) std::printf("%s%.9g", k ? ", " : "", c_abi[12 * b + k]);
      std::printf("]");
    }
    std::printf("], ");
  }
  std::printf("\"start\": [");
  for (int b = 0; b < n_bodies; ++b) {
    std::printf("%s[", b ? ", " : "");
    for (int k = 0; k < 12; ++k) std::printf("%s%.9g", k ? ", " : "", start[b].m[k]);
    std::printf("]");
  }
  std::printf("], ");
  PrintPoses("fused", fused);
  std::printf(", ");
  PrintPoses("object_wise", object_wise);
  std::printf("}\n");
  return 0;
}
