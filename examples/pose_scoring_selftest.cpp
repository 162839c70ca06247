// pose_scoring_selftest.cpp — the C++ mirror's EvaluationModel and the four evaluators' CalculatePoseResults on two
// small models: the corners of a 0.1 m cube, and a 5 x 5 x 5 grid with 0.02 m spacing reduced to 50 vertices. Checks the
// closed forms (a cube under a 90 degree turn has ADD-S 0, a pure translation t has ADD |t|, the diameters) and that
// bodies of two batches are refused, and prints one JSON line with every result (floats with 9 significant digits, so
// float32 values round-trip). Exit status 0 when every check holds.
//
//   pose_scoring_selftest
#include <cmath>
#include <cstdio>
#include <memory>
#include <vector>

#include "m3t_b200/m3t_b200.hpp"

using namespace m3t_b200;

static Transform3fA Pose(float r00, float r01, float r10, float r11, float tx, float ty, float tz) {
  Transform3fA p;
  p(0, 0) = r00; p(0, 1) = r01; p(1, 0) = r10; p(1, 1) = r11;
  p(0, 3) = tx; p(1, 3) = ty; p(2, 3) = tz;
  return p;
}

int main() {
  auto batch = std::make_shared<Batch>(0, 3, 1, 2);
  if (!batch->ok()) return 2;
  std::vector<float> cube, grid;
  for (int i = 0; i < 8; ++i)
    for (int k = 0; k < 3; ++k) cube.push_back((i >> k) & 1 ? 0.05f : -0.05f);
  for (int i = 0; i < 125; ++i)
    for (int k : {i % 5, (i / 5) % 5, i / 25}) grid.push_back(0.02f * float(k));
  EvaluationModel cube_model("cube", batch), grid_model("grid", batch);
  cube_model.set_vertices(cube);
  cube_model.set_n_vertices_evaluation(0);
  grid_model.set_vertices(grid);
  grid_model.set_n_vertices_evaluation(50);
  if (!cube_model.SetUp() || !grid_model.SetUp()) return 1;

  std::vector<std::shared_ptr<Body>> bodies;
  for (const char* name : {"cube", "grid", "grid_opt"}) bodies.push_back(std::make_shared<Body>(name, batch));
  const Transform3fA geometry2body = Pose(0.0f, -1.0f, 1.0f, 0.0f, 0.01f, 0.0f, 0.0f);
  if (!cube_model.AddBody(*bodies[0]) || !grid_model.AddBody(*bodies[1]) ||
      !grid_model.AddBody(*bodies[2], &geometry2body))
    return 1;
  for (auto& b : bodies) b->set_body2world_pose(Transform3fA::Identity());
  const std::vector<Transform3fA> gt = {Pose(0.0f, -1.0f, 1.0f, 0.0f, 0.0f, 0.0f, 0.0f),
                                        Pose(1.0f, 0.0f, 0.0f, 1.0f, 0.003f, 0.004f, 0.0f),
                                        Pose(1.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.002f)};

  float d_cube = 0.0f, d_grid = 0.0f;
  std::vector<YCBEvaluator::Result> ycb;
  std::vector<RBOTEvaluator::Result> rbot;
  std::vector<OPTEvaluator::Result> opt;
  RTBEvaluator::Result rtb;
  const std::vector<std::shared_ptr<Body>> opt_bodies = {bodies[2]};
  if (!cube_model.CalculateDiameter(&d_cube) || !grid_model.CalculateDiameter(&d_grid) ||
      !YCBEvaluator::CalculatePoseResults(bodies, gt, &ycb) || !RBOTEvaluator::CalculatePoseResults(bodies, gt, &rbot) ||
      !OPTEvaluator::CalculatePoseResults(opt_bodies, {gt[2]}, d_grid, &opt) ||
      !RTBEvaluator::CalculatePoseResults(bodies, gt, {{0}, {1, 2}}, 0.1f, &rtb))
    return 1;
  const int n_reduced = int(grid_model.reduced_vertices().size() / 3);
  // a body of another Batch (another context) is refused instead of being scored by its index in this one
  auto other = std::make_shared<Batch>(0, 1, 1, 1);
  const std::vector<std::shared_ptr<Body>> mixed = {bodies[0], std::make_shared<Body>("stranger", other)};
  std::vector<YCBEvaluator::Result> refused;
  const bool mixed_refused = !YCBEvaluator::CalculatePoseResults(mixed, {gt[0], gt[0]}, &refused);

  bool ok = true;
  auto expect = [&](bool c, const char* what) {
    if (!c) std::fprintf(stderr, "check failed: %s\n", what);
    ok = ok && c;
  };
  expect(ycb[0].adds_auc == 1.0f && ycb[0].add_auc < 1.0f, "cube: ADD-S 0 under a 90 degree turn, ADD above 0");
  expect(std::fabs(ycb[1].add_auc - 0.95f) < 1e-6f, "grid: ADD of a 0.005 m translation");
  expect(std::fabs(d_cube - std::sqrt(0.03f)) < 1e-6f, "cube diameter");
  expect(std::fabs(d_grid - std::sqrt(3.0f) * 0.08f) < 1e-6f, "grid diameter");
  expect(n_reduced == 50, "reduced set size");
  expect(mixed_refused, "bodies of two batches are refused");
  expect(std::fabs(rbot[1].translation_error - 0.005f) < 1e-7f && rbot[1].tracking_success == 1.0f, "RBOT translation");
  expect(std::fabs(rbot[0].rotation_error - 1.5707964f) < 1e-6f && rbot[0].tracking_success == 0.0f, "RBOT rotation");

  std::printf("{\"diameters\": [%.9g, %.9g], \"n_reduced\": %d, \"ycb\": [", d_cube, d_grid, n_reduced);
  for (size_t i = 0; i < ycb.size(); ++i) {
    int add_first = 0, adds_first = 0;  // index of the first curve value 1
    while (add_first < 100 && ycb[i].add_curve[add_first] == 0.0f) ++add_first;
    while (adds_first < 100 && ycb[i].adds_curve[adds_first] == 0.0f) ++adds_first;
    std::printf("%s[%.9g, %.9g, %d, %d]", i ? ", " : "", ycb[i].add_auc, ycb[i].adds_auc, add_first, adds_first);
  }
  std::printf("], \"rbot\": [");
  for (size_t i = 0; i < rbot.size(); ++i)
    std::printf("%s[%.9g, %.9g, %.9g]", i ? ", " : "", rbot[i].translation_error, rbot[i].rotation_error,
                rbot[i].tracking_success);
  int opt_first = 0;
  while (opt_first < 100 && opt[0].curve_values[opt_first] == 0.0f) ++opt_first;
  std::printf("], \"opt\": [%.9g, %d], \"rtb\": [%.9g, %.9g], \"ok\": %s}\n", opt[0].area_under_curve, opt_first,
              rtb.add_auc, rtb.adds_auc, ok ? "true" : "false");
  return ok ? 0 : 1;
}
