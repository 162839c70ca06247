// host_mirror_selftest.cpp — the set-up / error conventions of the C++ mirror that do not need a device, after the
// reference's own tests (OptimizerTest.TestWithoutSetUp / TestWithoutSetUpLink, TrackerTest.TestWithoutSetUp,
// M3T/test/optimizer_test.cpp:88-95, tracker_test.cpp:160-162): every method returns false instead of throwing,
// objects that are not set up refuse to run, structural setters clear set_up. Runs on a machine without GPU: the Batch
// then has no context (there is no CPU fallback) and everything that would need it must fail cleanly.
#include <iostream>
#include <limits>
#include <memory>

#include "m3t_b200/m3t_b200.hpp"

using namespace m3t_b200;

static int failures = 0;
#define EXPECT(cond)                                                                  \
  do {                                                                                \
    if (!(cond)) { std::cout << "FAILED: " #cond " (line " << __LINE__ << ")\n"; ++failures; } \
  } while (0)

int main() {
  auto batch = std::make_shared<Batch>(0, 4, 4, 1);
  const bool have_device = batch->ok();
  std::cout << "{\"have_device\": " << (have_device ? "true" : "false");

  auto body = std::make_shared<Body>("body", batch);
  auto body2 = std::make_shared<Body>("body2", batch);
  EXPECT(body->index() == 0 && body2->index() == 1);

  // Link tree bookkeeping
  auto root = std::make_shared<Link>("root", body);
  auto child = std::make_shared<Link>("child", body2);
  EXPECT(root->AddChildLink(child));
  EXPECT(!root->AddChildLink(child));                 // "Child link ... already exists"
  EXPECT(!root->set_up());                            // structural change clears set_up
  EXPECT(root->SetUp() && root->set_up());
  child->set_free_directions({true, false, false, false, false, false});
  EXPECT(child->DegreesOfFreedom() == 1 && root->DegreesOfFreedom() == 6);
  EXPECT(!child->set_up());

  // Optimizer: referenced links in pre-order, degrees of freedom, refuses without set-up links / modalities
  auto optimizer = std::make_shared<Optimizer>("optimizer", batch, root);
  EXPECT(optimizer->ReferencedLinks().size() == 2 && optimizer->ReferencedLinks()[0] == root);
  EXPECT(optimizer->DegreesOfFreedom() == 7);
  EXPECT(!optimizer->SetUp());                        // "Link child was not set up"
  EXPECT(child->SetUp());
  EXPECT(!optimizer->SetUp());                        // "No modalities were assigned ..."
  EXPECT(!optimizer->set_up());
  EXPECT(!optimizer->CalculateOptimization(0, 0, 0)); // "Set up optimizer ... first"
  EXPECT(!optimizer->CalculateConsistentPoses());

  // Depth modality schedule: a malformed value is refused by its setter whatever the order of the calls; a considered
  // distance below half the stride length, or 2^31 strides or more, is refused by SetUp (as by m3tb_set_body)
  auto depth = std::make_shared<DepthModality>("depth", batch, body, nullptr, nullptr);
  EXPECT(!depth->set_considered_distances({0.05f, 0.0f}) && !depth->set_considered_distances({-0.01f}));
  EXPECT(!depth->set_considered_distances({std::numeric_limits<float>::quiet_NaN()}));
  EXPECT(!depth->set_considered_distances({std::numeric_limits<float>::infinity()}));
  EXPECT(!depth->set_stride_length(0.0f) && !depth->set_stride_length(std::numeric_limits<float>::infinity()));
  EXPECT(depth->params().n_considered_distances == 3 && depth->params().stride_length == 0.005f);
  EXPECT(depth->set_stride_length(0.1f));              // 0.01 / 0.1 + 0.5 < 1 until the schedule follows
  EXPECT(!depth->SetUp() && !depth->set_up());
  EXPECT(depth->set_stride_length(1e-12f));            // 0.05 / 1e-12 strides overflow an int
  EXPECT(!depth->SetUp());
  EXPECT(depth->set_considered_distances({0.2f, 0.1f}) && depth->set_stride_length(0.1f));
  EXPECT(depth->params().n_considered_distances == 2 && depth->params().stride_length == 0.1f);

  // Constraints
  auto constraint = std::make_shared<Constraint>("constraint", root, child);
  constraint->set_constraint_directions({false, true, true, true, true, true});
  EXPECT(constraint->NumberOfConstraints() == 5);
  EXPECT(!constraint->set_up() && constraint->SetUp() && constraint->set_up());
  auto dangling = std::make_shared<Constraint>("dangling", root, nullptr);
  EXPECT(!dangling->SetUp());
  EXPECT(optimizer->AddConstraint(constraint));
  EXPECT(optimizer->NumberOfConstraints() == 5);
  auto soft = std::make_shared<SoftConstraint>("soft", root, child);
  EXPECT(soft->standard_deviation_rotation() == 0.01f && soft->standard_deviation_translation() == 0.001f);
  EXPECT(soft->max_distance_rotation() == 0.0f);

  // Shared colour histograms (region_modality.cpp:168-203): the object's parameters replace the modality's, the modality's
  // own setters refuse while it is shared, and SetUp needs the object set up first
  {
    Intrinsics intr{600.0f, 600.0f, 320.0f, 240.0f, 640, 480};
    auto camera = std::make_shared<ColorCamera>("camera_h", batch, intr, Transform3fA::Identity());
    auto model = std::make_shared<RegionModel>("model_h", batch);
    auto modality = std::make_shared<RegionModality>("region_h", batch, body, camera, model);
    auto histograms = std::make_shared<ColorHistograms>("histograms", 32, 0.3f, 0.1f);
    EXPECT(modality->set_n_histogram_bins(16));
    modality->UseSharedColorHistograms(histograms);
    EXPECT(!modality->set_n_histogram_bins(8) && !modality->set_learning_rate_f(0.5f) && !modality->set_learning_rate_b(0.5f));
    EXPECT(!modality->SetUp());                        // "Color histograms histograms was not set up"
    EXPECT(histograms->SetUp() && modality->SetUp());
    EXPECT(modality->params().n_histogram_bins == 32 && modality->params().learning_rate_f == 0.3f &&
           modality->params().learning_rate_b == 0.1f);
    EXPECT(histograms->owner_body() == -1);            // claimed by the first Optimizer::SetUp that sees it
    modality->DoNotUseSharedColorHistograms();
    EXPECT(!modality->set_up() && modality->set_n_histogram_bins(16) && modality->SetUp());
  }

  // Tracker refuses to run before SetUp (tracker.cpp:224-228)
  Tracker tracker("tracker", batch);
  EXPECT(!tracker.ExecuteTrackingStep(0));

  // Without a device nothing that needs the context may succeed (no CPU fallback)
  if (!have_device) {
    Intrinsics intr{600.0f, 600.0f, 320.0f, 240.0f, 640, 480};
    auto camera = std::make_shared<ColorCamera>("camera", batch, intr, Transform3fA::Identity());
    EXPECT(!camera->SetUp());
    EXPECT(!body->set_body2world_pose(Transform3fA::Identity()));
  }
  std::cout << ", \"failures\": " << failures << "}" << std::endl;
  return failures == 0 ? 0 : 1;
}
