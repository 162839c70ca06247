// texture_orb_mirror_selftest.cpp — the conventions of the C++ mirror's device ORB detection that need no device: the
// orb_* settings start at the reference's (300, 1.2, 3), their setters clear set_up as the reference's do, and
// DetectFeatures refuses, before touching the device, a modality that is not set up; an empty list is nothing to do.
// Runs with or without a GPU.
#include <iostream>
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
  std::cout << "{\"have_device\": " << (batch->ok() ? "true" : "false");
  auto body = std::make_shared<Body>("body", batch);
  Intrinsics intr{600.0f, 600.0f, 320.0f, 240.0f, 640, 480};
  auto camera = std::make_shared<ColorCamera>("camera", batch, intr, Transform3fA::Identity());
  auto geometry = std::make_shared<RendererGeometry>("geometry", batch);
  auto silhouette = std::make_shared<FocusedSilhouetteRenderer>("silhouette", batch, geometry, camera, IDType::BODY);

  // the reference's detector settings (texture_modality.h:410-412) and m3tb_orb_params_default agree
  auto texture = std::make_shared<TextureModality>("texture", batch, body, camera, silhouette);
  m3tb_orb_params defaults;
  m3tb_orb_params_default(&defaults);
  EXPECT(texture->orb_n_features() == 300 && texture->orb_scale_factor() == 1.2f && texture->orb_n_levels() == 3);
  EXPECT(defaults.n_features == 300 && defaults.scale_factor == 1.2f && defaults.n_levels == 3);
  // setters change what DetectFeatures hands over
  texture->set_orb_n_features(500);
  texture->set_orb_scale_factor(2.0f);
  texture->set_orb_n_levels(8);
  EXPECT(texture->orb_n_features() == 500 && texture->orb_scale_factor() == 2.0f && texture->orb_n_levels() == 8);
  EXPECT(texture->orb_params().n_features == 500 && texture->orb_params().scale_factor == 2.0f &&
         texture->orb_params().n_levels == 8);
  // the silhouette renderer is not set up (and without a device cannot be): SetUp refuses, and so does detection
  EXPECT(!texture->SetUp() && !texture->set_up());
  EXPECT(!texture->DetectFeatures());
  EXPECT(!TextureModality::DetectFeatures({texture}));
  // an empty list is nothing to do
  EXPECT(TextureModality::DetectFeatures({}));

  std::cout << ", \"failures\": " << failures << "}" << std::endl;
  return failures == 0 ? 0 : 1;
}
