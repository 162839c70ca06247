// texture_mirror_selftest.cpp — the set-up conventions of the C++ mirror's TextureModality that need no device: SetUp
// refuses without a focused silhouette renderer and for a descriptor type other than ORB, a link refuses a texture
// modality of another body, and the modality has no correspondence renderers (the Tracker must not render its
// silhouette renderer before every correspondence iteration). Runs with or without a GPU.
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
  auto other = std::make_shared<Body>("other", batch);
  Intrinsics intr{600.0f, 600.0f, 320.0f, 240.0f, 640, 480};
  auto camera = std::make_shared<ColorCamera>("camera", batch, intr, Transform3fA::Identity());
  auto geometry = std::make_shared<RendererGeometry>("geometry", batch);
  auto silhouette = std::make_shared<FocusedSilhouetteRenderer>("silhouette", batch, geometry, camera, IDType::BODY);
  auto depth_renderer = std::make_shared<FocusedBasicDepthRenderer>("depth_renderer", batch, geometry, camera);

  // no silhouette renderer: TextureModality::SetUp fails (texture_modality.cpp:50-55)
  auto bare = std::make_shared<TextureModality>("bare", batch, body, camera, nullptr);
  EXPECT(!bare->SetUp() && !bare->set_up());
  EXPECT(!bare->StartModality(0, 0) && !bare->CalculateCorrespondences(0, 0));  // "Set up modality ... first"

  // only ORB is implemented
  auto brisk = std::make_shared<TextureModality>("brisk", batch, body, camera, silhouette);
  brisk->set_descriptor_type(TextureModality::DescriptorType::BRISK);
  EXPECT(!brisk->SetUp());
  EXPECT(brisk->params().descriptor_type == M3TB_DESCRIPTOR_ORB);

  // the setters change the parameters handed to m3tb_set_texture_modality and clear set_up
  auto texture = std::make_shared<TextureModality>("texture", batch, body, camera, silhouette);
  texture->set_n_keyframes(3);
  texture->set_standard_deviations({20.0f, 10.0f, 5.0f});
  texture->set_max_keyframe_age(7);
  EXPECT(texture->params().n_keyframes == 3 && texture->params().n_standard_deviations == 3 &&
         texture->params().standard_deviations[2] == 5.0f && texture->params().max_keyframe_age == 7);
  texture->ModelOcclusions(depth_renderer);
  EXPECT(texture->params().model_occlusions == 1 && texture->depth_renderer_ptr() == depth_renderer);
  // no correspondence renderers, even with a silhouette and a depth renderer (texture_modality.h)
  EXPECT(texture->correspondence_renderer_ptrs().empty());
  const Modality& as_modality = *texture;
  EXPECT(as_modality.correspondence_renderer_ptrs().empty());
  texture->DoNotModelOcclusions();
  EXPECT(texture->params().model_occlusions == 0 && !texture->depth_renderer_ptr());
  // the silhouette renderer is not set up (and without a device cannot be): SetUp refuses
  EXPECT(!texture->SetUp());

  // a texture modality of another body on a link: Link::SetUp fails (link.cpp:37-58)
  auto foreign = std::make_shared<TextureModality>("foreign", batch, other, camera, silhouette);
  auto link = std::make_shared<Link>("link", body);
  EXPECT(link->AddModality(foreign));
  EXPECT(!link->SetUp() && !link->set_up());
  auto own = std::make_shared<Link>("own", other);
  EXPECT(own->AddModality(foreign) && own->SetUp());

  std::cout << ", \"failures\": " << failures << "}" << std::endl;
  return failures == 0 ? 0 : 1;
}
