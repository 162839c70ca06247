// texture_l2_mirror_selftest.cpp — the set-up conventions of the C++ mirror's TextureModality for SIFT and DAISY that
// need no device: SetUp passes the descriptor type on to the parameters it hands to m3tb_set_texture_modality only
// once the modality is set up, still refuses without a focused silhouette renderer, and the float SetFeatures
// overload refuses a descriptor count that does not match the keypoints. Runs with or without a GPU.
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

  for (auto type : {TextureModality::DescriptorType::SIFT, TextureModality::DescriptorType::DAISY}) {
    // no silhouette renderer: SetUp fails as for ORB (texture_modality.cpp:50-55)
    auto bare = std::make_shared<TextureModality>("bare", batch, body, camera, nullptr);
    bare->set_descriptor_type(type);
    EXPECT(!bare->SetUp() && !bare->set_up());
    EXPECT(!bare->CalculateCorrespondences(0, 0));
    // the descriptor type is kept; the silhouette renderer is not set up (and without a device cannot be)
    auto texture = std::make_shared<TextureModality>("texture", batch, body, camera, silhouette);
    texture->set_descriptor_type(type);
    EXPECT(texture->descriptor_type() == type);
    EXPECT(!texture->SetUp());
    EXPECT(texture->params().descriptor_type == M3TB_DESCRIPTOR_ORB);  // not handed on before SetUp succeeds
    // the float overload: one descriptor of `length` floats per keypoint, length at least 1
    const std::array<int32_t, 4> roi{0, 0, 100, 100};
    EXPECT(!texture->SetFeatures(std::vector<float>(4, 0.0f), std::vector<float>(3 * 128, 0.0f), 128, roi, 1.0f));
    EXPECT(!texture->SetFeatures(std::vector<float>(4, 0.0f), std::vector<float>(), 0, roi, 1.0f));
  }
  // BRISK, FREAK and ORB_CUDA stay refused
  for (auto type : {TextureModality::DescriptorType::BRISK, TextureModality::DescriptorType::FREAK,
                    TextureModality::DescriptorType::ORB_CUDA}) {
    auto other = std::make_shared<TextureModality>("other", batch, body, camera, silhouette);
    other->set_descriptor_type(type);
    EXPECT(!other->SetUp());
  }
  EXPECT(M3TB_DESCRIPTOR_SIFT == int(TextureModality::DescriptorType::SIFT) &&
         M3TB_DESCRIPTOR_DAISY == int(TextureModality::DescriptorType::DAISY));

  std::cout << ", \"failures\": " << failures << "}" << std::endl;
  return failures == 0 ? 0 : 1;
}
