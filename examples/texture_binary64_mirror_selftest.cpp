// texture_binary64_mirror_selftest.cpp — the set-up conventions of the C++ mirror's TextureModality for BRISK and
// FREAK that need no device: SetUp takes the descriptor type (it stops only at the silhouette renderer, which is not
// set up here), ORB_CUDA is still refused by its type, the descriptor type reaches the parameters handed to
// m3tb_set_texture_modality only once the modality is set up, and the binary SetFeatures refuses anything but one
// 64-byte descriptor per keypoint for BRISK and FREAK. Runs with or without a GPU.
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

  const std::array<int32_t, 4> roi{0, 0, 100, 100};
  for (auto [name, type] : {std::make_pair("brisk", TextureModality::DescriptorType::BRISK),
                            std::make_pair("freak", TextureModality::DescriptorType::FREAK)}) {
    auto texture = std::make_shared<TextureModality>(name, batch, body, camera, silhouette);
    texture->set_descriptor_type(type);
    EXPECT(texture->descriptor_type() == type);
    EXPECT(!texture->SetUp() && !texture->set_up());  // the silhouette renderer is not set up
    EXPECT(texture->params().descriptor_type == M3TB_DESCRIPTOR_ORB);  // not handed on before SetUp succeeds
    EXPECT(!texture->SetFeatures(std::vector<float>(4, 0.0f), std::vector<uint8_t>(2 * 32, 0), roi, 1.0f));
    EXPECT(!texture->SetFeatures(std::vector<float>(4, 0.0f), std::vector<uint8_t>(3 * 64, 0), roi, 1.0f));
  }
  auto orb_cuda = std::make_shared<TextureModality>("orb_cuda", batch, body, camera, silhouette);
  orb_cuda->set_descriptor_type(TextureModality::DescriptorType::ORB_CUDA);
  EXPECT(!orb_cuda->SetUp());
  EXPECT(M3TB_DESCRIPTOR_BRISK == int(TextureModality::DescriptorType::BRISK) &&
         M3TB_DESCRIPTOR_FREAK == int(TextureModality::DescriptorType::FREAK));
  EXPECT(std::string(TextureModality::DescriptorName(TextureModality::DescriptorType::FREAK)) == "FREAK");

  std::cout << ", \"failures\": " << failures << "}" << std::endl;
  return failures == 0 ? 0 : 1;
}
