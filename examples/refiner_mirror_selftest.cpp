// refiner_mirror_selftest.cpp — the set-up conventions of the C++ mirror's Refiner that need no device, after the
// reference's Refiner (refiner.h / refiner.cpp): default iteration counts, setters, one optimizer name per refiner,
// RefinePoses refused before SetUp, SetUp refused while an optimizer is not set up, and names that match no optimizer
// ignored without any device work. Runs with or without a GPU.
#include <iostream>
#include <memory>
#include <set>
#include <string>

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

  // defaults and setters (refiner.h:40)
  Refiner refiner("refiner");
  EXPECT(refiner.name() == "refiner" && refiner.n_corr_iterations() == 7 && refiner.n_update_iterations() == 2);
  refiner.set_n_corr_iterations(4);
  refiner.set_n_update_iterations(3);
  EXPECT(refiner.n_corr_iterations() == 4 && refiner.n_update_iterations() == 3);

  // an empty refiner sets up; RefinePoses is refused before SetUp and does nothing for names it does not know
  EXPECT(!refiner.set_up() && !refiner.RefinePoses({"body"}));
  EXPECT(refiner.SetUp() && refiner.set_up());
  EXPECT(refiner.RefinePoses({"body"}) && refiner.RefinePoses({}));

  // optimizers: one per name, one batch per refiner, and SetUp needs them set up
  auto body = std::make_shared<Body>("body", batch);
  auto link = std::make_shared<Link>("link", body);
  auto optimizer = std::make_shared<Optimizer>("optimizer", batch, link);
  EXPECT(refiner.AddOptimizer(optimizer));
  EXPECT(!refiner.set_up());                             // a new optimizer clears set_up
  EXPECT(!refiner.AddOptimizer(optimizer));              // "Optimizer optimizer already exists"
  auto other_batch = std::make_shared<Batch>(0, 4, 4, 1);
  auto other = std::make_shared<Optimizer>("other", other_batch,
                                           std::make_shared<Link>("other_link", std::make_shared<Body>("b", other_batch)));
  EXPECT(!refiner.AddOptimizer(other));
  EXPECT(refiner.optimizer_ptrs().size() == 1);
  EXPECT(!optimizer->set_up() && !refiner.SetUp());      // "Optimizer optimizer was not set up"
  EXPECT(!refiner.RefinePoses({"optimizer"}));

  std::cout << ", \"failures\": " << failures << "}" << std::endl;
  return failures == 0 ? 0 : 1;
}
