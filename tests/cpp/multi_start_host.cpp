// A multi-start solve through the C++ host layer (include/trajopt_b200.hpp): ProblemConstructionInfo with
// seeds_per_problem / stop_seeds_on_converged -> ConstructProblem -> OptimizeProblemMultiStart.
//   multi_start_host <problem file> dump|solve <seeds_per_problem> <stop_seeds_on_converged>
// reads the problem file (host_input.hpp) with the seeded initial trajectories, builds the configs[2] description and
// either dumps what the flattened description says about groups (mode "dump", no device needed) or solves it (mode
// "solve": one line per problem).
#include <cstdio>
#include <cstdlib>

#include "host_input.hpp"

namespace tb = trajopt_b200;
using namespace tb::trajopt;

int main(int argc, char** argv) {
  if (argc < 5) return 2;
  HostProblem hp = readProblem(argv[1]);
  const std::string mode = argv[2];
  ProblemConstructionInfo& pci = hp.pci;
  pci.seeds_per_problem = std::atoi(argv[3]);
  pci.stop_seeds_on_converged = std::atoi(argv[4]) != 0;
  appendConfig2Terms(hp);

  try {
    if (mode == "dump") {
      auto fp = FlattenProblem(pci);
      std::printf("batch %d group_size %d group_stop %d\n", fp->desc.batch, fp->desc.group_size, fp->desc.group_stop);
      return 0;
    }
    TrajOptProb::Ptr prob = ConstructProblem(pci);
    for (const MultiStartResult& r : OptimizeProblemMultiStart(*prob)) {
      std::printf("problem %d %d %.17g", r.best, static_cast<int>(r.result.status), r.result.total_cost);
      for (tb::sco::OptStatus s : r.seed_status) std::printf(" %d", static_cast<int>(s));
      std::printf("\n");
    }
    return 0;
  } catch (const std::runtime_error& e) {
    std::fprintf(stderr, "runtime_error: %s\n", e.what());
    return 3;
  }
}
