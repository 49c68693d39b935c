// The trajectory collision check through the C++ host layer (include/trajopt_b200.hpp): ProblemConstructionInfo ->
// ConstructProblem -> checkTrajectories with a CollisionCheckConfig.
//   check_host <problem file> <type> <longest_valid_segment_length> <contact_margin>
// checks the trajectories of the problem file (host_input.hpp) and prints one line per trajectory: found, first_slot,
// min_distance, the slot minima, the slot contact counts.
#include <cstdio>
#include <cstdlib>

#include "host_input.hpp"

namespace tb = trajopt_b200;
using namespace tb::trajopt;

int main(int argc, char** argv) {
  if (argc < 5) return 2;
  HostProblem hp = readProblem(argv[1]);
  const ProblemConstructionInfo& pci = hp.pci;
  CollisionCheckConfig cfg;
  cfg.type = std::atoi(argv[2]);
  cfg.longest_valid_segment_length = std::strtod(argv[3], nullptr);
  cfg.contact_margin = std::strtod(argv[4], nullptr);
  const size_t N = static_cast<size_t>(pci.basic_info.n_steps) * pci.kin->numJoints();
  std::vector<TrajArray> trajs;
  for (auto t = pci.init_info.data.begin(); t != pci.init_info.data.end(); t += N) trajs.emplace_back(t, t + N);
  try {
    TrajOptProb::Ptr prob = ConstructProblem(pci);
    for (const TrajectoryCheckResult& r : checkTrajectories(*prob, cfg, &trajs)) {
      std::printf("%d %d %.17g", r.found ? 1 : 0, r.first_slot, r.min_distance);
      for (double v : r.step_min_distance) std::printf(" %.17g", v);
      for (int c : r.step_contacts) std::printf(" %d", c);
      std::printf("\n");
    }
    return 0;
  } catch (const std::runtime_error& e) {
    std::fprintf(stderr, "runtime_error: %s\n", e.what());
    return 3;
  }
}
