// The trajectory collision check through the C++ host layer (include/trajopt_b200.hpp): ProblemConstructionInfo ->
// ConstructProblem -> checkTrajectories with a CollisionCheckConfig.  Reads the robot, the trajectories, the obstacles and
// the check settings from a text file written by tests/test_check_trajectories.py and prints one line per trajectory:
// found, first_slot, min_distance, the slot minima, the slot contact counts.
#include <cstdio>
#include <fstream>

#include "trajopt_b200.hpp"

namespace tb = trajopt_b200;
using namespace tb::trajopt;

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  std::ifstream in(argv[1]);
  int B, T, D, nseg;
  CollisionCheckConfig cfg;
  in >> B >> T >> D >> nseg >> cfg.type >> cfg.longest_valid_segment_length >> cfg.contact_margin;
  auto kin = std::make_shared<RobotModel>();
  for (int s = 0; s < nseg; ++s) {
    RobotModel::Joint j;
    in >> j.parent >> j.type >> j.q_index >> j.origin.xyz[0] >> j.origin.xyz[1] >> j.origin.xyz[2] >> j.origin.wxyz[0] >>
        j.origin.wxyz[1] >> j.origin.wxyz[2] >> j.origin.wxyz[3] >> j.axis[0] >> j.axis[1] >> j.axis[2];
    j.child_link = "link" + std::to_string(s);
    kin->joints.push_back(j);
  }
  kin->lower.resize(D);
  kin->upper.resize(D);
  for (double& v : kin->lower) in >> v;
  for (double& v : kin->upper) in >> v;
  int nsph;
  in >> nsph;
  for (int s = 0; s < nsph; ++s) {
    RobotModel::Sphere sp;
    int seg;
    in >> seg >> sp.center[0] >> sp.center[1] >> sp.center[2] >> sp.radius;
    sp.link = "link" + std::to_string(seg);
    kin->spheres.push_back(sp);
  }
  std::vector<TrajArray> trajs(B, TrajArray(static_cast<size_t>(T) * D));
  for (TrajArray& t : trajs)
    for (double& v : t) in >> v;
  ProblemConstructionInfo pci;
  pci.kin = kin;
  pci.batch = B;
  pci.basic_info.n_steps = T;
  pci.init_info.type = InitInfo::GIVEN_TRAJ;
  for (const TrajArray& t : trajs) pci.init_info.data.insert(pci.init_info.data.end(), t.begin(), t.end());
  in >> pci.n_obstacles;
  pci.obstacles.resize(static_cast<size_t>(B) * pci.n_obstacles * 4);
  for (double& v : pci.obstacles) in >> v;
  if (!in) { std::fprintf(stderr, "bad input file\n"); return 2; }
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
