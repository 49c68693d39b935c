// AvoidSingularityTermInfo of the C++ host layer (include/trajopt_b200.hpp) for tests/test_avoid_singularity.py: hatches
// one term on a 2-joint arm through FlattenProblem (no device needed) and prints the tb200_term it became, or the
// message hatch threw.  argv[1]: ok | two_coeffs | unknown_link | default_steps | past_the_end | reversed | cnt
#include <cstdio>
#include <string>

#include "trajopt_b200.hpp"

namespace tb = trajopt_b200;
using namespace tb::trajopt;

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string mode = argv[1];
  auto kin = std::make_shared<RobotModel>();
  RobotModel::Joint j0, j1, tip;
  j0.child_link = "link0"; j0.type = TB200_JOINT_REVOLUTE; j0.q_index = 0;
  j1.child_link = "link1"; j1.parent = 0; j1.type = TB200_JOINT_REVOLUTE; j1.q_index = 1; j1.origin.xyz[0] = 0.5;
  j1.axis[0] = 0; j1.axis[1] = 1; j1.axis[2] = 0;
  tip.child_link = "tool"; tip.parent = 1; tip.origin.xyz[0] = 0.4;
  kin->joints = {j0, j1, tip};
  kin->lower = {-3, -3};
  kin->upper = {3, 3};
  ProblemConstructionInfo pci;
  pci.kin = kin;
  pci.basic_info.n_steps = 5;
  pci.init_info.type = InitInfo::STATIONARY;
  pci.init_info.start = {0.1, 0.2};
  auto t = std::make_shared<AvoidSingularityTermInfo>();
  t->term_type = mode == "cnt" ? TT_CNT : TT_COST;
  t->link = mode == "unknown_link" ? "nowhere" : "tool";
  if (mode != "default_steps") { t->first_step = 1; t->last_step = 4; }
  if (mode == "past_the_end") t->last_step = 5;
  if (mode == "reversed") { t->first_step = 3; t->last_step = 2; }
  if (mode == "two_coeffs") t->coeffs = {1.0, 2.0};
  if (mode == "ok") { t->coeffs = {2.5}; t->lambda = 0.05; }
  (mode == "cnt" ? pci.cnt_infos : pci.cost_infos).push_back(t);
  try {
    auto fp = FlattenProblem(pci);
    const tb200_term& r = fp->terms.at(0);
    std::printf("kind %d role %d link %d first %d last %d coeff %.17g lambda %.17g\n", r.kind, r.role, r.link, r.first_step,
                r.last_step, r.coeffs[0], r.lambda);
    return 0;
  } catch (const std::runtime_error& e) {
    std::printf("runtime_error: %s\n", e.what());
    return 3;
  }
}
