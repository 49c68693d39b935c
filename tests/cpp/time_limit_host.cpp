// The time limit through the C++ host layer (include/trajopt_b200.hpp, trajopt_b200_json.hpp): a problem in the
// reference's JSON schema (argv[1]) on a three-joint planar arm, two problems that differ in their start state.
//   mode "params": print the flattened description's opt_info.max_time (no device needed);
//   mode "solve":  ConstructProblem + OptimizeWithParams, one line per problem:
//                  status n_qp_solves n_func_evals n_cnts max(cnt_viols) cnt_tolerance
#include <algorithm>
#include <cstdio>
#include <fstream>
#include <sstream>

#include "trajopt_b200_json.hpp"

namespace tb = trajopt_b200;
using namespace tb::trajopt;

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  const std::string mode = argv[2];
  auto kin = std::make_shared<RobotModel>();
  for (int j = 0; j < 3; ++j) {
    RobotModel::Joint jt;
    jt.child_link = "link" + std::to_string(j);
    jt.parent = j - 1;
    jt.type = TB200_JOINT_REVOLUTE;
    jt.q_index = j;
    jt.origin.xyz[0] = j ? 0.3 : 0.0;
    kin->joints.push_back(jt);
  }
  kin->lower.assign(3, -3.0);
  kin->upper.assign(3, 3.0);
  try {
    std::ifstream jf(argv[1]);
    std::stringstream ss;
    ss << jf.rdbuf();
    ProblemConstructionInfo pci;
    pci.kin = kin;
    pci.batch = 2;
    fromJson(pci, tb::json::parse(ss.str()));
    pci.init_info.start = {0.1, -0.2, 0.3, -0.4, 0.5, -0.6};
    if (mode == "params") {
      auto fp = FlattenProblem(pci);
      std::printf("max_time %.17g\n", fp->desc.sqp.max_time);
      return 0;
    }
    TrajOptProb::Ptr prob = ConstructProblem(pci);
    for (const auto& r : OptimizeWithParams(*prob)) {
      const double mx = r.cnt_viols.empty() ? 0.0 : *std::max_element(r.cnt_viols.begin(), r.cnt_viols.end());
      std::printf("%d %d %d %zu %.17g %.17g\n", static_cast<int>(r.status), r.n_qp_solves, r.n_func_evals, r.cnt_viols.size(),
                  mx, pci.opt_info.cnt_tolerance);
    }
    return 0;
  } catch (const std::runtime_error& e) {
    std::fprintf(stderr, "runtime_error: %s\n", e.what());
    return 3;
  }
}
