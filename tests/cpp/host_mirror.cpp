// Exercises the C++ host layer (include/trajopt_b200.hpp) the way a caller of the reference writes a problem:
// ProblemConstructionInfo + TermInfo objects -> ConstructProblem -> OptimizeProblem.  Reads the problem file
// (host_input.hpp), builds the configs[2] description and either dumps the flattened POD description (mode "dump", no
// device needed) or solves it (mode "solve").
#include <cstdio>
#include <fstream>
#include <sstream>

#include "host_input.hpp"
#include "trajopt_b200_json.hpp"

namespace tb = trajopt_b200;
using namespace tb::trajopt;

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  HostProblem hp = readProblem(argv[1]);
  const std::string mode = argv[2];
  ProblemConstructionInfo& pci = hp.pci;
  // JOINT_INTERPOLATED from the first to the last waypoint of the file's trajectories
  const int B = pci.batch, T = pci.basic_info.n_steps, D = pci.kin->numJoints();
  tb::DblVec traj;
  traj.swap(pci.init_info.data);
  pci.init_info.type = InitInfo::JOINT_INTERPOLATED;
  for (int b = 0; b < B; ++b) {
    const auto first = traj.begin() + static_cast<size_t>(b) * T * D, last = first + (T - 1) * D;
    pci.init_info.start.insert(pci.init_info.start.end(), first, first + D);
    pci.init_info.data.insert(pci.init_info.data.end(), last, last + D);
  }

  if (mode == "json") {  // the description comes from a JSON document in the reference's schema (argv[3])
    try {
      std::ifstream jf(argv[3]);
      std::stringstream ss;
      ss << jf.rdbuf();
      ProblemConstructionInfo jp;
      jp.kin = pci.kin;
      jp.batch = B;
      jp.obstacles = pci.obstacles;
      jp.n_obstacles = pci.n_obstacles;
      fromJson(jp, tb::json::parse(ss.str()));
      jp.init_info.start = pci.init_info.start;  // the environment's current joint values, one state per problem
      auto fp = FlattenProblem(jp);
      std::printf("n_terms %d n_cart_targets %d n_fixed %d max_iter %d trust %.17g\n", fp->desc.n_terms, fp->desc.n_cart_targets,
                  fp->desc.n_fixed_timesteps, fp->desc.sqp.max_iter, fp->desc.sqp.trust_box_size);
      const unsigned char* p = reinterpret_cast<const unsigned char*>(fp->terms.data());
      std::printf("terms ");
      for (size_t i = 0; i < fp->terms.size() * sizeof(tb200_term); ++i) std::printf("%02x", p[i]);
      std::printf("\ninit");
      for (double v : fp->init_traj) std::printf(" %.17g", v);
      std::printf("\ntargets");
      for (double v : fp->cart_targets) std::printf(" %.17g", v);
      std::printf("\n");
      return 0;
    } catch (const std::runtime_error& e) {
      std::fprintf(stderr, "runtime_error: %s\n", e.what());
      return 3;
    }
  }

  appendConfig2Terms(hp);
  try {
    if (mode == "dump") {
      auto fp = FlattenProblem(pci);
      std::printf("n_terms %d n_cart_targets %d n_fixed %d\n", fp->desc.n_terms, fp->desc.n_cart_targets, fp->desc.n_fixed_timesteps);
      const unsigned char* p = reinterpret_cast<const unsigned char*>(fp->terms.data());
      std::printf("terms ");
      for (size_t i = 0; i < fp->terms.size() * sizeof(tb200_term); ++i) std::printf("%02x", p[i]);
      std::printf("\ninit");
      for (double v : fp->init_traj) std::printf(" %.17g", v);
      std::printf("\ntargets");
      for (double v : fp->cart_targets) std::printf(" %.17g", v);
      std::printf("\n");
      return 0;
    }
    TrajOptProb::Ptr prob = ConstructProblem(pci);
    // "solve": with the description's own parameters (pci.opt_info); "solve_ref": trajopt::OptimizeProblem, which
    // overrides four of them on top of the optimizer's defaults (problem_description.cpp:394-408)
    std::vector<tb::sco::OptResults> res = (mode == "solve_ref") ? OptimizeProblem(*prob) : OptimizeWithParams(*prob);
    for (const auto& r : res) {
      std::printf("result %d %.17g %d %d", static_cast<int>(r.status), r.total_cost, r.n_qp_solves, r.n_func_evals);
      for (double v : r.x) std::printf(" %.17g", v);
      std::printf("\n");
    }
    return 0;
  } catch (const std::runtime_error& e) {  // PRINT_AND_THROW in the reference
    std::fprintf(stderr, "runtime_error: %s\n", e.what());
    return 3;
  }
}
