// Per-problem optimizer parameters through the C++ host layer (include/trajopt_b200.hpp): SqpParamRows,
// OptimizeWithParams and OptimizeProblemMultiStart with one sco::BasicTrustRegionSQPParameters per problem.
// Mode "rows" (no device): the size check and the order of the flattened rows.
// Mode "solve <problem file> <K> <seeds_per_problem> <stop_seeds_on_converged>": the configs[2] description of the
// problem file (host_input.hpp); gives problem b the parameter set b % K (set_params below) and prints one line per
// problem, then, with groups, one line per group of the multi-start overload.
#include <cstdio>
#include <cstdlib>

#include "host_input.hpp"

namespace tb = trajopt_b200;
using namespace tb::trajopt;

// Parameter set k of the solve mode (tests/test_sqp_params_per_traj.py restates it)
static tb::sco::BasicTrustRegionSQPParameters set_params(int k) {
  tb::sco::BasicTrustRegionSQPParameters p;
  const double trust[4] = {0.1, 0.02, 0.3, 0.05};
  const double shrink[4] = {0.1, 0.5, 0.1, 0.3};
  const int max_iter[4] = {50, 8, 30, 50};
  p.trust_box_size = trust[k % 4];
  p.trust_shrink_ratio = shrink[k % 4];
  p.max_iter = max_iter[k % 4];
  return p;
}

static int rows_mode() {
  std::vector<tb::sco::BasicTrustRegionSQPParameters> ps(3);
  for (int b = 0; b < 3; ++b) {
    ps[b].trust_box_size = 0.1 * (b + 1);
    ps[b].max_iter = 10 + b;
    ps[b].cnt_tolerance = 1e-3 * (b + 1);
    ps[b].max_time = b == 1 ? -1.0 : ps[b].max_time;
    ps[b].inflate_constraints_individually = b != 2;
  }
  try {
    SqpParamRows(4, ps);
    std::printf("no throw\n");
  } catch (const std::invalid_argument& e) {
    std::printf("invalid_argument %s\n", e.what());
  }
  for (const tb200_sqp_params& r : SqpParamRows(3, ps))
    std::printf("row %.17g %d %.17g %.17g %d %.17g\n", r.trust_box_size, r.max_iter, r.cnt_tolerance, r.max_time,
                r.inflate_constraints_individually, r.initial_merit_error_coeff);
  return 0;
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string mode = argv[1];
  if (mode == "rows") return rows_mode();
  if (mode != "solve" || argc < 6) return 2;
  HostProblem hp = readProblem(argv[2]);
  const int K = std::atoi(argv[3]), G = std::atoi(argv[4]);
  ProblemConstructionInfo& pci = hp.pci;
  pci.seeds_per_problem = G;
  pci.stop_seeds_on_converged = std::atoi(argv[5]) != 0;
  appendConfig2Terms(hp);

  try {
    TrajOptProb::Ptr prob = ConstructProblem(pci);
    std::vector<tb::sco::BasicTrustRegionSQPParameters> params;
    for (int b = 0; b < pci.batch; ++b) params.push_back(set_params(b % K));
    try {
      OptimizeWithParams(*prob, std::vector<tb::sco::BasicTrustRegionSQPParameters>(params.begin(), params.end() - 1));
      std::printf("no throw\n");
    } catch (const std::invalid_argument&) {
      std::printf("throws\n");
    }
    const std::vector<tb::sco::OptResults> r = OptimizeWithParams(*prob, params);
    for (const tb::sco::OptResults& o : r)
      std::printf("traj %d %.17g %d %d\n", static_cast<int>(o.status), o.total_cost, o.n_qp_solves, o.n_func_evals);
    if (G > 1)
      for (const MultiStartResult& m : OptimizeProblemMultiStart(*prob, params))
        std::printf("problem %d %d %.17g\n", m.best, static_cast<int>(m.result.status), m.result.total_cost);
    return 0;
  } catch (const std::runtime_error& e) {
    std::fprintf(stderr, "runtime_error: %s\n", e.what());
    return 3;
  }
}
