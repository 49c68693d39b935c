// Per-problem optimizer parameters through the C++ host layer (include/trajopt_b200.hpp): SqpParamRows,
// OptimizeWithParams and OptimizeProblemMultiStart with one sco::BasicTrustRegionSQPParameters per problem.
// Mode "rows" (no device): the size check and the order of the flattened rows.  Mode "solve <file> <K>": reads the
// configs[2] description written by tests/test_sqp_params_per_traj.py (the format of multi_start_host.cpp), gives
// problem b the parameter set b % K (set_params below) and prints one line per problem, then, with groups, one line per
// group of the multi-start overload.
#include <cstdio>
#include <fstream>

#include "trajopt_b200.hpp"

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
  if (mode != "solve" || argc < 4) return 2;
  std::ifstream in(argv[2]);
  const int K = std::atoi(argv[3]);
  int B, T, D, nseg, G, stop;
  in >> B >> T >> D >> nseg >> G >> stop;
  auto kin = std::make_shared<RobotModel>();
  for (int s = 0; s < nseg; ++s) {
    RobotModel::Joint j;
    in >> j.parent >> j.type >> j.q_index >> j.origin.xyz[0] >> j.origin.xyz[1] >> j.origin.xyz[2] >> j.origin.wxyz[0] >>
        j.origin.wxyz[1] >> j.origin.wxyz[2] >> j.origin.wxyz[3] >> j.axis[0] >> j.axis[1] >> j.axis[2] >> j.child_link;
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
    in >> sp.link >> sp.center[0] >> sp.center[1] >> sp.center[2] >> sp.radius;
    kin->spheres.push_back(sp);
  }
  std::string tool;
  in >> tool;
  ProblemConstructionInfo pci;
  pci.kin = kin;
  pci.batch = B;
  pci.seeds_per_problem = G;
  pci.stop_seeds_on_converged = stop != 0;
  pci.basic_info.n_steps = T;
  pci.basic_info.manip = "right_arm";
  pci.basic_info.fixed_timesteps = {0};
  pci.init_info.type = InitInfo::GIVEN_TRAJ;
  pci.init_info.data.resize(static_cast<size_t>(B) * T * D);
  for (double& v : pci.init_info.data) in >> v;
  std::vector<Pose> goals(B);
  for (Pose& g : goals) in >> g.xyz[0] >> g.xyz[1] >> g.xyz[2] >> g.wxyz[0] >> g.wxyz[1] >> g.wxyz[2] >> g.wxyz[3];
  in >> pci.n_obstacles;
  pci.obstacles.resize(static_cast<size_t>(B) * pci.n_obstacles * 4);
  for (double& v : pci.obstacles) in >> v;
  if (!in) { std::fprintf(stderr, "bad input file\n"); return 2; }

  auto vel = std::make_shared<JointVelTermInfo>();
  vel->term_type = TT_COST;
  vel->first_step = 0; vel->last_step = T - 1;
  auto acc = std::make_shared<JointAccTermInfo>();
  acc->term_type = TT_COST;
  acc->first_step = 0; acc->last_step = T - 1;
  pci.cost_infos = {vel, acc};
  auto pose = std::make_shared<CartPoseTermInfo>();
  pose->term_type = TT_CNT;
  pose->timestep = T - 1;
  pose->source_frame = tool;
  pose->target = goals;
  auto coll = std::make_shared<CollisionTermInfo>();
  coll->term_type = TT_CNT;
  coll->first_step = 0; coll->last_step = T - 1;
  coll->fixed_steps = {0};
  coll->evaluator_type = TB200_COLL_DISCRETE;
  coll->collision_margin = 0.02; coll->collision_coeff = 20.0; coll->collision_margin_buffer = 0.01;
  coll->longest_valid_segment_length = 0.5;
  pci.cnt_infos = {pose, coll};

  try {
    TrajOptProb::Ptr prob = ConstructProblem(pci);
    std::vector<tb::sco::BasicTrustRegionSQPParameters> params;
    for (int b = 0; b < B; ++b) params.push_back(set_params(b % K));
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
