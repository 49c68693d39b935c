// A multi-start solve through the C++ host layer (include/trajopt_b200.hpp): ProblemConstructionInfo with
// seeds_per_problem / stop_seeds_on_converged -> ConstructProblem -> OptimizeProblemMultiStart.  Reads the robot, the
// seeded initial trajectories and the per-trajectory data from a text file written by tests/test_multi_start.py, builds
// the configs[2] description and either dumps what the flattened description says about groups (mode "dump", no
// device needed) or solves it (mode "solve": one line per problem).
#include <cstdio>
#include <fstream>

#include "trajopt_b200.hpp"

namespace tb = trajopt_b200;
using namespace tb::trajopt;

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  std::ifstream in(argv[1]);
  const std::string mode = argv[2];
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
