// The problem file of tests/cpp_host.py (write_problem) read into the C++ host layer (include/trajopt_b200.hpp), and
// the configs[2] description of trajopt_b200.problems.config2 written with the layer's TermInfo objects.  Shared by the
// host programs in this directory.
#pragma once

#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <string>
#include <vector>

#include "trajopt_b200.hpp"

struct HostProblem {
  trajopt_b200::trajopt::ProblemConstructionInfo pci;  // kin, batch, n_steps, GIVEN_TRAJ init_traj and obstacles
  std::string tool;                                     // the name of the tool link
  std::vector<trajopt_b200::trajopt::Pose> goals;       // the cart target of every problem, or none
};

// Exits with status 2 when the file cannot be read.
inline HostProblem readProblem(const char* path) {
  using namespace trajopt_b200::trajopt;
  std::ifstream in(path);
  HostProblem p;
  ProblemConstructionInfo& pci = p.pci;
  int B = 0, T = 0, D = 0, nseg = 0, nsph = 0, ngoals = 0;
  in >> B >> T >> D >> nseg;
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
  in >> nsph;
  for (int s = 0; s < nsph; ++s) {
    RobotModel::Sphere sp;
    in >> sp.link >> sp.center[0] >> sp.center[1] >> sp.center[2] >> sp.radius;
    kin->spheres.push_back(sp);
  }
  in >> p.tool;
  pci.kin = kin;
  pci.batch = B;
  pci.basic_info.n_steps = T;
  pci.init_info.type = InitInfo::GIVEN_TRAJ;
  pci.init_info.data.resize(static_cast<size_t>(B) * T * D);
  for (double& v : pci.init_info.data) in >> v;
  in >> ngoals;
  p.goals.resize(ngoals);
  for (Pose& g : p.goals) in >> g.xyz[0] >> g.xyz[1] >> g.xyz[2] >> g.wxyz[0] >> g.wxyz[1] >> g.wxyz[2] >> g.wxyz[3];
  in >> pci.n_obstacles;
  pci.obstacles.resize(static_cast<size_t>(B) * pci.n_obstacles * 4);
  for (double& v : pci.obstacles) in >> v;
  if (!in) {
    std::fprintf(stderr, "bad input file\n");
    std::exit(2);
  }
  return p;
}

// configs[2] (manip "right_arm", the OSQP solver): step 0 fixed, JointVel and JointAcc costs over the whole trajectory,
// a CartPose constraint of the tool at the last step towards p.goals, and a discrete collision constraint (margin 0.02,
// coeff 20, buffer 0.01, longest_valid_segment_length 0.5 as in trajopt_b200.problems.collision_term).
inline void appendConfig2Terms(HostProblem& p) {
  using namespace trajopt_b200::trajopt;
  ProblemConstructionInfo& pci = p.pci;
  const int T = pci.basic_info.n_steps;
  pci.basic_info.manip = "right_arm";
  pci.basic_info.fixed_timesteps = {0};
  pci.basic_info.convex_solver = trajopt_b200::sco::modelTypeFromName("OSQP");
  auto vel = std::make_shared<JointVelTermInfo>();
  vel->term_type = TT_COST;
  vel->first_step = 0; vel->last_step = T - 1;
  auto acc = std::make_shared<JointAccTermInfo>();
  acc->term_type = TT_COST;
  acc->first_step = 0; acc->last_step = T - 1;
  pci.cost_infos.push_back(vel);
  pci.cost_infos.push_back(acc);
  auto pose = std::make_shared<CartPoseTermInfo>();
  pose->term_type = TT_CNT;
  pose->timestep = T - 1;
  pose->source_frame = p.tool;
  pose->target = p.goals;
  auto coll = std::make_shared<CollisionTermInfo>();
  coll->term_type = TT_CNT;
  coll->first_step = 0; coll->last_step = T - 1;
  coll->fixed_steps = {0};
  coll->evaluator_type = TB200_COLL_DISCRETE;
  coll->collision_margin = 0.02; coll->collision_coeff = 20.0; coll->collision_margin_buffer = 0.01;
  coll->longest_valid_segment_length = 0.5;
  pci.cnt_infos.push_back(pose);
  pci.cnt_infos.push_back(coll);
}
