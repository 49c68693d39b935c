// The SQP iteration log through the C++ host layer (include/trajopt_b200.hpp), driven by tests/test_sqp_log.py.
//   sqp_log_host synth <dir>          no device: a synthetic log (two problems, written below) is replayed through
//                                     ReplayCallbacks, printing one "cb" line per callback, and written by WriteLogResults
//                                     into <dir>/<problem>
//   sqp_log_host solve <input> <dir>  configs[2] on the problem file (host_input.hpp) with log_results on:
//                                     OptimizeWithParams with a printing callback and a WriteCallback into
//                                     <dir>/write.csv; prints the callbacks and the final results of the logged and
//                                     the plain solve
//   sqp_log_host fk <input>           no device: RobotFK of every waypoint of trajectory 0 ("fk t joint R[9] p[3]")
//   sqp_log_host write <input> <csv>  no device: WriteCallback over the input's robot with synthetic names and results
//                                     (x = trajectory 0), called twice
#include <cstdio>
#include <fstream>

#include "host_input.hpp"

namespace tb = trajopt_b200;
using namespace tb::trajopt;

static void printResults(const char* tag, std::size_t b, const tb::sco::OptResults& r) {
  std::printf("%s %zu %d %d %d %.17g %zu %zu %zu", tag, b, static_cast<int>(r.status), r.n_qp_solves, r.n_func_evals,
              r.total_cost, r.x.size(), r.cost_vals.size(), r.cnt_viols.size());
  for (double v : r.x) std::printf(" %.17g", v);
  for (double v : r.cost_vals) std::printf(" %.17g", v);
  for (double v : r.cnt_viols) std::printf(" %.17g", v);
  std::printf("\n");
}

static Callback printer() {
  return [](TrajOptProb*, std::size_t b, tb::sco::OptResults& r) { printResults("cb", b, r); };
}

// Two problems, T*D = 2, one cost and one constraint, R = 6.  Problem 0: kind 0, a QP failure, a shrink, an accept
// (round 0 iter 1), an accept (iter 2), a converged-by-small-improvement (iter 3, ends).  Problem 1: kind 0, an accept
// and a shrink in round 0 iter 1, then round 1 iter 1: an accept; two records were dropped.
static SqpLog synthetic() {
  SqpLog L;
  L.B = 2; L.R = 6; L.n_costs = 1; L.n_cnts = 1; L.N = 2; L.with_x = true;
  const size_t BR = 12;
  for (auto* v : {&L.kind, &L.merit_round, &L.iter, &L.qp_status, &L.admm_iters, &L.polish, &L.action, &L.ended}) v->assign(BR, 0);
  for (auto* v : {&L.trust_box_size, &L.old_merit, &L.model_merit, &L.new_merit, &L.merit_coeffs, &L.model_cost_vals,
                  &L.model_cnt_viols, &L.old_cost_vals, &L.old_cnt_viols, &L.new_cost_vals, &L.new_cnt_viols})
    v->assign(BR, std::nan(""));
  L.new_x.assign(BR * 2, std::nan(""));
  L.n_records = {6, 4};
  L.n_dropped = {0, 2};
  struct Rec { int b, r, kind, round, iter, action, ended; double mu, mc, mk, nc, nk, x0, x1; };
  const Rec recs[] = {
      {0, 0, 0, 0, 1, -1, -1, 10, NAN, NAN, 5.0, 0.5, 0.1, 0.2},
      {0, 1, 1, 0, 1, 3, -1, 10, NAN, NAN, NAN, NAN, NAN, NAN},
      {0, 2, 1, 0, 1, 0, -1, 10, 1.0, 0.1, 7.0, 0.4, 0.3, 0.3},
      {0, 3, 1, 0, 1, 1, -1, 10, 3.0, 0.2, 4.0, 0.25, 0.15, 0.25},
      {0, 4, 1, 0, 2, 1, -1, 10, 2.5, 0.1, 3.5, 0.125, 0.175, 0.3},
      {0, 5, 1, 0, 3, 2, 0, 10, 3.4999999999, 0.125, 3.5, 0.125, 0.175, 0.3},
      {1, 0, 0, 0, 1, -1, -1, 10, NAN, NAN, 1.0, 2.0, -0.5, 0.5},
      {1, 1, 1, 0, 1, 1, -1, 10, 0.5, 1.0, 0.75, 1.5, -0.25, 0.5},
      {1, 2, 1, 0, 2, 0, -1, 10, 0.5, 1.0, 0.8, 1.6, -0.2, 0.4},
      {1, 3, 1, 1, 1, 1, -1, 100, 0.5, 0.5, 0.6, 0.75, -0.1, 0.3},
  };
  for (const Rec& q : recs) {
    const size_t i = L.at(q.b, q.r);
    L.kind[i] = q.kind; L.merit_round[i] = q.round; L.iter[i] = q.iter; L.action[i] = q.action; L.ended[i] = q.ended;
    L.merit_coeffs[i] = q.mu; L.model_cost_vals[i] = q.mc; L.model_cnt_viols[i] = q.mk;
    L.new_cost_vals[i] = q.nc; L.new_cnt_viols[i] = q.nk; L.new_x[2 * i] = q.x0; L.new_x[2 * i + 1] = q.x1;
  }
  // the derived values of tb200_fetch_sqp_log: old = the last accepted record's new values (or kind 0's)
  for (int b = 0; b < L.B; ++b) {
    size_t last = L.at(b, 0);
    for (int r = 1; r < L.n_records[b]; ++r) {
      const size_t i = L.at(b, r);
      L.old_cost_vals[i] = L.new_cost_vals[last];
      L.old_cnt_viols[i] = L.new_cnt_viols[last];
      if (L.action[i] != 3) {
        L.old_merit[i] = L.old_cost_vals[i] + L.old_cnt_viols[i] * L.merit_coeffs[i];
        L.model_merit[i] = L.model_cost_vals[i] + L.model_cnt_viols[i] * L.merit_coeffs[i];
        L.new_merit[i] = L.new_cost_vals[i] + L.new_cnt_viols[i] * L.merit_coeffs[i];
      }
      if (L.action[i] == 1) last = i;
    }
  }
  return L;
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  const std::string mode = argv[1];
  try {
    if (mode == "synth") {
      const SqpLog L = synthetic();
      const std::vector<std::string> vars = VarNames(1, 2), costs = {"joint_vel"}, cnts = {"collision_3"};
      for (int b = 0; b < L.B; ++b) {
        tb::sco::OptResults fin;
        fin.status = tb::sco::OPT_CONVERGED;
        fin.n_qp_solves = 99;
        ReplayCallbacks(nullptr, L, b, fin, {printer()}, /*allow_truncated=*/b == 1);
        WriteLogResults(L, b, std::string(argv[2]) + "/" + std::to_string(b), vars, costs, cnts);
      }
      try {  // problem 1 dropped records: refused without allow_truncated
        ReplayCallbacks(nullptr, L, 1, tb::sco::OptResults{}, {printer()});
      } catch (const std::runtime_error& e) {
        std::printf("refused %s\n", e.what());
      }
      return 0;
    }
    HostProblem hp = readProblem(argv[2]);
    ProblemConstructionInfo& pci = hp.pci;
    const int T = pci.basic_info.n_steps, D = pci.kin->numJoints();
    const double* x0 = pci.init_info.data.data();
    if (mode == "fk") {
      for (int t = 0; t < T; ++t) {
        const std::vector<Frame> fr = RobotFK(*pci.kin, x0 + static_cast<size_t>(t) * D);
        for (size_t j = 0; j < fr.size(); ++j) {
          std::printf("fk %d %zu", t, j);
          for (double v : fr[j].R) std::printf(" %.17g", v);
          for (double v : fr[j].p) std::printf(" %.17g", v);
          std::printf("\n");
        }
      }
      return 0;
    }
    if (mode == "write") {
      auto file = std::make_shared<std::ofstream>(argv[3]);
      Callback cb = WriteCallback(file, pci.kin, {"joint_vel", "joint_acc"}, {"cart_pose", "collision_3"});
      tb::sco::OptResults r;
      r.x.assign(x0, x0 + static_cast<size_t>(T) * D);
      r.cost_vals = {1.5, 0.0625};
      r.cnt_viols = {0.25, 1e-7};
      cb(nullptr, 0, r);
      r.cost_vals[0] = 3.0;
      cb(nullptr, 0, r);
      return 0;
    }
    if (mode != "solve" || argc < 4) return 2;
    appendConfig2Terms(hp);
    pci.opt_info.log_results = true;
    pci.opt_info.log_dir = argv[3];
    TrajOptProb::Ptr prob = ConstructProblem(pci);
    const std::vector<tb::sco::OptResults> plain = OptimizeWithParams(*prob);
    std::filesystem::create_directories(argv[3]);
    auto csv = std::make_shared<std::ofstream>(std::string(argv[3]) + "/write.csv");
    const std::vector<tb::sco::OptResults> res = OptimizeWithParams(*prob, {printer(), WriteCallback(csv, *prob)});
    for (size_t b = 0; b < res.size(); ++b) {
      printResults("final", b, res[b]);
      printResults("plain", b, plain[b]);
    }
    return 0;
  } catch (const std::runtime_error& e) {
    std::fprintf(stderr, "runtime_error: %s\n", e.what());
    return 3;
  }
}
