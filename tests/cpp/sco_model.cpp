// The reference's solver-interface tests (trajopt_sco/test/solver-interface-unit.cpp:33-73, 136-237) written against
// include/trajopt_b200_sco.hpp exactly as they are written against trajopt_sco: createModel(ModelType), addVar, update,
// setVarBounds, setObjective(exprSquare / exprMult), optimize, getVarValue, removeVar.  Mode "dump": print the canonical QP
// of the setup_problem case (no device needed).  Mode "solve": run the three cases on the GPU and print their results.
#include <cstdio>
#include <iostream>

#include "trajopt_b200_sco.hpp"

using namespace sco;

static Model::Ptr setupProblem(VarVector& vars, AffExpr& aff) {
  const Model::Ptr solver = createModel(ModelType::OSQP);
  for (int i = 0; i < 3; ++i) {
    char namebuf[8];
    std::snprintf(namebuf, sizeof(namebuf), "v%i", i);
    vars.push_back(solver->addVar(namebuf));
  }
  solver->update();
  for (std::size_t i = 0; i < 3; ++i) {
    exprInc(aff, vars[i]);
    solver->setVarBounds(vars[i], 0, 10);
  }
  aff.constant -= 3;
  solver->setObjective(exprSquare(aff));
  solver->update();
  return solver;
}

static double exprMultCase(double v1_val, double v2_val, double v1_coeff, double v2_coeff, double c1, double c2, double& answer) {
  const Model::Ptr solver = createModel(ModelType("OSQP"));
  VarVector vars;
  vars.push_back(solver->addVar("v1"));
  vars.push_back(solver->addVar("v2"));
  solver->update();
  AffExpr aff1, aff2;
  exprInc(aff1, vars[0]);
  solver->setVarBounds(vars[0], v1_val, v1_val);
  aff1.constant = c1;
  aff1.coeffs[0] = v1_coeff;
  exprInc(aff2, vars[1]);
  solver->setVarBounds(vars[1], v2_val, v2_val);
  aff2.constant = c2;
  aff2.coeffs[0] = v2_coeff;
  const QuadExpr aff12 = exprMult(aff1, aff2);
  solver->setObjective(aff12);
  solver->update();
  solver->writeToFile("solver-interface-test.lp");  // in the working directory the test gives
  solver->optimize();
  DblVec soln(2);
  for (std::size_t i = 0; i < 2; ++i) soln[i] = solver->getVarValue(vars[i]);
  answer = (v1_coeff * v1_val + c1) * (v2_coeff * v2_val + c2);
  return aff12.value(soln);
}

int main(int argc, char** argv) {
  const std::string mode = argc > 1 ? argv[1] : "dump";
  VarVector vars;
  AffExpr aff;
  const Model::Ptr solver = setupProblem(vars, aff);
  if (mode == "dump") {
    std::size_t n, m;
    DblVec P, q, A, l, u;
    std::dynamic_pointer_cast<B200Model>(solver)->canonicalForm(n, m, P, q, A, l, u);
    std::printf("%zu %zu\n", n, m);
    for (double v : P) std::printf("%.17g ", v);
    std::printf("\n");
    for (double v : q) std::printf("%.17g ", v);
    std::printf("\n");
    for (double v : A) std::printf("%.17g ", v);
    std::printf("\n");
    for (double v : l) std::printf("%.17g ", v);
    std::printf("\n");
    for (double v : u) std::printf("%.17g ", v);
    std::printf("\n");
    // removal bookkeeping (solver-interface-unit.cpp:70-72)
    solver->removeVar(vars[2]);
    solver->update();
    std::printf("%zu\n", solver->getVars().size());
    try {
      solver->addIneqCnt(QuadExpr(1.0), "q");
      std::printf("no throw\n");
    } catch (const std::runtime_error& e) {
      std::printf("%s\n", e.what());
    }
    return 0;
  }
  // ---- solve: setup_problem -> aff(soln) ~ 0 within 1e-6; ExprMult_test2 -> 400; ExprMult_test3 -> 945
  const CvxOptStatus st = solver->optimize();
  DblVec soln(3);
  for (std::size_t i = 0; i < 3; ++i) soln[i] = solver->getVarValue(vars[i]);
  std::printf("setup_problem status %d aff %.12g x %.9g %.9g %.9g\n", static_cast<int>(st), aff.value(soln), soln[0], soln[1], soln[2]);
  solver->removeVar(vars[2]);
  solver->update();
  std::printf("vars_after_remove %zu\n", solver->getVars().size());
  double answer = 0;
  double got = exprMultCase(10, 20, 2, 1, 0, 0, answer);
  std::printf("ExprMult_test2 %.12g expect %.12g\n", got, answer);
  got = exprMultCase(10, 20, 3, 2, -3, -5, answer);
  std::printf("ExprMult_test3 %.12g expect %.12g\n", got, answer);
  // an infeasible model: x <= -1 and x >= 1  -> CVX_INFEASIBLE (status map of osqp_interface.cpp:565-614)
  {
    const Model::Ptr m2 = createModel();
    Var x = m2->addVar("x", -10, 10);
    m2->update();
    AffExpr a(x), b2(x);
    a.constant = 1.0;          // x + 1 <= 0
    exprScale(b2, -1.0);
    b2.constant = 1.0;         // -x + 1 <= 0
    m2->addIneqCnt(a, "a");
    m2->addIneqCnt(b2, "b");
    m2->setObjective(exprSquare(AffExpr(x)));
    m2->update();
    std::printf("infeasible status %d\n", static_cast<int>(m2->optimize()));
  }
  return 0;
}
