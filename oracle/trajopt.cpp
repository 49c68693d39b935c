// ORACLE — TEST INFRASTRUCTURE ONLY (see trajopt.hpp / sco.hpp header comments).
#include "trajopt.hpp"

#include <algorithm>
#include <cmath>
#include <functional>
#include <limits>
#include <cstdlib>
#include <cstring>
#include <stdexcept>

namespace oracle {

// ============================================================================ small rigid-body algebra
Pose poseIdentity() {
  Pose t{};
  t.R[0] = t.R[4] = t.R[8] = 1.0;
  return t;
}
Pose poseMul(const Pose& a, const Pose& b) {
  Pose o{};
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += a.R[i * 3 + k] * b.R[k * 3 + j];
      o.R[i * 3 + j] = s;
    }
    o.p[i] = a.R[i * 3] * b.p[0] + a.R[i * 3 + 1] * b.p[1] + a.R[i * 3 + 2] * b.p[2] + a.p[i];
  }
  return o;
}
Pose poseInv(const Pose& a) {
  Pose o{};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) o.R[i * 3 + j] = a.R[j * 3 + i];
  for (int i = 0; i < 3; ++i) o.p[i] = -(o.R[i * 3] * a.p[0] + o.R[i * 3 + 1] * a.p[1] + o.R[i * 3 + 2] * a.p[2]);
  return o;
}
static void quatToRot(const double* q, double* R) {  // wxyz, normalised here
  double w = q[0], x = q[1], y = q[2], z = q[3];
  const double n = std::sqrt(w * w + x * x + y * y + z * z);
  w /= n; x /= n; y /= n; z /= n;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - z * w);     R[2] = 2 * (x * z + y * w);
  R[3] = 2 * (x * y + z * w);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - x * w);
  R[6] = 2 * (x * z - y * w);     R[7] = 2 * (y * z + x * w);     R[8] = 1 - 2 * (x * x + y * y);
}
Pose poseFromXyzWxyz(const double* xyz, const double* wxyz) {
  Pose t{};
  quatToRot(wxyz, t.R);
  for (int i = 0; i < 3; ++i) t.p[i] = xyz[i];
  return t;
}
void rotToQuatWxyz(const double* m, double* q) {
  // Eigen::Quaterniond(Matrix3d) (trace / largest-diagonal branches) [EXT]
  double t = m[0] + m[4] + m[8];
  if (t > 0) {
    t = std::sqrt(t + 1.0);
    q[0] = 0.5 * t;
    t = 0.5 / t;
    q[1] = (m[7] - m[5]) * t;
    q[2] = (m[2] - m[6]) * t;
    q[3] = (m[3] - m[1]) * t;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[i * 3 + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0);
    q[1 + i] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m[k * 3 + j] - m[j * 3 + k]) * t;
    q[1 + j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
    q[1 + k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
  }
}
// axis (unit) and signed angle in [-pi, pi]; axis = (1,0,0), angle 0 for the identity.
static void rotErrDecomposed(const double* R, double axis[3], double& angle) {
  double q[4];
  rotToQuatWxyz(R, q);
  // Eigen::AngleAxisd(q): angle = 2 atan2(|v|, |w|) in [0, pi], axis = v/|v| * sign(w).  The
  // tesseract helper then flips the pair so the axis always equals +v/|v| and the sign lives in the
  // angle ("not ideal for numerical differentiation" otherwise) and wraps the angle to [-pi, pi].
  const double n = std::sqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (n == 0.0) {
    axis[0] = 1; axis[1] = 0; axis[2] = 0;
    angle = 0;
    return;
  }
  double ang = 2.0 * std::atan2(n, std::fabs(q[0]));
  const double s = (q[0] < 0) ? -1.0 : 1.0;
  for (int i = 0; i < 3; ++i) axis[i] = q[1 + i] / n;
  ang *= s;
  const double two_pi = 2.0 * M_PI;
  ang = std::copysign(std::fmod(std::fabs(ang), two_pi), ang);
  if (ang < -M_PI)
    ang += two_pi;
  else if (ang > M_PI)
    ang -= two_pi;
  angle = ang;
}
void calcRotationalError(const double* R, double out[3]) {
  double axis[3], angle;
  rotErrDecomposed(R, axis, angle);
  for (int i = 0; i < 3; ++i) out[i] = axis[i] * angle;
}
void calcTransformError(const Pose& t1, const Pose& t2, double out[6]) {
  const Pose e = poseMul(poseInv(t1), t2);
  for (int i = 0; i < 3; ++i) out[i] = e.p[i];
  calcRotationalError(e.R, out + 3);
}
void calcJacobianTransformErrorDiff(const Pose& target, const Pose& source, const Pose& source_pert, double out[6]) {
  const Pose tinv = poseInv(target);
  const Pose e0 = poseMul(tinv, source);
  const Pose e1 = poseMul(tinv, source_pert);
  double a0[3], a1[3], g0, g1;
  rotErrDecomposed(e0.R, a0, g0);
  rotErrDecomposed(e1.R, a1, g1);
  // keep the perturbed axis on the same side as the nominal one, and the angle on the same branch
  if (a1[0] * a0[0] + a1[1] * a0[1] + a1[2] * a0[2] < 0) {
    for (double& v : a1) v = -v;
    g1 = -g1;
  }
  const double diff = g1 - g0;
  if (diff > M_PI)
    g1 -= 2.0 * M_PI;
  else if (diff < -M_PI)
    g1 += 2.0 * M_PI;
  for (int i = 0; i < 3; ++i) {
    out[i] = e1.p[i] - e0.p[i];
    out[3 + i] = a1[i] * g1 - a0[i] * g0;
  }
}

// ============================================================================ robot
Robot::Robot(const tb200_robot& r) : n_dof(r.n_dof) {
  segs.assign(r.segments, r.segments + r.n_segments);
  if (r.n_spheres > 0) spheres.assign(r.spheres, r.spheres + r.n_spheres);
  lower.assign(r.lower, r.lower + r.n_dof);
  upper.assign(r.upper, r.upper + r.n_dof);
}
void Robot::fk(const double* q, std::vector<Pose>& frames) const {
  frames.resize(segs.size());
  for (size_t s = 0; s < segs.size(); ++s) {
    const tb200_segment& g = segs[s];
    Pose t = poseFromXyzWxyz(g.origin_xyz, g.origin_wxyz);
    if (g.joint_type == TB200_JOINT_REVOLUTE) {
      const double a = q[g.q_index], c = std::cos(a), sn = std::sin(a), v = 1 - c;
      const double x = g.axis[0], y = g.axis[1], z = g.axis[2];
      Pose m = poseIdentity();  // Rodrigues
      m.R[0] = c + x * x * v;     m.R[1] = x * y * v - z * sn; m.R[2] = x * z * v + y * sn;
      m.R[3] = y * x * v + z * sn; m.R[4] = c + y * y * v;     m.R[5] = y * z * v - x * sn;
      m.R[6] = z * x * v - y * sn; m.R[7] = z * y * v + x * sn; m.R[8] = c + z * z * v;
      t = poseMul(t, m);
    } else if (g.joint_type == TB200_JOINT_PRISMATIC) {
      Pose m = poseIdentity();
      for (int i = 0; i < 3; ++i) m.p[i] = g.axis[i] * q[g.q_index];
      t = poseMul(t, m);
    }
    frames[s] = (g.parent < 0) ? t : poseMul(frames[g.parent], t);
  }
}
void Robot::jacobian(const std::vector<Pose>& frames, int link, const double* point, std::vector<Vec>& J) const {
  J.assign(6, Vec(n_dof, 0.0));
  for (int s = link; s >= 0; s = segs[s].parent) {
    const tb200_segment& g = segs[s];
    if (g.joint_type == TB200_JOINT_FIXED) continue;
    const Pose& f = frames[s];
    double a[3];
    for (int i = 0; i < 3; ++i) a[i] = f.R[i * 3] * g.axis[0] + f.R[i * 3 + 1] * g.axis[1] + f.R[i * 3 + 2] * g.axis[2];
    const int c = g.q_index;
    if (g.joint_type == TB200_JOINT_REVOLUTE) {
      const double r[3] = {point[0] - f.p[0], point[1] - f.p[1], point[2] - f.p[2]};
      J[0][c] = a[1] * r[2] - a[2] * r[1];
      J[1][c] = a[2] * r[0] - a[0] * r[2];
      J[2][c] = a[0] * r[1] - a[1] * r[0];
      J[3][c] = a[0]; J[4][c] = a[1]; J[5][c] = a[2];
    } else {
      J[0][c] = a[0]; J[1][c] = a[1]; J[2][c] = a[2];
    }
  }
}

// ============================================================================ joint-space terms
namespace {
// order 0/1/2 = position / velocity / acceleration stencil on rows first..last (inclusive)
struct JointStencil {
  int order, first, last, D;
  Vec coeffs, targets, upper, lower;
  int nRows() const { return last - first + 1 - order; }
  AffExpr expr(int i, int j) const {  // e = stencil(x) - target, trajectory_costs.cpp:151-160, 277-286, 522-533
    AffExpr a;
    static const double w[3][3] = {{1, 0, 0}, {-1, 1, 0}, {1, -2, 1}};
    for (int k = 0; k <= order; ++k) {
      a.vars.push_back((i + k) * D + j);
      a.coeffs.push_back(w[order][k]);
    }
    a.constant = -targets[j];
    return a;
  }
  double err(const Vec& x, int i, int j) const { return expr(i, j).value(x.data()); }
};

class JointEqCost : public Cost {  // JointPosEqCost / JointVelEqCost / JointAccEqCost
public:
  explicit JointEqCost(JointStencil s) : s_(std::move(s)) {
    if (s_.nRows() <= 0) throw std::runtime_error("joint cost: trajectory is too short");
    for (int i = s_.first; i < s_.first + s_.nRows(); ++i)
      for (int j = 0; j < s_.D; ++j) {
        QuadExpr q = exprSquare(s_.expr(i, j));
        exprScale(q, s_.coeffs[j]);
        exprInc(expr_, q);
      }
  }
  double value(const Vec& x) override {
    double out = 0;
    for (int i = s_.first; i < s_.first + s_.nRows(); ++i)
      for (int j = 0; j < s_.D; ++j) {
        const double e = s_.err(x, i, j);
        out += e * e * s_.coeffs[j];
      }
    return out;
  }
  std::shared_ptr<ConvexObjective> convex(const Vec&, Model* m) override {
    auto out = std::make_shared<ConvexObjective>(m);
    out->addQuadExpr(expr_);
    return out;
  }

private:
  JointStencil s_;
  QuadExpr expr_;
};
class JointEqConstraint : public Constraint {  // rows c*e, value c*e^2 (quirk kept, trajectory_costs.cpp:160,173)
public:
  explicit JointEqConstraint(JointStencil s) : s_(std::move(s)) {
    if (s_.nRows() <= 0) throw std::runtime_error("joint constraint: trajectory is too short");
  }
  CntType type() const override { return EQ; }
  Vec value(const Vec& x) override {
    Vec out;
    for (int i = s_.first; i < s_.first + s_.nRows(); ++i)
      for (int j = 0; j < s_.D; ++j) {
        const double e = s_.err(x, i, j);
        out.push_back(e * e * s_.coeffs[j]);
      }
    return out;
  }
  std::shared_ptr<ConvexConstraints> convex(const Vec&, Model*) override {
    auto out = std::make_shared<ConvexConstraints>();
    for (int i = s_.first; i < s_.first + s_.nRows(); ++i)
      for (int j = 0; j < s_.D; ++j) {
        AffExpr a = s_.expr(i, j);
        exprScale(a, s_.coeffs[j]);
        out->eqs.push_back(a);
      }
    return out;
  }

private:
  JointStencil s_;
};
// two rows per (step, joint): (e - upper_tol)*c and (lower_tol - e)*c   (trajectory_costs.cpp:185-254, 303-374)
static void ineqRows(const JointStencil& s, std::vector<AffExpr>& rows) {
  for (int i = s.first; i < s.first + s.nRows(); ++i)
    for (int j = 0; j < s.D; ++j) {
      AffExpr up = s.expr(i, j);
      up.constant -= s.upper[j];
      exprScale(up, s.coeffs[j]);
      rows.push_back(up);
      AffExpr lo = s.expr(i, j);
      exprScale(lo, -1.0);
      lo.constant += s.lower[j];
      exprScale(lo, s.coeffs[j]);
      rows.push_back(lo);
    }
}
class JointIneqCost : public Cost {
public:
  explicit JointIneqCost(JointStencil s) : s_(std::move(s)) { ineqRows(s_, rows_); }
  double value(const Vec& x) override {
    double out = 0;
    for (const AffExpr& r : rows_) out += std::max(r.value(x.data()), 0.0);
    return out;
  }
  std::shared_ptr<ConvexObjective> convex(const Vec&, Model* m) override {
    auto out = std::make_shared<ConvexObjective>(m);
    for (const AffExpr& r : rows_) out->addHinge(r, 1);
    return out;
  }

private:
  JointStencil s_;
  std::vector<AffExpr> rows_;
};
class JointIneqConstraint : public Constraint {
public:
  explicit JointIneqConstraint(JointStencil s) : s_(std::move(s)) { ineqRows(s_, rows_); }
  CntType type() const override { return INEQ; }
  Vec value(const Vec& x) override {
    // reference layout: all upper rows then all lower rows (out << diff1, diff2); only sums are consumed
    Vec out;
    for (const AffExpr& r : rows_) out.push_back(r.value(x.data()));
    return out;
  }
  std::shared_ptr<ConvexConstraints> convex(const Vec&, Model*) override {
    auto out = std::make_shared<ConvexConstraints>();
    out->ineqs = rows_;
    return out;
  }

private:
  JointStencil s_;
  std::vector<AffExpr> rows_;
};

// ============================================================================ collision (discrete)
// unit normal d / |d| from the robot sphere towards the obstacle; coincident centres (|d| = 0) take the fixed
// scene-frame normal (1, 0, 0) instead of 0/0 (DESIGN.md section 6, "Coincident centres"), as the kernel does
static void contactNormal(const double* d, double len, double* n) {
  if (len > 0.0) {
    for (int i = 0; i < 3; ++i) n[i] = d[i] / len;
  } else {
    n[0] = 1.0; n[1] = 0.0; n[2] = 0.0;
  }
}
struct Contact {
  int sphere, obstacle;
  double dist;
  double normal[3];   // from robot sphere centre (A) towards the obstacle (B)
  double point[3];    // robot sphere centre in the scene root (reference point of the gradient)
};
struct CollisionEval {
  std::shared_ptr<Robot> robot;
  Vec obstacles;  // [O][4]
  int t, D;
  double margin, coeff, buffer;
  // SingleTimestepCollisionEvaluator::CalcCollisions (collision_terms.cpp:655-691): all pairs with
  // distance <= margin + buffer, ordered by (robot sphere, obstacle).
  void contacts(const Vec& x, std::vector<Contact>& out, std::vector<Pose>& frames) const {
    robot->fk(x.data() + t * D, frames);
    out.clear();
    const int O = static_cast<int>(obstacles.size() / 4);
    for (size_t s = 0; s < robot->spheres.size(); ++s) {
      const tb200_sphere& sp = robot->spheres[s];
      const Pose& f = frames[sp.segment];
      double c[3];
      for (int i = 0; i < 3; ++i)
        c[i] = f.R[i * 3] * sp.center[0] + f.R[i * 3 + 1] * sp.center[1] + f.R[i * 3 + 2] * sp.center[2] + f.p[i];
      for (int o = 0; o < O; ++o) {
        const double* ob = &obstacles[o * 4];
        const double d[3] = {ob[0] - c[0], ob[1] - c[1], ob[2] - c[2]};
        const double len = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        const double dist = len - sp.radius - ob[3];
        if (dist > margin + buffer) continue;
        Contact ct;
        ct.sphere = static_cast<int>(s);
        ct.obstacle = o;
        ct.dist = dist;
        contactNormal(d, len, ct.normal);
        for (int i = 0; i < 3; ++i) ct.point[i] = c[i];
        out.push_back(ct);
      }
    }
  }
  // CollisionsToDistanceExpressions + CalcDistExpressionsSingleTimeStep (collision_terms.cpp:343-383, 540-556):
  // dist(q) ~ d0 + g.(q - q0), g = -n' J_lin (link A active, obstacle static => only gradients[0]).
  void distExpressions(const Vec& x, std::vector<AffExpr>& exprs) const {
    std::vector<Contact> cts;
    std::vector<Pose> frames;
    contacts(x, cts, frames);
    exprs.clear();
    std::vector<Vec> J;
    for (const Contact& ct : cts) {
      robot->jacobian(frames, robot->spheres[ct.sphere].segment, ct.point, J);
      AffExpr e;
      double dot = 0;
      for (int j = 0; j < D; ++j) {
        const double g = -(ct.normal[0] * J[0][j] + ct.normal[1] * J[1][j] + ct.normal[2] * J[2][j]);
        e.vars.push_back(t * D + j);
        e.coeffs.push_back(g);
        dot += g * x[t * D + j];
      }
      e.constant = -dot + ct.dist;
      exprs.push_back(e);  // (cleanupAff result is discarded in the reference: collision_terms.cpp:554)
    }
  }
  // every (sphere, obstacle) candidate; filtered ones carry weight 0 and a zero gradient (fixed GPU layout)
  void denseRows(const Vec& x, std::vector<Vec>& rows) const {
    std::vector<Pose> frames;
    robot->fk(x.data() + t * D, frames);
    const int O = static_cast<int>(obstacles.size() / 4);
    std::vector<Vec> J;
    for (size_t s = 0; s < robot->spheres.size(); ++s) {
      const tb200_sphere& sp = robot->spheres[s];
      const Pose& f = frames[sp.segment];
      double c[3];
      for (int i = 0; i < 3; ++i)
        c[i] = f.R[i * 3] * sp.center[0] + f.R[i * 3 + 1] * sp.center[1] + f.R[i * 3 + 2] * sp.center[2] + f.p[i];
      robot->jacobian(frames, sp.segment, c, J);
      for (int o = 0; o < O; ++o) {
        const double* ob = &obstacles[o * 4];
        const double d[3] = {ob[0] - c[0], ob[1] - c[1], ob[2] - c[2]};
        const double len = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        const double dist = len - sp.radius - ob[3];
        Vec row(D + 3, 0.0);
        const bool filtered = dist > margin + buffer;  // no expression is ever built for a filtered contact
        if (!filtered)  // (coincident centres: the normal (1, 0, 0) of contactNormal)
          for (int j = 0; j < D; ++j)
            row[j] = len > 0.0 ? -(d[0] * J[0][j] + d[1] * J[1][j] + d[2] * J[2][j]) / len : -J[0][j];
        row[D] = dist;
        row[D + 1] = margin;
        row[D + 2] = filtered ? 0.0 : coeff;
        rows.push_back(row);
      }
    }
  }
  Vec values(const Vec& x) const {  // collision_terms.cpp:1391-1412
    std::vector<Contact> cts;
    std::vector<Pose> frames;
    contacts(x, cts, frames);
    Vec out;
    for (const Contact& ct : cts) out.push_back(std::max(margin - ct.dist, 0.0) * coeff);
    return out;
  }
};
// ============================================================================ collision (continuous, "cast")
// CastCollisionEvaluator (collision_terms.cpp:1071-1173) + GetGradient(q0, q1, ...) (:262-323) +
// CalcDistExpressions{BothFree,StartFree,EndFree} (:468-538) + the fixed-state contact filter
// (trajopt_common/src/collision_utils.cpp:73-114), for the synthetic sphere model of SURVEY.md §8d:
// the swept robot sphere of a (sub-)segment is the capsule between its two centres; contact with a static
// obstacle sphere is closed form (closest point of the centre segment, parameter s clamped to [0,1]).
//   * LVS: ||q1-q0|| > longest_valid_segment_length  =>  ceil(dist/lvs) sub-segments between linearly
//     interpolated joint states (the reference's LinSpaced sub-trajectory, :1118-1155), unbounded as in the
//     reference.  The fixed-layout row output (denseRows, what the CUDA path is compared in) is the step pair's
//     ACTIVE contacts in canonical order (sphere, obstacle, sub-segment) followed by zero rows up to
//     the pair's row block (tb200inl_cast_rows_per_pair).
//     CONTINUOUS (evaluator 3) never subdivides (lvs = max double, problem_description.cpp:1782-1784).
//   * cc_time of a contact in sub-segment i of n: (i + s)/n  (addInterpolatedCollisionResults [EXT]);
//     type Time0 iff i == 0 and s == 0, Time1 iff i == n-1 and s == 1, else Between.
//   * filter: distance > margin + buffer; start fixed and Time0; end fixed and Time1.
//   * gradient: Jacobian of the link at q0 + (q1-q0)*cc_time, reference point moved by
//     R_link(sub-segment start | end) * c_local for the timestep-0 | timestep-1 expression
//     (jacobianChangeRefPoint with transform | cc_transform), g_k = -n' J_lin, scaled (1-cc_time) | cc_time.
//   * row: dist + g_0.(q_t - q0) + g_1.(q_t+1 - q1), coefficients |c| <= 1e-7 dropped (cleanupAff IS applied
//     on this path, :481,502,536); a fixed side contributes nothing.
struct CastContact {
  int sphere, obstacle, sub;
  double dist, cc_time;
  double normal[3];
  Vec g0, g1;  // scaled gradients over q_t and q_{t+1} (zero on a fixed side)
};
struct CastCollisionEval {
  std::shared_ptr<Robot> robot;
  Vec obstacles;  // [O][4]
  int t, D;
  double margin, coeff, buffer, lvs;
  bool start_fixed, end_fixed;
  int row_cap;  // rows of a step pair in the fixed-layout output (tb200inl_cast_rows_per_pair)
  // LVS_DISCRETE (DiscreteCollisionEvaluator, collision_terms.cpp:744-893): a discrete contact test at EVERY state of
  // the sub-trajectory (both waypoints included: cnt = ceil(dist/lvs) + 1 states, 2 when the step is short) instead of
  // a swept test per sub-segment.  cc_time of a contact at state i is i / (cnt - 1), type Time0 | Time1 at the two
  // waypoints, transform == cc_transform == the link frame at that state (addInterpolatedCollisionResults with
  // discrete = true [EXT]); filter, gradient and rows as for the swept evaluator.
  bool discrete_states = false;

  int subSegments(const double* q0, const double* q1) const {
    double d2 = 0;
    for (int j = 0; j < D; ++j) d2 += (q1[j] - q0[j]) * (q1[j] - q0[j]);
    const double dist = std::sqrt(d2);
    if (!(dist > lvs)) return 1;
    return static_cast<int>(std::ceil(dist / lvs));
  }
  void sphereCentre(const std::vector<Pose>& fr, int s, double* c) const {
    const tb200_sphere& sp = robot->spheres[s];
    const Pose& f = fr[sp.segment];
    for (int i = 0; i < 3; ++i)
      c[i] = f.R[i * 3] * sp.center[0] + f.R[i * 3 + 1] * sp.center[1] + f.R[i * 3 + 2] * sp.center[2] + f.p[i];
  }
  // every candidate (sphere, obstacle, sub-segment); `all` keeps the filtered ones too (flag active)
  struct Cand {
    bool exists, active;
    CastContact ct;
  };
  // out: [sphere][obstacle][n] with n = the sub-segments of this step pair (returned)
  int candidates(const Vec& x, std::vector<Cand>& out) const {
    const double* q0 = x.data() + t * D;
    const double* q1 = x.data() + (t + 1) * D;
    const int n = subSegments(q0, q1);
    const int O = static_cast<int>(obstacles.size() / 4), L = static_cast<int>(robot->spheres.size());
    std::vector<std::vector<Pose>> fr(n + 1);
    Vec u(D);
    for (int i = 0; i <= n; ++i) {
      for (int j = 0; j < D; ++j) u[j] = (i == n) ? q1[j] : q0[j] + (q1[j] - q0[j]) * (static_cast<double>(i) / n);
      robot->fk(u.data(), fr[i]);
    }
    const int n_slots = discrete_states ? n + 1 : n;  // states | sub-segments
    out.assign(static_cast<size_t>(L) * O * n_slots, Cand{});
    std::vector<Pose> frt;
    std::vector<Vec> J;
    for (int s = 0; s < L; ++s) {
      const tb200_sphere& sp = robot->spheres[s];
      for (int o = 0; o < O; ++o) {
        const double* ob = &obstacles[o * 4];
        for (int i = 0; i < n_slots; ++i) {
          Cand& cd = out[(static_cast<size_t>(s) * O + o) * n_slots + i];
          cd.exists = true;
          const int i_end = discrete_states ? i : i + 1;  // a state is a sub-segment of zero length
          double ca[3], cb[3], w[3], ww = 0, wd = 0;
          sphereCentre(fr[i], s, ca);
          sphereCentre(fr[i_end], s, cb);
          for (int k = 0; k < 3; ++k) {
            w[k] = cb[k] - ca[k];
            ww += w[k] * w[k];
            wd += (ob[k] - ca[k]) * w[k];
          }
          double sc = (ww > 0) ? wd / ww : 0.0;
          sc = sc < 0 ? 0.0 : (sc > 1 ? 1.0 : sc);
          double d[3], len2 = 0;
          for (int k = 0; k < 3; ++k) {
            d[k] = ob[k] - (ca[k] + sc * w[k]);
            len2 += d[k] * d[k];
          }
          const double len = std::sqrt(len2);
          CastContact& ct = cd.ct;
          ct.sphere = s; ct.obstacle = o; ct.sub = i;
          ct.dist = len - sp.radius - ob[3];
          ct.cc_time = (i + sc) / n;
          contactNormal(d, len, ct.normal);
          const bool time0 = (i == 0 && sc == 0.0), time1 = discrete_states ? (i == n) : (i == n - 1 && sc == 1.0);
          cd.active = !(ct.dist > margin + buffer) && !(start_fixed && time0) && !(end_fixed && time1);
          ct.g0.assign(D, 0.0);
          ct.g1.assign(D, 0.0);
          if (!cd.active) continue;
          // Jacobian at the contact-time state, reference point shifted with the sub-segment's start / end rotation
          Vec qt(D);
          for (int j = 0; j < D; ++j) qt[j] = (ct.cc_time == 1.0) ? q1[j] : q0[j] + (q1[j] - q0[j]) * ct.cc_time;
          robot->fk(qt.data(), frt);
          const Pose& lt = frt[sp.segment];
          for (int k = 0; k < 2; ++k) {
            if ((k == 0 && start_fixed) || (k == 1 && end_fixed)) continue;
            const Pose& lk = fr[discrete_states ? i : i + k][sp.segment];
            double pt[3];
            for (int a = 0; a < 3; ++a)
              pt[a] = lk.R[a * 3] * sp.center[0] + lk.R[a * 3 + 1] * sp.center[1] + lk.R[a * 3 + 2] * sp.center[2] + lt.p[a];
            robot->jacobian(frt, sp.segment, pt, J);
            const double scale = (k == 0) ? 1.0 - ct.cc_time : ct.cc_time;
            Vec& g = (k == 0) ? ct.g0 : ct.g1;
            for (int j = 0; j < D; ++j)
              g[j] = -(ct.normal[0] * J[0][j] + ct.normal[1] * J[1][j] + ct.normal[2] * J[2][j]) * scale;
          }
        }
      }
    }
    return n_slots;
  }
  void distExpressions(const Vec& x, std::vector<AffExpr>& exprs) const {
    std::vector<Cand> cands;
    candidates(x, cands);
    exprs.clear();
    for (const Cand& cd : cands) {
      if (!cd.exists || !cd.active) continue;
      AffExpr e;
      e.constant = cd.ct.dist;
      for (int k = 0; k < 2; ++k) {
        if ((k == 0 && start_fixed) || (k == 1 && end_fixed)) continue;
        const Vec& g = (k == 0) ? cd.ct.g0 : cd.ct.g1;
        double dot = 0;
        for (int j = 0; j < D; ++j) {
          e.vars.push_back((t + k) * D + j);
          e.coeffs.push_back(g[j]);
          dot += g[j] * x[(t + k) * D + j];
        }
        e.constant -= dot;
      }
      exprs.push_back(cleanupAff(e));
    }
  }
  // fixed GPU layout: the active contacts in canonical order -> {g0[D], g1[D], dist0, margin, coeff}, then zero rows
  void denseRows(const Vec& x, std::vector<Vec>& rows) const {
    std::vector<Cand> cands;
    candidates(x, cands);
    int n_act = 0;
    for (const Cand& cd : cands) {
      if (!cd.exists || !cd.active) continue;
      if (++n_act > row_cap) throw std::runtime_error("oracle: more active contacts in a step pair than its row block holds");
      Vec row(2 * D + 3, 0.0);
      for (int j = 0; j < D; ++j) {
        row[j] = cd.ct.g0[j];
        row[D + j] = cd.ct.g1[j];
      }
      row[2 * D] = cd.ct.dist;
      row[2 * D + 1] = margin;
      row[2 * D + 2] = coeff;
      rows.push_back(row);
    }
    for (; n_act < row_cap; ++n_act) rows.push_back(Vec(2 * D + 3, 0.0));
  }
  Vec values(const Vec& x) const {
    std::vector<Cand> cands;
    candidates(x, cands);
    Vec out;
    for (const Cand& cd : cands)
      if (cd.exists && cd.active) out.push_back(std::max(margin - cd.ct.dist, 0.0) * coeff);
    return out;
  }
};

// what CollisionCost / CollisionConstraint need from an evaluator (collision_terms.cpp:1283-1412)
struct CollisionCalc {
  std::function<void(const Vec&, std::vector<AffExpr>&)> distExpressions;
  std::function<Vec(const Vec&)> values;
  double margin, coeff;
};
template <class E>
CollisionCalc calcOf(const E& e) {
  return CollisionCalc{[e](const Vec& x, std::vector<AffExpr>& ex) { e.distExpressions(x, ex); },
                       [e](const Vec& x) { return e.values(x); }, e.margin, e.coeff};
}
class CollisionConstraint : public Constraint {
public:
  explicit CollisionConstraint(CollisionCalc e) : e_(std::move(e)) {}
  CntType type() const override { return INEQ; }
  Vec value(const Vec& x) override { return e_.values(x); }
  std::shared_ptr<ConvexConstraints> convex(const Vec& x, Model*) override {
    auto out = std::make_shared<ConvexConstraints>();
    std::vector<AffExpr> exprs;
    e_.distExpressions(x, exprs);
    for (AffExpr& d : exprs) {  // coeff * (margin - dist(q)) <= 0
      exprScale(d, -1.0);
      d.constant += e_.margin;
      exprScale(d, e_.coeff);
      out->ineqs.push_back(d);
    }
    return out;
  }

private:
  CollisionCalc e_;
};
class CollisionCost : public Cost {
public:
  explicit CollisionCost(CollisionCalc e) : e_(std::move(e)) {}
  double value(const Vec& x) override {
    double s = 0;
    for (double v : e_.values(x)) s += v;
    return s;
  }
  std::shared_ptr<ConvexObjective> convex(const Vec& x, Model* m) override {
    auto out = std::make_shared<ConvexObjective>(m);
    std::vector<AffExpr> exprs;
    e_.distExpressions(x, exprs);
    for (AffExpr& d : exprs) {  // hinge(margin - dist(q)) * coeff
      exprScale(d, -1.0);
      d.constant += e_.margin;
      out->addHinge(d, e_.coeff);
    }
    return out;
  }

private:
  CollisionCalc e_;
};
}  // namespace

// ============================================================================ avoid_singularity
// AvoidSingularityTermInfo (kinematic_terms.cpp:586-642): err = 1/(s + lambda) - 1/(0.1 + lambda), s the smallest
// singular value of the 6 x D geometric Jacobian of the link's origin, by a one-sided Jacobi SVD (the rotation order
// and stopping rule of the device's); the gradient is the reference's forward difference
// g_j = u' ((J(q + eps e_j) - J(q)) / eps) v, eps = 1e-6, times -1 / (s + lambda)^2.
namespace sing {
namespace {
constexpr double kEps = 1e-6, kUlp = 2.220446049250313e-16;  // rotations stop at |a_p.a_q| <= M kUlp |a_p||a_q|
constexpr int kSweeps = 32;
}  // namespace

void jacobiSvdMin(const double* J, int D, double& sigma, double* u, double* v) {
  const int NC = D < 6 ? D : 6, M = D < 6 ? 6 : D;
  std::vector<double> A(static_cast<size_t>(M) * NC), V(static_cast<size_t>(NC) * NC, 0.0);  // row-major
  for (int i = 0; i < M; ++i)
    for (int k = 0; k < NC; ++k) A[i * NC + k] = D < 6 ? J[i * D + k] : J[k * D + i];
  for (int k = 0; k < NC; ++k) V[k * NC + k] = 1.0;
  auto dot = [&](int p, int q) {
    double s = 0.0;
    for (int i = 0; i < M; ++i) s += A[i * NC + p] * A[i * NC + q];
    return s;
  };
  for (int sweep = 0; sweep < kSweeps; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < NC - 1; ++p)
      for (int q = p + 1; q < NC; ++q) {
        const double al = dot(p, p), be = dot(q, q), ga = dot(p, q);
        if (!(std::fabs(ga) > M * kUlp * std::sqrt(al * be))) continue;
        const double zeta = (be - al) / (2.0 * ga);
        const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / std::sqrt(1.0 + t * t), s = c * t;
        for (int i = 0; i < M; ++i) {
          const double ap = A[i * NC + p], aq = A[i * NC + q];
          A[i * NC + p] = c * ap - s * aq;
          A[i * NC + q] = s * ap + c * aq;
        }
        for (int i = 0; i < NC; ++i) {
          const double vp = V[i * NC + p], vq = V[i * NC + q];
          V[i * NC + p] = c * vp - s * vq;
          V[i * NC + q] = s * vp + c * vq;
        }
        rotated = true;
      }
    if (!rotated) break;
  }
  int kmin = 0;
  sigma = 0.0;
  for (int k = 0; k < NC; ++k) {
    const double sk = std::sqrt(dot(k, k));
    if (k == 0 || sk < sigma) {
      sigma = sk;
      kmin = k;
    }
  }
  double* w = D < 6 ? u : v;   // W_k / sigma
  double* vk = D < 6 ? v : u;  // V_k
  for (int i = 0; i < M; ++i) w[i] = sigma > 0.0 ? A[i * NC + kmin] / sigma : 0.0;
  for (int i = 0; i < NC; ++i) vk[i] = V[i * NC + kmin];
}

void jacobianAt(const Robot& robot, const double* q, int link, std::vector<double>& J) {
  std::vector<Pose> fr;
  robot.fk(q, fr);
  std::vector<Vec> Jv;
  robot.jacobian(fr, link, fr[link].p, Jv);
  const int D = robot.n_dof;
  J.assign(6 * D, 0.0);
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < D; ++j) J[i * D + j] = Jv[i][j];
}

void errGrad(const Robot& robot, const double* q, int link, double lambda, double* err, double* grad, double* sigma_out) {
  const int D = robot.n_dof;
  std::vector<double> J0, Jk;
  jacobianAt(robot, q, link, J0);
  double sigma, u[6], v[16];
  jacobiSvdMin(J0.data(), D, sigma, u, v);
  if (err) *err = 1.0 / (sigma + lambda) - 1.0 / (0.1 + lambda);
  if (sigma_out) *sigma_out = sigma;
  if (!grad) return;
  std::vector<double> qk(q, q + D), dJ(6 * D);
  for (int j = 0; j < D; ++j) {
    qk[j] = q[j] + kEps;
    jacobianAt(robot, qk.data(), link, Jk);
    qk[j] = q[j];
    for (int e = 0; e < 6 * D; ++e) dJ[e] = (Jk[e] - J0[e]) / kEps;  // difference matrix, then the division
    double g = 0.0;
    for (int c = 0; c < D; ++c) {  // (u' dJ) v
      double s = 0.0;
      for (int i = 0; i < 6; ++i) s += u[i] * dJ[i * D + c];
      g += s * v[c];
    }
    grad[j] = g;
  }
  const double scale = -1.0 / ((sigma + lambda) * (sigma + lambda));
  for (int j = 0; j < D; ++j) grad[j] *= scale;
}
}  // namespace sing

// ============================================================================ problem assembly
SQPParams sqpParamsFrom(const tb200_sqp_params& p) {
  SQPParams s;
  s.improve_ratio_threshold = p.improve_ratio_threshold;
  s.min_trust_box_size = p.min_trust_box_size;
  s.min_approx_improve = p.min_approx_improve;
  s.min_approx_improve_frac = p.min_approx_improve_frac;
  s.max_iter = p.max_iter;
  s.trust_shrink_ratio = p.trust_shrink_ratio;
  s.trust_expand_ratio = p.trust_expand_ratio;
  s.cnt_tolerance = p.cnt_tolerance;
  s.max_merit_coeff_increases = p.max_merit_coeff_increases;
  s.max_qp_solver_failures = p.max_qp_solver_failures;
  s.merit_coeff_increase_ratio = p.merit_coeff_increase_ratio;
  s.initial_merit_error_coeff = p.initial_merit_error_coeff;
  s.inflate_constraints_individually = p.inflate_constraints_individually != 0;
  s.trust_box_size = p.trust_box_size;
  return s;
}
QPSettings qpSettingsFrom(const tb200_qp_settings& q) {
  QPSettings s;
  s.rho = q.rho; s.sigma = q.sigma; s.alpha = q.alpha;
  s.eps_abs = q.eps_abs; s.eps_rel = q.eps_rel;
  s.eps_prim_inf = q.eps_prim_inf; s.eps_dual_inf = q.eps_dual_inf;
  s.delta = q.delta; s.adaptive_rho_tolerance = q.adaptive_rho_tolerance;
  s.max_iter = q.max_iter; s.scaling = q.scaling; s.check_termination = q.check_termination;
  s.adaptive_rho = q.adaptive_rho; s.adaptive_rho_interval = q.adaptive_rho_interval;
  s.polishing = q.polishing; s.polish_refine_iter = q.polish_refine_iter; s.warm_starting = q.warm_starting;
  s.early_polish_every = q.early_polish_every; s.early_polish_from = q.early_polish_from;
  // ORACLE_PLAIN_OSQP=1 (tests only): OSQP's own behaviour - no early polish (O1), the polish accepted by OSQP's rule
  // without verification rounds (D2), the next QP warm started from the polished duals (D1)
  if (const char* e = getenv("ORACLE_PLAIN_OSQP")) {
    if (atoi(e)) {
      s.early_polish_every = 0;
      s.verify_rounds = 0;
      s.warm_polished_duals = 1;
    }
  }
  if (const char* e = getenv("ORACLE_EARLY_STABLE")) s.early_polish_stable = atoi(e);
  if (const char* e = getenv("ORACLE_EARLY_EVERY")) s.early_polish_every = atoi(e);
  return s;
}

TrajProblem buildProblem(const tb200_problem_desc& desc, int b, int cast_cap) {
  if (cast_cap < 0) cast_cap = tb200inl_cast_rows_per_pair(&desc);
  TrajProblem tp;
  tp.robot = std::make_shared<Robot>(desc.robot);
  const int T = desc.n_steps, D = desc.robot.n_dof;
  tp.T = T;
  tp.D = D;
  tp.prob = std::make_shared<OptProb>(qpSettingsFrom(desc.qp));
  // TrajOptProb ctor: variables j_<t>_<d>, timestep-major, bounds = joint limits per step
  Vec lb(T * D), ub(T * D);
  for (int t = 0; t < T; ++t)
    for (int d = 0; d < D; ++d) {
      lb[t * D + d] = desc.robot.lower[d];
      ub[t * D + d] = desc.robot.upper[d];
    }
  tp.prob->createVariables(T * D, lb, ub);
  tp.init.assign(desc.init_traj + static_cast<size_t>(b) * T * D, desc.init_traj + static_cast<size_t>(b + 1) * T * D);
  // fixed_timesteps / fixed_dofs -> permanent model rows (problem_description.cpp:485-530)
  for (int k = 0; k < desc.n_fixed_timesteps; ++k) {
    const int t = desc.fixed_timesteps[k];
    for (int d = 0; d < D; ++d) {
      AffExpr e = AffExpr::var(t * D + d);
      e.constant = -tp.init[t * D + d];
      tp.prob->addLinearConstraint(e, EQ);
    }
  }
  for (int k = 0; k < desc.n_fixed_dofs; ++k) {
    const int d = desc.fixed_dofs[k];
    for (int t = 0; t < T; ++t) {
      bool skip = false;
      for (int f = 0; f < desc.n_fixed_timesteps; ++f) skip |= (desc.fixed_timesteps[f] == t);
      if (skip) continue;
      AffExpr e = AffExpr::var(t * D + d);
      e.constant = -tp.init[t * D + d];
      tp.prob->addLinearConstraint(e, EQ);
    }
  }
  Vec obstacles;
  if (desc.n_obstacles > 0) {
    const double* o = desc.obstacles + (desc.obstacles_per_traj ? static_cast<size_t>(b) * desc.n_obstacles * 4 : 0);
    obstacles.assign(o, o + desc.n_obstacles * 4);
  }

  // the collision rows of the cost objects come first, then those of the constraints (the objects' OptProb order, the
  // layout of tb200_convexify_batch)
  std::vector<std::function<void(const Vec& x, std::vector<Vec>& rows)>> cnt_coll_hooks;
  for (int k = 0; k < desc.n_terms; ++k) {
    const tb200_term& tm = desc.terms[k];
    const bool is_cost = tm.role == TB200_ROLE_COST;
    const std::string nm = "term" + std::to_string(k);
    auto addCost = [&](std::shared_ptr<Cost> c, const std::string& name, int step) {
      c->name = name;
      c->term = k;
      c->step = step;
      tp.prob->addCost(c);
    };
    auto addCnt = [&](std::shared_ptr<Constraint> c, const std::string& name, int step) {
      c->name = name;
      c->term = k;
      c->step = step;
      tp.prob->addConstraint(c);
    };
    switch (tm.kind) {
      case TB200_TERM_JOINT_POS:
      case TB200_TERM_JOINT_VEL:
      case TB200_TERM_JOINT_ACC: {
        JointStencil s;
        s.order = tm.kind - TB200_TERM_JOINT_POS;
        s.first = tm.first_step;
        s.last = tm.last_step;
        s.D = D;
        s.coeffs.assign(tm.coeffs, tm.coeffs + D);
        s.targets.assign(tm.targets, tm.targets + D);
        s.upper.assign(tm.upper_tols, tm.upper_tols + D);
        s.lower.assign(tm.lower_tols, tm.lower_tols + D);
        bool zero_tol = true;  // doubleEquals(tol, 0) for all joints => Eq flavour
        for (int d = 0; d < D; ++d) zero_tol &= std::fabs(s.upper[d]) < 1e-5 && std::fabs(s.lower[d]) < 1e-5;
        if (is_cost) {
          std::shared_ptr<Cost> c;
          if (zero_tol) c = std::make_shared<JointEqCost>(s);
          else c = std::make_shared<JointIneqCost>(s);
          addCost(c, nm, tm.first_step);
        } else {
          std::shared_ptr<Constraint> c;
          if (zero_tol) c = std::make_shared<JointEqConstraint>(s);
          else c = std::make_shared<JointIneqConstraint>(s);
          addCnt(c, nm, tm.first_step);
        }
        break;
      }
      case TB200_TERM_CART_POSE: {
        // CartPoseTermInfo::hatch (problem_description.cpp:901-987): rows with |coeff| <= 1e-5 dropped
        std::vector<int> idx;
        Vec coeff;
        for (int i = 0; i < 3; ++i)
          if (std::fabs(tm.pos_coeffs[i]) > 1e-5) { idx.push_back(i); coeff.push_back(tm.pos_coeffs[i]); }
        for (int i = 0; i < 3; ++i)
          if (std::fabs(tm.rot_coeffs[i]) > 1e-5) { idx.push_back(3 + i); coeff.push_back(tm.rot_coeffs[i]); }
        const double* tgt = (tm.target_slot >= 0)
                                ? desc.cart_targets + (static_cast<size_t>(b) * desc.n_cart_targets + tm.target_slot) * 7
                                : tm.target_pose;
        const Pose target = poseFromXyzWxyz(tgt, tgt + 3);
        const Pose src_off = poseFromXyzWxyz(tm.source_offset, tm.source_offset + 3);
        auto robot = tp.robot;
        const int link = tm.link;
        auto source_tf = [robot, link, src_off](const Vec& q) {
          std::vector<Pose> fr;
          robot->fk(q.data(), fr);
          return poseMul(fr[link], src_off);
        };
        VectorFn f = [=](const Vec& q) {  // CartPoseErrCalculator::operator(), kinematic_terms.cpp:250-263
          double e[6];
          calcTransformError(target, source_tf(q), e);
          Vec out;
          for (int i : idx) out.push_back(e[i]);
          return out;
        };
        MatrixFn dfdx = [=](const Vec& q) {  // CartPoseJacCalculator::operator(), kinematic_terms.cpp:348-366
          const double eps = 1e-5;
          const Pose src = source_tf(q);
          std::vector<Vec> J(idx.size(), Vec(q.size()));
          Vec qp = q;
          for (size_t i = 0; i < q.size(); ++i) {
            qp[i] = q[i] + eps;
            double diff[6];
            calcJacobianTransformErrorDiff(target, src, source_tf(qp), diff);
            for (size_t r = 0; r < idx.size(); ++r) J[r][i] = diff[idx[r]] / eps;
            qp[i] = q[i];
          }
          return J;
        };
        std::vector<int> vars(D);
        for (int d = 0; d < D; ++d) vars[d] = tm.first_step * D + d;
        tp.cart_hooks.push_back([=](const Vec& x, Vec& err, std::vector<Vec>& jac) {
          Vec q(x.begin() + vars[0], x.begin() + vars[0] + D);
          Vec e = f(q);
          std::vector<Vec> J = dfdx(q);
          for (size_t r = 0; r < e.size(); ++r) {
            err.push_back(e[r] * coeff[r]);
            for (double& v : J[r]) v *= coeff[r];
            jac.push_back(J[r]);
          }
        });
        if (is_cost)
          addCost(std::make_shared<CostFromErrFunc>(f, dfdx, vars, coeff, ABS), nm, tm.first_step);
        else
          addCnt(std::make_shared<ConstraintFromErrFunc>(f, dfdx, vars, coeff, EQ), nm, tm.first_step);
        break;
      }
      case TB200_TERM_CART_VEL: {
        // CartVelTermInfo::hatch (problem_description.cpp:1011-1057): one object per step pair
        auto robot = tp.robot;
        const int link = tm.link;
        const double lim = tm.max_displacement;
        for (int t = tm.first_step; t <= tm.last_step; ++t) {
          if (t + 1 >= T) throw std::runtime_error("cart_vel: step pair beyond the trajectory");
          VectorFn f = [=](const Vec& qq) {  // kinematic_terms.cpp:411-425
            std::vector<Pose> f0, f1;
            robot->fk(qq.data(), f0);
            robot->fk(qq.data() + robot->n_dof, f1);
            Vec out(6);
            for (int i = 0; i < 3; ++i) {
              out[i] = f1[link].p[i] - f0[link].p[i] - lim;
              out[3 + i] = f0[link].p[i] - f1[link].p[i] - lim;
            }
            return out;
          };
          MatrixFn dfdx = [=](const Vec& qq) {  // kinematic_terms.cpp:376-401
            const int n = robot->n_dof;
            std::vector<Pose> f0, f1;
            robot->fk(qq.data(), f0);
            robot->fk(qq.data() + n, f1);
            std::vector<Vec> J0, J1;
            robot->jacobian(f0, link, f0[link].p, J0);
            robot->jacobian(f1, link, f1[link].p, J1);
            std::vector<Vec> J(6, Vec(2 * n));
            for (int i = 0; i < 3; ++i)
              for (int j = 0; j < n; ++j) {
                J[i][j] = -J0[i][j];
                J[i][n + j] = J1[i][j];
                J[3 + i][j] = J0[i][j];
                J[3 + i][n + j] = -J1[i][j];
              }
            return J;
          };
          std::vector<int> vars(2 * D);
          for (int d = 0; d < D; ++d) {
            vars[d] = t * D + d;
            vars[D + d] = (t + 1) * D + d;
          }
          tp.cart_hooks.push_back([=](const Vec& x, Vec& err, std::vector<Vec>& jac) {
            Vec qq(x.begin() + vars[0], x.begin() + vars[0] + 2 * D);
            Vec e = f(qq);
            std::vector<Vec> J = dfdx(qq);
            for (size_t r = 0; r < e.size(); ++r) {
              err.push_back(e[r]);
              jac.push_back(J[r]);
            }
          });
          if (is_cost)
            addCost(std::make_shared<CostFromErrFunc>(f, dfdx, vars, Vec(), ABS), nm + "_" + std::to_string(t), t);
          else
            addCnt(std::make_shared<ConstraintFromErrFunc>(f, dfdx, vars, Vec(), INEQ), "CartVel", t);
        }
        break;
      }
      case TB200_TERM_COLLISION: {
        if (tm.evaluator_type != TB200_COLL_DISCRETE) {
          // CollisionTermInfo::hatch continuous branch (problem_description.cpp:1776-1819 / cost: 1714-1760):
          // one object per step pair [first, last), expression type from the fixed steps
          const double lvs = (tm.evaluator_type == TB200_COLL_CONTINUOUS) ? std::numeric_limits<double>::max()
                                                                          : tm.longest_valid_segment_length;
          for (int t = tm.first_step; t < tm.last_step; ++t) {
            bool cur_fixed = false, next_fixed = false;
            for (int f = 0; f < tm.n_fixed_steps; ++f) {
              cur_fixed |= (tm.fixed_steps[f] == t);
              next_fixed |= (tm.fixed_steps[f] == t + 1);
            }
            // (two adjacent fixed steps fall into the START_FIXED_END_FREE branch: the reference's throw is unreachable)
            CastCollisionEval e{tp.robot, obstacles, t, D, tm.margin, tm.coeff, tm.margin_buffer, lvs, cur_fixed,
                                !cur_fixed && next_fixed, cast_cap, tm.evaluator_type == TB200_COLL_LVS_DISCRETE};
            (is_cost ? tp.coll_hooks : cnt_coll_hooks).push_back([e](const Vec& x, std::vector<Vec>& rows) { e.denseRows(x, rows); });
            if (is_cost)
              addCost(std::make_shared<CollisionCost>(calcOf(e)), nm + "_" + std::to_string(t), t);
            else
              addCnt(std::make_shared<CollisionConstraint>(calcOf(e)), nm + "_" + std::to_string(t), t);
          }
          break;
        }
        // CollisionTermInfo::hatch discrete branch (problem_description.cpp:1762-1775, 1824-1833)
        for (int t = tm.first_step; t <= tm.last_step; ++t) {
          bool fixed = false;
          for (int f = 0; f < tm.n_fixed_steps; ++f) fixed |= (tm.fixed_steps[f] == t);
          if (fixed) continue;
          CollisionEval e{tp.robot, obstacles, t, D, tm.margin, tm.coeff, tm.margin_buffer};
          (is_cost ? tp.coll_hooks : cnt_coll_hooks).push_back([e](const Vec& x, std::vector<Vec>& rows) { e.denseRows(x, rows); });
          if (is_cost)
            addCost(std::make_shared<CollisionCost>(calcOf(e)), nm + "_" + std::to_string(t), t);
          else
            addCnt(std::make_shared<CollisionConstraint>(calcOf(e)), nm + "_" + std::to_string(t), t);
        }
        break;
      }
      case TB200_TERM_AVOID_SINGULARITY: {
        // AvoidSingularityTermInfo::hatch (problem_description.cpp:1900-1939): one object per step, ABS cost or INEQ
        // constraint, and one coefficient-scaled Cartesian row per step
        if (tm.link < 0 || tm.link >= desc.robot.n_segments) throw std::runtime_error("avoid_singularity link out of range");
        if (tm.first_step < 0 || tm.last_step >= T || tm.first_step > tm.last_step)
          throw std::runtime_error("avoid_singularity steps outside the trajectory");
        auto robot = tp.robot;
        const int link = tm.link;
        const double lambda = tm.lambda, coeff = tm.coeffs[0];
        for (int t = tm.first_step; t <= tm.last_step; ++t) {
          std::vector<int> vars(D);
          for (int j = 0; j < D; ++j) vars[j] = t * D + j;
          VectorFn f = [robot, link, lambda](const Vec& q) {
            Vec e(1);
            sing::errGrad(*robot, q.data(), link, lambda, &e[0], nullptr, nullptr);
            return e;
          };
          MatrixFn dfdx = [robot, link, lambda](const Vec& q) {
            std::vector<Vec> g(1, Vec(q.size()));
            sing::errGrad(*robot, q.data(), link, lambda, nullptr, g[0].data(), nullptr);
            return g;
          };
          tp.cart_hooks.push_back([=](const Vec& x, Vec& err, std::vector<Vec>& jac) {
            double e;
            Vec g(D);
            sing::errGrad(*robot, x.data() + t * D, link, lambda, &e, g.data(), nullptr);
            err.push_back(coeff * e);
            for (double& v : g) v = coeff * v;
            jac.push_back(g);
          });
          if (is_cost)
            addCost(std::make_shared<CostFromErrFunc>(f, dfdx, vars, Vec{coeff}, ABS), nm + "_" + std::to_string(t), t);
          else
            addCnt(std::make_shared<ConstraintFromErrFunc>(f, dfdx, vars, Vec{coeff}, INEQ), nm + "_" + std::to_string(t), t);
        }
        break;
      }
      default:
        throw std::runtime_error("unknown term kind");
    }
  }
  tp.coll_hooks.insert(tp.coll_hooks.end(), cnt_coll_hooks.begin(), cnt_coll_hooks.end());
  for (auto& c : tp.prob->getCosts()) tp.cost_names.push_back(c->name);
  for (auto& c : tp.prob->getConstraints()) tp.cnt_names.push_back(c->name);
  return tp;
}

}  // namespace oracle
