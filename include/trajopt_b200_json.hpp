// trajopt_b200_json.hpp — the JSON front end of the problem description:
// ProblemConstructionInfo::fromJson (trajopt/src/problem_description.cpp:118-308) and the fromJson of the TermInfo
// subclasses the device path implements (:832-899 cart_pose, :989-1009 cart_vel, :1059-1076 / 1178-1195 / 1374-1391
// joint_pos / joint_vel / joint_acc, :1617-1712 collision), key for key (SURVEY.md Appendix A), including
// ensure_only_members (:32-51: an unknown key inside "params" throws) and the registry names of :53-66.
// The reference parses with jsoncpp (absent here): json::Value below is a minimal stand-in with the same accessors.
// One JSON document describes ONE problem; a batch repeats it for pci.batch problems, whose per-problem start states
// (and, if wanted, endpoints / targets / obstacles) the caller fills in afterwards.
// Not on the device path (std::runtime_error, as an unregistered type is in the reference): joint_jerk, total_time,
// dynamic_cart_pose, use_time terms and collision "pairs" overrides.
#pragma once
#include <cctype>
#include <cstdlib>
#include <initializer_list>
#include <utility>

#include "trajopt_b200.hpp"

namespace trajopt_b200 {
namespace json {

class Value {
public:
  enum Type { Null, Bool, Number, String, Array, Object };
  Type type = Null;
  bool b = false;
  double num = 0;
  std::string str;
  std::vector<Value> arr;
  std::vector<std::pair<std::string, Value>> obj;

  bool isMember(const std::string& k) const {
    for (const auto& kv : obj)
      if (kv.first == k) return true;
    return false;
  }
  const Value& operator[](const std::string& k) const {
    for (const auto& kv : obj)
      if (kv.first == k) return kv.second;
    throw std::runtime_error("missing field: " + k);  // json_marshal::childFromJson without a default
  }
  const Value& operator[](size_t i) const { return arr.at(i); }
  size_t size() const { return type == Array ? arr.size() : obj.size(); }
  bool isArray() const { return type == Array; }
  double asDouble() const {
    if (type != Number) throw std::runtime_error("expected a number");
    return num;
  }
  int asInt() const { return static_cast<int>(asDouble()); }
  bool asBool() const {
    if (type != Bool) throw std::runtime_error("expected a boolean");
    return b;
  }
  const std::string& asString() const {
    if (type != String) throw std::runtime_error("expected a string");
    return str;
  }
};

namespace detail {
struct Parser {
  const std::string& s;
  size_t i = 0;
  explicit Parser(const std::string& text) : s(text) {}
  [[noreturn]] void fail(const std::string& what) const { throw std::runtime_error("JSON: " + what + " at offset " + std::to_string(i)); }
  void ws() {
    while (i < s.size() && std::isspace(static_cast<unsigned char>(s[i]))) ++i;
  }
  char peek() {
    ws();
    if (i >= s.size()) fail("unexpected end");
    return s[i];
  }
  void expect(char c) {
    if (peek() != c) fail(std::string("expected '") + c + "'");
    ++i;
  }
  std::string string() {
    expect('"');
    std::string out;
    while (i < s.size() && s[i] != '"') {
      if (s[i] == '\\' && i + 1 < s.size()) {
        const char e = s[++i];
        out += (e == 'n') ? '\n' : (e == 't') ? '\t' : e;
      } else {
        out += s[i];
      }
      ++i;
    }
    if (i >= s.size()) fail("unterminated string");
    ++i;
    return out;
  }
  Value value() {
    Value v;
    const char c = peek();
    if (c == '{') {
      v.type = Value::Object;
      ++i;
      if (peek() == '}') { ++i; return v; }
      for (;;) {
        std::string k = string();
        expect(':');
        v.obj.emplace_back(std::move(k), value());
        if (peek() == ',') { ++i; continue; }
        expect('}');
        return v;
      }
    }
    if (c == '[') {
      v.type = Value::Array;
      ++i;
      if (peek() == ']') { ++i; return v; }
      for (;;) {
        v.arr.push_back(value());
        if (peek() == ',') { ++i; continue; }
        expect(']');
        return v;
      }
    }
    if (c == '"') {
      v.type = Value::String;
      v.str = string();
      return v;
    }
    if (s.compare(i, 4, "true") == 0) { v.type = Value::Bool; v.b = true; i += 4; return v; }
    if (s.compare(i, 5, "false") == 0) { v.type = Value::Bool; v.b = false; i += 5; return v; }
    if (s.compare(i, 4, "null") == 0) { i += 4; return v; }
    char* end = nullptr;
    v.num = std::strtod(s.c_str() + i, &end);
    if (end == s.c_str() + i) fail("unexpected character");
    v.type = Value::Number;
    i = static_cast<size_t>(end - s.c_str());
    return v;
  }
};
}  // namespace detail

inline Value parse(const std::string& text) {
  detail::Parser p(text);
  Value v = p.value();
  p.ws();
  if (p.i != text.size()) p.fail("trailing characters");
  return v;
}

}  // namespace json

namespace trajopt {
namespace json_marshal {  // trajopt_common/include/trajopt_common/json_marshal.hpp
inline void fromJson(const json::Value& v, double& out) { out = v.asDouble(); }
inline void fromJson(const json::Value& v, int& out) { out = v.asInt(); }
inline void fromJson(const json::Value& v, bool& out) { out = v.asBool(); }
inline void fromJson(const json::Value& v, std::string& out) { out = v.asString(); }
template <class T>
void fromJson(const json::Value& v, std::vector<T>& out) {
  if (!v.isArray()) throw std::runtime_error("expected an array");
  out.resize(v.size());
  for (size_t i = 0; i < v.size(); ++i) fromJson(v[i], out[i]);
}
template <class T>
void childFromJson(const json::Value& parent, T& out, const char* name) {  // required
  if (!parent.isMember(name)) throw std::runtime_error(std::string("missing field: ") + name);
  fromJson(parent[name], out);
}
template <class T>
void childFromJson(const json::Value& parent, T& out, const char* name, const T& def) {
  if (parent.isMember(name)) fromJson(parent[name], out);
  else out = def;
}
}  // namespace json_marshal

namespace detail {
// ensure_only_members, problem_description.cpp:32-51
inline void ensureOnlyMembers(const json::Value& v, std::initializer_list<const char*> fields) {
  for (const auto& kv : v.obj) {
    bool ok = false;
    for (const char* f : fields) ok = ok || kv.first == f;
    if (!ok) throw std::runtime_error("illegal field \"" + kv.first + "\"");
  }
}
inline void fillVec3(const json::Value& params, const char* key, double* out, std::initializer_list<double> def) {
  DblVec v;
  json_marshal::childFromJson(params, v, key, DblVec(def));
  if (v.size() != def.size()) throw std::runtime_error(std::string(key) + " has the wrong size");
  for (size_t i = 0; i < v.size(); ++i) out[i] = v[i];
}
inline void jointFromJson(JointTermInfoBase& t, const ProblemConstructionInfo& pci, const json::Value& v) {
  if (!v.isMember("params")) throw std::runtime_error(t.name + ": missing params");
  const json::Value& params = v["params"];
  const size_t n_dof = static_cast<size_t>(pci.kin->numJoints());
  json_marshal::childFromJson(params, t.targets, "targets");
  json_marshal::childFromJson(params, t.coeffs, "coeffs", DblVec(n_dof, 1));
  json_marshal::childFromJson(params, t.upper_tols, "upper_tols", DblVec(n_dof, 0));
  json_marshal::childFromJson(params, t.lower_tols, "lower_tols", DblVec(n_dof, 0));
  json_marshal::childFromJson(params, t.first_step, "first_step", 0);
  json_marshal::childFromJson(params, t.last_step, "last_step", pci.basic_info.n_steps - 1);
  ensureOnlyMembers(params, {"coeffs", "first_step", "last_step", "targets", "lower_tols", "upper_tols", "use_time"});
  // checkParameterSize(..., apply_first = true): a single value is broadcast to every joint
  for (DblVec* p : {&t.targets, &t.coeffs, &t.upper_tols, &t.lower_tols})
    if (p->size() == 1 && n_dof > 1) p->assign(n_dof, (*p)[0]);
}
}  // namespace detail

// TermInfo::fromName + term->fromJson, problem_description.cpp:53-66, 162-220.  root_frame: the name the reference's
// JSON uses for a static target frame (its pose is the scene root here).
inline TermInfo::Ptr termFromJson(ProblemConstructionInfo& pci, const json::Value& v, int term_type,
                                  const std::string& root_frame) {
  std::string type;
  json_marshal::childFromJson(v, type, "type");
  bool use_time = false;
  json_marshal::childFromJson(v, use_time, "use_time", false);
  if (use_time) throw std::runtime_error(type + ": use_time terms are not on the device path");
  TermInfo::Ptr out;
  if (type == "joint_pos" || type == "joint_vel" || type == "joint_acc") {
    std::shared_ptr<JointTermInfoBase> t;
    if (type == "joint_pos") t = std::make_shared<JointPosTermInfo>();
    else if (type == "joint_vel") t = std::make_shared<JointVelTermInfo>();
    else t = std::make_shared<JointAccTermInfo>();
    detail::jointFromJson(*t, pci, v);
    out = t;
  } else if (type == "cart_pose") {
    auto t = std::make_shared<CartPoseTermInfo>();
    const json::Value& params = v["params"];
    json_marshal::childFromJson(params, t->timestep, "timestep", pci.basic_info.n_steps - 1);
    detail::fillVec3(params, "pos_coeffs", t->pos_coeffs, {1, 1, 1});
    detail::fillVec3(params, "rot_coeffs", t->rot_coeffs, {1, 1, 1});
    std::string target_frame;
    json_marshal::childFromJson(params, t->source_frame, "source_frame");
    json_marshal::childFromJson(params, target_frame, "target_frame");
    detail::fillVec3(params, "source_frame_offset_xyz", t->source_frame_offset.xyz, {0, 0, 0});
    detail::fillVec3(params, "source_frame_offset_wxyz", t->source_frame_offset.wxyz, {1, 0, 0, 0});
    Pose target;
    detail::fillVec3(params, "target_frame_offset_xyz", target.xyz, {0, 0, 0});
    detail::fillVec3(params, "target_frame_offset_wxyz", target.wxyz, {1, 0, 0, 0});
    detail::ensureOnlyMembers(params, {"timestep", "pos_coeffs", "rot_coeffs", "source_frame", "target_frame",
                                       "source_frame_offset_xyz", "source_frame_offset_wxyz", "target_frame_offset_xyz",
                                       "target_frame_offset_wxyz"});
    // :877-887: exactly one of the two frames is an active link; here the source, and the target is the static root
    if (target_frame != root_frame)
      throw std::runtime_error("cart_pose: target_frame must be the static frame \"" + root_frame + "\" on the device path");
    t->target.assign(static_cast<size_t>(pci.batch), target);
    out = t;
  } else if (type == "cart_vel") {
    auto t = std::make_shared<CartVelTermInfo>();
    const json::Value& params = v["params"];
    json_marshal::childFromJson(params, t->first_step, "first_step");
    json_marshal::childFromJson(params, t->last_step, "last_step");
    json_marshal::childFromJson(params, t->max_displacement, "max_displacement");
    json_marshal::childFromJson(params, t->link, "link");
    if (!(t->first_step >= 0 && t->first_step <= pci.basic_info.n_steps - 1 && t->last_step >= t->first_step &&
          t->last_step <= pci.basic_info.n_steps - 1 && t->first_step < t->last_step))
      throw std::runtime_error("cart_vel: invalid first_step / last_step");
    pci.kin->linkIndex(t->link);  // "invalid link name" otherwise
    // (hatch pairs (iStep, iStep + 1) for iStep in [first_step, last_step], :1025,1040; last_step = n_steps - 1 would
    // index past the trajectory in the reference, the host layer clamps it to the last pair)
    detail::ensureOnlyMembers(params, {"first_step", "last_step", "max_displacement", "link"});
    out = t;
  } else if (type == "collision") {
    auto t = std::make_shared<CollisionTermInfo>();
    const json::Value& params = v["params"];
    const int n_steps = pci.basic_info.n_steps;
    json_marshal::childFromJson(params, t->first_step, "first_step", 0);
    json_marshal::childFromJson(params, t->last_step, "last_step", n_steps - 1);
    json_marshal::childFromJson(params, t->fixed_steps, "fixed_steps", IntVec());
    json_marshal::childFromJson(params, t->evaluator_type, "evaluator_type", static_cast<int>(TB200_COLL_DISCRETE));
    json_marshal::childFromJson(params, t->longest_valid_segment_length, "longest_valid_segment_length", 0.5);
    json_marshal::childFromJson(params, t->collision_coeff, "coeffs");
    json_marshal::childFromJson(params, t->collision_margin, "dist_pen");
    t->collision_margin_buffer = 0.5;  // the JSON path's default; supplying "safety_margin_buffer" throws (:1625-1630, 1700-1711)
    if (t->evaluator_type > TB200_COLL_LVS_CONTINUOUS) throw std::runtime_error("collision: invalid evaluator_type");
    if (!(t->first_step >= 0 && t->first_step < n_steps && t->last_step >= t->first_step && t->last_step < n_steps))
      throw std::runtime_error("collision: invalid first_step / last_step");
    for (int f : t->fixed_steps)
      if (f < t->first_step || f > t->last_step) throw std::runtime_error("collision: fixed_steps outside [first_step, last_step]");
    if (params.isMember("pairs")) throw std::runtime_error("collision: per-pair overrides are not on the device path");
    detail::ensureOnlyMembers(params, {"evaluator_type", "first_step", "last_step", "fixed_steps", "contact_test_type",
                                       "longest_valid_segment_length", "coeffs", "dist_pen", "pairs"});
    out = t;
  } else if (type == "joint_jerk" || type == "total_time" || type == "dynamic_cart_pose") {
    throw std::runtime_error("term type \"" + type + "\" is not on the device path");
  } else {
    throw std::runtime_error("failed to construct cost named " + type);  // problem_description.cpp:205-206
  }
  json_marshal::childFromJson(v, out->name, "name", type);
  out->term_type = term_type;
  return out;
}

// ProblemConstructionInfo::fromJson, problem_description.cpp:272-308 (pci.kin and pci.batch must be set before).
inline void fromJson(ProblemConstructionInfo& pci, const json::Value& v, const std::string& root_frame = "base_footprint") {
  if (!pci.kin) throw std::runtime_error("fromJson: pci.kin must be set first");
  {  // readBasicInfo, :118-134
    const json::Value& b = v["basic_info"];
    json_marshal::childFromJson(b, pci.basic_info.n_steps, "n_steps");
    json_marshal::childFromJson(b, pci.basic_info.manip, "manip");
    json_marshal::childFromJson(b, pci.basic_info.fixed_timesteps, "fixed_timesteps", IntVec());
    json_marshal::childFromJson(b, pci.basic_info.fixed_dofs, "fixed_dofs", IntVec());
    std::string solver;
    json_marshal::childFromJson(b, solver, "convex_solver", std::string("AUTO_SOLVER"));
    pci.basic_info.convex_solver = sco::modelTypeFromName(solver);
    json_marshal::childFromJson(b, pci.basic_info.use_time, "use_time", false);
    double lo = 1.0, hi = 1.0;
    json_marshal::childFromJson(b, lo, "dt_lower_lim", 1.0);
    json_marshal::childFromJson(b, hi, "dt_upper_lim", 1.0);
    if (lo <= 0 || hi < lo)
      throw std::runtime_error("dt limits (Basic Info) invalid. The lower limit must be positive, and the minimum upper limit is equal to the lower limit.");
  }
  if (v.isMember("opt_info")) {  // readOptInfo, :136-160
    const json::Value& o = v["opt_info"];
    sco::BasicTrustRegionSQPParameters& p = pci.opt_info;
    const sco::BasicTrustRegionSQPParameters d = p;
    json_marshal::childFromJson(o, p.improve_ratio_threshold, "improve_ratio_threshold", d.improve_ratio_threshold);
    json_marshal::childFromJson(o, p.min_trust_box_size, "min_trust_box_size", d.min_trust_box_size);
    json_marshal::childFromJson(o, p.min_approx_improve, "min_approx_improve", d.min_approx_improve);
    json_marshal::childFromJson(o, p.min_approx_improve_frac, "min_approx_improve_frac", d.min_approx_improve_frac);
    json_marshal::childFromJson(o, p.max_iter, "max_iter", d.max_iter);
    json_marshal::childFromJson(o, p.trust_shrink_ratio, "trust_shrink_ratio", d.trust_shrink_ratio);
    json_marshal::childFromJson(o, p.trust_expand_ratio, "trust_expand_ratio", d.trust_expand_ratio);
    json_marshal::childFromJson(o, p.cnt_tolerance, "cnt_tolerance", d.cnt_tolerance);
    json_marshal::childFromJson(o, p.max_merit_coeff_increases, "max_merit_coeff_increases", d.max_merit_coeff_increases);
    json_marshal::childFromJson(o, p.merit_coeff_increase_ratio, "merit_coeff_increase_ratio", d.merit_coeff_increase_ratio);
    json_marshal::childFromJson(o, p.max_time, "max_time", d.max_time);
    json_marshal::childFromJson(o, p.initial_merit_error_coeff, "initial_merit_error_coeff", d.initial_merit_error_coeff);
    json_marshal::childFromJson(o, p.inflate_constraints_individually, "inflate_constraints_individually", d.inflate_constraints_individually);
    json_marshal::childFromJson(o, p.trust_box_size, "trust_box_size", d.trust_box_size);
  }
  if (v.isMember("costs"))  // readCosts, :162-190
    for (const json::Value& c : v["costs"].arr) pci.cost_infos.push_back(termFromJson(pci, c, TT_COST, root_frame));
  if (v.isMember("constraints"))  // readConstraints, :192-220
    for (const json::Value& c : v["constraints"].arr) pci.cnt_infos.push_back(termFromJson(pci, c, TT_CNT, root_frame));
  {  // readInitInfo, :222-270
    const json::Value& ii = v["init_info"];
    std::string type_str;
    json_marshal::childFromJson(ii, type_str, "type");
    for (char& c : type_str) c = static_cast<char>(std::tolower(static_cast<unsigned char>(c)));
    const int T = pci.basic_info.n_steps, D = pci.kin->numJoints(), B = pci.batch;
    if (type_str == "stationary") {
      pci.init_info.type = InitInfo::STATIONARY;
    } else if (type_str == "given_traj") {
      pci.init_info.type = InitInfo::GIVEN_TRAJ;
      const json::Value& data = ii["data"];
      if (static_cast<int>(data.size()) != T) throw std::runtime_error("given initialization traj has wrong length");
      DblVec one;
      for (int t = 0; t < T; ++t) {
        DblVec row;
        json_marshal::fromJson(data[t], row);
        if (static_cast<int>(row.size()) != D) throw std::runtime_error("given initialization traj has wrong width");
        one.insert(one.end(), row.begin(), row.end());
      }
      pci.init_info.data.clear();
      for (int b = 0; b < B; ++b) pci.init_info.data.insert(pci.init_info.data.end(), one.begin(), one.end());
    } else if (type_str == "joint_interpolated") {
      pci.init_info.type = InitInfo::JOINT_INTERPOLATED;
      DblVec endpoint;
      json_marshal::childFromJson(ii, endpoint, "endpoint");
      if (static_cast<int>(endpoint.size()) != D)
        throw std::runtime_error("wrong number of dof values in initialization. expected " + std::to_string(D) + " got " +
                                 std::to_string(endpoint.size()));
      pci.init_info.data.clear();
      for (int b = 0; b < B; ++b) pci.init_info.data.insert(pci.init_info.data.end(), endpoint.begin(), endpoint.end());
    } else {
      throw std::runtime_error("init_info did not have a valid type from Json. Valid types are stationary, joint_interpolated, or given_traj");
    }
  }
}

}  // namespace trajopt
}  // namespace trajopt_b200
