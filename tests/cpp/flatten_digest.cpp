// FNV-1a digest of everything trajopt_b200/csrc/flatten.h makes of a description (tests/test_flatten.py): the tables
// in the order the library uploads them, then the counts the kernels' layout is planned from.
#include <cstdint>
#include <cstring>

#include "../../trajopt_b200/csrc/flatten.h"

namespace {
struct Fnv {
  uint64_t h = 1469598103934665603ull;
  void bytes(const void* p, size_t n) {
    const unsigned char* c = static_cast<const unsigned char*>(p);
    for (size_t i = 0; i < n; ++i) {
      h ^= c[i];
      h *= 1099511628211ull;
    }
  }
  template <class T>
  void vec(const std::vector<T>& v) { bytes(v.data(), v.size() * sizeof(T)); }
  void i32(int v) { bytes(&v, sizeof v); }
};
}  // namespace

extern "C" int flatten_digest(const tb200_problem_desc* d, uint64_t* digest, char* msg, int msg_len) {
  tb200::FlatProblem F;
  std::string err;
  const int rc = tb200::flatten(*d, F, err);
  std::strncpy(msg, err.c_str(), msg_len - 1);
  msg[msg_len - 1] = 0;
  if (rc != TB200_OK) return rc;
  Fnv h;
  h.vec(F.segs); h.vec(F.spheres);
  h.bytes(F.sphere_jmask, sizeof F.sphere_jmask); h.bytes(F.qtype, sizeof F.qtype); h.bytes(F.joint_seg, sizeof F.joint_seg);
  h.vec(F.link_chain);
  h.vec(F.cost_objs); h.vec(F.cnt_objs); h.vec(F.cart_objs); h.vec(F.vel_objs); h.vec(F.coll_objs);
  h.vec(F.obj_src);
  h.vec(F.joint_terms); h.vec(F.cart_terms); h.vec(F.fixed_vars);
  h.vec(F.Pband); h.vec(F.qlin);
  h.i32(F.n_band); h.bytes(F.band_offs, sizeof F.band_offs);
  h.i32(F.n_cart_rows); h.i32(F.n_coll_cand); h.i32(F.max_rows); h.i32(F.has_vel); h.i32(F.has_cast); h.i32(F.cast_cap);
  h.i32(F.n_joint_objs); h.bytes(F.joint_obj_idx, sizeof F.joint_obj_idx);
  *digest = h.h;
  return TB200_OK;
}
