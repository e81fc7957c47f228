// mpl_host.hpp — host side of the planner above the libmplx C ABI, C++17, no Eigen/Boost.
//
// Mirrors the reference's C++ surface for the node-expansion path and its caller, with the
// reference's names and argument meaning (citations are path:line in the reference checkout):
//   MPL::MapUtil<Dim>          include/mpl_collision/map_util.h
//   Waypoint<Dim>, hash_value  include/mpl_basis/waypoint.h
//   MPL::env_base<Dim>         include/mpl_planner/common/env_base.h   (params, is_goal, get_heur, get_succ)
//   MPL::env_map_gpu<Dim>      replaces env_map<Dim> (include/mpl_planner/env/env_map.h): get_succ via libmplx
//   MPL::StateSpace / State    include/mpl_planner/common/state_space.h (A* part)
//   MPL::GraphSearch::Astar    include/mpl_planner/common/graph_search.h:39-182, recoverTraj :369-455
//   MPL::MapPlanner::plan      include/mpl_planner/common/planner_base.h:275-325, src/mpl_planner/map_planner.cpp:14-18
// The search bookkeeping (hash map, priority queue) stays on the host, as in the reference; only
// get_succ crosses the boundary.  The only addition is env_base::prefetch(): a hint that lets a
// batching env expand the likely-next open nodes in the same launch.  get_succ is a pure function
// of (node, env), so speculation cannot change which nodes A* expands or in which order.
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <cmath>
#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <type_traits>
#include <deque>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>

#include "iterative_rounds.hpp"
#include <vector>

#include "../../include/mplx.h"

typedef double decimal_t;

namespace Control {
enum Control { NONE = 0, VEL = 0x01, ACC = 0x03, JRK = 0x07, SNP = 0x0f, VELxYAW = 0x11, ACCxYAW = 0x13, JRKxYAW = 0x17, SNPxYAW = 0x1f };
}

template <int N>
struct Vecf {
  decimal_t d[N];
  Vecf() { for (int i = 0; i < N; i++) d[i] = 0; }
  decimal_t &operator()(int i) { return d[i]; }
  const decimal_t &operator()(int i) const { return d[i]; }
  Vecf operator-(const Vecf &o) const { Vecf r; for (int i = 0; i < N; i++) r.d[i] = d[i] - o.d[i]; return r; }
  Vecf operator+(const Vecf &o) const { Vecf r; for (int i = 0; i < N; i++) r.d[i] = d[i] + o.d[i]; return r; }
  Vecf operator*(decimal_t k) const { Vecf r; for (int i = 0; i < N; i++) r.d[i] = d[i] * k; return r; }
  Vecf operator/(decimal_t k) const { Vecf r; for (int i = 0; i < N; i++) r.d[i] = d[i] / k; return r; }
  decimal_t lpNormInf() const { decimal_t m = 0; for (int i = 0; i < N; i++) m = std::max(m, std::abs(d[i])); return m; }
  /// Eigen's unrolled fixed-size reduction: a0 + a1 for two elements, a0 + (a1 + a2) for three
  decimal_t dot(const Vecf &o) const {
    if (N == 2) return d[0] * o.d[0] + d[1] * o.d[1];
    return d[0] * o.d[0] + (d[1] * o.d[1] + d[N - 1] * o.d[N - 1]);
  }
  decimal_t norm() const { return std::sqrt(dot(*this)); }
};
template <int N>
struct Veci {
  int d[N];
  Veci() { for (int i = 0; i < N; i++) d[i] = 0; }
  int &operator()(int i) { return d[i]; }
  const int &operator()(int i) const { return d[i]; }
  bool operator!=(const Veci &o) const { for (int i = 0; i < N; i++) if (d[i] != o.d[i]) return true; return false; }
};
template <typename T>
using vec_E = std::vector<T>;
using VecDf = std::vector<decimal_t>;

/// Waypoint<Dim>: include/mpl_basis/waypoint.h:23-58
template <int Dim>
struct Waypoint {
  Vecf<Dim> pos, vel, acc, jrk;
  decimal_t yaw{0}, t{0};
  int control{Control::NONE};
  bool enable_t{false};
  Waypoint() {}
  explicit Waypoint(int c) : control(c) {}
  bool use_pos() const { return control & 1; }
  bool use_vel() const { return control & 2; }
  bool use_acc() const { return control & 4; }
  bool use_jrk() const { return control & 8; }
  bool use_yaw() const { return control & 16; }
};

/// boost::hash_combine, 64-bit, Boost 1.56-1.80 (see DESIGN.md §2 for the version caveat)
inline void hash_combine(std::size_t &h, int v) {
  std::uint64_t k = (std::uint64_t)(std::int64_t)v;
  const std::uint64_t m = 0xc6a4a7935bd1e995ULL;
  k *= m; k ^= k >> 47; k *= m; h ^= k; h *= m; h += 0xe6546b64ULL;
}
/// hash_value(Waypoint): include/mpl_basis/waypoint.h:93-125 (host copy: start/goal nodes only;
/// successor keys come back from the device)
template <int Dim>
std::size_t hash_value(const Waypoint<Dim> &key) {
  std::size_t val = 0;
  for (int i = 0; i < Dim; i++) {
    if (key.use_pos()) { int id = std::round(key.pos(i) / 0.01); hash_combine(val, id); }
    if (key.use_vel()) { int id = std::round(key.vel(i) / 0.1); hash_combine(val, id); }
    if (key.use_acc()) { int id = std::round(key.acc(i) / 0.1); hash_combine(val, id); }
    if (key.use_jrk()) { int id = std::round(key.jrk(i) / 0.1); hash_combine(val, id); }
  }
  if (key.use_yaw()) { int id = std::round(key.yaw / 0.1); hash_combine(val, id); }
  if (key.enable_t) { int id = std::round(key.t / 0.1); hash_combine(val, id); }
  return val;
}

/// power: include/mpl_basis/math.h:197-205
inline decimal_t power(decimal_t t, int n) {
  decimal_t tn = 1;
  while (n > 0) { tn *= t; n--; }
  return tn;
}
/// normalize_angle: include/mpl_basis/math.h:15-19
inline decimal_t normalize_angle(decimal_t angle) {
  while (angle > M_PI) angle -= 2.0 * M_PI;
  while (angle < -M_PI) angle += 2.0 * M_PI;
  return angle;
}

/// The closed-form real-root solvers of include/mpl_basis/math.h:21-131, operation by operation: quad for
/// b t^2 + c t + d, cubic for a t^3 + b t^2 + c t + d, quartic for a t^4 + ... + e, and solve(a, b, c, d, e),
/// which drops zero leading coefficients.  Roots come in the reference's order; repeated and NaN roots are
/// kept as it keeps them.
inline std::vector<decimal_t> quad(decimal_t b, decimal_t c, decimal_t d) {
  std::vector<decimal_t> dts;
  const decimal_t p = c * c - 4 * b * d;
  if (p < 0) return dts;
  dts.push_back((-c - std::sqrt(p)) / (2 * b));
  dts.push_back((-c + std::sqrt(p)) / (2 * b));
  return dts;
}
inline std::vector<decimal_t> cubic(decimal_t a, decimal_t b, decimal_t c, decimal_t d) {
  std::vector<decimal_t> dts;
  const decimal_t a2 = b / a, a1 = c / a, a0 = d / a;
  const decimal_t Q = (3 * a1 - a2 * a2) / 9;
  const decimal_t R = (9 * a1 * a2 - 27 * a0 - 2 * a2 * a2 * a2) / 54;
  const decimal_t D = Q * Q * Q + R * R;
  if (D > 0) {
    const decimal_t S = std::cbrt(R + std::sqrt(D));
    const decimal_t T = std::cbrt(R - std::sqrt(D));
    dts.push_back(-a2 / 3 + (S + T));
  } else if (D == 0) {
    const decimal_t S = std::cbrt(R);
    dts.push_back(-a2 / 3 + S + S);
    dts.push_back(-a2 / 3 - S);
  } else {
    const decimal_t theta = std::acos(R / std::sqrt(-Q * Q * Q));
    dts.push_back(2 * std::sqrt(-Q) * std::cos(theta / 3) - a2 / 3);
    dts.push_back(2 * std::sqrt(-Q) * std::cos((theta + 2 * M_PI) / 3) - a2 / 3);
    dts.push_back(2 * std::sqrt(-Q) * std::cos((theta + 4 * M_PI) / 3) - a2 / 3);
  }
  return dts;
}
inline std::vector<decimal_t> quartic(decimal_t a, decimal_t b, decimal_t c, decimal_t d, decimal_t e) {
  std::vector<decimal_t> dts;
  const decimal_t a3 = b / a, a2 = c / a, a1 = d / a, a0 = e / a;
  const std::vector<decimal_t> ys = cubic(1, -a2, a1 * a3 - 4 * a0, 4 * a2 * a0 - a1 * a1 - a3 * a3 * a0);
  const decimal_t y1 = ys.front();
  const decimal_t r = a3 * a3 / 4 - a2 + y1;
  if (r < 0) return dts;
  const decimal_t R = std::sqrt(r);
  decimal_t D, E;
  if (R != 0) {
    D = std::sqrt(0.75 * a3 * a3 - R * R - 2 * a2 + 0.25 * (4 * a3 * a2 - 8 * a1 - a3 * a3 * a3) / R);
    E = std::sqrt(0.75 * a3 * a3 - R * R - 2 * a2 - 0.25 * (4 * a3 * a2 - 8 * a1 - a3 * a3 * a3) / R);
  } else {
    D = std::sqrt(0.75 * a3 * a3 - 2 * a2 + 2 * std::sqrt(y1 * y1 - 4 * a0));
    E = std::sqrt(0.75 * a3 * a3 - 2 * a2 - 2 * std::sqrt(y1 * y1 - 4 * a0));
  }
  if (!std::isnan(D)) {
    dts.push_back(-a3 / 4 + R / 2 + D / 2);
    dts.push_back(-a3 / 4 + R / 2 - D / 2);
  }
  if (!std::isnan(E)) {
    dts.push_back(-a3 / 4 - R / 2 + E / 2);
    dts.push_back(-a3 / 4 - R / 2 - E / 2);
  }
  return dts;
}
inline std::vector<decimal_t> solve(decimal_t a, decimal_t b, decimal_t c, decimal_t d, decimal_t e) {
  if (a != 0) return quartic(a, b, c, d, e);
  if (b != 0) return cubic(b, c, d, e);
  if (c != 0) return quad(c, d, e);
  if (d != 0) return std::vector<decimal_t>(1, -e / d);
  return std::vector<decimal_t>();
}

/// Primitive1D: include/mpl_basis/primitive.h:25-197 — the evaluators and the effort integral of one
/// axis, with the reference's operand order (these run on the host, after planning: sampling a
/// recovered trajectory is not on the expansion path).
struct Primitive1D {
  decimal_t c[6] = {0, 0, 0, 0, 0, 0};  // highest order first (primitive.h:34-50)
  /// primitive.h:128-145
  decimal_t p(decimal_t t) const {
    return c[0] / 120 * power(t, 5) + c[1] / 24 * power(t, 4) + c[2] / 6 * power(t, 3) + c[3] / 2 * t * t + c[4] * t + c[5];
  }
  decimal_t v(decimal_t t) const { return c[0] / 24 * power(t, 4) + c[1] / 6 * power(t, 3) + c[2] / 2 * t * t + c[3] * t + c[4]; }
  decimal_t a(decimal_t t) const { return c[0] / 6 * power(t, 3) + c[1] / 2 * t * t + c[2] * t + c[3]; }
  decimal_t j(decimal_t t) const { return c[0] / 2 * t * t + c[1] * t + c[2]; }
  /// primitive.h:152-162: the roots of a(t) in (0, t), in solver order, stopping at the first root >= t
  std::vector<decimal_t> extrema_v(decimal_t t) const {
    const std::vector<decimal_t> roots = solve(0, c[0] / 6, c[1] / 2, c[2], c[3]);
    std::vector<decimal_t> ts;
    for (const decimal_t it : roots) {
      if (it > 0 && it < t) ts.push_back(it);
      else if (it >= t) break;
    }
    return ts;
  }
  /// primitive.h:169-179: the roots of j(t) in (0, t), in solver order, stopping at the first root >= t
  std::vector<decimal_t> extrema_a(decimal_t t) const {
    const std::vector<decimal_t> roots = solve(0, 0, c[0] / 2, c[1], c[2]);
    std::vector<decimal_t> ts;
    for (const decimal_t it : roots) {
      if (it > 0 && it < t) ts.push_back(it);
      else if (it >= t) break;
    }
    return ts;
  }
  /// primitive.h:186-193: the root of the snap's linear jerk derivative in (0, t)
  std::vector<decimal_t> extrema_j(decimal_t t) const {
    std::vector<decimal_t> ts;
    if (c[0] != 0) {
      const decimal_t t_sol = -c[1] * 2 / c[0];
      if (t_sol > 0 && t_sol < t) ts.push_back(t_sol);
    }
    return ts;
  }
  /// primitive.h:92-122
  decimal_t J(decimal_t t, int control) const {
    const int o = control & 15;
    if (o == Control::VEL)
      return c[0] * c[0] / 5184 * power(t, 9) + c[0] * c[1] / 576 * power(t, 8) +
             (c[1] * c[1] / 252 + c[0] * c[2] / 168) * power(t, 7) + (c[0] * c[3] / 72 + c[1] * c[2] / 36) * power(t, 6) +
             (c[2] * c[2] / 20 + c[0] * c[4] / 60 + c[1] * c[3] / 15) * power(t, 5) +
             (c[2] * c[3] / 4 + c[1] * c[4] / 12) * power(t, 4) + (c[3] * c[3] / 3 + c[2] * c[4] / 3) * power(t, 3) +
             c[3] * c[4] * t * t + c[4] * c[4] * t;
    else if (o == Control::ACC)
      return c[0] * c[0] / 252 * power(t, 7) + c[0] * c[1] / 36 * power(t, 6) +
             (c[1] * c[1] / 20 + c[0] * c[2] / 15) * power(t, 5) + (c[0] * c[3] / 12 + c[1] * c[2] / 4) * power(t, 4) +
             (c[2] * c[2] / 3 + c[1] * c[3] / 3) * power(t, 3) + c[2] * c[3] * t * t + c[3] * c[3] * t;
    else if (o == Control::JRK)
      return c[0] * c[0] / 20 * power(t, 5) + c[0] * c[1] / 4 * power(t, 4) + (c[1] * c[1] + c[0] * c[2]) / 3 * power(t, 3) +
             c[1] * c[2] * t * t + c[2] * c[2] * t;
    else if (o == Control::SNP)
      return c[0] * c[0] / 3 * power(t, 3) + c[0] * c[1] * t * t + c[1] * c[1] * t;
    return 0;
  }
};

/// Primitive<Dim> built from a state and a control input: include/mpl_basis/primitive.h:220-256
template <int Dim>
class Primitive {
 public:
  Primitive() {}
  Primitive(const Waypoint<Dim> &p, const VecDf &u, decimal_t t) : t_(t), control_(p.control) {
    const int o = control_ & 15;
    for (int i = 0; i < Dim; i++) {
      decimal_t *c = prs_[i].c;
      if (o == Control::SNP) { c[1] = u[i]; c[2] = p.jrk(i); c[3] = p.acc(i); c[4] = p.vel(i); c[5] = p.pos(i); }
      else if (o == Control::JRK) { c[2] = u[i]; c[3] = p.acc(i); c[4] = p.vel(i); c[5] = p.pos(i); }
      else if (o == Control::ACC) { c[3] = u[i]; c[4] = p.vel(i); c[5] = p.pos(i); }
      else if (o == Control::VEL) { c[4] = u[i]; c[5] = p.pos(i); }
    }
    if (control_ & 16) { pr_yaw_.c[4] = u[Dim]; pr_yaw_.c[5] = p.yaw; }
  }
  /// From coefficients (each highest order first) and a duration: primitive.h:309-313.  cs holds Dim
  /// axes, then optionally the yaw axis.
  Primitive(const vec_E<Vecf<6>> &cs, decimal_t t, int control) : t_(t), control_(control) {
    for (int i = 0; i < Dim; i++)
      for (int k = 0; k < 6; k++) prs_[i].c[k] = cs[i](k);
    if ((int)cs.size() == Dim + 1)
      for (int k = 0; k < 6; k++) pr_yaw_.c[k] = cs[Dim](k);
  }
  /// primitive.h:321-331
  Waypoint<Dim> evaluate(decimal_t t) const {
    Waypoint<Dim> p(control_);
    for (int k = 0; k < Dim; k++) {
      p.pos(k) = prs_[k].p(t);
      p.vel(k) = prs_[k].v(t);
      p.acc(k) = prs_[k].a(t);
      p.jrk(k) = prs_[k].j(t);
      if (p.use_yaw()) p.yaw = normalize_angle(pr_yaw_.p(t));
    }
    return p;
  }
  decimal_t t() const { return t_; }
  int control() const { return control_; }
  const Primitive1D &pr(int k) const { return prs_[k]; }
  const Primitive1D &pr_yaw() const { return pr_yaw_; }
  /// primitive.h:403-410
  decimal_t J(int control) const {
    decimal_t j = 0;
    for (int k = 0; k < Dim; k++) j += prs_[k].J(t_, control);
    return j;
  }
  decimal_t Jyaw() const { return pr_yaw_.J(t_, Control::VEL); }
  /// primitive.h:353-363: max |v| along axis k over [0, t] from the ends and extrema_v
  decimal_t max_vel(int k) const {
    const std::vector<decimal_t> ts = prs_[k].extrema_v(t_);
    decimal_t max_v = std::max(std::abs(prs_[k].v(0)), std::abs(prs_[k].v(t_)));
    for (const decimal_t it : ts) {
      if (it > 0 && it < t_) {
        const decimal_t v = std::abs(prs_[k].v(it));
        max_v = v > max_v ? v : max_v;
      }
    }
    return max_v;
  }
  /// primitive.h:369-379: max |a| along axis k over [0, t] from the ends and extrema_a
  decimal_t max_acc(int k) const {
    const std::vector<decimal_t> ts = prs_[k].extrema_a(t_);
    decimal_t max_a = std::max(std::abs(prs_[k].a(0)), std::abs(prs_[k].a(t_)));
    for (const decimal_t it : ts) {
      if (it > 0 && it < t_) {
        const decimal_t a = std::abs(prs_[k].a(it));
        max_a = a > max_a ? a : max_a;
      }
    }
    return max_a;
  }
  /// primitive.h:384-394: max |j| along axis k over [0, t] from the ends and extrema_j
  decimal_t max_jrk(int k) const {
    const std::vector<decimal_t> ts = prs_[k].extrema_j(t_);
    decimal_t max_j = std::max(std::abs(prs_[k].j(0)), std::abs(prs_[k].j(t_)));
    for (const decimal_t it : ts) {
      if (it > 0 && it < t_) {
        const decimal_t j = std::abs(prs_[k].j(it));
        max_j = j > max_j ? j : max_j;
      }
    }
    return max_j;
  }

 private:
  decimal_t t_{0};
  int control_{Control::NONE};
  Primitive1D prs_[Dim];
  Primitive1D pr_yaw_;
};

/// validate_xxx: primitive.h:476-493 — every axis's max_vel (xxx VEL), max_acc (ACC) or max_jrk (JRK) within
/// max; a max <= 0 passes
template <int Dim>
bool validate_xxx(const Primitive<Dim> &pr, decimal_t max, int xxx) {
  if (max <= 0) return true;
  for (int i = 0; i < Dim; i++) {
    if (xxx == Control::VEL && pr.max_vel(i) > max) return false;
    else if (xxx == Control::ACC && pr.max_acc(i) > max) return false;
    else if (xxx == Control::JRK && pr.max_jrk(i) > max) return false;
  }
  return true;
}

/// validate_yaw: primitive.h:503-525 — at both ends, a nonzero planar velocity's direction against the yaw:
/// v.normalized().dot((cos yaw, sin yaw)) >= cos(my); a my <= 0 passes
template <int Dim>
bool validate_yaw(const Primitive<Dim> &pr, decimal_t my) {
  if (my <= 0) return true;
  const Waypoint<Dim> ws[2] = {pr.evaluate(0), pr.evaluate(pr.t())};
  for (const auto &w : ws) {
    decimal_t v0 = w.vel(0), v1 = w.vel(1);
    if (v0 != 0 || v1 != 0) {
      const decimal_t z = v0 * v0 + v1 * v1;  // Eigen's normalized(): divide by sqrt(squaredNorm) when > 0
      if (z > 0) {
        const decimal_t n = std::sqrt(z);
        v0 = v0 / n;
        v1 = v1 / n;
      }
      const decimal_t d = v0 * std::cos(w.yaw) + v1 * std::sin(w.yaw);
      if (d < std::cos(my)) return false;
    }
  }
  return true;
}

/// validate_primitive: primitive.h:449-470 — the checks the primitive's control names
template <int Dim>
bool validate_primitive(const Primitive<Dim> &pr, decimal_t mv = 0, decimal_t ma = 0, decimal_t mj = 0,
                        decimal_t myaw = 0) {
  switch (pr.control()) {
    case Control::ACC: return validate_xxx(pr, mv, Control::VEL);
    case Control::JRK: return validate_xxx(pr, mv, Control::VEL) && validate_xxx(pr, ma, Control::ACC);
    case Control::SNP:
      return validate_xxx(pr, mv, Control::VEL) && validate_xxx(pr, ma, Control::ACC) && validate_xxx(pr, mj, Control::JRK);
    case Control::VELxYAW: return validate_yaw(pr, myaw);
    case Control::ACCxYAW: return validate_yaw(pr, myaw) && validate_xxx(pr, mv, Control::VEL);
    case Control::JRKxYAW:
      return validate_yaw(pr, myaw) && validate_xxx(pr, mv, Control::VEL) && validate_xxx(pr, ma, Control::ACC);
    case Control::SNPxYAW:
      return validate_yaw(pr, myaw) && validate_xxx(pr, mv, Control::VEL) && validate_xxx(pr, ma, Control::ACC) &&
             validate_xxx(pr, mj, Control::JRK);
    default: return true;
  }
}

/// Command<Dim>: include/mpl_basis/trajectory.h:19-28
template <int Dim>
struct Command {
  Vecf<Dim> pos, vel, acc, jrk;
  decimal_t yaw{0}, yaw_dot{0}, t{0};
};

/// VirtualPoint: include/mpl_basis/lambda.h:15-19 — a knot of the time-scaling factor lambda(tau)
struct VirtualPoint {
  decimal_t p{0}, v{0}, t{0};
};

/// LambdaSeg: lambda.h:24-71 — the cubic lambda(tau) = a3 tau^3 + a2 tau^2 + a1 tau + a0 between two knots
/// (value and slope at each end), fitted by inverting the 4 x 4 Hermite matrix.  The inverse is Gauss-Jordan
/// with partial pivoting (the pivot of a column is the first row of largest |value|), the same operations as
/// the Eigen stand-in the reference is compiled against in the tests; a = inv * b sums each element in
/// increasing k from 0.  Coefficients with |a| < 1e-5 become 0, as in the reference.
struct LambdaSeg {
  decimal_t a[4] = {0, 0, 0, 0};  // a3, a2, a1, a0
  decimal_t ti{0}, tf{0}, dT{0};
  LambdaSeg() {}
  LambdaSeg(const VirtualPoint &v1, const VirtualPoint &v2) {
    decimal_t A[4][4] = {{power(v1.t, 3), v1.t * v1.t, v1.t, 1},
                         {3 * v1.t * v1.t, 2 * v1.t, 1, 0},
                         {power(v2.t, 3), v2.t * v2.t, v2.t, 1},
                         {3 * v2.t * v2.t, 2 * v2.t, 1, 0}};
    decimal_t inv[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
    for (int col = 0; col < 4; col++) {
      int piv = col;
      for (int r = col + 1; r < 4; r++)
        if (std::abs(A[r][col]) > std::abs(A[piv][col])) piv = r;
      for (int k = 0; k < 4; k++) {
        std::swap(A[col][k], A[piv][k]);
        std::swap(inv[col][k], inv[piv][k]);
      }
      const decimal_t d = A[col][col];
      for (int k = 0; k < 4; k++) {
        A[col][k] /= d;
        inv[col][k] /= d;
      }
      for (int r = 0; r < 4; r++) {
        if (r == col) continue;
        const decimal_t f = A[r][col];
        for (int k = 0; k < 4; k++) {
          A[r][k] -= f * A[col][k];
          inv[r][k] -= f * inv[col][k];
        }
      }
    }
    const decimal_t b[4] = {v1.p, v1.v, v2.p, v2.v};
    for (int i = 0; i < 4; i++) {
      decimal_t acc = 0;
      for (int k = 0; k < 4; k++) acc += inv[i][k] * b[k];
      a[i] = acc;
    }
    for (int i = 0; i < 4; i++)
      if (std::abs(a[i]) < 1e-5) a[i] = 0;
    ti = v1.t;
    tf = v2.t;
    dT = getT(tf) - getT(ti);
  }
  VirtualPoint evaluate(decimal_t tau) const {
    VirtualPoint vt;
    vt.t = tau;
    vt.p = a[0] * power(tau, 3) + a[1] * tau * tau + a[2] * tau + a[3];
    vt.v = 3 * a[0] * tau * tau + 2 * a[1] * tau + a[2];
    return vt;
  }
  /// the integral of lambda from 0 to t
  decimal_t getT(decimal_t t) const { return a[0] / 4 * power(t, 4) + a[1] / 3 * power(t, 3) + a[2] / 2 * t * t + a[3] * t; }
};

/// Lambda: lambda.h:76-184 (without sample / sampleT) — the piecewise-cubic time-scaling factor: real time
/// t = integral of lambda over the polynomial's time tau.
///  * evaluate(tau) takes the first segment with ti <= tau < tf.  At tau equal to the last tf the reference
///    finds none and returns an uninitialised point; here the last segment is evaluated instead.
///  * getTau(t) scans the segments with a running T += dT (left to right) and returns the first root of the
///    quartic T + integral = t that lies in [ti, tf] of the first segment whose [T, T + dT] holds t, going on
///    to the next segment when none fits, and -1 when no segment gives one.  t = N * (total / N) can land an
///    ulp past the last segment; the caller then clamps -1 to 0 and evaluates the trajectory's start, as the
///    reference does.
class Lambda {
 public:
  Lambda() {}
  explicit Lambda(const std::vector<VirtualPoint> &vs) {
    for (int i = 0; i < (int)vs.size() - 1; i++) segs.push_back(LambdaSeg(vs[i], vs[i + 1]));
  }
  bool exist() const { return !segs.empty(); }
  VirtualPoint evaluate(decimal_t tau) const {
    for (const auto &seg : segs)
      if (tau >= seg.ti && tau < seg.tf) return seg.evaluate(tau);
    return segs.empty() ? VirtualPoint() : segs.back().evaluate(tau);
  }
  decimal_t getT(decimal_t tau) const {
    if (segs.empty()) return tau;
    decimal_t T = 0;
    for (const auto &seg : segs) {
      if (tau >= seg.ti && tau <= seg.tf) {
        T += seg.getT(tau) - seg.getT(seg.ti);
        return T;
      }
      T += seg.dT;
    }
    return T;
  }
  decimal_t getTau(decimal_t t) const {
    if (!exist()) return t;
    decimal_t T = 0;
    for (const auto &seg : segs) {
      if (t >= T && t <= T + seg.dT) {
        const decimal_t a = seg.a[0] / 4, b = seg.a[1] / 3, c = seg.a[2] / 2, d = seg.a[3];
        const decimal_t e = T - t - seg.getT(seg.ti);
        for (const decimal_t it : solve(a, b, c, d, e))
          if (it >= seg.ti && it <= seg.tf) return it;
      }
      T += seg.dT;
    }
    return -1;
  }
  decimal_t getTotalTime() const {
    decimal_t t = 0;
    for (const auto &seg : segs) t += seg.dT;
    return t;
  }
  std::vector<LambdaSeg> segs;
};

/// Trajectory<Dim>: include/mpl_basis/trajectory.h:42-318 with the Lambda time scaling.  Without a lambda
/// (no scale, or a scale_down that found nothing to slow), getTau(t) = t, lambda = 1 and lambda_dot = 0.
template <int Dim>
class Trajectory {
 public:
  Trajectory() {}
  explicit Trajectory(const vec_E<Primitive<Dim>> &prs) : segs(prs) {
    taus.push_back(0);
    for (const auto &pr : prs) taus.push_back(pr.t() + taus.back());
    Ts = taus;
    total_t_ = taus.back();
  }
  /// trajectory.h:67-91
  Waypoint<Dim> evaluate(decimal_t time) const {
    decimal_t tau = lambda_.getTau(time);
    if (tau < 0) tau = 0;
    if (tau > total_t_) tau = total_t_;
    for (std::size_t id = 0; id < segs.size(); id++) {
      if ((tau >= taus[id] && tau < taus[id + 1]) || id == segs.size() - 1) {
        tau -= taus[id];
        Waypoint<Dim> p(segs[id].control());
        for (int j = 0; j < Dim; j++) {
          const Primitive1D &pr = segs[id].pr(j);
          p.pos(j) = pr.p(tau);
          p.vel(j) = pr.v(tau);
          p.acc(j) = pr.a(tau);
          p.jrk(j) = pr.j(tau);
          p.yaw = normalize_angle(segs[id].pr_yaw().p(tau));
        }
        return p;
      }
    }
    return Waypoint<Dim>();
  }
  /// trajectory.h:100-137
  bool evaluate(decimal_t time, Command<Dim> &p) const {
    decimal_t tau = lambda_.getTau(time);
    if (tau < 0) tau = 0;
    if (tau > total_t_) tau = total_t_;
    decimal_t lambda = 1, lambda_dot = 0;
    if (lambda_.exist()) {
      const VirtualPoint vt = lambda_.evaluate(tau);
      lambda = vt.p;
      lambda_dot = vt.v;
    }
    for (std::size_t id = 0; id < segs.size(); id++) {
      if (tau >= taus[id] && tau <= taus[id + 1]) {
        tau -= taus[id];
        for (int j = 0; j < Dim; j++) {
          const Primitive1D &pr = segs[id].pr(j);
          p.pos(j) = pr.p(tau);
          p.vel(j) = pr.v(tau) / lambda;
          p.acc(j) = pr.a(tau) / lambda / lambda - p.vel(j) * lambda_dot / lambda / lambda / lambda;
          p.jrk(j) = pr.j(tau) / lambda / lambda - 3 / power(lambda, 3) * p.acc(j) * p.acc(j) * lambda_dot +
                     3 / power(lambda, 4) * p.vel(j) * lambda_dot * lambda_dot;
          p.yaw = normalize_angle(segs[id].pr_yaw().p(tau));
          p.yaw_dot = normalize_angle(segs[id].pr_yaw().v(tau));
          p.t = time;
        }
        return true;
      }
    }
    return false;
  }
  /// trajectory.h:142-168: lambda from (0, 1/ri, slope 0) to (taus.back(), 1/rf, slope 0); Ts and the total
  /// time become the scaled ones
  bool scale(decimal_t ri, decimal_t rf) {
    VirtualPoint vi, vf;
    vi.p = 1.0 / ri;
    vi.v = 0;
    vi.t = 0;
    vf.p = 1.0 / rf;
    vf.v = 0;
    vf.t = taus.back();
    lambda_ = Lambda(std::vector<VirtualPoint>{vi, vf});
    set_scaled_times();
    return true;
  }
  /// trajectory.h:173-228, which does not compile in the reference (nothing instantiates it): it is defined
  /// here as that text with extrema_v for extrema_vel, v(t) for evaluate(t)(1), and the axes i < Dim for
  /// i < 3.  Every segment and axis whose max_vel exceeds mv adds a knot at each of its extrema_v roots, at
  /// its start (except segment 0) and at its end where |v| / mv > 1; the knots, between (0, ri) and
  /// (taus.back(), rf), are sorted by time, every interior one takes the largest ratio max_l, and equal
  /// times keep their first knot.  false (and no lambda) when max_l <= 1.  Note p = ri, rf here where
  /// scale uses 1/ri, 1/rf, as in the reference.
  bool scale_down(decimal_t mv, decimal_t ri, decimal_t rf) {
    std::vector<VirtualPoint> vs;
    VirtualPoint vi, vf;
    vi.p = ri;
    vi.v = 0;
    vi.t = 0;
    vf.p = rf;
    vf.v = 0;
    vf.t = taus.back();
    vs.push_back(vi);
    for (int id = 0; id < (int)segs.size(); id++) {
      for (int i = 0; i < Dim; i++) {
        if (segs[id].max_vel(i) > mv) {
          std::vector<decimal_t> ts = segs[id].pr(i).extrema_v(segs[id].t());
          if (id != 0) ts.push_back(0);
          ts.push_back(segs[id].t());
          for (const decimal_t tv : ts) {
            const decimal_t v = segs[id].pr(i).v(tv);
            const decimal_t lambda_v = std::abs(v) / mv;
            if (lambda_v <= 1) continue;
            VirtualPoint vt;
            vt.p = lambda_v;
            vt.v = 0;
            vt.t = tv + taus[id];
            vs.push_back(vt);
          }
        }
      }
    }
    vs.push_back(vf);
    std::sort(vs.begin(), vs.end(), [](const VirtualPoint &a, const VirtualPoint &b) { return a.t < b.t; });
    decimal_t max_l = 1;
    for (const auto &v : vs)
      if (v.p > max_l) max_l = v.p;
    if (max_l <= 1) return false;
    for (int i = 1; i < (int)vs.size() - 1; i++) vs[i].p = max_l;
    std::vector<VirtualPoint> vs_s;
    vs_s.push_back(vs.front());
    for (const auto &v : vs)
      if (v.t > vs_s.back().t) vs_s.push_back(v);
    lambda_ = Lambda(vs_s);
    set_scaled_times();
    return true;
  }
  const Lambda &lambda() const { return lambda_; }
  /// A lambda fitted elsewhere (mplx_traj_scale's segments) and the total time it gives, in place of
  /// scale / scale_down
  void set_lambda(const Lambda &lambda, decimal_t total_t) {
    lambda_ = lambda;
    set_scaled_times();
    total_t_ = total_t;
  }
  /// trajectory.h:230-237
  vec_E<Command<Dim>> sample(int N) const {
    vec_E<Command<Dim>> ps(N + 1);
    decimal_t dt = total_t_ / N;
    for (int i = 0; i <= N; i++) evaluate(i * dt, ps[i]);
    return ps;
  }
  /// trajectory.h:251-266
  decimal_t J(int control) const {
    decimal_t j = 0;
    for (const auto &seg : segs) j += seg.J(control);
    return j;
  }
  decimal_t Jyaw() const {
    decimal_t j = 0;
    for (const auto &seg : segs) j += seg.Jyaw();
    return j;
  }
  /// trajectory.h:269-289
  std::vector<decimal_t> getSegmentTimes() const {
    std::vector<decimal_t> dts;
    for (int i = 0; i < (int)Ts.size() - 1; i++) dts.push_back(Ts[i + 1] - Ts[i]);
    return dts;
  }
  vec_E<Waypoint<Dim>> getWaypoints() const {
    vec_E<Waypoint<Dim>> ws;
    if (segs.empty()) return ws;
    decimal_t t = 0;
    for (const auto &seg : segs) {
      ws.push_back(seg.evaluate(0));
      ws.back().t = t;
      t += seg.t();
    }
    ws.push_back(segs.back().evaluate(segs.back().t()));
    ws.back().t = t;
    return ws;
  }
  vec_E<Primitive<Dim>> getPrimitives() const { return segs; }
  decimal_t getTotalTime() const { return total_t_; }

  vec_E<Primitive<Dim>> segs;
  std::vector<decimal_t> taus, Ts;
  decimal_t total_t_{0};

 private:
  void set_scaled_times() {
    std::vector<decimal_t> ts;
    for (const auto &tau : taus) ts.push_back(lambda_.getT(tau));
    Ts = ts;
    total_t_ = Ts.back();
  }
  Lambda lambda_;
};

/// factorial: include/mpl_basis/math.h:187-194
inline int factorial(int n) {
  int nf = 1;
  while (n > 0) { nf *= n; n--; }
  return nf;
}

namespace MPL {
/// The dense linear algebra of PolySolver: a column-major matrix, products that sum each element in
/// increasing k from 0, and LU with row partial pivoting.  The reference calls Eigen here; the Eigen
/// stand-in the tests compile the reference against implements the same operations in the same order,
/// so the restatement is pinned to the reference bit for bit under that stand-in.
namespace dense {
struct Mat {
  int r = 0, c = 0;
  std::vector<decimal_t> d;
  Mat() {}
  Mat(int rows, int cols) : r(rows), c(cols), d((size_t)rows * cols, 0.0) {}
  decimal_t &operator()(int i, int j) { return d[i + (size_t)j * r]; }
  const decimal_t &operator()(int i, int j) const { return d[i + (size_t)j * r]; }
  Mat block(int i0, int j0, int rows, int cols) const {
    Mat b(rows, cols);
    for (int j = 0; j < cols; j++)
      for (int i = 0; i < rows; i++) b(i, j) = (*this)(i0 + i, j0 + j);
    return b;
  }
  Mat transpose() const {
    Mat t(c, r);
    for (int j = 0; j < c; j++)
      for (int i = 0; i < r; i++) t(j, i) = (*this)(i, j);
    return t;
  }
};
/// a * b, element (i, j) = ((0 + a(i,0) b(0,j)) + a(i,1) b(1,j)) + ...
inline Mat mul(const Mat &a, const Mat &b) {
  Mat p(a.r, b.c);
  for (int j = 0; j < b.c; j++)
    for (int k = 0; k < a.c; k++) {
      const decimal_t bkj = b(k, j);
      for (int i = 0; i < a.r; i++) p(i, j) += a(i, k) * bkj;
    }
  return p;
}
/// Doolittle LU with row partial pivoting: the pivot of column k is the first row >= k of largest |value|.
/// A zero pivot is divided by, so a singular matrix gives non-finite solutions.
struct LU {
  Mat lu;
  std::vector<int> swap;  // row k was exchanged with row swap[k]
  explicit LU(Mat a) : lu(std::move(a)), swap(lu.r) {
    const int n = lu.r;
    for (int k = 0; k < n; k++) {
      int p = k;
      decimal_t amax = std::abs(lu(k, k));
      for (int i = k + 1; i < n; i++)
        if (std::abs(lu(i, k)) > amax) { amax = std::abs(lu(i, k)); p = i; }
      swap[k] = p;
      if (p != k)
        for (int j = 0; j < n; j++) std::swap(lu(k, j), lu(p, j));
      for (int i = k + 1; i < n; i++) lu(i, k) = lu(i, k) / lu(k, k);
      for (int j = k + 1; j < n; j++)
        for (int i = k + 1; i < n; i++) lu(i, j) = lu(i, j) - lu(i, k) * lu(k, j);
    }
  }
  /// lu^-1 b: the row exchanges, then forward (unit lower) and back substitution, each sum in increasing index
  Mat solve(const Mat &b) const {
    Mat x(b);
    const int n = lu.r;
    for (int k = 0; k < n; k++)
      if (swap[k] != k)
        for (int j = 0; j < x.c; j++) std::swap(x(k, j), x(swap[k], j));
    for (int j = 0; j < x.c; j++) {
      for (int i = 0; i < n; i++)
        for (int k = 0; k < i; k++) x(i, j) = x(i, j) - lu(i, k) * x(k, j);
      for (int i = n - 1; i >= 0; i--) {
        for (int k = i + 1; k < n; k++) x(i, j) = x(i, j) - lu(i, k) * x(k, j);
        x(i, j) = x(i, j) / lu(i, i);
      }
    }
    return x;
  }
};
}  // namespace dense

/// PolySolver<Dim>: src/mpl_traj_solver/poly_solver.cpp:4-219 and PolyTraj::toPrimitives
/// (poly_traj.cpp:72-88).  Fits N = 2 (smooth_derivative_order + 1) coefficients per segment through the
/// waypoints, minimising the integral of the squared minimize_derivative-th derivative, by the reference's
/// dense formulation, operation by operation: the A, Q and M assembly, A^-1 M by LU, R = ((A^-1 M)^T Q) A^-1 M,
/// Dp = -Rpp^-1 (Rpf Df), d = M D and one N x N LU solve per segment.  The cost is cubic in the number of
/// segments; libmplx's mplx_traj_solve solves the same problem in linear time on the device.
///
/// Where the reference is undefined:
///  * two waypoints with free derivatives (the reference skips the free solve, poly_solver.cpp:205, and leaves
///    those rows of D uninitialised): they are 0;
///  * a zero-length or non-finite segment time makes A singular: the coefficients are not all finite.
template <int Dim>
class PolySolver {
 public:
  PolySolver(unsigned smooth_derivative_order, unsigned minimize_derivative)
      : N_(2 * (smooth_derivative_order + 1)), R_(minimize_derivative) {}

  /// false (and no coefficients) for fewer than two waypoints; dts[i] is segment i's duration
  bool solve(const vec_E<Waypoint<Dim>> &waypoints, const std::vector<decimal_t> &dts) {
    coeffs_.clear();
    waypoints_ = waypoints;
    dts_ = dts;
    const int W = (int)waypoints.size(), S = W - 1, N = (int)N_, h = N / 2, R = (int)R_;
    if (W < 2) return false;
    dense::Mat A(S * N, S * N), Q(S * N, S * N);
    for (int i = 0; i < S; i++) {
      const decimal_t seg_time = dts[i];
      for (int n = 0; n < N; n++) {
        if (n < h) {
          int val = 1;
          for (int m = 0; m < n; m++) val *= (n - m);
          A(i * N + n, i * N + n) = val;
        }
        for (int r = 0; r < h; r++)
          if (r <= n) {
            int val = 1;
            for (int m = 0; m < r; m++) val *= (n - m);
            A(i * N + h + r, i * N + n) = val * power(seg_time, n - r);
          }
        for (int r = 0; r < N; r++)
          if (r >= R && n >= R) {
            int val = 1;
            for (int m = 0; m < R; m++) val *= (r - m) * (n - m);
            Q(i * N + r, i * N + n) = val * power(seg_time, r + n - 2 * R + 1) / (unsigned)(r + n - 2 * R + 1);
          }
      }
    }
    // derivative k < h of a waypoint is fixed when its control flag says so (use_pos, use_vel, use_acc)
    auto fixed = [&](const Waypoint<Dim> &w, int k) { return ((w.control >> k) & 1) != 0; };
    int nfix = 0;
    for (const auto &w : waypoints)
      for (int k = 0; k < h; k++) nfix += fixed(w, k) ? 1 : 0;
    const int nfree = W * h - nfix;
    // (row of the raw per-segment derivative vector, column of D): fixed derivatives first, then the free
    // ones, each in waypoint order; an interior waypoint ends one segment and starts the next
    std::vector<std::pair<int, int>> perm;
    int raw = 0, fix_cnt = 0, free_cnt = 0;
    for (int id = 0; id < W; id++) {
      const bool interior = id > 0 && id < W - 1;
      for (int k = 0; k < h; k++) {
        const int col = fixed(waypoints[id], k) ? fix_cnt++ : nfix + free_cnt++;
        perm.push_back({raw, col});
        if (interior) perm.push_back({raw + h, col});
        raw++;
      }
      if (interior) raw += h;
    }
    dense::Mat M(S * N, W * h);
    for (const auto &pc : perm) M(pc.first, pc.second) = 1;
    const dense::Mat AinvM = dense::LU(A).solve(M);
    const dense::Mat Rm = dense::mul(dense::mul(AinvM.transpose(), Q), AinvM);
    const dense::Mat Rpp = Rm.block(nfix, nfix, nfree, nfree), Rpf = Rm.block(nfix, 0, nfree, nfix);
    dense::Mat Df(nfix, Dim);
    for (const auto &pc : perm)
      if (pc.second < nfix) {
        const Waypoint<Dim> &w = waypoints[(pc.first + h) / N];
        const int k = pc.first % h;
        for (int a = 0; a < Dim; a++) Df(pc.second, a) = k == 0 ? w.pos(a) : k == 1 ? w.vel(a) : k == 2 ? w.acc(a) : w.jrk(a);
      }
    dense::Mat D(W * h, Dim);
    for (int a = 0; a < Dim; a++)
      for (int i = 0; i < nfix; i++) D(i, a) = Df(i, a);
    if (W > 2 && nfree > 0) {
      const dense::Mat Dp = dense::LU(Rpp).solve(dense::mul(Rpf, Df));
      for (int a = 0; a < Dim; a++)
        for (int i = 0; i < nfree; i++) D(nfix + i, a) = -Dp(i, a);
    }
    const dense::Mat d = dense::mul(M, D);
    for (int i = 0; i < S; i++) coeffs_.push_back(dense::LU(A.block(i * N, i * N, N, N)).solve(d.block(i * N, 0, N, Dim)));
    return true;
  }

  /// PolyTraj::toPrimitives: Primitive1D coefficient k! p_k at index 5 - k, control = the first waypoint's
  vec_E<Primitive<Dim>> toPrimitives() const {
    vec_E<Primitive<Dim>> prs;
    for (std::size_t i = 0; i < coeffs_.size(); i++) {
      const dense::Mat &p = coeffs_[i];
      vec_E<Vecf<6>> cs;
      for (int j = 0; j < p.c; j++) {
        Vecf<6> c;
        for (int k = 0; k < p.r; k++) c(5 - k) = p(k, j) * factorial(k);
        cs.push_back(c);
      }
      prs.push_back(Primitive<Dim>(cs, dts_[i], waypoints_.front().control));
    }
    return prs;
  }

 private:
  unsigned N_, R_;
  vec_E<Waypoint<Dim>> waypoints_;
  std::vector<decimal_t> dts_;
  std::vector<dense::Mat> coeffs_;  // per segment: N x Dim, p(k, axis) multiplies t^k
};

/// TrajSolver<Dim>: include/mpl_traj_solver/traj_solver.h.  control VEL / ACC / JRK (with or without YAW)
/// minimises velocity / acceleration / jerk; SNP, or a yaw_control other than VEL / ACC / JRK, leaves the
/// solver unset and solve() returns an empty Trajectory, as in the reference.  The yaw axis comes from a
/// PolySolver<1> pass over the waypoints' yaw (endpoints yaw_control, interior VEL).
/// Where the reference is undefined (see also PolySolver): solve() without usable segment times (no
/// setDts of n - 1 entries and v <= 0, for two or more waypoints) throws std::invalid_argument.
template <int Dim>
class TrajSolver {
 public:
  explicit TrajSolver(int control, int yaw_control = Control::VEL) : control_(control), yaw_control_(yaw_control) {
    if (control == Control::VEL || control == Control::VELxYAW) poly_solver_.reset(new PolySolver<Dim>(0, 1));
    else if (control == Control::ACC || control == Control::ACCxYAW) poly_solver_.reset(new PolySolver<Dim>(1, 2));
    else if (control == Control::JRK || control == Control::JRKxYAW) poly_solver_.reset(new PolySolver<Dim>(2, 3));
    if (yaw_control == Control::VEL) yaw_solver_.reset(new PolySolver<1>(0, 1));
    else if (yaw_control == Control::ACC) yaw_solver_.reset(new PolySolver<1>(1, 2));
    else if (yaw_control == Control::JRK) yaw_solver_.reset(new PolySolver<1>(2, 3));
  }
  /// waypoints with their own control flags (which derivatives are fixed) and yaw
  void setWaypoints(const vec_E<Waypoint<Dim>> &ws) {
    path_.resize(ws.size());
    for (std::size_t i = 0; i < ws.size(); i++) path_[i] = ws[i].pos;
    waypoints_ = ws;
  }
  /// velocity of the L-inf time allocation used when no segment times are set
  void setV(decimal_t v) { v_ = v; }
  void setDts(const std::vector<decimal_t> &dts) { dts_ = dts; }
  /// positions only: the endpoints take the solver's control, the interior waypoints VEL (position fixed)
  void setPath(const vec_E<Vecf<Dim>> &path) {
    path_ = path;
    waypoints_.assign(path.size(), Waypoint<Dim>(Control::VEL));
    for (std::size_t i = 0; i < path.size(); i++) waypoints_[i].pos = path[i];
    if (!waypoints_.empty()) waypoints_.front().control = waypoints_.back().control = control_;
  }
  Trajectory<Dim> solve() {
    if (waypoints_.size() != dts_.size() + 1) dts_ = allocate_time(path_, v_);
    if (!poly_solver_ || !yaw_solver_) return Trajectory<Dim>();
    if (waypoints_.size() >= 2 && dts_.size() + 1 != waypoints_.size())
      throw std::invalid_argument("TrajSolver: no segment times (setDts with n - 1 entries, or setV with v > 0)");
    poly_solver_->solve(waypoints_, dts_);
    vec_E<Waypoint<1>> yaws(waypoints_.size(), Waypoint<1>(Control::VEL));
    for (std::size_t i = 0; i < waypoints_.size(); i++) yaws[i].pos(0) = waypoints_[i].yaw;
    if (!yaws.empty()) yaws.front().control = yaws.back().control = yaw_control_;
    yaw_solver_->solve(yaws, dts_);
    vec_E<Primitive<Dim>> prs = poly_solver_->toPrimitives();
    const vec_E<Primitive<1>> yaw_prs = yaw_solver_->toPrimitives();
    for (std::size_t i = 0; i < prs.size(); i++) {
      vec_E<Vecf<6>> cs(Dim + 1);
      for (int a = 0; a < Dim; a++)
        for (int k = 0; k < 6; k++) cs[a](k) = prs[i].pr(a).c[k];
      for (int k = 0; k < 6; k++) cs[Dim](k) = yaw_prs[i].pr(0).c[k];
      prs[i] = Primitive<Dim>(cs, prs[i].t(), prs[i].control());
    }
    return Trajectory<Dim>(prs);
  }
  vec_E<Vecf<Dim>> getPath() const { return path_; }
  vec_E<Waypoint<Dim>> getWaypoints() const { return waypoints_; }
  std::vector<decimal_t> getDts() const { return dts_; }

 private:
  /// traj_solver.h allocate_time: |p_i - p_{i-1}|_inf / v; empty for fewer than two points or v <= 0
  static std::vector<decimal_t> allocate_time(const vec_E<Vecf<Dim>> &pts, decimal_t v) {
    if (pts.size() < 2 || v <= 0) return std::vector<decimal_t>();
    std::vector<decimal_t> dts(pts.size() - 1);
    for (std::size_t i = 1; i < pts.size(); i++) {
      decimal_t d = 0;
      for (int a = 0; a < Dim; a++) {
        const decimal_t x = std::abs(pts[i](a) - pts[i - 1](a));
        if (x > d) d = x;
      }
      dts[i - 1] = d / v;
    }
    return dts;
  }
  vec_E<Vecf<Dim>> path_;
  vec_E<Waypoint<Dim>> waypoints_;
  std::vector<decimal_t> dts_;
  decimal_t v_{1};
  int control_, yaw_control_;
  std::unique_ptr<PolySolver<Dim>> poly_solver_;
  std::unique_ptr<PolySolver<1>> yaw_solver_;
};
}  // namespace MPL

namespace MPL {
using Tmap = std::vector<signed char>;

/// MapUtil<Dim>: include/mpl_collision/map_util.h (storage + the lookups the planner's host side uses)
template <int Dim>
class MapUtil {
 public:
  Tmap getMap() { return map_; }
  const Tmap &map() const { return map_; }
  decimal_t getRes() { return res_; }
  Veci<Dim> getDim() { return dim_; }
  Vecf<Dim> getOrigin() { return origin_d_; }
  int getIndex(const Veci<Dim> &pn) {
    return Dim == 2 ? pn(0) + dim_(0) * pn(1) : pn(0) + dim_(0) * pn(1) + dim_(0) * dim_(1) * pn(Dim - 1);
  }
  bool isFree(int idx) { return map_[idx] < val_occ && map_[idx] >= val_free; }
  bool isOccupied(int idx) { return map_[idx] == val_occ; }
  bool isOutside(const Veci<Dim> &pn) {
    for (int i = 0; i < Dim; i++) if (pn(i) < 0 || pn(i) >= dim_(i)) return true;
    return false;
  }
  bool isFree(const Veci<Dim> &pn) { return isOutside(pn) ? false : isFree(getIndex(pn)); }
  bool isOccupied(const Veci<Dim> &pn) { return isOutside(pn) ? false : isOccupied(getIndex(pn)); }
  void setMap(const Vecf<Dim> &ori, const Veci<Dim> &dim, const Tmap &map, decimal_t res) {
    map_ = map; dim_ = dim; origin_d_ = ori; res_ = res; version_++;
    resetJournal();
  }
  /// Set voxel cells[k] to values[k], in order (a later entry for the same voxel wins): one version
  /// bump per call.  Every (index, value) entry is journalled with the new version, so an env holding
  /// the grid of an older version can apply just the change (changesSince) instead of copying the whole
  /// grid.  Throws, with nothing changed, when a cell lies outside the map.  The reference's MapUtil
  /// has no per-cell setter; its users copy the map, edit it and call setMap.
  void setCells(const vec_E<Veci<Dim>> &cells, const std::vector<int8_t> &values) {
    if (values.size() != cells.size()) throw std::invalid_argument("MapUtil::setCells: one value per cell");
    for (const auto &c : cells)
      if (isOutside(c)) throw std::out_of_range("MapUtil::setCells: cell outside the map");
    version_++;
    for (std::size_t k = 0; k < cells.size(); k++) {
      const int idx = getIndex(cells[k]);
      map_[idx] = values[k];
      journal_idx_.push_back(idx);
      journal_val_.push_back(values[k]);
      journal_ver_.push_back(version_);
    }
    if (journal_idx_.size() > journalLimit()) resetJournal();  // an edit this large is sent as a whole grid
  }
  /// Journal entries [first, end) turn the grid of version `since` into the current one.  False when the
  /// journal does not reach back to `since` (setMap, freeUnknown or a truncation came after it): the
  /// consumer must copy the whole grid.  At most journalLimit() entries follow any covered version.
  bool changesSince(unsigned long since, std::size_t &first) const {
    if (since < journal_base_ || since > version_) return false;
    first = std::upper_bound(journal_ver_.begin(), journal_ver_.end(), since) - journal_ver_.begin();
    return true;
  }
  const std::vector<int32_t> &journalIndex() const { return journal_idx_; }
  const std::vector<int8_t> &journalValue() const { return journal_val_; }
  /// Journal entries kept before it is truncated: 1/kJournalFraction of the voxels; a consumer behind a
  /// larger edit copies the whole grid.  map_update_bench.py, on one H100 80GB HBM3 at a
  /// 700 W power limit, medians of three runs: mplx_set_map takes 14.6-23.7 ms (512^3) and 1.12-1.52 ms
  /// (256^3); mplx_update_cells of 1/64 of the voxels takes 3.2-4.7 ms and 0.42-0.54 ms (random voxels
  /// or one box), and of 1/16 of them 12.1-20.5 ms and 1.5-2.3 ms, at or past the full upload on the
  /// 256^3 map.  1/64 is the largest measured fraction at which the sparse update wins on both maps and
  /// patterns.
  static constexpr std::size_t kJournalFraction = 64;
  std::size_t journalLimit() const { return map_.size() / kJournalFraction; }
  Veci<Dim> floatToInt(const Vecf<Dim> &pt) {
    Veci<Dim> pn;
    for (int i = 0; i < Dim; i++) pn(i) = std::round((pt(i) - origin_d_(i)) / res_ - 0.5);
    return pn;
  }
  /// Cells crossed by the segment pt1 -> pt2, the way MapUtil::rayTrace samples it (map_util.h:120-137):
  /// the segment is cut into floor(Linf(diff/res)/0.8) equal steps and the interior points
  /// pt1 + (diff/steps)*i, i = 1..steps-1, are converted with floatToInt; the walk ends at the first
  /// point outside the map, and a cell is reported once per run of consecutive equal cells.  `visit`
  /// returns false to stop early (is_goal stops at the first occupied cell).  The sample points must
  /// be these exact doubles for the goal test / tunnel to agree with the reference, hence the same
  /// three operations per point (scale, multiply by i, add).
  template <typename Visit>
  void walkRay(const Vecf<Dim> &pt1, const Vecf<Dim> &pt2, Visit visit) {
    const Vecf<Dim> span = pt2 - pt1;
    const int steps = (span / res_).lpNormInf() / 0.8;
    const Vecf<Dim> inc = span * (1.0 / steps);
    bool have_last = false;
    Veci<Dim> last;
    for (int i = 1; i < steps; i++) {
      const Veci<Dim> cell = floatToInt(pt1 + inc * i);
      if (isOutside(cell)) return;
      if (!have_last || cell != last) {
        if (!visit(cell)) return;
      }
      last = cell;
      have_last = true;
    }
  }
  vec_E<Veci<Dim>> rayTrace(const Vecf<Dim> &pt1, const Vecf<Dim> &pt2) {
    vec_E<Veci<Dim>> cells;
    walkRay(pt1, pt2, [&](const Veci<Dim> &c) { cells.push_back(c); return true; });
    return cells;
  }
  void freeUnknown() { for (auto &v : map_) if (v == val_unknown) v = val_free; version_++; resetJournal(); }
  unsigned long version() const { return version_; }

 protected:
  void resetJournal() {
    journal_idx_.clear(); journal_val_.clear(); journal_ver_.clear();
    journal_base_ = version_;
  }
  // (index, value, version) of every setCells entry since version journal_base_
  std::vector<int32_t> journal_idx_;
  std::vector<int8_t> journal_val_;
  std::vector<unsigned long> journal_ver_;
  unsigned long journal_base_{0};
  decimal_t res_{1};
  Vecf<Dim> origin_d_;
  Veci<Dim> dim_;
  Tmap map_;
  unsigned long version_{0};
  int8_t val_occ = 100, val_free = 0, val_unknown = -1;
};
typedef MapUtil<2> OccMapUtil;
typedef MapUtil<3> VoxelMapUtil;

/// env_base<Dim>: include/mpl_planner/common/env_base.h (the members the A* path touches)
template <int Dim>
class env_base {
 public:
  virtual ~env_base() {}
  /// env_base.h:23-41
  virtual bool is_goal(const Waypoint<Dim> &state) const {
    if (state.t >= t_max_) return true;
    bool goaled = (state.pos - goal_node_.pos).lpNormInf() <= tol_pos_;
    if (goaled && tol_vel_ >= 0) goaled = (state.vel - goal_node_.vel).lpNormInf() <= tol_vel_;
    if (goaled && tol_acc_ >= 0) goaled = (state.acc - goal_node_.acc).lpNormInf() <= tol_acc_;
    if (goaled && tol_yaw_ >= 0) goaled = std::abs(state.yaw - goal_node_.yaw) <= tol_yaw_;
    return goaled;
  }
  /// env_base.h:48-64 (heur_ignore_dynamics_ == true, the default: :368)
  virtual decimal_t get_heur(const Waypoint<Dim> &state) const { return get_heur(state, hash_value(state)); }
  /// the same with the state's lattice key already known (the device returns it with the successor);
  /// `goal_node_ == state` is hash equality (waypoint.h:133-135), the goal's hash is cached by set_goal
  virtual decimal_t get_heur(const Waypoint<Dim> &state, std::size_t state_key) const {
    if (goal_key_ == state_key) return 0;
    return cal_heur(state, goal_node_);
  }
  /// cal_heur: env_base.h:55-64, the heur_ignore_dynamics_ branch (the reference's default, :368): the Linf
  /// distance over v_max.  The minimum-time heuristics with dynamics (env_base.h:66-211: closed-form
  /// quartic for ACC states, Eigen's PolynomialSolver for JRK) are outside the expansion path this
  /// library rebuilds (SURVEY.md §2) and are not provided: set_heur_ignore_dynamics(false) is ignored.
  virtual decimal_t cal_heur(const Waypoint<Dim> &state, const Waypoint<Dim> &goal) const {
    if (v_max_ > 0) return w_ * (state.pos - goal.pos).lpNormInf() / v_max_;
    return w_ * (state.pos - goal.pos).lpNormInf();
  }
  /// env_base.h:305-306
  /// Only the default (true) is supported; false is reported and ignored (the reference's style: a
  /// message and no exception, planner_base.h:283-287), the search keeps the admissible Linf heuristic.
  bool set_heur_ignore_dynamics(bool ignore) {
    if (!ignore) {
      std::fprintf(stderr, "[mpl_host] setHeurIgnoreDynamics(false): the minimum-time heuristic with dynamics "
                           "(env_base.h:66-211) is not provided; keeping the default Linf heuristic\n");
      return false;
    }
    heur_ignore_dynamics_ = true;
    return true;
  }
  /// env_base.h:228-231
  void forward_action(const Waypoint<Dim> &curr, int action_id, Primitive<Dim> &pr) const {
    pr = Primitive<Dim>(curr, U_[action_id], dt_);
  }
  void set_u(const vec_E<VecDf> &U) { U_ = U; touch(); }
  void set_v_max(decimal_t v) { v_max_ = v; touch(); }
  void set_a_max(decimal_t a) { a_max_ = a; touch(); }
  void set_j_max(decimal_t j) { j_max_ = j; touch(); }
  void set_yaw_max(decimal_t yaw) { yaw_max_ = yaw; touch(); }
  void set_dt(decimal_t dt) { dt_ = dt; touch(); }
  void set_tol_pos(decimal_t pos) { tol_pos_ = pos; }
  void set_tol_vel(decimal_t vel) { tol_vel_ = vel; }
  void set_tol_acc(decimal_t acc) { tol_acc_ = acc; }
  void set_tol_yaw(decimal_t yaw) { tol_yaw_ = yaw; }
  void set_w(decimal_t w) { w_ = w; touch(); }
  void set_wyaw(decimal_t wyaw) { wyaw_ = wyaw; touch(); }
  void set_t_max(int t) { t_max_ = t; }
  bool set_goal(const Waypoint<Dim> &state) { goal_node_ = state; goal_key_ = hash_value(state); return true; }
  virtual void set_potential_weight(decimal_t) {}
  virtual void set_gradient_weight(decimal_t) {}
  virtual void set_potential_map(const std::vector<int8_t> &) {}
  virtual void set_search_region(const std::vector<bool> &r) { search_region_ = r; touch(); }
  decimal_t get_dt() const { return dt_; }
  virtual bool is_free(const Vecf<Dim> &) const { return true; }
  /// env_base.h:358-362
  virtual void get_succ(const Waypoint<Dim> &curr, vec_E<Waypoint<Dim>> &succ, std::vector<decimal_t> &succ_cost,
                        std::vector<int> &action_idx) const = 0;
  /// Extensions for batching envs (results of get_succ are pure, so none of this can change what
  /// the search expands):
  ///  - wants_candidates(key): true when the env would have to launch for this node and could take
  ///    more nodes in the same launch;
  ///  - prefetch(cands, keys): the open nodes the search is likely to pop next;
  ///  - last_succ_keys(): lattice keys of the successors returned by the last get_succ call, if the
  ///    env already has them (the device computes them); nullptr = hash on the host.
  /// Stored-edge queries of the incremental planner, batched.  Edge k is the primitive
  /// forward_action(parents[k], actions[k]) (env_base.h:228-231):
  ///  - is_free_edges: is_free(pr) (env_base.h:338-341, env_map.h:60-76) and
  ///    calculate_intrinsic_cost(pr) (env_base.h:343-345) per edge;
  ///  - edge_cells: the cells getLinkedNodes visits along each edge (map_planner.cpp:135-151),
  ///    edge k owning cells[offset[k]*Dim .. offset[k+1]*Dim); an env that can also returns the
  ///    inverted table (table_voxel sorted, table_edge the edge of each entry, edges of one voxel in
  ///    emission order), else leaves both empty and the planner sorts on the host.
  virtual void is_free_edges(const vec_E<Waypoint<Dim>> &, const std::vector<int> &, std::vector<uint8_t> &,
                             std::vector<decimal_t> &) const {
    throw std::runtime_error("this env does not serve edge re-validation");
  }
  virtual void edge_cells(const vec_E<Waypoint<Dim>> &, const std::vector<int> &, std::vector<long long> &,
                          std::vector<int> &, std::vector<int> &, std::vector<int> &) const {
    throw std::runtime_error("this env does not serve edge re-validation");
  }
  /// MapPlanner::setSearchRegion(path, dense) (src/mpl_planner/map_planner.cpp:46-95) served by the
  /// env that owns the grids: build the tunnel of half-width ceil(radius/res) cells around the path
  /// and install it as the search region.
  virtual void search_region_from_path(const vec_E<Vecf<Dim>> &, const Vecf<Dim> &, bool) {
    throw std::runtime_error("this env does not build search regions");
  }
  virtual bool wants_candidates(std::size_t) const { return false; }
  virtual void prefetch(const vec_E<Waypoint<Dim>> &, const std::vector<std::size_t> &) const {}
  virtual const std::size_t *last_succ_keys() const { return nullptr; }
  virtual void begin_plan() const {}

  bool heur_ignore_dynamics_{true};
  decimal_t w_{10.0}, wyaw_{1.0};
  decimal_t tol_pos_{0.5}, tol_vel_{-1.0}, tol_acc_{-1.0}, tol_yaw_{-1.0};
  decimal_t v_max_{-1.0}, a_max_{-1.0}, j_max_{-1.0}, yaw_max_{-1.0};
  decimal_t t_max_{std::numeric_limits<decimal_t>::infinity()};
  decimal_t dt_{1.0};
  vec_E<VecDf> U_;
  Waypoint<Dim> goal_node_;
  std::size_t goal_key_{hash_value(Waypoint<Dim>())};
  std::vector<bool> search_region_;
  mutable vec_E<Vecf<Dim>> expanded_nodes_;

 protected:
  void touch() { params_version_++; }
  unsigned long params_version_{1};
};

/// The host-only members of env_map<Dim> (include/mpl_planner/env/env_map.h:25-51): goal test with
/// ray-trace and the start-point free test.  They run on the host against the MapUtil copy.
template <int Dim>
class env_map_host : public env_base<Dim> {
 public:
  explicit env_map_host(std::shared_ptr<MapUtil<Dim>> map_util) : map_util_(map_util) {}
  /// env_map.h:25-45
  bool is_goal(const Waypoint<Dim> &state) const override {
    bool goaled = (state.pos - this->goal_node_.pos).lpNormInf() <= this->tol_pos_;
    if (goaled && this->tol_vel_ >= 0) goaled = (state.vel - this->goal_node_.vel).lpNormInf() <= this->tol_vel_;
    if (goaled && this->tol_acc_ >= 0) goaled = (state.acc - this->goal_node_.acc).lpNormInf() <= this->tol_acc_;
    if (goaled && this->tol_yaw_ >= 0) goaled = std::abs(state.yaw - this->goal_node_.yaw) <= this->tol_yaw_;
    if (goaled) {
      // env_map.h:31-35: the straight line to the goal must not cross an occupied cell
      map_util_->walkRay(state.pos, this->goal_node_.pos, [&](const Veci<Dim> &c) {
        if (map_util_->isOccupied(c)) goaled = false;
        return goaled;
      });
    }
    return goaled;
  }
  /// env_map.h:48-51
  bool is_free(const Vecf<Dim> &pt) const override { return map_util_->isFree(map_util_->floatToInt(pt)); }
  void set_potential_map(const std::vector<int8_t> &map) override { potential_map_ = map; this->touch(); }
  void set_potential_weight(decimal_t w) override { potential_weight_ = w; this->touch(); }
  void set_gradient_weight(decimal_t w) override { gradient_weight_ = w; this->touch(); }

  /// env_map.h:60-76: the n + 1 samples of pr.sample(n), n = ceil(max_v * t / res), each one in a free cell of
  /// the map and, with a search region, inside it.  A stationary primitive (n = 0) samples at t = 0 * inf = NaN,
  /// which floatToInt makes INT_MIN (x86-64): outside, not free.  n above MPLX_SAMPLE_N_MAX, where the reference
  /// would allocate the samples: not free.
  bool is_free(const Primitive<Dim> &pr) const {
    decimal_t max_v = 0;
    for (int i = 0; i < Dim; i++)
      if (pr.max_vel(i) > max_v) max_v = pr.max_vel(i);
    const decimal_t nd = std::ceil(max_v * pr.t() / map_util_->getRes());
    if (!(nd <= MPLX_SAMPLE_N_MAX)) return false;
    const int n = (int)nd;
    const decimal_t dt = pr.t() / n;
    for (int i = 0; i <= n; i++) {
      const Veci<Dim> pn = map_util_->floatToInt(pr.evaluate(i * dt).pos);
      if (map_util_->isOccupied(pn) || map_util_->isOutside(pn)) return false;
      if (!this->search_region_.empty() && !this->search_region_[map_util_->getIndex(pn)]) return false;
    }
    return true;
  }

  /// traverse_trajectory's sample count N = ceil(v_max * total / res) (env_map.h:230-231), or 0 where it is not
  /// in [1, MPLX_SAMPLE_N_MAX]: with the default v_max < 0 the reference asks for a vector of negative size, at
  /// N = 0 it samples t = 0 * inf = NaN, and above the bound it would allocate the samples.
  int traverse_samples(const Trajectory<Dim> &traj) const {
    const decimal_t nd = std::ceil(this->v_max_ * traj.getTotalTime() / map_util_->getRes());
    return nd >= 1 && nd <= MPLX_SAMPLE_N_MAX ? (int)nd : 0;
  }

  /// env_map.h:228-255: the cost of traj.sample(N).  A sample counts when its cell index differs from the
  /// previous sample's (-1 before the first; getIndex before any bounds test, in 32-bit arithmetic that wraps
  /// as on the reference's targets).  A counted sample outside the map, or with a potential map at a potential
  /// >= 100, or without one in an occupied cell, returns +inf; with a potential map a counted sample with
  /// 0 < potential < 100 adds potential_weight * potential + gradient_weight * |vel|, in sample order.  Throws
  /// std::domain_error where traverse_samples is 0.
  decimal_t traverse_trajectory(const Trajectory<Dim> &traj) const {
    const int n = traverse_samples(traj);
    if (n < 1) throw std::domain_error("traverse_trajectory: N = ceil(v_max * total / res) outside [1, MPLX_SAMPLE_N_MAX]");
    const Veci<Dim> dim = map_util_->getDim();
    decimal_t c = 0;
    const auto pts = traj.sample(n);
    uint32_t prev_idx = ~0u;
    for (const auto &pt : pts) {
      const Veci<Dim> pn = map_util_->floatToInt(pt.pos);
      uint32_t idx = (uint32_t)pn(0) + (uint32_t)dim(0) * (uint32_t)pn(1);
      if (Dim == 3) idx += (uint32_t)dim(0) * (uint32_t)dim(1) * (uint32_t)pn(Dim - 1);
      if (prev_idx == idx) continue;
      prev_idx = idx;
      if (map_util_->isOutside(pn)) return std::numeric_limits<decimal_t>::infinity();
      if (!potential_map_.empty()) {
        if (potential_map_[idx] < 100 && potential_map_[idx] > 0)
          c += potential_weight_ * potential_map_[idx] + gradient_weight_ * pt.vel.norm();
        else if (potential_map_[idx] >= 100)
          return std::numeric_limits<decimal_t>::infinity();
      } else if (map_util_->isOccupied(pn)) {
        return std::numeric_limits<decimal_t>::infinity();
      }
    }
    return c;
  }

 protected:
  std::shared_ptr<MapUtil<Dim>> map_util_;
  std::vector<int8_t> potential_map_;
  decimal_t potential_weight_{0.1}, gradient_weight_{0.0};
};

/// env_map_gpu<Dim>: env_map<Dim> (include/mpl_planner/env/env_map.h) with get_succ served by
/// libmplx (CUDA).  Throws std::runtime_error when the engine cannot be created: no CPU fallback.
template <int Dim>
class env_map_gpu : public env_map_host<Dim> {
  using env_map_host<Dim>::map_util_;
  using env_map_host<Dim>::potential_map_;
  using env_map_host<Dim>::potential_weight_;
  using env_map_host<Dim>::gradient_weight_;

 public:
  explicit env_map_gpu(std::shared_ptr<MapUtil<Dim>> map_util, int device = 0) : env_map_host<Dim>(map_util) {
    if (mplx_create(Dim, device, &ctx_) != MPLX_OK) throw std::runtime_error(mplx_last_error());
  }
  ~env_map_gpu() override { mplx_destroy(ctx_); }
  env_map_gpu(const env_map_gpu &) = delete;

  void set_potential_map(const std::vector<int8_t> &map) override { potential_map_ = map; potential_on_device_ = false; this->touch(); }
  void set_search_region(const std::vector<bool> &r) override { region_on_device_ = false; env_base<Dim>::set_search_region(r); }
  void set_potential_weight(decimal_t w) override { potential_weight_ = w; this->touch(); }
  void set_gradient_weight(decimal_t w) override { gradient_weight_ = w; this->touch(); }
  void set_control(int control) { control_ = control; this->touch(); }
  /// nodes speculatively expanded per launch (1 = plain one-node get_succ)
  void set_speculation(int k) { speculate_ = std::max(1, k); }
  /// record the node of every get_succ call, in call order = the A* pop order (graph_search.h:66-75);
  /// the replay frontier of the benchmark (SURVEY.md §8d i)
  void set_trace(std::vector<mplx_waypoint> *trace) { trace_ = trace; }

  void begin_plan() const override { cache_.clear(); stats_nodes_ = stats_calls_ = stats_hits_ = 0; }

  /// env_map.h:147-172.  Served from the speculation cache when possible.
  void get_succ(const Waypoint<Dim> &curr, vec_E<Waypoint<Dim>> &succ, std::vector<decimal_t> &succ_cost,
                std::vector<int> &action_idx) const override {
    succ.clear(); succ_cost.clear(); action_idx.clear();
    this->expanded_nodes_.push_back(curr.pos);  // env_map.h:154, at real pop time
    if (trace_) trace_->push_back(to_pod(curr));
    const std::size_t key = hash_value(curr);
    auto it = cache_.find(key);
    if (it == cache_.end()) {
      batch_.clear(); batch_keys_.clear();
      batch_.push_back(curr); batch_keys_.push_back(key);
      for (std::size_t c = 0; c < pending_.size() && (int)batch_.size() < speculate_; c++) {
        const std::size_t k = pending_keys_[c];
        if (k != key && !cache_.count(k)) { batch_.push_back(pending_[c]); batch_keys_.push_back(k); }
      }
      pending_.clear(); pending_keys_.clear();
      expand_batch();
      it = cache_.find(key);
    } else {
      stats_hits_++;
    }
    Entry &e = it->second;
    for (std::size_t j = 0; j < e.cost.size(); j++) succ.push_back(from_pod(e.succ[j], curr.control));
    succ_cost.assign(e.cost.begin(), e.cost.end());
    action_idx.assign(e.action.begin(), e.action.end());
    last_keys_.swap(e.key);
    cache_.erase(it);  // A* expands a node once
  }
  bool wants_candidates(std::size_t key) const override { return speculate_ > 1 && !cache_.count(key); }
  void prefetch(const vec_E<Waypoint<Dim>> &cands, const std::vector<std::size_t> &keys) const override {
    pending_ = cands;
    pending_keys_ = keys;
  }
  const std::size_t *last_succ_keys() const override { return last_keys_.data(); }

  /// MapPlanner::updatePotentialMap on the device (mplx_update_potential_map): the MapUtil grid is
  /// replaced by the potential field, which also becomes the potential map (map_planner.cpp:387-388).
  void update_potential_map(const Vecf<Dim> &radius, decimal_t pow_, const Vecf<Dim> &range, const Vecf<Dim> &pos) {
    sync();
    Tmap out(map_util_->map().size());
    check(mplx_update_potential_map(ctx_, radius.d, pow_, range.d, pos.d, potential_weight_, gradient_weight_,
                                    (int8_t *)out.data()));
    map_util_->setMap(map_util_->getOrigin(), map_util_->getDim(), out, map_util_->getRes());
    map_version_ = map_util_->version();  // the device already holds this grid
    potential_map_.assign(out.begin(), out.end());
    potential_on_device_ = true;
  }
  /// The points setSearchRegion traces for `path`: the path itself, or for an empty path (the waypoints of a plan
  /// whose start is already a goal) one point two cells below the map's origin, whose region is empty as the
  /// reference's is for an empty path (map_planner.cpp:49-58 traces nothing).
  vec_E<Vecf<Dim>> region_points(const vec_E<Vecf<Dim>> &path) const {
    if (!path.empty()) return path;
    Vecf<Dim> p = map_util_->getOrigin();
    for (int k = 0; k < Dim; k++) p(k) -= 2 * map_util_->getRes();
    return vec_E<Vecf<Dim>>{p};
  }
  /// MapPlanner::setSearchRegion on the device (mplx_set_search_region_path)
  void search_region_from_path(const vec_E<Vecf<Dim>> &path, const Vecf<Dim> &radius, bool dense) override {
    set_search_region_path(path, radius, dense);
  }
  void set_search_region_path(const vec_E<Vecf<Dim>> &path, const Vecf<Dim> &radius, bool dense) {
    sync();
    std::vector<double> flat;
    for (const auto &p : region_points(path)) for (int k = 0; k < Dim; k++) flat.push_back(p(k));
    std::vector<uint8_t> out(map_util_->map().size());
    check(mplx_set_search_region_path(ctx_, flat.data(), (int)(flat.size() / Dim), radius.d, dense ? 1 : 0,
                                      out.data()));
    this->search_region_.assign(out.begin(), out.end());
    region_on_device_ = true;
  }

  /// env_map::is_free(pr) for stored edges on the device (mplx_edges_is_free)
  void is_free_edges(const vec_E<Waypoint<Dim>> &parents, const std::vector<int> &actions, std::vector<uint8_t> &free,
                     std::vector<decimal_t> &cost) const override {
    sync();
    std::vector<mplx_waypoint> in(parents.size());
    for (std::size_t i = 0; i < parents.size(); i++) in[i] = to_pod(parents[i]);
    free.assign(parents.size(), 0);
    cost.assign(parents.size(), 0);
    check(mplx_edges_is_free(ctx_, in.data(), actions.data(), (int)parents.size(), free.data(), cost.data()));
  }
  /// the getLinkedNodes voxel walk for stored edges on the device (mplx_edges_cells)
  void edge_cells(const vec_E<Waypoint<Dim>> &parents, const std::vector<int> &actions, std::vector<long long> &offset,
                  std::vector<int> &cells, std::vector<int> &table_voxel, std::vector<int> &table_edge) const override {
    sync();
    std::vector<mplx_waypoint> in(parents.size());
    for (std::size_t i = 0; i < parents.size(); i++) in[i] = to_pod(parents[i]);
    offset.assign(parents.size() + 1, 0);
    int64_t total = 0;
    std::size_t cap = std::max<std::size_t>(1, 32 * parents.size());
    for (int attempt = 0;; attempt++) {
      cells.resize(cap * Dim); table_voxel.resize(cap); table_edge.resize(cap);
      const int rc = mplx_edges_cells(ctx_, in.data(), actions.data(), (int)parents.size(), (int64_t *)offset.data(),
                                      cells.data(), (int64_t)cap, &total, table_voxel.data(), table_edge.data());
      if (rc == MPLX_OK) break;
      if (attempt > 0 || total <= (int64_t)cap) check(rc);
      cap = (std::size_t)total;  // sized from the reported total
    }
    cells.resize((std::size_t)total * Dim); table_voxel.resize((std::size_t)total); table_edge.resize((std::size_t)total);
  }

  /// Packed batched expansion for lock-step drivers (mplx_expand_packed, +inf successors dropped
  /// on the device: A* skips them, graph_search.h:81).  Results stay in the env's buffers until the
  /// next call: record r of node i is r in [p_offset[i], p_offset[i] + p_count[i]).
  ///
  /// keys_only: per record only {key, action} cross PCIe (10 B instead of 66 B for 3-D ACC).  Possible
  /// for occupancy planning (keys_only_possible()): the finite edge cost is calculate_intrinsic_cost,
  /// a function of the action alone (action_cost()), and the coordinates of a successor are needed only
  /// when its key is new to the search (graph_search.h:84-88), where forward_from_pod() evaluates them
  /// on the host with the reference's own operand order (the same bits the device produces).
  void expand_packed(const std::vector<mplx_waypoint> &nodes, bool keys_only = false) const {
    sync();
    const int n = (int)nodes.size(), nU = (int)this->U_.size();
    const std::size_t cap = (std::size_t)n * nU;
    const int nstate = Dim * __builtin_popcount(control_ & 15) + ((control_ & 16) ? 1 : 0);
    p_count.reserve(n); p_offset.reserve(n); p_action.reserve(cap); p_key.reserve(cap);
    if (!keys_only) { p_state.reserve(cap * nstate); p_cost.reserve(cap); }
    mplx_packed_out out{p_count.data(), (int64_t *)p_offset.data(), keys_only ? nullptr : p_state.data(),
                        keys_only ? nullptr : p_cost.data(), p_action.data(), p_key.data(), (int64_t)cap, 0, 0};
    check(mplx_expand_packed(ctx_, nodes.data(), n, MPLX_PACK_DROP_INF, &out));
    p_nstate = out.nstate;
    stats_nodes_ += n;
    stats_calls_++;
  }
  /// No potential field and no yaw control: traverse_primitive contributes 0 to every finite cost.
  bool keys_only_possible() const { return potential_map_.empty() && !(control_ & 16); }
  /// calculate_intrinsic_cost (env_base.h:343-345) of Primitive(., U[action], dt): for a primitive built
  /// from a state and a control only the control's own term of Primitive1D::J is non-zero
  /// (primitive.h:92-122), so the cost does not depend on the state.
  decimal_t action_cost(int action) const {
    if (action_cost_version_ != this->params_version_ || action_cost_.size() != this->U_.size()) {
      action_cost_.resize(this->U_.size());
      const Waypoint<Dim> zero(control_);
      for (std::size_t a = 0; a < this->U_.size(); a++) {
        const Primitive<Dim> pr(zero, this->U_[a], this->dt_);
        action_cost_[a] = pr.J(control_ & 15) + this->w_ * this->dt_;
      }
      action_cost_version_ = this->params_version_;
    }
    return action_cost_[action];
  }
  /// env_map.h:156-161 on the host for one successor: tn = Primitive(curr, U[action], dt).evaluate(dt),
  /// tn.t = curr.t + dt.
  Waypoint<Dim> forward_from_pod(const mplx_waypoint &curr, int action) const {
    const Waypoint<Dim> c = from_pod(curr, control_);
    const Primitive<Dim> pr(c, this->U_[action], this->dt_);
    Waypoint<Dim> tn = pr.evaluate(this->dt_);
    tn.t = c.t + this->dt_;
    return tn;
  }
  /// Rebuild the successor Waypoint of packed record r (parent `curr`): the state fields come from
  /// the record; the rest are copies, not results (include/mplx.h, mplx_packed_out): the first
  /// derivative above the state order is 0 + U[action] (Primitive1D::v/a/j at T with literal-zero
  /// higher coefficients, primitive.h:134-145), higher ones 0, yaw 0 without a yaw control,
  /// t = curr.t + dt (env_map.h:161).
  Waypoint<Dim> packed_waypoint(std::size_t r, const mplx_waypoint &curr) const {
    Waypoint<Dim> w(control_);
    const double *st = p_state.data() + r * p_nstate;
    const int nf = __builtin_popcount(control_ & 15);
    const VecDf &u = this->U_[p_action[r]];
    int c = 0;
    for (int d = 0; d < Dim; d++) w.pos(d) = st[c++];
    for (int d = 0; d < Dim; d++) w.vel(d) = nf >= 2 ? st[c++] : 0.0 + u[d];
    for (int d = 0; d < Dim; d++) w.acc(d) = nf >= 3 ? st[c++] : (nf == 2 ? 0.0 + u[d] : 0.0);
    for (int d = 0; d < Dim; d++) w.jrk(d) = nf >= 4 ? st[c++] : (nf == 3 ? 0.0 + u[d] : 0.0);
    w.yaw = (control_ & 16) ? st[c++] : 0.0;
    w.t = curr.t + this->dt_;
    return w;
  }
  /// page-locked host array (mplx_host_alloc): the packed records cross PCIe by DMA straight into
  /// it; grows, never shrinks
  template <typename T>
  struct Pinned {
    T *p = nullptr;
    std::size_t cap = 0;
    Pinned() {}
    Pinned(const Pinned &) = delete;
    ~Pinned() { if (p) mplx_host_free(p); }
    void reserve(std::size_t n) {
      if (n <= cap) return;
      if (p) mplx_host_free(p);
      cap = n + n / 4;
      p = (T *)mplx_host_alloc(cap * sizeof(T));
      if (!p) { cap = 0; throw std::runtime_error(mplx_last_error()); }
    }
    T *data() const { return p; }
    T &operator[](std::size_t i) const { return p[i]; }
  };
  mutable Pinned<int32_t> p_count;
  mutable Pinned<long long> p_offset;
  mutable Pinned<double> p_state, p_cost;
  mutable Pinned<uint16_t> p_action;
  mutable Pinned<uint64_t> p_key;
  mutable int p_nstate = 0;
  mutable std::vector<decimal_t> action_cost_;
  mutable unsigned long action_cost_version_ = ~0ul;
  static mplx_waypoint pod(const Waypoint<Dim> &w) { return to_pod(w); }
  /// the waypoint of a device state, with the env's control flag
  Waypoint<Dim> unpod(const mplx_waypoint &p) const { return from_pod(p, control_); }
  int control() const { return control_; }

  /// bring the device copy of the map (sparse edits as sparse updates), the parameters, the potential
  /// map and the tunnel up to date, for callers of the ctx's other entry points (mplx_plan_batch)
  void prepare_device() const { sync(); }
  mplx_ctx *ctx() const { return ctx_; }

  long stats_nodes() const { return stats_nodes_; }
  long stats_calls() const { return stats_calls_; }
  long stats_hits() const { return stats_hits_; }
  long launches() const { return (long)mplx_launch_count(ctx_); }
  /// grid transfers to the device so far: whole grids (mplx_set_map) and setCells edits (mplx_update_cells)
  long full_uploads() const { return full_uploads_; }
  long delta_uploads() const { return delta_uploads_; }

 private:
  struct Entry { std::vector<mplx_waypoint> succ; std::vector<double> cost; std::vector<int> action; std::vector<std::size_t> key; };
  static void check(int rc) { if (rc != MPLX_OK) throw std::runtime_error(mplx_last_error()); }
  static mplx_waypoint to_pod(const Waypoint<Dim> &w) {
    mplx_waypoint p{};
    for (int d = 0; d < Dim; d++) { p.pos[d] = w.pos(d); p.vel[d] = w.vel(d); p.acc[d] = w.acc(d); p.jrk[d] = w.jrk(d); }
    p.yaw = w.yaw; p.t = w.t;
    return p;
  }
  static Waypoint<Dim> from_pod(const mplx_waypoint &p, int control) {
    Waypoint<Dim> w(control);
    for (int d = 0; d < Dim; d++) { w.pos(d) = p.pos[d]; w.vel(d) = p.vel[d]; w.acc(d) = p.acc[d]; w.jrk(d) = p.jrk[d]; }
    w.yaw = p.yaw; w.t = p.t;
    return w;
  }
  void sync() const {
    std::size_t first = 0;
    if (map_version_ != map_util_->version() && map_util_->changesSince(map_version_, first)) {
      // only setCells edits since the device copy: patch it (O(edit), the potential map and the tunnel stay)
      const auto &idx = map_util_->journalIndex();
      check(mplx_update_cells(ctx_, idx.data() + first, map_util_->journalValue().data() + first, (int)(idx.size() - first)));
      map_version_ = map_util_->version();
      delta_uploads_++;
    }
    if (map_version_ != map_util_->version()) {
      full_uploads_++;
      const Veci<Dim> dim = map_util_->getDim();
      const Vecf<Dim> ori = map_util_->getOrigin();
      check(mplx_set_map(ctx_, map_util_->map().data(), dim.d, ori.d, map_util_->getRes()));
      map_version_ = map_util_->version();
      sent_version_ = 0;
      // mplx_set_map drops the device's potential map and tunnel (their sizes are tied to the grid); the
      // reference keeps both across MapUtil::setMap, so they are re-sent from the host copies below
      potential_on_device_ = region_on_device_ = false;
    }
    if (sent_version_ != this->params_version_) {
      if (this->U_.empty()) throw std::runtime_error("env_map_gpu: set_u() was not called");
      const int udim = (int)this->U_.front().size();
      std::vector<double> U;
      for (const auto &u : this->U_) for (int k = 0; k < udim; k++) U.push_back(u[k]);
      check(mplx_set_params(ctx_, control_, this->dt_, this->w_, this->wyaw_, this->v_max_, this->a_max_,
                            this->j_max_, this->yaw_max_, U.data(), (int)this->U_.size(), udim));
      if (!potential_on_device_)
        check(mplx_set_potential(ctx_, potential_map_.empty() ? nullptr : potential_map_.data(), potential_weight_,
                                 gradient_weight_));
      else  // the field was built on the device: only the weights may have changed
        check(mplx_set_potential_weights(ctx_, potential_weight_, gradient_weight_));
      if (!region_on_device_) {
        if (this->search_region_.empty()) check(mplx_set_search_region(ctx_, nullptr));
        else {
          std::vector<uint8_t> r(this->search_region_.begin(), this->search_region_.end());
          check(mplx_set_search_region(ctx_, r.data()));
        }
      }
      sent_version_ = this->params_version_;
    }
  }
  void expand_batch() const {
    sync();
    const int n = (int)batch_.size(), nU = (int)this->U_.size();
    in_.resize(n);
    for (int i = 0; i < n; i++) in_[i] = to_pod(batch_[i]);
    const std::size_t slots = (std::size_t)n * nU;
    count_.resize(n); succ_.resize(slots); cost_.resize(slots); action_.resize(slots); key_.resize(slots);
    mplx_succ_out out{count_.data(), succ_.data(), cost_.data(), action_.data(), key_.data(), nullptr};
    check(mplx_expand(ctx_, in_.data(), n, &out));
    for (int i = 0; i < n; i++) {
      Entry &e = cache_[batch_keys_[i]];
      const std::size_t o = (std::size_t)i * nU;
      e.succ.assign(succ_.begin() + o, succ_.begin() + o + count_[i]);
      e.cost.assign(cost_.begin() + o, cost_.begin() + o + count_[i]);
      e.action.assign(action_.begin() + o, action_.begin() + o + count_[i]);
      e.key.assign(key_.begin() + o, key_.begin() + o + count_[i]);
    }
    stats_nodes_ += n;
    stats_calls_++;
  }

  mplx_ctx *ctx_ = nullptr;
  std::vector<mplx_waypoint> *trace_ = nullptr;
  int control_ = Control::NONE, speculate_ = 1;
  mutable bool potential_on_device_ = false, region_on_device_ = false;
  mutable unsigned long map_version_ = ~0ul, sent_version_ = 0;
  mutable std::unordered_map<std::size_t, Entry> cache_;
  mutable vec_E<Waypoint<Dim>> pending_, batch_;
  mutable std::vector<std::size_t> pending_keys_, batch_keys_, last_keys_;
  mutable std::vector<uint64_t> key_;
  mutable std::vector<mplx_waypoint> in_, succ_;
  mutable std::vector<int32_t> count_, action_;
  mutable std::vector<double> cost_;
  mutable long stats_nodes_ = 0, stats_calls_ = 0, stats_hits_ = 0;
  mutable long full_uploads_ = 0, delta_uploads_ = 0;
};

/// Bump allocator for the overflow buffers of a search's predecessor lists: one rewind() returns
/// everything at once, so recycling the states of a finished search costs nothing per state.
class BumpPool {
 public:
  BumpPool() {}
  BumpPool(const BumpPool &) = delete;
  BumpPool &operator=(const BumpPool &) = delete;
  ~BumpPool() {
    for (char *b : blocks_) std::free(b);
    for (char *b : big_) std::free(b);
  }
  void *alloc(std::size_t n) {
    n = (n + 15) & ~(std::size_t)15;
    if (n > kBytes) {  // never for predecessor lists; kept correct
      char *p = (char *)std::malloc(n);
      if (!p) throw std::bad_alloc();
      big_.push_back(p);
      return p;
    }
    if (blocks_.empty() || used_ + n > kBytes) {
      if (!blocks_.empty() && cur_ + 1 < blocks_.size()) {
        cur_++;
      } else {
        char *b = (char *)std::malloc(kBytes);
        if (!b) throw std::bad_alloc();
        blocks_.push_back(b);
        cur_ = blocks_.size() - 1;
      }
      used_ = 0;
    }
    void *p = blocks_[cur_] + used_;
    used_ += n;
    return p;
  }
  void rewind() {
    cur_ = 0;
    used_ = 0;
    for (char *b : big_) std::free(b);
    big_.clear();
  }

 private:
  static constexpr std::size_t kBytes = 1 << 16;
  std::vector<char *> blocks_, big_;
  std::size_t cur_ = 0, used_ = 0;
};
/// The pool the SmallVecs of the calling thread grow into (set for the duration of one relax step by
/// PoolScope); null = malloc.
inline BumpPool *&tl_pred_pool() {
  static thread_local BumpPool *p = nullptr;
  return p;
}
struct PoolScope {
  BumpPool *prev;
  explicit PoolScope(BumpPool *p) : prev(tl_pred_pool()) { tl_pred_pool() = p; }
  ~PoolScope() { tl_pred_pool() = prev; }
};

/// A vector with room for N elements inside the object: most states have one or two predecessors,
/// so the common case needs no heap allocation.  Only what the planner uses.  A buffer grown while a
/// PoolScope is active lives in that pool (never freed individually); otherwise it is malloc'ed.
template <typename T, int N>
class SmallVec {
 public:
  SmallVec() {}
  SmallVec(const SmallVec &) = delete;
  SmallVec &operator=(const SmallVec &) = delete;
  ~SmallVec() { if (heap_ && owned_) std::free(heap_); }
  std::size_t size() const { return n_; }
  bool empty() const { return n_ == 0; }
  void clear() { n_ = 0; }
  T *begin() { return data(); }
  T *end() { return data() + n_; }
  const T *begin() const { return data(); }
  const T *end() const { return data() + n_; }
  T &operator[](std::size_t i) { return data()[i]; }
  const T &operator[](std::size_t i) const { return data()[i]; }
  void push_back(const T &v) {
    if (n_ == cap_) grow();
    data()[n_++] = v;
  }

 private:
  static_assert(std::is_trivially_copyable<T>::value, "SmallVec holds plain records");
  T *data() { return heap_ ? heap_ : inl_; }
  const T *data() const { return heap_ ? heap_ : inl_; }
  void grow() {
    const unsigned nc = cap_ * 2;
    BumpPool *pool = tl_pred_pool();
    T *p = (T *)(pool ? pool->alloc(sizeof(T) * nc) : std::malloc(sizeof(T) * nc));
    if (!p) throw std::bad_alloc();
    std::memcpy(p, data(), sizeof(T) * n_);
    if (heap_ && owned_) std::free(heap_);
    heap_ = p;
    owned_ = pool == nullptr;
    cap_ = nc;
  }
  T inl_[N];
  T *heap_ = nullptr;
  unsigned n_ = 0, cap_ = N;
  bool owned_ = false;
};

/// State: include/mpl_planner/common/state_space.h:36-74 (A* members)
template <int Dim>
struct State {
  Waypoint<Dim> coord;
  std::size_t key;
  /// pred_coord / pred_action_id / pred_action_cost of the reference (state_space.h:47-52), kept as
  /// one array of records (a predecessor is identified by its lattice key)
  struct Pred {
    State *node;
    decimal_t action_cost;
    int action_id;
  };
  SmallVec<Pred, 1> pred;
  /// succ_coord / succ_action_id / succ_action_cost (state_space.h:40-45), LPA* only.  The
  /// successor is looked up again by its lattice key when the node is re-expanded (hm_[succ_coord],
  /// graph_search.h:282), so a state pruned from the space in between is re-created, as there.
  struct Succ {
    State *node;
    decimal_t action_cost;
    int action_id;
  };
  std::vector<Succ> succ;
  int heap_idx = -1;
  decimal_t g = std::numeric_limits<decimal_t>::infinity();
  decimal_t rhs = std::numeric_limits<decimal_t>::infinity();
  decimal_t h = std::numeric_limits<decimal_t>::infinity();
  bool iterationopened = false, iterationclosed = false;
  State(const Waypoint<Dim> &c, std::size_t k) : coord(c), key(k) {}
};

/// priorityQueue: boost::heap::d_ary_heap<pair<f, State*>, arity<2>, mutable_<true>,
/// compare<compare_pair>> (state_space.h:16-34) restated: binary heap of (key, state) pairs with
/// position handles; push = append + sift up, pop = swap root with last + sift down, increase =
/// sift up, erase = move the element to the root, then pop; a child replaces its parent unless it
/// compares strictly lower.
template <int Dim>
class PriorityQueue {
 public:
  using S = State<Dim>;
  using Item = std::pair<decimal_t, S *>;
  /// compare_pair (state_space.h:16-27): true when p1 has LOWER priority than p2; ties on the key
  /// are broken on the states' current min(g, rhs)
  static bool lower(const Item &p1, const Item &p2) {
    if (p1.first == p2.first) return std::min(p1.second->g, p1.second->rhs) > std::min(p2.second->g, p2.second->rhs);
    return p1.first > p2.first;
  }
  bool empty() const { return q_.empty(); }
  std::size_t size() const { return q_.size(); }
  const Item &top() const { return q_.front(); }
  const std::vector<Item> &raw() const { return q_; }
  void clear() { q_.clear(); }
  void push(decimal_t key, S *s) { s->heap_idx = (int)q_.size(); q_.emplace_back(key, s); siftup(s->heap_idx); }
  void pop() {
    swap_at(0, (int)q_.size() - 1);
    q_.back().second->heap_idx = -1;
    q_.pop_back();
    if (!q_.empty()) siftdown(0);
  }
  /// (*heapkey).first = key; pq_.increase(heapkey)  (graph_search.h:118-119)
  void increase(S *s, decimal_t key) { q_[s->heap_idx].first = key; siftup(s->heap_idx); }
  void erase(S *s) {
    int i = s->heap_idx;
    while (i != 0) {
      const int p = (i - 1) / 2;
      swap_at(p, i);
      i = p;
    }
    pop();
  }

 private:
  void swap_at(int a, int b) { std::swap(q_[a], q_[b]); q_[a].second->heap_idx = a; q_[b].second->heap_idx = b; }
  void siftup(int i) {
    while (i != 0) {
      int p = (i - 1) / 2;
      if (lower(q_[p], q_[i])) { swap_at(p, i); i = p; } else return;
    }
  }
  void siftdown(int i) {
    const int n = (int)q_.size();
    while (2 * i + 1 < n) {
      int c = 2 * i + 1;
      if (c + 1 < n && lower(q_[c], q_[c + 1])) c = c + 1;  // first maximum among the children
      if (!lower(q_[c], q_[i])) { swap_at(c, i); i = c; } else return;
    }
  }
  std::vector<Item> q_;
};

/// lattice key -> state, open addressing with linear probing (the keys are already well-mixed 64-bit
/// hashes).  Only what the state space needs of the reference's hashMap (state_space.h:77-79):
/// look-up, insert-if-absent, swap; iteration goes through StateSpace::order_.  A slot is empty
/// while its value is null, so a key is only present once a state has been stored for it.
template <typename V>
class KeyMap {
 public:
  KeyMap() { rehash(64); }
  V *find(std::size_t k) const {
    for (std::size_t i = slot_of(k);; i = (i + 1) & mask_) {
      if (!tab_[i].second) return nullptr;
      if (tab_[i].first == k) return tab_[i].second;
    }
  }
  /// the value slot of k, entered (null) if absent; the caller must store a non-null value before the
  /// next call when `created`
  V *&obtain(std::size_t k, bool &created) {
    if ((size_ + 1) * 2 > tab_.size()) rehash(tab_.size() * 2);
    for (std::size_t i = slot_of(k);; i = (i + 1) & mask_) {
      if (!tab_[i].second) {
        tab_[i].first = k;
        size_++;
        created = true;
        return tab_[i].second;
      }
      if (tab_[i].first == k) {
        created = false;
        return tab_[i].second;
      }
    }
  }
  std::size_t size() const { return size_; }
  /// forget every key, keep the table
  void clear() {
    std::fill(tab_.begin(), tab_.end(), std::pair<std::size_t, V *>(0, nullptr));
    size_ = 0;
  }
  void swap(KeyMap &o) { tab_.swap(o.tab_); std::swap(mask_, o.mask_); std::swap(size_, o.size_); }

 private:
  std::size_t slot_of(std::size_t k) const { return ((k * 0x9e3779b97f4a7c15ULL) >> 20) & mask_; }
  void rehash(std::size_t n) {
    std::vector<std::pair<std::size_t, V *>> old(n);
    old.swap(tab_);
    mask_ = n - 1;
    for (const auto &e : old)
      if (e.second) {
        std::size_t i = slot_of(e.first);
        while (tab_[i].second) i = (i + 1) & mask_;
        tab_[i] = e;
      }
  }
  std::vector<std::pair<std::size_t, V *>> tab_;
  std::size_t mask_ = 0, size_ = 0;
};

/// StateSpace: include/mpl_planner/common/state_space.h:81-287
template <int Dim>
struct StateSpace {
  using S = State<Dim>;
  PriorityQueue<Dim> pq_;
  /// hashMap (state_space.h:77-79): lattice key -> state.  The states live in an arena owned by the
  /// space; order_ lists the states of hm_ in insertion order, which is the iteration order this
  /// planner defines for `for (it : hm_)` (boost::unordered_map leaves it unspecified; the loops
  /// of getSubStateSpace :184-192 and getLinkedNodes depend on it).
  KeyMap<S> hm_;
  std::vector<S *> order_;
  /// states are carved out of 256-state blocks: one allocation per block, addresses never move; blocks
  /// survive reset() and are handed out again
  struct Arena {
    static constexpr std::size_t kBlock = 256;
    std::vector<S *> blocks;
    std::size_t in_use = 0;  // blocks holding states
    std::size_t used = kBlock;
    S *emplace(const Waypoint<Dim> &c, std::size_t k) {
      if (used == kBlock) {
        if (in_use == blocks.size()) blocks.push_back((S *)::operator new(sizeof(S) * kBlock));
        in_use++;
        used = 0;
      }
      return new (blocks[in_use - 1] + used++) S(c, k);
    }
    /// end the life of every state; `trivial`: no state owns memory (A*-only search whose predecessor
    /// lists grew into the space's pool), so nothing has to be visited
    void rewind(bool trivial) {
      if (!trivial)
        for (std::size_t b = 0; b < in_use; b++) {
          const std::size_t n = b + 1 == in_use ? used : kBlock;
          for (std::size_t i = 0; i < n; i++) blocks[b][i].~S();
        }
      in_use = 0;
      used = kBlock;
    }
    ~Arena() {
      for (S *b : blocks) ::operator delete(b);
    }
  } arena_;
  /// overflow buffers of the predecessor lists of an A* search (AstarStepper::consume)
  BumpPool pred_pool_;
  /// true while only AstarStepper touched the states: none of them owns memory
  bool trivial_states_ = true;
  ~StateSpace() { arena_.rewind(trivial_states_); }
  /// Forget the search but keep every allocation (state blocks, predecessor pool, hash table, heap and
  /// order arrays) for the next one on this space.
  void reset(decimal_t eps) {
    arena_.rewind(trivial_states_);
    pred_pool_.rewind();
    trivial_states_ = true;
    hm_.clear();
    order_.clear();
    pq_.clear();
    best_child_.clear();
    expand_iteration_ = 0;
    eps_ = eps;
    start_t_ = start_g_ = start_rhs_ = 0;
  }
  /// hm_[coord] of a key that is not in the map yet: create the state and enter it
  S *make_state(const Waypoint<Dim> &c, std::size_t k) {
    S *n = arena_.emplace(c, k);
    bool created;
    hm_.obtain(k, created) = n;
    order_.push_back(n);
    return n;
  }
  S *find(std::size_t k) const { return hm_.find(k); }
  /// `StatePtr &p = hm_[coord]; if (!p) p = make_shared<State>(coord)` (graph_search.h:84-87) with
  /// one hash-map operation; coord() is only evaluated for a new state
  template <typename MakeCoord>
  S *get_or_make(std::size_t k, MakeCoord coord, bool &created) {
    S *&slot = hm_.obtain(k, created);
    if (created) {
      slot = arena_.emplace(coord(), k);
      order_.push_back(slot);
    }
    return slot;
  }
  decimal_t eps_;
  decimal_t dt_{1};
  std::vector<S *> best_child_;
  int expand_iteration_ = 0;
  /// state_space.h:96-100
  decimal_t start_t_{0}, start_g_{0}, start_rhs_{0};
  explicit StateSpace(decimal_t eps = 1) : eps_(eps) {}

  /// state_space.h:106-111
  decimal_t getInitTime() const { return best_child_.empty() ? 0 : best_child_.front()->coord.t; }

  /// calculateKey: state_space.h:283-285
  decimal_t calculateKey(const S *node) const { return std::min(node->g, node->rhs) + eps_ * node->h; }

  /// updateNode: state_space.h:254-280
  void updateNode(S *currNode_ptr) {
    if (currNode_ptr->rhs != start_rhs_) {  // compares VALUES, as the reference does
      currNode_ptr->rhs = std::numeric_limits<decimal_t>::infinity();
      for (const auto &pr : currNode_ptr->pred)
        if (currNode_ptr->rhs > pr.node->g + pr.action_cost) currNode_ptr->rhs = pr.node->g + pr.action_cost;
    }
    if (currNode_ptr->iterationopened && !currNode_ptr->iterationclosed) {
      pq_.erase(currNode_ptr);
      currNode_ptr->iterationclosed = true;
    }
    if (currNode_ptr->g != currNode_ptr->rhs) {
      pq_.push(calculateKey(currNode_ptr), currNode_ptr);
      currNode_ptr->iterationopened = true;
      currNode_ptr->iterationclosed = false;
    }
  }

  /// getSubStateSpace: state_space.h:116-197 — re-root the graph at best_child_[time_step]
  void getSubStateSpace(int time_step) {
    if (best_child_.empty()) return;
    const decimal_t inf = std::numeric_limits<decimal_t>::infinity();
    S *currNode_ptr = best_child_[time_step];
    start_g_ = currNode_ptr->g;
    start_rhs_ = currNode_ptr->rhs;
    start_t_ = currNode_ptr->coord.t;
    currNode_ptr->pred.clear();
    for (S *it : order_) {
      it->g = inf;
      it->rhs = inf;
      it->pred.clear();
    }
    currNode_ptr->g = start_g_;
    currNode_ptr->rhs = start_rhs_;

    KeyMap<S> new_hm;
    std::vector<S *> new_order;
    PriorityQueue<Dim> epq;
    epq.push(currNode_ptr->rhs, currNode_ptr);
    bool fresh;
    new_hm.obtain(currNode_ptr->key, fresh) = currNode_ptr;
    new_order.push_back(currNode_ptr);
    while (!epq.empty()) {
      currNode_ptr = epq.top().second;
      epq.pop();
      for (std::size_t i = 0; i < currNode_ptr->succ.size(); i++) {
        const std::size_t skey = currNode_ptr->succ[i].node->key;
        S *&slot = new_hm.obtain(skey, fresh);
        if (fresh) {
          slot = find(skey);  // hm_[succ_coord]; the reference reports a "critical bug" when absent
          if (!slot) throw std::logic_error("getSubStateSpace: successor is not in the state space");
          new_order.push_back(slot);
        }
        S *succNode_ptr = slot;
        int id = -1;
        for (std::size_t k = 0; k < succNode_ptr->pred.size(); k++)
          if (succNode_ptr->pred[k].node->key == currNode_ptr->key) { id = (int)k; break; }
        if (id == -1)
          succNode_ptr->pred.push_back(typename S::Pred{currNode_ptr, currNode_ptr->succ[i].action_cost,
                                                        currNode_ptr->succ[i].action_id});
        const decimal_t tentative_rhs = currNode_ptr->rhs + currNode_ptr->succ[i].action_cost;
        if (tentative_rhs < succNode_ptr->rhs) {
          succNode_ptr->rhs = tentative_rhs;
          if (succNode_ptr->iterationclosed) {
            succNode_ptr->g = succNode_ptr->rhs;
            epq.push(succNode_ptr->rhs, succNode_ptr);
          }
        }
      }
    }
    hm_.swap(new_hm);
    order_.swap(new_order);
    pq_.clear();
    for (S *it : order_)
      if (it->iterationopened && !it->iterationclosed) pq_.push(calculateKey(it), it);
  }

  /// One (state, i-th predecessor) reference: std::pair<Coord, int> of the reference (state_space.h:200,225)
  using EdgeRef = std::pair<S *, int>;

  /// increaseCost: state_space.h:200-221
  void increaseCost(const std::vector<EdgeRef> &states) {
    const decimal_t inf = std::numeric_limits<decimal_t>::infinity();
    for (const auto &affected_node : states) {
      S *succNode_ptr = affected_node.first;
      const int i = affected_node.second;
      if (!std::isinf(succNode_ptr->pred[i].action_cost)) {
        succNode_ptr->pred[i].action_cost = inf;
        updateNode(succNode_ptr);
        S *parent = succNode_ptr->pred[i].node;
        const int succ_act_id = succNode_ptr->pred[i].action_id;
        for (auto &sc : parent->succ)
          if (succ_act_id == sc.action_id) { sc.action_cost = inf; break; }
      }
    }
  }

  /// decreaseCost: state_space.h:223-251.  is_free(pr) of every still-blocked edge is asked in ONE
  /// batched query up front (the map does not change during the call, so the answers are the ones
  /// the reference's per-edge calls would get); the updates are then applied in list order.
  template <typename Env>
  void decreaseCost(const std::vector<EdgeRef> &states, const Env &ENV) {
    vec_E<Waypoint<Dim>> parents;
    std::vector<int> actions;
    std::vector<int> slot(states.size(), -1);
    for (std::size_t k = 0; k < states.size(); k++) {
      const auto &pr = states[k].first->pred[states[k].second];
      if (std::isinf(pr.action_cost)) {
        slot[k] = (int)parents.size();
        parents.push_back(pr.node->coord);  // forward_action(parent_key, action_id): env_base.h:228-231
        actions.push_back(pr.action_id);
      }
    }
    std::vector<uint8_t> free;
    std::vector<decimal_t> cost;
    if (!parents.empty()) ENV.is_free_edges(parents, actions, free, cost);
    for (std::size_t k = 0; k < states.size(); k++) {
      S *succNode_ptr = states[k].first;
      const int i = states[k].second;
      if (std::isinf(succNode_ptr->pred[i].action_cost) && free[slot[k]]) {
        succNode_ptr->pred[i].action_cost = cost[slot[k]];  // calculate_intrinsic_cost(pr)
        updateNode(succNode_ptr);
        S *parent = succNode_ptr->pred[i].node;
        const int succ_act_id = succNode_ptr->pred[i].action_id;
        for (auto &sc : parent->succ)
          if (succ_act_id == sc.action_id) { sc.action_cost = succNode_ptr->pred[i].action_cost; break; }
      }
    }
  }
};

/// One edge of the recovered trajectory (the reference stores Primitive<Dim>; a primitive built
/// by the state+control constructor is fully described by its start node and action id,
/// env_base.h:228-231).
template <int Dim>
struct Edge { Waypoint<Dim> from; int action_id; };

/// recoverTraj: graph_search.h:369-455 (shared by Astar and LPAstar)
template <int Dim>
bool recoverTraj(State<Dim> *currNode_ptr, StateSpace<Dim> &ss, std::size_t start_key, std::vector<Edge<Dim>> &traj) {
  using S = State<Dim>;
  const decimal_t inf = std::numeric_limits<decimal_t>::infinity();
  ss.best_child_.clear();
  bool find_traj = false;
  std::vector<Edge<Dim>> prs;
  while (!currNode_ptr->pred.empty()) {
    ss.best_child_.push_back(currNode_ptr);
    int min_id = -1;
    decimal_t min_rhs = inf, min_g = inf;
    for (unsigned int i = 0; i < currNode_ptr->pred.size(); i++) {
      const S *pred = currNode_ptr->pred[i].node;
      const decimal_t ac = currNode_ptr->pred[i].action_cost;
      if (min_rhs > pred->g + ac) {
        min_rhs = pred->g + ac;
        min_g = pred->g;
        min_id = i;
      } else if (!std::isinf(ac) && min_rhs == pred->g + ac) {
        if (min_g < pred->g) {
          min_g = pred->g;
          min_id = i;
        }
      }
    }
    if (min_id >= 0) {
      int action_idx = currNode_ptr->pred[min_id].action_id;
      currNode_ptr = currNode_ptr->pred[min_id].node;
      prs.push_back(Edge<Dim>{currNode_ptr->coord, action_idx});  // forward_action(coord, action): env_base.h:228-231
    } else
      break;
    if (currNode_ptr->key == start_key) {
      ss.best_child_.push_back(currNode_ptr);
      find_traj = true;
      break;
    }
  }
  std::reverse(prs.begin(), prs.end());
  std::reverse(ss.best_child_.begin(), ss.best_child_.end());
  traj = find_traj ? prs : std::vector<Edge<Dim>>();
  return find_traj;
}

/// The A* loop of include/mpl_planner/common/graph_search.h:39-182 cut at the get_succ call, so
/// that a driver can either run it to completion for one query (GraphSearch::Astar below) or
/// advance many queries in lock-step and expand their current nodes in ONE device launch
/// (MultiQueryPlanner).  The order of operations inside an iteration is the reference's:
/// pop + close (:66-68) -> get_succ (:75) -> relax successors (:79-143) -> goal test (:146) ->
/// max_expand (:149-155) -> empty queue (:157-161).
template <int Dim>
class AstarStepper {
 public:
  using S = State<Dim>;
  AstarStepper(const env_base<Dim> *env, std::shared_ptr<StateSpace<Dim>> ss, int max_expand)
      : ENV(env), ss_ptr(ss), max_expand_(max_expand) {}

  /// graph_search.h:43-61
  void start(const Waypoint<Dim> &start_coord) {
    start_key_ = hash_value(start_coord);
    if (ENV->is_goal(start_coord)) {
      status_ = DONE_TRIVIAL;
      return;
    }
    if (ss_ptr->pq_.empty()) {
      S *n = ss_ptr->make_state(start_coord, start_key_);
      n->g = 0;
      n->h = ss_ptr->eps_ == 0 ? 0 : ENV->get_heur(start_coord);
      ss_ptr->pq_.push(n->g + ss_ptr->eps_ * n->h, n);
      n->iterationopened = true;
      n->iterationclosed = false;
    }
    status_ = RUNNING;
  }
  bool active() const { return status_ == RUNNING; }
  const std::vector<std::pair<decimal_t, S *>> &open_heap() const { return ss_ptr->pq_.raw(); }

  /// graph_search.h:64-68: the node this iteration expands
  const Waypoint<Dim> &pop() {
    expand_iteration_++;
    curr_ = ss_ptr->pq_.top().second;
    ss_ptr->pq_.pop();
    curr_->iterationclosed = true;
    return curr_->coord;
  }

  /// graph_search.h:79-161 with the successors of the node returned by pop()
  template <typename SuccAt, typename KeyAt>
  void consume(int n_succ, SuccAt succ_at, const decimal_t *succ_cost, const int *succ_act_id, KeyAt key_at) {
    const PoolScope pool(&ss_ptr->pred_pool_);  // predecessor lists grow into the space's pool
    for (int s = 0; s < n_succ; ++s) {
      if (std::isinf(succ_cost[s])) continue;  // graph_search.h:81
      const std::size_t skey = key_at(s);
      bool created;
      S *succNode_ptr = ss_ptr->get_or_make(skey, [&] { return succ_at(s); }, created);
      if (created) succNode_ptr->h = ss_ptr->eps_ == 0 ? 0 : ENV->get_heur(succNode_ptr->coord, skey);
      succNode_ptr->pred.push_back(typename S::Pred{curr_, succ_cost[s], succ_act_id[s]});
      const decimal_t tentative_gval = curr_->g + succ_cost[s];
      if (tentative_gval < succNode_ptr->g) {
        succNode_ptr->g = tentative_gval;
        const decimal_t fval = succNode_ptr->g + (ss_ptr->eps_) * succNode_ptr->h;
        if (succNode_ptr->iterationopened && !succNode_ptr->iterationclosed) {
          ss_ptr->pq_.increase(succNode_ptr, fval);
        } else {
          ss_ptr->pq_.push(fval, succNode_ptr);
          succNode_ptr->iterationopened = true;
        }
      }
    }
    if (ENV->is_goal(curr_->coord)) {
      status_ = DONE_GOAL;
    } else if (max_expand_ > 0 && expand_iteration_ >= max_expand_) {
      status_ = FAILED;
    } else if (ss_ptr->pq_.empty()) {
      status_ = FAILED;
    }
    if (status_ != RUNNING) ss_ptr->expand_iteration_ = expand_iteration_;
  }

  /// graph_search.h:163-181: cost + recovered trajectory
  decimal_t finish(std::vector<Edge<Dim>> &traj) {
    const decimal_t inf = std::numeric_limits<decimal_t>::infinity();
    traj.clear();
    if (status_ == DONE_TRIVIAL) return 0;
    if (status_ != DONE_GOAL) return inf;
    if (recoverTraj<Dim>(curr_, *ss_ptr, start_key_, traj)) return curr_->g;
    return inf;
  }
  int expanded() const { return expand_iteration_; }

 private:
  enum Status { IDLE, RUNNING, DONE_TRIVIAL, DONE_GOAL, FAILED };
  const env_base<Dim> *ENV;
  std::shared_ptr<StateSpace<Dim>> ss_ptr;
  int max_expand_;
  Status status_ = IDLE;
  int expand_iteration_ = 0;
  std::size_t start_key_ = 0;
  S *curr_ = nullptr;
};

/// GraphSearch::Astar: include/mpl_planner/common/graph_search.h:39-182
template <int Dim>
class GraphSearch {
 public:
  explicit GraphSearch(bool verbose = false, int lookahead = 0) : verbose_(verbose), lookahead_(lookahead) {}

  decimal_t Astar(const Waypoint<Dim> &start_coord, const std::shared_ptr<env_base<Dim>> &ENV,
                  std::shared_ptr<StateSpace<Dim>> &ss_ptr, std::vector<Edge<Dim>> &traj, int max_expand = -1) {
    AstarStepper<Dim> st(ENV.get(), ss_ptr, max_expand);
    st.start(start_coord);
    vec_E<Waypoint<Dim>> succ_coord;
    std::vector<decimal_t> succ_cost;
    std::vector<int> succ_act_id;
    vec_E<Waypoint<Dim>> cands;
    std::vector<std::size_t> cand_keys;
    while (st.active()) {
      const auto &raw = st.open_heap();
      if (lookahead_ > 0 && !raw.empty() && ENV->wants_candidates(raw[0].second->key)) {
        // hint: the open nodes nearest the root of the heap are the likeliest next pops
        cands.clear();
        cand_keys.clear();
        for (std::size_t i = 1; i < raw.size() && (int)cands.size() < lookahead_; i++) {
          cands.push_back(raw[i].second->coord);
          cand_keys.push_back(raw[i].second->key);
        }
        ENV->prefetch(cands, cand_keys);
      }
      const Waypoint<Dim> &curr = st.pop();
      ENV->get_succ(curr, succ_coord, succ_cost, succ_act_id);
      const std::size_t *keys = ENV->last_succ_keys();
      st.consume((int)succ_coord.size(), [&](int s) -> const Waypoint<Dim> & { return succ_coord[s]; },
                 succ_cost.data(), succ_act_id.data(),
                 [&](int s) { return keys ? keys[s] : hash_value(succ_coord[s]); });
    }
    if (verbose_ && std::isinf(st.finish(traj))) printf("[GraphSearch] no trajectory (max expansions or empty queue)\n");
    return st.finish(traj);
  }

  /// LPAstar: include/mpl_planner/common/graph_search.h:194-365.  +inf successors are kept (they
  /// may be re-opened by decreaseCost).  An empty queue at entry reads as a +inf top key (the
  /// reference dereferences pq_.top() there).
  decimal_t LPAstar(const Waypoint<Dim> &start_coord, const std::shared_ptr<env_base<Dim>> &ENV,
                    std::shared_ptr<StateSpace<Dim>> &ss_ptr, std::vector<Edge<Dim>> &traj, int max_expand = -1) {
    ss_ptr->trivial_states_ = false;  // LPA* keeps successor lists and malloc'ed predecessor lists in the states
    using S = State<Dim>;
    const decimal_t inf = std::numeric_limits<decimal_t>::infinity();
    traj.clear();
    if (ENV->is_goal(start_coord)) return 0;
    const std::size_t start_key = hash_value(start_coord);
    S *currNode_ptr = ss_ptr->find(start_key);
    if (!currNode_ptr) {
      currNode_ptr = ss_ptr->make_state(start_coord, start_key);
      currNode_ptr->g = inf;
      currNode_ptr->rhs = 0;
      currNode_ptr->h = ss_ptr->eps_ == 0 ? 0 : ENV->get_heur(start_coord);
      ss_ptr->pq_.push(ss_ptr->calculateKey(currNode_ptr), currNode_ptr);
      currNode_ptr->iterationopened = true;
      currNode_ptr->iterationclosed = false;
    }
    // goal node: the previous goal if it still is one, else a detached placeholder (:222-240)
    S goal_placeholder{Waypoint<Dim>(), 0};
    S *goalNode_ptr = &goal_placeholder;
    if (!ss_ptr->best_child_.empty() && ENV->is_goal(ss_ptr->best_child_.back()->coord)) {
      goalNode_ptr = ss_ptr->best_child_.back();
    } else {
      goalNode_ptr->g = inf;
      goalNode_ptr->rhs = inf;
      goalNode_ptr->h = 0;
    }

    int expand_iteration = 0;
    vec_E<Waypoint<Dim>> succ_coord, cands;
    std::vector<decimal_t> succ_cost;
    std::vector<int> succ_act_id;
    std::vector<std::size_t> succ_key, cand_keys;
    auto top_key = [&] { return ss_ptr->pq_.empty() ? inf : ss_ptr->pq_.top().first; };
    while (top_key() < ss_ptr->calculateKey(goalNode_ptr) || goalNode_ptr->rhs != goalNode_ptr->g) {
      if (ss_ptr->pq_.empty()) return inf;
      expand_iteration++;
      const auto &raw = ss_ptr->pq_.raw();
      if (lookahead_ > 0 && raw[0].second->succ.empty() && ENV->wants_candidates(raw[0].second->key)) {
        cands.clear();
        cand_keys.clear();
        for (std::size_t i = 1; i < raw.size() && (int)cands.size() < lookahead_; i++)
          if (raw[i].second->succ.empty()) {
            cands.push_back(raw[i].second->coord);
            cand_keys.push_back(raw[i].second->key);
          }
        ENV->prefetch(cands, cand_keys);
      }
      currNode_ptr = ss_ptr->pq_.top().second;
      ss_ptr->pq_.pop();
      currNode_ptr->iterationclosed = true;
      if (currNode_ptr->g > currNode_ptr->rhs)
        currNode_ptr->g = currNode_ptr->rhs;
      else {
        currNode_ptr->g = inf;
        ss_ptr->updateNode(currNode_ptr);
      }

      // successors: stored ones if the node was explored before, else get_succ (:259-271)
      const bool explored = !currNode_ptr->succ.empty();
      succ_key.clear();
      if (explored) {
        succ_coord.clear(); succ_cost.clear(); succ_act_id.clear();
        for (const auto &sc : currNode_ptr->succ) {
          succ_coord.push_back(sc.node->coord);
          succ_key.push_back(sc.node->key);
          succ_cost.push_back(sc.action_cost);
          succ_act_id.push_back(sc.action_id);
        }
      } else {
        ENV->get_succ(currNode_ptr->coord, succ_coord, succ_cost, succ_act_id);
        const std::size_t *keys = ENV->last_succ_keys();
        for (std::size_t s = 0; s < succ_coord.size(); s++) succ_key.push_back(keys ? keys[s] : hash_value(succ_coord[s]));
        currNode_ptr->succ.resize(succ_coord.size());
      }

      for (std::size_t s = 0; s < succ_coord.size(); ++s) {
        bool created;
        S *succNode_ptr = ss_ptr->get_or_make(succ_key[s], [&] { return succ_coord[s]; }, created);
        if (created) succNode_ptr->h = ss_ptr->eps_ == 0 ? 0 : ENV->get_heur(succNode_ptr->coord, succ_key[s]);
        currNode_ptr->succ[s] = typename S::Succ{succNode_ptr, succ_cost[s], succ_act_id[s]};
        int id = -1;
        for (std::size_t i = 0; i < succNode_ptr->pred.size(); i++)
          if (succNode_ptr->pred[i].node->key == currNode_ptr->key) { id = (int)i; break; }
        if (id == -1) succNode_ptr->pred.push_back(typename S::Pred{currNode_ptr, succ_cost[s], succ_act_id[s]});
        ss_ptr->updateNode(succNode_ptr);
      }

      if (ENV->is_goal(currNode_ptr->coord)) goalNode_ptr = currNode_ptr;
      if (max_expand > 0 && expand_iteration >= max_expand) return inf;
      if (ss_ptr->pq_.empty()) return inf;
    }
    ss_ptr->expand_iteration_ = expand_iteration;
    if (recoverTraj<Dim>(goalNode_ptr, *ss_ptr, start_key, traj)) return goalNode_ptr->g - ss_ptr->start_g_;
    return inf;
  }

 private:
  bool verbose_;
  int lookahead_;
};

/// PlannerBase + MapPlanner: include/mpl_planner/common/planner_base.h, planner/map_planner.h
template <int Dim>
class PlannerBase {
 public:
  explicit PlannerBase(bool verbose = false) : planner_verbose_(verbose) {}
  virtual ~PlannerBase() {}
  bool initialized() { return !(ss_ptr_ == nullptr); }
  std::vector<Edge<Dim>> getTraj() const { return traj_; }
  /// planner_base.h getTraj(): the recovered trajectory as piece-wise polynomials
  /// (recoverTraj's forward_action per edge, graph_search.h:417-419)
  Trajectory<Dim> getTrajectory() const {
    vec_E<Primitive<Dim>> prs;
    for (const auto &e : traj_) {
      Primitive<Dim> pr;
      ENV_->forward_action(e.from, e.action_id, pr);
      prs.push_back(pr);
    }
    return Trajectory<Dim>(prs);
  }
  decimal_t getTrajCost() const { return traj_cost_; }
  int getExpandedNum() const { return ss_ptr_ ? ss_ptr_->expand_iteration_ : 0; }
  vec_E<Vecf<Dim>> getExpandedNodes() const { return ENV_->expanded_nodes_; }
  /// getCloseSet (planner_base.h): states with iterationclosed
  std::vector<const State<Dim> *> getCloseSetStates() const {
    std::vector<const State<Dim> *> v;
    for (const auto *st : ss_ptr_->order_) if (st->iterationclosed) v.push_back(st);
    return v;
  }
  std::size_t getOpenSetSize() const {
    std::size_t n = 0;
    for (const auto *st : ss_ptr_->order_) if (st->iterationopened && !st->iterationclosed) n++;
    return n;
  }
  void setVmax(decimal_t v) { ENV_->set_v_max(v); }
  void setAmax(decimal_t a) { ENV_->set_a_max(a); }
  void setJmax(decimal_t j) { ENV_->set_j_max(j); }
  void setYawmax(decimal_t yaw) { ENV_->set_yaw_max(yaw); }
  void setTmax(decimal_t t) { ENV_->set_t_max(t); }
  void setDt(decimal_t dt) { ENV_->set_dt(dt); }
  void setW(decimal_t w) { ENV_->set_w(w); }
  void setWyaw(decimal_t w) { ENV_->set_wyaw(w); }
  void setEpsilon(decimal_t eps) { epsilon_ = eps; }
  void setMaxNum(int num) { max_num_ = num; }
  void setU(const vec_E<VecDf> &U) { ENV_->set_u(U); }
  void setTol(decimal_t tol_pos, decimal_t tol_vel = -1, decimal_t tol_acc = -1) {
    ENV_->set_tol_pos(tol_pos); ENV_->set_tol_vel(tol_vel); ENV_->set_tol_acc(tol_acc);
  }
  void setLookahead(int k) { lookahead_ = k; }
  /// planner_base.h:233-237
  void setHeurIgnoreDynamics(bool ignore) { ENV_->set_heur_ignore_dynamics(ignore); }
  /// planner_base.h:170-176
  void setLPAstar(bool use_lpastar) { use_lpastar_ = use_lpastar; }
  /// planner_base.h:155: prune the state space to the subtree under best_child_[time_step]
  void getSubStateSpace(int time_step) { ss_ptr_->getSubStateSpace(time_step); }
  /// planner_base.h:164-167
  void reset() { ss_ptr_ = nullptr; traj_.clear(); }
  const std::shared_ptr<StateSpace<Dim>> &stateSpace() const { return ss_ptr_; }

  /// planner_base.h:275-325
  bool plan(const Waypoint<Dim> &start, const Waypoint<Dim> &goal) {
    if (!ENV_->is_free(start.pos)) {
      printf("[PlannerBase] start is not free!\n");
      return false;
    }
    GraphSearch<Dim> planner(planner_verbose_, lookahead_);
    // A*: a fresh state space per plan; LPA*: only at the first plan (planner_base.h:293-303)
    if (!use_lpastar_ || !initialized()) ss_ptr_.reset(new StateSpace<Dim>(epsilon_));
    ENV_->set_goal(goal);
    ENV_->expanded_nodes_.clear();
    ENV_->begin_plan();
    ss_ptr_->dt_ = ENV_->get_dt();
    if (use_lpastar_)
      traj_cost_ = planner.LPAstar(start, ENV_, ss_ptr_, traj_, max_num_);
    else
      traj_cost_ = planner.Astar(start, ENV_, ss_ptr_, traj_, max_num_);
    if (std::isinf(traj_cost_)) return false;
    return true;
  }

 protected:
  std::shared_ptr<env_base<Dim>> ENV_;
  std::shared_ptr<StateSpace<Dim>> ss_ptr_;
  std::vector<Edge<Dim>> traj_;
  decimal_t traj_cost_ = 0;
  decimal_t epsilon_ = 1.0;
  int max_num_ = -1;
  int lookahead_ = 0;
  bool planner_verbose_;
  bool use_lpastar_ = false;
};

template <int Dim>
class MapPlanner : public PlannerBase<Dim> {
 public:
  explicit MapPlanner(bool verbose = false) : PlannerBase<Dim>(verbose) {}
  /// src/mpl_planner/map_planner.cpp:14-18 — installs the GPU env instead of env_map<Dim>
  virtual void setMapUtil(const std::shared_ptr<MapUtil<Dim>> &map_util, int device = 0) {
    gpu_env_.reset(new env_map_gpu<Dim>(map_util, device));
    this->ENV_ = gpu_env_;
    map_util_ = map_util;
    // One launch per popped node costs ~40 us of launch + PCIe latency against ~25 us of CPU get_succ, so the
    // default expands the node together with the best open nodes it is likely to pop next (results are
    // identical for any value: get_succ is a pure function of the node); setSpeculation(1) = one node per call.
    setSpeculation(kDefaultSpeculation);
  }
  static constexpr int kDefaultSpeculation = 32;
  /// Any env_base implementation (the closed-set equality tests install a CPU checker env here).
  void setEnv(const std::shared_ptr<env_base<Dim>> &env, const std::shared_ptr<MapUtil<Dim>> &map_util = nullptr) {
    this->ENV_ = env;
    gpu_env_.reset();
    if (map_util) map_util_ = map_util;
  }
  void setControl(int control) { if (gpu_env_) gpu_env_->set_control(control); }
  void setSpeculation(int k) { if (gpu_env_) gpu_env_->set_speculation(k); this->setLookahead(k > 1 ? 4 * k : 0); }
  /// map_planner.cpp:20-43
  void setPotentialRadius(const Vecf<Dim> &radius) { potential_radius_ = radius; }
  void setPotentialMapRange(const Vecf<Dim> &range) { potential_map_range_ = range; }
  void setSearchRadius(const Vecf<Dim> &radius) { search_radius_ = radius; }
  /// map_planner.cpp:323-391, on the device
  void updatePotentialMap(const Vecf<Dim> &pos) {
    if (!gpu_env_) throw std::runtime_error("updatePotentialMap needs the GPU env (setMapUtil)");
    gpu_env_->update_potential_map(potential_radius_, pow_, potential_map_range_, pos);
  }
  /// map_planner.cpp:46-95, on the device
  void setSearchRegion(const vec_E<Vecf<Dim>> &path, bool dense = false) {
    this->ENV_->search_region_from_path(path, search_radius_, dense);
  }
  /// Trajectory::getWaypoints() positions of the last plan (trajectory.h:277-289): the start state of
  /// every primitive and the end state of the last one = the states recoverTraj walked, start to goal
  vec_E<Vecf<Dim>> getWaypointPositions() const {
    vec_E<Vecf<Dim>> path;
    if (this->ss_ptr_)
      for (const auto *st : this->ss_ptr_->best_child_) path.push_back(st->coord.pos);
    return path;
  }
  /// iterativePlan: src/mpl_planner/map_planner.cpp:393-433 — replan inside a tunnel around the previous
  /// trajectory until the cost stops changing (or max_num iterations).  raw_path = the waypoint
  /// positions of the trajectory to start from (getWaypointPositions() of an earlier plan).
  bool iterativePlan(const Waypoint<Dim> &start, const Waypoint<Dim> &goal, const vec_E<Vecf<Dim>> &raw_path,
                     int max_num = 3) {
    vec_E<Vecf<Dim>> path = raw_path;
    double prev_traj_cost = 0;
    iterations_ = 0;
    int cnt = 0;
    while (cnt < max_num) {
      cnt++;
      iterations_ = cnt;
      setSearchRegion(path, false);
      if (!this->plan(start, goal)) return false;
      if (prev_traj_cost == this->traj_cost_) break;
      prev_traj_cost = this->traj_cost_;
      path = getWaypointPositions();
    }
    return true;
  }
  /// plan() calls made by the last iterativePlan
  int iterations() const { return iterations_; }
  void setPotentialWeight(decimal_t w) { this->ENV_->set_potential_weight(w); }
  void setGradientWeight(decimal_t w) { this->ENV_->set_gradient_weight(w); }
  env_map_gpu<Dim> *gpu_env() { return gpu_env_.get(); }

  /// The reference's lhm_ (map_planner.h:15-16,101: voxel index -> the (state, i-th predecessor)
  /// edges through it) kept as a table sorted by voxel index; the edges of one voxel are in the
  /// order getLinkedNodes' push_backs would have left them.
  struct LinkedTable {
    std::vector<int> voxel, edge;                          // sorted by voxel (stable)
    std::vector<std::pair<State<Dim> *, int>> owner;       // edge -> (state, pred index)
    void clear() { voxel.clear(); edge.clear(); owner.clear(); }
    /// append the edges through voxel `id`, in lhm_[id] order
    void collect(int id, std::vector<std::pair<State<Dim> *, int>> &out) const {
      auto r = std::equal_range(voxel.begin(), voxel.end(), id);
      for (auto it = r.first; it != r.second; ++it) out.push_back(owner[edge[it - voxel.begin()]]);
    }
  };

  /// getLinkedNodes: src/mpl_planner/map_planner.cpp:124-157.  Every stored edge (state, i-th
  /// predecessor) is walked through the grid — on the device for the GPU env, all edges in one
  /// batch, which also sorts the (voxel, edge) pairs into the table — and the voxel centres are
  /// returned in the reference's order.
  vec_E<Vecf<Dim>> getLinkedNodes() const {
    using S = State<Dim>;
    const auto t_begin = std::chrono::steady_clock::now();
    lhm_.clear();
    vec_E<Vecf<Dim>> linked_pts;
    vec_E<Waypoint<Dim>> parents;
    std::vector<int> actions;
    std::size_t n_edges = 0;
    for (const S *st : this->ss_ptr_->order_) n_edges += st->pred.size();
    parents.reserve(n_edges); actions.reserve(n_edges); lhm_.owner.reserve(n_edges);
    for (S *st : this->ss_ptr_->order_)
      for (std::size_t i = 0; i < st->pred.size(); i++) {
        parents.push_back(st->pred[i].node->coord);
        actions.push_back(st->pred[i].action_id);
        lhm_.owner.emplace_back(st, (int)i);
      }
    std::vector<long long> offset;
    std::vector<int> cells;
    if (parents.empty()) return linked_pts;
    const auto t_env0 = std::chrono::steady_clock::now();
    this->ENV_->edge_cells(parents, actions, offset, cells, lhm_.voxel, lhm_.edge);
    const auto t_env1 = std::chrono::steady_clock::now();
    const std::size_t total = cells.size() / Dim;
    const decimal_t res = map_util_->getRes();
    const Vecf<Dim> ori = map_util_->getOrigin();
    const bool host_table = lhm_.voxel.size() != total;
    std::vector<int> ids;
    if (host_table) ids.resize(total);
    linked_pts.resize(total);
    for (std::size_t c = 0; c < total; c++) {
      Veci<Dim> pn;
      for (int k = 0; k < Dim; k++) pn(k) = cells[c * Dim + k];
      for (int k = 0; k < Dim; k++) linked_pts[c](k) = (pn(k) + 0.5) * res + ori(k);  // intToFloat: map_util.h:110-113
      if (host_table) ids[c] = map_util_->getIndex(pn);
    }
    if (host_table) {  // an env without the device sort: stable sort of the (voxel, edge) pairs here
      std::vector<int> owner_of(total), perm(total);
      for (std::size_t e = 0; e < parents.size(); e++)
        for (long long c = offset[e]; c < offset[e + 1]; c++) owner_of[c] = (int)e;
      for (std::size_t c = 0; c < total; c++) perm[c] = (int)c;
      std::stable_sort(perm.begin(), perm.end(), [&](int x, int y) { return ids[x] < ids[y]; });
      lhm_.voxel.resize(total); lhm_.edge.resize(total);
      for (std::size_t c = 0; c < total; c++) { lhm_.voxel[c] = ids[perm[c]]; lhm_.edge[c] = owner_of[perm[c]]; }
    }
    if (std::getenv("MPLH_TRACE")) {
      auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
        return std::chrono::duration<double, std::milli>(b - a).count();
      };
      std::fprintf(stderr, "[getLinkedNodes] %zu edges, %zu voxels: gather %.1f ms, env walk %.1f ms, points/table %.1f ms\n",
                   parents.size(), total, ms(t_begin, t_env0), ms(t_env0, t_env1), ms(t_env1, std::chrono::steady_clock::now()));
    }
    return linked_pts;
  }
  /// updateBlockedNodes: map_planner.cpp:159-171
  void updateBlockedNodes(const vec_E<Veci<Dim>> &blocked_pns) {
    std::vector<std::pair<State<Dim> *, int>> blocked_nodes;
    for (const auto &it : blocked_pns) lhm_.collect(map_util_->getIndex(it), blocked_nodes);
    this->ss_ptr_->increaseCost(blocked_nodes);
  }
  /// updateClearedNodes: map_planner.cpp:173-185; the is_free(pr) re-validation runs batched in the env
  void updateClearedNodes(const vec_E<Veci<Dim>> &cleared_pns) {
    std::vector<std::pair<State<Dim> *, int>> cleared_nodes;
    for (const auto &it : cleared_pns) lhm_.collect(map_util_->getIndex(it), cleared_nodes);
    this->ss_ptr_->decreaseCost(cleared_nodes, *this->ENV_);
  }
  const LinkedTable &linkedTable() const { return lhm_; }

 protected:
  mutable LinkedTable lhm_;
  int iterations_ = 0;
  std::shared_ptr<MapUtil<Dim>> map_util_;
  std::shared_ptr<env_map_gpu<Dim>> gpu_env_;
  Vecf<Dim> potential_radius_, potential_map_range_, search_radius_;
  decimal_t pow_{1.0};  // map_planner.h:113
};
typedef MapPlanner<2> OccMapPlanner;
typedef MapPlanner<3> VoxelMapPlanner;

/// CPUs this process may actually use: the hardware thread count capped by the cgroup v2 CPU quota
/// (/sys/fs/cgroup/cpu.max = "<quota> <period>"); oversubscribing a quota only adds throttling.
inline int effective_cpus() {
  int n = (int)std::thread::hardware_concurrency();
  if (n < 1) n = 1;
  if (FILE *f = std::fopen("/sys/fs/cgroup/cpu.max", "r")) {
    char q[64];
    long period = 0;
    if (std::fscanf(f, "%63s %ld", q, &period) == 2 && period > 0 && q[0] != 'm') {
      const long quota = std::atol(q);
      const int cap = (int)((quota + period - 1) / period);
      if (cap >= 1 && cap < n) n = cap;
    }
    std::fclose(f);
  }
  return n;
}

/// Minimal persistent worker pool for the host side of the lock-step driver: the per-query
/// bookkeeping (hash map, heap) of different queries is independent, so it is spread over the host
/// cores while the device expands the next batch's nodes.
class WorkerPool {
 public:
  explicit WorkerPool(int n_threads) {
    n_ = n_threads < 1 ? 1 : n_threads;
    for (int t = 1; t < n_; t++) th_.emplace_back([this] { loop(); });
  }
  ~WorkerPool() {
    {
      std::lock_guard<std::mutex> lk(m_);
      stop_ = true;
      gen_++;
    }
    cv_.notify_all();
    for (auto &t : th_) t.join();
  }
  int size() const { return n_; }
  /// fn(i) for i in [0, count), dynamically chunked; returns when all are done
  void run(std::size_t count, const std::function<void(std::size_t)> &fn) {
    if (count == 0) return;
    if (n_ == 1 || count < 64) {
      for (std::size_t i = 0; i < count; i++) fn(i);
      return;
    }
    {
      std::lock_guard<std::mutex> lk(m_);
      fn_ = &fn;
      count_ = count;
      next_.store(0);
      pending_ = n_ - 1;
      gen_++;
    }
    cv_.notify_all();
    work();
    std::unique_lock<std::mutex> lk(m_);
    done_.wait(lk, [this] { return pending_ == 0; });
  }

 private:
  void work() {
    const std::size_t chunk = 16;
    for (;;) {
      const std::size_t b = next_.fetch_add(chunk);
      if (b >= count_) break;
      const std::size_t e = b + chunk < count_ ? b + chunk : count_;
      for (std::size_t i = b; i < e; i++) (*fn_)(i);
    }
  }
  void loop() {
    unsigned long seen = 0;
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(m_);
        cv_.wait(lk, [&] { return gen_ != seen; });
        seen = gen_;
        if (stop_) return;
      }
      work();
      {
        std::lock_guard<std::mutex> lk(m_);
        if (--pending_ == 0) done_.notify_one();
      }
    }
  }
  int n_;
  std::vector<std::thread> th_;
  std::mutex m_;
  std::condition_variable cv_, done_;
  const std::function<void(std::size_t)> *fn_ = nullptr;
  std::size_t count_ = 0;
  std::atomic<std::size_t> next_{0};
  int pending_ = 0;
  unsigned long gen_ = 0;
  bool stop_ = false;
};

/// Lock-step batched A* over many independent (start, goal) queries on one map — BASELINE.json
/// config 5.  Every iteration pops the best open node of each live query (AstarStepper::pop) and
/// expands all of them in ONE device launch (env_map_gpu::expand_packed); each query then relaxes
/// its own successors.  Per query the sequence of expanded nodes is exactly the one
/// MapPlanner::plan() produces for that query alone.
template <int Dim>
class MultiQueryPlanner {
 public:
  struct Result {
    bool valid = false;
    decimal_t cost = std::numeric_limits<decimal_t>::infinity();
    int expanded = 0;
    std::size_t n_closed = 0;
    std::vector<int> actions;
    std::vector<uint64_t> closed_keys;  // sorted; only with setCollectClosed(true)
    /// only with setCollectTrajectories(true): recoverTraj's edges (segment k = forward_action(traj[k].from,
    /// traj[k].action_id), `from` the stored coordinates of the path's k-th state) and the stored coordinates of
    /// the goal state the last one leads to; empty without a trajectory of at least one segment
    std::vector<Edge<Dim>> traj;
    Waypoint<Dim> traj_end;
  };
  /// Which loop plan() runs.  AUTO picks, for max_expand > 0 and |U| <= 256 when the batch's worst-case
  /// search memory fits the device-memory budget:
  ///   - occupancy planning: the device search (mplx_plan_batch) once the batch has
  ///     kDeviceSearchMinQueries queries;
  ///   - plans with per-sample cost terms (a potential map or a yaw control): the device search that sums
  ///     them (mplx_plan_batch_cost_terms) once the batch has kDeviceCostTermsMinQueries queries;
  /// and the lock-step loop otherwise.  For an unbounded search (max_expand <= 0, the reference's default)
  /// and |U| <= 256, AUTO takes the growing device search (mplx_plan_batch_grow, whose arenas are sized for
  /// the batch and grow for the queries that outgrow them) from the same batch sizes.  LOCKSTEP always runs
  /// the lock-step loop.  DEVICE takes mplx_plan_batch whenever the plan, the control and the cap allow it,
  /// whatever the batch size; DEVICE_COST_TERMS takes mplx_plan_batch_cost_terms for every plan the cap and
  /// |U| allow; DEVICE_GROW takes mplx_plan_batch_grow for every plan |U| allows, bounded or not.  The
  /// forced paths run the lock-step loop for the plans they cannot take, and fail when the memory does
  /// not fit.  Queries the growing search could not fit in its largest arena run through the lock-step
  /// loop.  Every loop gives every query the same result.
  enum Path { AUTO = 0, LOCKSTEP = 1, DEVICE = 2, DEVICE_COST_TERMS = 3, DEVICE_GROW = 4 };
  /// Smallest batch AUTO sends to the device search.  search_bench.py, one H100 80GB HBM3 (the
  /// measurements are cited in DESIGN.md §7): the device search was faster at every measured batch size.
  static constexpr std::size_t kDeviceSearchMinQueries = 16;
  /// Smallest cost-term batch AUTO sends to mplx_plan_batch_cost_terms.  search_bench.py --workload cfg4,
  /// one H100 80GB HBM3 at 400 W (DESIGN.md §7): the device search was faster at every measured batch size,
  /// 2.1x at 16 queries (0.059 s against 0.125 s) and 4.8x at 4 096.
  static constexpr std::size_t kDeviceCostTermsMinQueries = 16;
  explicit MultiQueryPlanner(const std::shared_ptr<MapUtil<Dim>> &map_util, int device = 0)
      : map_util_(map_util), gpu_(new env_map_gpu<Dim>(map_util, device)) {}
  /// the shared env: set U, limits, weights, control, tolerances on it
  env_map_gpu<Dim> &env() { return *gpu_; }
  /// the session's map: edits made with setCells reach the device as sparse updates at the next plan()
  MapUtil<Dim> &map_util() { return *map_util_; }
  long iterations() const { return iterations_; }
  /// seconds spent in the three phases of the last plan(): pop, device expansion (incl. PCIe), relax
  double t_pop() const { return t_pop_; }
  double t_device() const { return t_dev_; }
  double t_relax() const { return t_relax_; }
  long nodes_expanded() const { return nodes_; }

  /// host threads used for the per-query bookkeeping (default: all cores)
  void setHostThreads(int n) { host_threads_ = n; }
  /// keys-only result stream for occupancy planning (default on; see env_map_gpu::expand_packed)
  void setKeysOnly(bool on) { keys_only_ = on; }
  /// diagnostics: force a path (Path); AUTO is the default
  void setPath(int p) { path_ = p; }
  /// diagnostics: the growing search's first and largest arena capacity (records; 0 = automatic, see
  /// mplx_plan_batch_grow)
  void setGrowCaps(long long first_cap, long long max_cap) {
    grow_first_cap_set_ = first_cap;
    grow_max_cap_set_ = max_cap;
  }
  /// also return each query's closed set (sorted lattice keys) in Result::closed_keys
  void setCollectClosed(bool on) { collect_closed_ = on; }
  /// also return each query's trajectory in Result::traj / traj_end, on every path: the lock-step loop takes
  /// recoverTraj's edges, the device searches record the stored coordinates of the path's states
  /// (mplx_set_batch_trajectories, mplx_plan_batch_trajectories)
  void setCollectTrajectories(bool on) { collect_traj_ = on; }
  /// One tunnel per query of the following plans (MapPlanner::setSearchRegion(paths[q], dense) with
  /// setSearchRadius(radius) for query q alone, in place of the env's own region); an empty list clears them, and
  /// a plan must then have paths.size() queries.  The device searches build them all at once
  /// (mplx_set_batch_regions).  The lock-step loop (small batches, LOCKSTEP and the growing search's fallback) runs
  /// tunnelled queries one at a time, each with its tunnel installed env-wide (set_search_region_path), and then
  /// restores the env's region: correct, and as slow as planning the queries one by one.
  void setSearchRegions(const std::vector<vec_E<Vecf<Dim>>> &paths, const Vecf<Dim> &radius, bool dense) {
    region_paths_ = paths;
    region_radius_ = radius;
    region_dense_ = dense;
  }
  /// a query's trajectory as PlannerBase::getTrajectory builds it: forward_action per edge
  Trajectory<Dim> trajectory(const Result &r) const {
    vec_E<Primitive<Dim>> prs;
    for (const auto &e : r.traj) {
      Primitive<Dim> pr;
      gpu_->forward_action(e.from, e.action_id, pr);
      prs.push_back(pr);
    }
    return Trajectory<Dim>(prs);
  }
  /// the path the last plan() ran: true = a device search
  bool lastPlanOnDevice() const { return last_device_ != 0; }
  /// the path the last plan() ran: 0 = lock-step, 1 = mplx_plan_batch, 2 = mplx_plan_batch_cost_terms,
  /// 3 = mplx_plan_batch_grow
  int lastDevicePath() const { return last_device_; }
  /// device search of the last plan(): arena slots and bytes per slot (0 after a lock-step plan); for the
  /// growing search those of its first round
  int searchSlots() const { return slots_; }
  long long searchArenaBytes() const { return arena_bytes_; }
  /// growing search of the last plan() (0 otherwise): kernel launches, abandoned and repeated query
  /// searches, records per arena in the first and the last round, and the queries it handed to the
  /// lock-step loop because they outgrew its largest arena
  int growRounds() const { return grow_rounds_; }
  long long growReruns() const { return grow_reruns_; }
  long long growFirstCap() const { return grow_first_cap_; }
  long long growLastCap() const { return grow_last_cap_; }
  int growLockstep() const { return grow_lockstep_; }

  /// the device search serves this plan: occupancy planning, a bounded search, |U| within one CTA
  bool deviceSearchPossible(int max_expand) const {
    return gpu_->keys_only_possible() && max_expand > 0 && gpu_->U_.size() <= 256;
  }
  /// the cost-term device search serves this plan: a bounded search, |U| within one CTA (any plan)
  bool costTermsSearchPossible(int max_expand) const { return max_expand > 0 && gpu_->U_.size() <= 256; }

  /// One query's outcome of iterativePlan.
  struct IterativeResult {
    bool ok = true;      // what MapPlanner::iterativePlan returns
    int iterations = 0;  // plan() calls made (MapPlanner::iterations())
    Result last;         // the query's last plan (traj / traj_end with setCollectTrajectories(true))
  };
  /// MapPlanner::iterativePlan(starts[q], goals[q], raw_paths[q], max_num) with setSearchRadius(radius) for every
  /// query (map_planner.cpp:393-433): replan inside the tunnel around the last trajectory until the cost stops
  /// changing, the plan fails or max_num plans were made.  Round r plans the queries still running as one batch,
  /// through plan(), so every path serves it.  Round 1 tunnels around raw_paths; later rounds around each query's
  /// last trajectory: a query the previous round's device search recorded gets its tunnel traced on the device from
  /// that recording (mplx_set_batch_regions_recorded), the others (lock-step results) from their host points in the
  /// same call.  Each query gives what MapPlanner::iterativePlan gives for it alone.  The env's own region, the
  /// setSearchRegions tunnels and setCollectTrajectories are restored however the call ends.
  std::vector<IterativeResult> iterativePlan(const vec_E<Waypoint<Dim>> &starts, const vec_E<Waypoint<Dim>> &goals,
                                             const std::vector<vec_E<Vecf<Dim>>> &raw_paths, const Vecf<Dim> &radius,
                                             decimal_t eps, int max_expand, int max_num) {
    const std::size_t Q = starts.size();
    if (goals.size() != Q || raw_paths.size() != Q)
      throw std::runtime_error("iterativePlan: one start, goal and raw path per query");
    const RestoreRegion restore_region{*gpu_, gpu_->search_region_};
    struct RestoreSettings {
      MultiQueryPlanner &p;
      std::vector<vec_E<Vecf<Dim>>> paths;
      Vecf<Dim> radius;
      bool dense, traj;
      ~RestoreSettings() {
        p.region_paths_ = std::move(paths);
        p.region_radius_ = radius;
        p.region_dense_ = dense;
        p.region_from_.clear();
        p.collect_traj_ = traj;
      }
    } restore{*this, region_paths_, region_radius_, region_dense_, collect_traj_};
    const bool want_traj = collect_traj_;
    collect_traj_ = true;  // the next round's tunnels follow this round's trajectories
    std::vector<IterativeResult> out(Q);
    std::vector<IterativeQuery> st(Q, iterative_begin(max_num));
    std::vector<vec_E<Vecf<Dim>>> path = raw_paths;
    std::vector<int32_t> from(Q, -1);  // the query's place in the last round's device search; -1: host points
    std::vector<std::size_t> run;
    for (;;) {
      run.clear();
      for (std::size_t q = 0; q < Q; q++)
        if (st[q].running) run.push_back(q);
      if (run.empty()) break;
      vec_E<Waypoint<Dim>> S, G;
      region_paths_.clear();
      region_from_.clear();
      for (const std::size_t q : run) {
        S.push_back(starts[q]);
        G.push_back(goals[q]);
        region_paths_.push_back(path[q]);
        region_from_.push_back(from[q]);
      }
      region_radius_ = radius;
      region_dense_ = false;
      std::vector<Result> res = plan(S, G, eps, max_expand);
      for (std::size_t i = 0; i < run.size(); i++) {
        const std::size_t q = run[i];
        iterative_round(st[q], res[i].valid, res[i].cost, max_num);
        if (st[q].running) {
          path[q].clear();
          for (const auto &e : res[i].traj) path[q].push_back(e.from.pos);
          if (!res[i].traj.empty()) path[q].push_back(res[i].traj_end.pos);
          from[q] = recorded_[i] ? (int32_t)i : -1;
        }
        out[q].last = std::move(res[i]);
      }
    }
    for (std::size_t q = 0; q < Q; q++) {
      out[q].ok = st[q].ok;
      out[q].iterations = st[q].iterations;
      if (!want_traj) {
        out[q].last.traj.clear();
        out[q].last.traj_end = Waypoint<Dim>();
      }
    }
    return out;
  }

  std::vector<Result> plan(const vec_E<Waypoint<Dim>> &starts, const vec_E<Waypoint<Dim>> &goals, decimal_t eps,
                           int max_expand) {
    recorded_.assign(starts.size(), 0);
    last_device_ = 0;
    slots_ = 0;
    arena_bytes_ = 0;
    grow_rounds_ = grow_lockstep_ = 0;
    grow_reruns_ = grow_first_cap_ = grow_last_cap_ = 0;
    if (!region_paths_.empty() && region_paths_.size() != starts.size())
      throw std::runtime_error("setSearchRegions: one path per query");
    const bool unbounded_auto =
        path_ == AUTO && max_expand <= 0 &&
        starts.size() >= (gpu_->keys_only_possible() ? kDeviceSearchMinQueries : kDeviceCostTermsMinQueries);
    int device = 0;  // lastDevicePath() of the device search that serves the plan, 0 for none
    if ((path_ == DEVICE_GROW || unbounded_auto) && gpu_->U_.size() <= 256) {
      device = 3;
    } else if ((path_ == AUTO || path_ == DEVICE) && deviceSearchPossible(max_expand) &&
        (path_ == DEVICE || starts.size() >= kDeviceSearchMinQueries)) {
      device = 1;
    } else if (costTermsSearchPossible(max_expand) &&
               (path_ == DEVICE_COST_TERMS ||
                (path_ == AUTO && !gpu_->keys_only_possible() && starts.size() >= kDeviceCostTermsMinQueries))) {
      device = 2;
    }
    if (device) {
      std::vector<Result> res;
      if (plan_device(starts, goals, eps, max_expand, device, res)) return res;
    }
    last_device_ = 0;
    return plan_lockstep(starts, goals, eps, max_expand, region_paths_);
  }

  /// The tunnels of setSearchRegions on the ctx for the next device search (cleared without them).  Within
  /// iterativePlan a query with region_from_ >= 0 takes the path the last device search recorded for that query.
  void install_tunnels() const {
    const bool recorded = std::any_of(region_from_.begin(), region_from_.end(), [](int32_t f) { return f >= 0; });
    std::vector<int64_t> off(region_paths_.size() + 1, 0);
    std::vector<double> pts;
    for (std::size_t q = 0; q < region_paths_.size(); q++) {
      if (!recorded || region_from_[q] < 0)
        for (const auto &p : gpu_->region_points(region_paths_[q]))
          for (int k = 0; k < Dim; k++) pts.push_back(p(k));
      off[q + 1] = (int64_t)(pts.size() / Dim);
    }
    const int n = (int)region_paths_.size(), dense = region_dense_ ? 1 : 0;
    const int rc = recorded ? mplx_set_batch_regions_recorded(gpu_->ctx(), n, region_from_.data(), off.data(),
                                                              pts.data(), region_radius_.d, dense)
                            : mplx_set_batch_regions(gpu_->ctx(), n, off.data(), pts.data(), region_radius_.d, dense);
    if (rc != MPLX_OK) throw std::runtime_error(mplx_last_error());
  }

  /// The queries in the device's form, with the start-is-free test run on the host map as the lock-step
  /// loop runs it (env_map.h:48-51).
  void device_queries(const vec_E<Waypoint<Dim>> &starts, const vec_E<Waypoint<Dim>> &goals,
                      std::vector<mplx_waypoint> &S, std::vector<mplx_waypoint> &G, std::vector<uint8_t> &fr) const {
    const std::size_t Q = starts.size();
    S.resize(Q);
    G.resize(Q);
    fr.resize(Q);
    for (std::size_t q = 0; q < Q; q++) {
      S[q] = env_map_gpu<Dim>::pod(starts[q]);
      G[q] = env_map_gpu<Dim>::pod(goals[q]);
      fr[q] = map_util_->isFree(map_util_->floatToInt(starts[q].pos)) ? 1 : 0;
    }
  }

  /// A device search's per-query results; query q's trajectory is acts[aoff[q], aoff[q+1]) and its closed
  /// keys are keys[coff[q], coff[q+1]).
  struct DeviceOut {
    std::vector<int32_t> valid, expd, ncl, acts;
    std::vector<double> cost;
    std::vector<int64_t> aoff, coff;
    std::vector<uint64_t> keys;
    explicit DeviceOut(std::size_t Q) : valid(Q), expd(Q), ncl(Q), cost(Q), aoff(Q + 1), coff(Q + 1) {}
  };

  /// Query q's result from a device search, its expansions counted in iterations_ and nodes_.
  void take_device_result(const DeviceOut &d, std::size_t q, Result &r) {
    r.valid = d.valid[q] != 0;
    r.cost = d.cost[q];
    r.expanded = d.expd[q];
    r.n_closed = (std::size_t)d.ncl[q];
    r.actions.assign(d.acts.begin() + d.aoff[q], d.acts.begin() + d.aoff[q + 1]);
    if (collect_closed_) r.closed_keys.assign(d.keys.begin() + d.coff[q], d.keys.begin() + d.coff[q + 1]);
    iterations_ = std::max<long>(iterations_, d.expd[q]);
    nodes_ += d.expd[q];
  }

  /// Trajectory recording for the next device search on the ctx: on with setCollectTrajectories(true).
  void record_trajectories() const {
    if (mplx_set_batch_trajectories(gpu_->ctx(), collect_traj_ ? 1 : 0, 0) != MPLX_OK)
      throw std::runtime_error(mplx_last_error());
  }

  /// Result::traj / traj_end of the queries the last device search gave a trajectory (res[q].actions set), from
  /// the stored coordinates it recorded (mplx_plan_batch_trajectories).
  void take_device_trajectories(std::vector<Result> &res) const {
    const std::size_t Q = res.size();
    int64_t cap = 0;
    for (const Result &r : res)
      if (!r.actions.empty()) cap += (int64_t)r.actions.size() + 1;
    cap = std::max<int64_t>(cap, 1);
    std::vector<int64_t> off(Q + 1);
    std::vector<mplx_waypoint> nodes((std::size_t)cap);
    std::vector<double> seg((std::size_t)cap), coeff((std::size_t)cap * (Dim + 1) * 6);
    mplx_batch_traj_out out{off.data(), nodes.data(), seg.data(), coeff.data(), nullptr, cap, 0, 0.0};
    if (mplx_plan_batch_trajectories(gpu_->ctx(), 0, &out) != MPLX_OK) throw std::runtime_error(mplx_last_error());
    for (std::size_t q = 0; q < Q; q++) {
      const int64_t n = off[q + 1] - off[q];
      if (n == 0) continue;
      if (n != (int64_t)res[q].actions.size() + 1) throw std::runtime_error("device trajectory length mismatch");
      for (int64_t j = 0; j + 1 < n; j++)
        res[q].traj.push_back(Edge<Dim>{gpu_->unpod(nodes[(std::size_t)(off[q] + j)]), res[q].actions[(std::size_t)j]});
      res[q].traj_end = gpu_->unpod(nodes[(std::size_t)(off[q] + n - 1)]);
    }
  }

  /// plan() on the device: every query's whole A* in one call of the device search `path` (lastDevicePath():
  /// 1 = mplx_plan_batch, 2 = mplx_plan_batch_cost_terms, 3 = mplx_plan_batch_grow, cost_terms for every plan that
  /// is not occupancy planning).  The start-is-free test runs here on the host map, as in the lock-step loop.  The
  /// queries the growing search could not fit in its largest arena (searched = 0) run through the lock-step loop,
  /// and their results are merged.  Returns false, with nothing planned, when the search memory does not fit the
  /// device-memory budget (MPLX_ERR_ALLOC: the worst-case arenas, or for the growing search a one-record arena)
  /// under AUTO: the caller then runs the lock-step loop, which served such plans before.  The forced paths report
  /// it as an error.
  bool plan_device(const vec_E<Waypoint<Dim>> &starts, const vec_E<Waypoint<Dim>> &goals, decimal_t eps,
                   int max_expand, int path, std::vector<Result> &res) {
    const std::size_t Q = starts.size();
    const bool grow = path == 3;
    res.assign(Q, Result());
    iterations_ = nodes_ = 0;
    t_pop_ = t_dev_ = t_relax_ = 0;
    gpu_->prepare_device();
    install_tunnels();
    DeviceOut d(Q);
    if (!grow) {
      // sized before any result buffer exists: the host arrays below are as large as the device's
      const int fit = (path == 2 ? mplx_plan_batch_cost_terms_fits : mplx_plan_batch_fits)(
          gpu_->ctx(), (int)Q, max_expand, collect_closed_ ? 1 : 0, nullptr, nullptr);
      if (fit == MPLX_ERR_ALLOC && path_ == AUTO) return false;
      if (fit != MPLX_OK) throw std::runtime_error(mplx_last_error());
      last_device_ = path;
      if (Q == 0) return true;
      d.acts.resize(Q * (std::size_t)max_expand);
      d.keys.resize(collect_closed_ ? Q * (std::size_t)max_expand : 0);
    }
    std::vector<mplx_waypoint> S, G;
    std::vector<uint8_t> fr;
    device_queries(starts, goals, S, G, fr);
    std::vector<int32_t> nact(Q), searched(Q, 1);
    mplx_batch_out out{d.valid.data(), d.cost.data(), d.expd.data(), d.ncl.data(), d.aoff.data(), d.acts.data(),
                       (int64_t)d.acts.size(), collect_closed_ ? d.coff.data() : nullptr,
                       collect_closed_ ? d.keys.data() : nullptr, (int64_t)d.keys.size(), 0, 0, 0.0};
    mplx_grow_out gout{d.valid.data(), d.cost.data(), d.expd.data(), d.ncl.data(), nact.data(), searched.data(), 0, 0, 0,
                       0, 0, 0, 0.0};
    record_trajectories();
    const auto t0 = std::chrono::steady_clock::now();
    const int rc =
        grow ? mplx_plan_batch_grow(gpu_->ctx(), gpu_->keys_only_possible() ? 0 : 1, S.data(), G.data(), fr.data(),
                                    (int)Q, eps, max_expand, gpu_->tol_pos_, gpu_->tol_vel_, gpu_->tol_acc_,
                                    gpu_->tol_yaw_, collect_closed_ ? 1 : 0, grow_first_cap_set_, grow_max_cap_set_, 0,
                                    &gout)
             : (path == 2 ? mplx_plan_batch_cost_terms : mplx_plan_batch)(
                   gpu_->ctx(), S.data(), G.data(), fr.data(), (int)Q, eps, max_expand, gpu_->tol_pos_,
                   gpu_->tol_vel_, gpu_->tol_acc_, gpu_->tol_yaw_, &out);
    // the device allocation itself can still fail when other users of the card took memory in between
    if (rc == MPLX_ERR_ALLOC && path_ == AUTO) {
      last_device_ = 0;
      return false;
    }
    if (rc != MPLX_OK) throw std::runtime_error(mplx_last_error());
    if (grow) {
      int64_t na = 0, nc = 0;
      for (std::size_t q = 0; q < Q; q++) {
        na += nact[q];
        nc += collect_closed_ ? d.ncl[q] : 0;
      }
      d.acts.resize(std::max<int64_t>(na, 1));
      d.keys.resize(std::max<int64_t>(nc, 1));
      if (mplx_plan_batch_grow_results(gpu_->ctx(), d.aoff.data(), d.acts.data(), (int64_t)d.acts.size(),
                                       d.coff.data(), collect_closed_ ? d.keys.data() : nullptr,
                                       (int64_t)d.keys.size()) != MPLX_OK)
        throw std::runtime_error(mplx_last_error());
    }
    t_dev_ = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    vec_E<Waypoint<Dim>> restS, restG;
    std::vector<std::size_t> rest;
    std::vector<vec_E<Vecf<Dim>>> restP;  // their tunnels, with setSearchRegions
    for (std::size_t q = 0; q < Q; q++) {
      if (searched[q]) {
        take_device_result(d, q, res[q]);
        recorded_[q] = collect_traj_ && !res[q].actions.empty();
        continue;
      }
      rest.push_back(q);
      restS.push_back(starts[q]);
      restG.push_back(goals[q]);
      if (!region_paths_.empty()) restP.push_back(region_paths_[q]);
    }
    // the device's trajectories before the lock-step loop takes the rest (unsearched queries have none)
    if (collect_traj_) take_device_trajectories(res);
    if (!rest.empty()) {
      std::vector<Result> sub = plan_lockstep(restS, restG, eps, max_expand, restP);
      for (std::size_t i = 0; i < rest.size(); i++) res[rest[i]] = std::move(sub[i]);
      iterations_ = nodes_ = 0;
      for (const Result &r : res) {
        iterations_ = std::max<long>(iterations_, r.expanded);
        nodes_ += r.expanded;
      }
    }
    last_device_ = path;
    slots_ = grow ? gout.slots : out.slots;
    arena_bytes_ = grow ? gout.arena_bytes : out.arena_bytes;
    if (grow) {
      grow_rounds_ = gout.rounds;
      grow_reruns_ = gout.reruns;
      grow_first_cap_ = gout.first_cap;
      grow_last_cap_ = gout.last_cap;
      grow_lockstep_ = (int)rest.size();
    }
    return true;
  }
  /// Free the search states of the last plan() (tens of millions of states for a large batch), on
  /// the host cores.  Called by the next plan() and the destructor.
  void release() {
    if (ss_.empty()) return;
    WorkerPool pool(host_threads_ > 0 ? host_threads_ : effective_cpus());
    pool.run(ss_.size(), [&](std::size_t q) {
      st_[q].reset();
      ss_[q].reset();
      envs_[q].reset();
    });
    st_.clear(); ss_.clear(); envs_.clear();
  }
  ~MultiQueryPlanner() { release(); }

 private:
  /// The lock-step loop over the queries.  With tunnels (one path per query; empty for none) it runs one query at a
  /// time with its tunnel as the env's region, and the env's own region comes back however the loop ends.
  std::vector<Result> plan_lockstep(const vec_E<Waypoint<Dim>> &starts, const vec_E<Waypoint<Dim>> &goals,
                                    decimal_t eps, int max_expand, const std::vector<vec_E<Vecf<Dim>>> &tunnels) {
    if (!tunnels.empty()) {
      const RestoreRegion restore{*gpu_, gpu_->search_region_};
      std::vector<Result> res(starts.size());
      long its = 0, nodes = 0;
      double tp = 0, td = 0, tr = 0;
      for (std::size_t q = 0; q < starts.size(); q++) {
        gpu_->set_search_region_path(tunnels[q], region_radius_, region_dense_);
        res[q] = std::move(plan_lockstep(vec_E<Waypoint<Dim>>{starts[q]}, vec_E<Waypoint<Dim>>{goals[q]}, eps,
                                         max_expand, {})[0]);
        its += iterations_;
        nodes += nodes_;
        tp += t_pop_;
        td += t_dev_;
        tr += t_relax_;
      }
      iterations_ = its;
      nodes_ = nodes;
      t_pop_ = tp;
      t_dev_ = td;
      t_relax_ = tr;
      return res;
    }
    // the search states of the previous plan() are recycled, not freed: a planner that answers batch
    // after batch allocates (and page-faults) its state memory once
    if (ss_.size() != starts.size()) release();
    WorkerPool pool(host_threads_ > 0 ? host_threads_ : effective_cpus());
    const std::size_t Q = starts.size();
    auto &envs = envs_;
    auto &ss = ss_;
    auto &st = st_;
    envs.resize(Q); ss.resize(Q); st.resize(Q);
    std::vector<Result> res(Q);
    pool.run(Q, [&](std::size_t q) {
      if (!envs[q]) envs[q].reset(new QueryEnv(map_util_));
      QueryEnv &e = *envs[q];
      // every env_base parameter the goal test and the heuristic read (the expansion itself runs on gpu_)
      e.w_ = gpu_->w_; e.wyaw_ = gpu_->wyaw_; e.v_max_ = gpu_->v_max_; e.a_max_ = gpu_->a_max_; e.j_max_ = gpu_->j_max_;
      e.yaw_max_ = gpu_->yaw_max_; e.dt_ = gpu_->dt_; e.t_max_ = gpu_->t_max_;
      e.tol_pos_ = gpu_->tol_pos_; e.tol_vel_ = gpu_->tol_vel_; e.tol_acc_ = gpu_->tol_acc_; e.tol_yaw_ = gpu_->tol_yaw_;
      e.set_goal(goals[q]);
      if (ss[q]) ss[q]->reset(eps);
      else ss[q].reset(new StateSpace<Dim>(eps));
      st[q].reset(new AstarStepper<Dim>(&e, ss[q], max_expand));
      if (e.is_free(starts[q].pos)) st[q]->start(starts[q]);  // planner_base.h:283-287
    });
    std::vector<mplx_waypoint> batch;
    std::vector<std::size_t> who;
    iterations_ = nodes_ = 0;
    t_pop_ = t_dev_ = t_relax_ = 0;
    for (;;) {
      // pop phase: one node per live query (independent heaps -> parallel), then compact
      who.clear();
      for (std::size_t q = 0; q < Q; q++)
        if (st[q]->active()) who.push_back(q);
      if (who.empty()) break;
      batch.resize(who.size());
      auto t0 = std::chrono::steady_clock::now();
      pool.run(who.size(), [&](std::size_t b) { batch[b] = env_map_gpu<Dim>::pod(st[who[b]]->pop()); });
      auto t1 = std::chrono::steady_clock::now();
      const bool keys_only = keys_only_ && gpu_->keys_only_possible();
      if (keys_only) gpu_->action_cost(0);  // build the table before the parallel phase
      gpu_->expand_packed(batch, keys_only);
      auto t2 = std::chrono::steady_clock::now();
      iterations_++;
      nodes_ += (long)batch.size();
      // relax phase: every query consumes its own successors (independent state spaces -> parallel)
      pool.run(who.size(), [&](std::size_t b) {
        const std::size_t r0 = (std::size_t)gpu_->p_offset[b];
        const int cnt = gpu_->p_count[b];
        int act[kMaxSucc];
        for (int j = 0; j < cnt; j++) act[j] = gpu_->p_action[r0 + j];
        if (keys_only) {
          decimal_t cst[kMaxSucc];
          for (int j = 0; j < cnt; j++) cst[j] = gpu_->action_cost(act[j]);
          st[who[b]]->consume(cnt, [&](int s) { return gpu_->forward_from_pod(batch[b], act[s]); }, cst, act,
                              [&](int s) { return (std::size_t)gpu_->p_key[r0 + s]; });
        } else {
          st[who[b]]->consume(cnt, [&](int s) { return gpu_->packed_waypoint(r0 + s, batch[b]); },
                              gpu_->p_cost.data() + r0, act, [&](int s) { return (std::size_t)gpu_->p_key[r0 + s]; });
        }
      });
      auto t3 = std::chrono::steady_clock::now();
      t_pop_ += std::chrono::duration<double>(t1 - t0).count();
      t_dev_ += std::chrono::duration<double>(t2 - t1).count();
      t_relax_ += std::chrono::duration<double>(t3 - t2).count();
    }
    // trace back and count on the pool; the state spaces stay until release() / the next plan()
    pool.run(Q, [&](std::size_t q) {
      std::vector<Edge<Dim>> traj;
      res[q].cost = st[q]->finish(traj);
      res[q].valid = !std::isinf(res[q].cost);
      res[q].expanded = st[q]->expanded();
      for (const auto &e : traj) res[q].actions.push_back(e.action_id);
      if (collect_traj_ && !traj.empty()) {
        res[q].traj = traj;
        res[q].traj_end = ss[q]->best_child_.back()->coord;
      }
      for (const auto *stt : ss[q]->order_)
        if (stt->iterationclosed) {
          res[q].n_closed++;
          if (collect_closed_) res[q].closed_keys.push_back((uint64_t)stt->key);
        }
      std::sort(res[q].closed_keys.begin(), res[q].closed_keys.end());
    });
    return res;
  }


  /// Puts the env's own search region back however the scope ends: the lock-step loop and iterativePlan install
  /// tunnels env-wide.
  struct RestoreRegion {
    env_map_gpu<Dim> &gpu;
    const std::vector<bool> region;
    ~RestoreRegion() { gpu.set_search_region(region); }
  };

  // per-query host env: goal test + heuristic only (its get_succ is never called)
  struct QueryEnv : env_map_host<Dim> {
    using env_map_host<Dim>::env_map_host;
    void get_succ(const Waypoint<Dim> &, vec_E<Waypoint<Dim>> &, std::vector<decimal_t> &, std::vector<int> &) const override {}
  };
  std::vector<std::unique_ptr<QueryEnv>> envs_;
  std::vector<std::shared_ptr<StateSpace<Dim>>> ss_;
  std::vector<std::unique_ptr<AstarStepper<Dim>>> st_;
  std::shared_ptr<MapUtil<Dim>> map_util_;
  std::unique_ptr<env_map_gpu<Dim>> gpu_;
  long iterations_ = 0, nodes_ = 0;
  double t_pop_ = 0, t_dev_ = 0, t_relax_ = 0;
  int host_threads_ = 0;
  bool keys_only_ = true;
  int path_ = AUTO;
  bool collect_closed_ = false;
  bool collect_traj_ = false;
  std::vector<vec_E<Vecf<Dim>>> region_paths_;  // setSearchRegions
  std::vector<int32_t> region_from_;  // within iterativePlan: per query, its recorded path's query, or -1
  std::vector<uint8_t> recorded_;     // per query of the last plan(): the device search recorded its path
  Vecf<Dim> region_radius_;
  bool region_dense_ = false;
  int last_device_ = 0;  // lastDevicePath()
  int slots_ = 0;
  long long arena_bytes_ = 0;
  int grow_rounds_ = 0, grow_lockstep_ = 0;
  long long grow_reruns_ = 0, grow_first_cap_ = 0, grow_last_cap_ = 0;
  long long grow_first_cap_set_ = 0, grow_max_cap_set_ = 0;  // setGrowCaps
  static constexpr int kMaxSucc = 1024;  // |U| upper bound of libmplx
};
}  // namespace MPL
