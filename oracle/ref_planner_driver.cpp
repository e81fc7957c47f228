// ref_planner_driver.cpp — the UNMODIFIED reference planner (include/mpl_planner/planner/map_planner.h,
// src/mpl_planner/map_planner.cpp, graph_search.h, state_space.h, planner_base.h) compiled where it
// lies, behind the same flat C interface as the product's host planner (host/plan_capi.hpp), plus
// MapPlanner::updatePotentialMap / setSearchRegion for pinning the generators.  TEST INFRASTRUCTURE.
#include <mpl_planner/planner/map_planner.h>

#include <algorithm>
#include <chrono>

#include "../motion_primitive_library_b200/host/plan_capi_types.h"
#include "../motion_primitive_library_b200/host/traj_rows.hpp"

namespace {
template <int Dim>
std::shared_ptr<MPL::MapUtil<Dim>> make_map(const mplh_plan_args *a) {
  std::shared_ptr<MPL::MapUtil<Dim>> mu(new MPL::MapUtil<Dim>);
  Vecf<Dim> ori;
  Veci<Dim> dim;
  size_t n = 1;
  for (int k = 0; k < Dim; k++) {
    ori(k) = a->origin[k];
    dim(k) = a->mdim[k];
    n *= (size_t)a->mdim[k];
  }
  mu->setMap(ori, dim, MPL::Tmap(a->map, a->map + n), a->res);
  return mu;
}
template <int Dim>
Waypoint<Dim> wp_from(const mplx_waypoint &p, int control) {
  Waypoint<Dim> w((Control::Control)control);
  for (int d = 0; d < Dim; d++) {
    w.pos(d) = p.pos[d];
    w.vel(d) = p.vel[d];
    w.acc(d) = p.acc[d];
    w.jrk(d) = p.jrk[d];
  }
  w.yaw = p.yaw;
  w.t = p.t;
  return w;
}

// exposes the protected state space of PlannerBase for the closed-set export
template <int Dim>
struct Planner : MPL::MapPlanner<Dim> {
  explicit Planner(bool v) : MPL::MapPlanner<Dim>(v) {}
  using MPL::MapPlanner<Dim>::ss_ptr_;
  using MPL::MapPlanner<Dim>::ENV_;
  using MPL::MapPlanner<Dim>::lhm_;
  using MPL::MapPlanner<Dim>::pow_;  // createMask's exponent: protected, no setter in the reference
};

template <int Dim>
int plan(const mplh_plan_args *a, mplh_plan_result *r, uint64_t *closed_keys, int cap_closed, int32_t *actions,
         int cap_actions) {
  Planner<Dim> planner(false);
  planner.setMapUtil(make_map<Dim>(a));
  vec_E<VecDf> U;
  for (int i = 0; i < a->nU; i++) {
    VecDf u(a->udim);
    for (int k = 0; k < a->udim; k++) u(k) = a->U[(size_t)i * a->udim + k];
    U.push_back(u);
  }
  planner.setU(U);
  planner.setVmax(a->v_max);
  planner.setAmax(a->a_max);
  planner.setJmax(a->j_max);
  planner.setYawmax(a->yaw_max);
  planner.setDt(a->T);
  planner.setW(a->w);
  planner.setWyaw(a->wyaw);
  planner.setEpsilon(a->eps);
  planner.setTol(a->tol_pos, a->tol_vel, a->tol_acc);
  planner.setMaxNum(a->max_num);
  planner.setHeurIgnoreDynamics(a->heur_ignore_dynamics != 0);
  const Waypoint<Dim> start = wp_from<Dim>(a->start, a->control), goal = wp_from<Dim>(a->goal, a->control);
  auto t0 = std::chrono::steady_clock::now();
  r->valid = planner.plan(start, goal) ? 1 : 0;
  r->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  r->cost = planner.getTrajCost();
  r->expanded = planner.initialized() ? planner.getExpandedNum() : 0;
  std::vector<uint64_t> keys;
  int n_open = 0;
  if (planner.initialized()) {
    for (const auto &it : planner.ss_ptr_->hm_) {
      if (!it.second) continue;
      if (it.second->iterationclosed) keys.push_back((uint64_t)hash_value(it.second->coord));
      else if (it.second->iterationopened) n_open++;
    }
  }
  std::sort(keys.begin(), keys.end());
  r->n_closed = (int)keys.size();
  r->n_open = n_open;
  for (int i = 0; i < (int)keys.size() && i < cap_closed; i++) closed_keys[i] = keys[i];
  // action ids of the recovered trajectory: match each primitive's control against U
  const auto prs = planner.getTraj().getPrimitives();
  r->n_actions = (int)prs.size();
  const int order = __builtin_popcount(a->control & 15);  // coefficient index of the control: 5 - order
  for (int i = 0; i < (int)prs.size() && i < cap_actions; i++) {
    int found = -1;
    for (int u = 0; u < a->nU && found < 0; u++) {
      bool same = true;
      for (int d = 0; d < Dim; d++) same = same && prs[i].pr(d).coeff()(5 - order) == a->U[(size_t)u * a->udim + d];
      if (same && (a->control & 16)) same = prs[i].pr_yaw().coeff()(4) == a->U[(size_t)u * a->udim + Dim];
      if (same) found = u;
    }
    actions[i] = found;
  }
  return 0;
}

template <int Dim>
int potential(const mplh_plan_args *a, const double *radius, double pow, const double *range, const double *pos,
              int8_t *out) {
  Planner<Dim> planner(false);
  planner.pow_ = pow;
  auto mu = make_map<Dim>(a);
  planner.setMapUtil(mu);
  Vecf<Dim> rad, rng, p;
  for (int k = 0; k < Dim; k++) {
    rad(k) = radius[k];
    rng(k) = range ? range[k] : 0;
    p(k) = pos ? pos[k] : 0;
  }
  planner.setPotentialRadius(rad);
  planner.setPotentialMapRange(rng);
  planner.updatePotentialMap(p);
  const MPL::Tmap m = mu->getMap();
  std::copy(m.begin(), m.end(), out);
  return 0;
}

template <int Dim>
int region(const mplh_plan_args *a, const double *path, int n_path, const double *radius, int dense, uint8_t *out) {
  Planner<Dim> planner(false);
  planner.setMapUtil(make_map<Dim>(a));
  Vecf<Dim> rad;
  for (int k = 0; k < Dim; k++) rad(k) = radius[k];
  planner.setSearchRadius(rad);
  vec_Vecf<Dim> pts;
  for (int i = 0; i < n_path; i++) {
    Vecf<Dim> p;
    for (int k = 0; k < Dim; k++) p(k) = path[(size_t)i * Dim + k];
    pts.push_back(p);
  }
  planner.setSearchRegion(pts, dense != 0);
  const std::vector<bool> reg = planner.ENV_->get_search_region();
  for (size_t i = 0; i < reg.size(); i++) out[i] = reg[i] ? 1 : 0;
  return 0;
}
// plan(), then the reference's MapPlanner::iterativePlan(start, goal, getTraj(), max_iter) inside a tunnel
// of the given radius; same outputs as the host planner's run_iterative (host/plan_capi.hpp).
template <int Dim>
void export_result(Planner<Dim> &planner, const mplh_plan_args *a, bool valid, mplh_plan_result *r, uint64_t *closed_keys,
                   int cap_closed, int32_t *actions, int cap_actions) {
  r->valid = valid ? 1 : 0;
  r->cost = planner.getTrajCost();
  r->expanded = planner.initialized() ? planner.getExpandedNum() : 0;
  std::vector<uint64_t> keys;
  int n_open = 0;
  if (planner.initialized())
    for (const auto &it : planner.ss_ptr_->hm_) {
      if (!it.second) continue;
      if (it.second->iterationclosed)
        keys.push_back((uint64_t)hash_value(it.second->coord));
      else if (it.second->iterationopened)
        n_open++;
    }
  std::sort(keys.begin(), keys.end());
  r->n_closed = (int)keys.size();
  r->n_open = n_open;
  if (closed_keys)
    for (int i = 0; i < (int)keys.size() && i < cap_closed; i++) closed_keys[i] = keys[i];
  const auto prs = planner.getTraj().getPrimitives();
  r->n_actions = (int)prs.size();
  const int order = __builtin_popcount(a->control & 15);
  if (actions)
    for (int i = 0; i < (int)prs.size() && i < cap_actions; i++) {
      int found = -1;
      for (int u = 0; u < a->nU && found < 0; u++) {
        bool same = true;
        for (int d = 0; d < Dim; d++) same = same && prs[i].pr(d).coeff()(5 - order) == a->U[(size_t)u * a->udim + d];
        if (same && (a->control & 16)) same = prs[i].pr_yaw().coeff()(4) == a->U[(size_t)u * a->udim + Dim];
        if (same) found = u;
      }
      actions[i] = found;
    }
}

template <int Dim>
int iterative(const mplh_plan_args *a, const double *search_radius, int max_iter, mplh_plan_result *first,
              mplh_plan_result *last, int32_t *info, uint64_t *closed_keys, int cap_closed, int32_t *actions,
              int cap_actions) {
  Planner<Dim> planner(false);
  planner.setMapUtil(make_map<Dim>(a));
  vec_E<VecDf> U;
  for (int i = 0; i < a->nU; i++) {
    VecDf u(a->udim);
    for (int k = 0; k < a->udim; k++) u(k) = a->U[(size_t)i * a->udim + k];
    U.push_back(u);
  }
  planner.setU(U);
  planner.setVmax(a->v_max);
  planner.setAmax(a->a_max);
  planner.setJmax(a->j_max);
  planner.setYawmax(a->yaw_max);
  planner.setDt(a->T);
  planner.setW(a->w);
  planner.setWyaw(a->wyaw);
  planner.setEpsilon(a->eps);
  planner.setTol(a->tol_pos, a->tol_vel, a->tol_acc);
  planner.setMaxNum(a->max_num);
  planner.setHeurIgnoreDynamics(a->heur_ignore_dynamics != 0);
  if (a->potential) {
    size_t n = 1;
    for (int k = 0; k < Dim; k++) n *= (size_t)a->mdim[k];
    planner.ENV_->set_potential_map(std::vector<int8_t>(a->potential, a->potential + n));
    planner.setPotentialWeight(a->potential_weight);
    planner.setGradientWeight(a->gradient_weight);
  }
  const Waypoint<Dim> start = wp_from<Dim>(a->start, a->control), goal = wp_from<Dim>(a->goal, a->control);
  auto t0 = std::chrono::steady_clock::now();
  const bool ok0 = planner.plan(start, goal);
  first->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  export_result<Dim>(planner, a, ok0, first, nullptr, 0, nullptr, 0);
  info[0] = info[1] = 0;
  *last = *first;
  if (!ok0) return 0;
  Vecf<Dim> rad;
  for (int k = 0; k < Dim; k++) rad(k) = search_radius[k];
  planner.setSearchRadius(rad);
  // the reference does not report how many plan() calls iterativePlan made: count them through the
  // expanded-nodes log, which plan() clears (planner_base.h:308) — not needed for parity, so 0 here
  t0 = std::chrono::steady_clock::now();
  const bool ok = planner.iterativePlan(start, goal, planner.getTraj(), max_iter);
  last->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  info[1] = ok ? 1 : 0;
  export_result<Dim>(planner, a, ok, last, closed_keys, cap_closed, actions, cap_actions);
  return 0;
}

// plan(), then the reference's own Trajectory: sample(N), totals, getWaypoints, evaluate(t) — the layouts of
// run_trajectory in host/plan_capi.hpp.
template <int Dim>
int trajectory(const mplh_plan_args *a, int N, mplh_plan_result *r, double *samples, double *totals, double *waypoints,
               int cap_wp, int32_t *n_wp, double *mids) {
  Planner<Dim> planner(false);
  planner.setMapUtil(make_map<Dim>(a));
  vec_E<VecDf> U;
  for (int i = 0; i < a->nU; i++) {
    VecDf u(a->udim);
    for (int k = 0; k < a->udim; k++) u(k) = a->U[(size_t)i * a->udim + k];
    U.push_back(u);
  }
  planner.setU(U);
  planner.setVmax(a->v_max);
  planner.setAmax(a->a_max);
  planner.setJmax(a->j_max);
  planner.setYawmax(a->yaw_max);
  planner.setDt(a->T);
  planner.setW(a->w);
  planner.setWyaw(a->wyaw);
  planner.setEpsilon(a->eps);
  planner.setTol(a->tol_pos, a->tol_vel, a->tol_acc);
  planner.setMaxNum(a->max_num);
  planner.setHeurIgnoreDynamics(a->heur_ignore_dynamics != 0);
  const Waypoint<Dim> start = wp_from<Dim>(a->start, a->control), goal = wp_from<Dim>(a->goal, a->control);
  const bool ok = planner.plan(start, goal);
  export_result<Dim>(planner, a, ok, r, nullptr, 0, nullptr, 0);
  *n_wp = 0;
  totals[0] = totals[1] = totals[2] = totals[3] = 0;
  if (!ok) return 0;
  const Trajectory<Dim> traj = planner.getTraj();
  totals[0] = traj.getTotalTime();
  totals[1] = traj.J((Control::Control)a->control);
  totals[2] = traj.Jyaw();
  totals[3] = (double)traj.segs.size();
  const auto cmds = traj.sample(N);
  for (int i = 0; i <= N; i++) mplh::put_command_row<Dim>(samples, i, cmds[i]);
  const auto ws = traj.getWaypoints();
  *n_wp = (int)ws.size();
  for (int i = 0; i < (int)ws.size() && i < cap_wp; i++) mplh::put_waypoint_row<Dim>(waypoints, i, ws[i]);
  const decimal_t dt = traj.getTotalTime() / N;
  for (int i = 0; i <= N; i++) mplh::put_waypoint_row<Dim>(mids, i, traj.evaluate(i * dt));
  return 0;
}

inline void fnv(uint64_t &h, const void *p, size_t n) {
  const unsigned char *b = (const unsigned char *)p;
  for (size_t i = 0; i < n; i++) {
    h ^= b[i];
    h *= 0x100000001b3ULL;
  }
}

template <int Dim>
void snapshot(Planner<Dim> &planner, mplh_lpa_out *o) {
  struct Rec {
    uint64_t key;
    double g, rhs;
    uint64_t flags;
  };
  std::vector<Rec> recs;
  o->n_closed = o->n_open = 0;
  if (planner.initialized())
    for (const auto &it : planner.ss_ptr_->hm_) {
      if (!it.second) continue;
      const auto &s = it.second;
      Rec r = {(uint64_t)hash_value(s->coord), s->g, s->rhs,
               (uint64_t)((s->iterationopened ? 1 : 0) | (s->iterationclosed ? 2 : 0))};
      recs.push_back(r);
      if (s->iterationclosed)
        o->n_closed++;
      else if (s->iterationopened)
        o->n_open++;
    }
  std::sort(recs.begin(), recs.end(), [](const Rec &a, const Rec &b) { return a.key < b.key; });
  o->n_states = (int)recs.size();
  uint64_t h = 0xcbf29ce484222325ULL;
  for (const auto &r : recs) fnv(h, &r, sizeof r);
  o->state_hash = h;
}

// The scripted LPA* session of plan_capi_types.h through the reference's own planner API:
// setLPAstar / plan / getLinkedNodes / setMap + updateBlockedNodes / updateClearedNodes / getSubStateSpace.
template <int Dim>
int lpa_run(const mplh_plan_args *a, const mplh_lpa_step *steps, int n_steps, mplh_lpa_out *outs, int32_t *actions,
            int cap_actions) {
  Planner<Dim> planner(false);
  auto mu = make_map<Dim>(a);
  planner.setMapUtil(mu);
  vec_E<VecDf> U;
  for (int i = 0; i < a->nU; i++) {
    VecDf u(a->udim);
    for (int k = 0; k < a->udim; k++) u(k) = a->U[(size_t)i * a->udim + k];
    U.push_back(u);
  }
  planner.setU(U);
  planner.setVmax(a->v_max);
  planner.setAmax(a->a_max);
  planner.setJmax(a->j_max);
  planner.setYawmax(a->yaw_max);
  planner.setDt(a->T);
  planner.setW(a->w);
  planner.setWyaw(a->wyaw);
  planner.setEpsilon(a->eps);
  planner.setTol(a->tol_pos, a->tol_vel, a->tol_acc);
  planner.setMaxNum(a->max_num);
  planner.setHeurIgnoreDynamics(a->heur_ignore_dynamics != 0);
  planner.setLPAstar(true);
  Waypoint<Dim> start = wp_from<Dim>(a->start, a->control);
  const Waypoint<Dim> goal = wp_from<Dim>(a->goal, a->control);
  const int order = __builtin_popcount(a->control & 15);
  for (int k = 0; k < n_steps; k++) {
    mplh_lpa_out *o = &outs[k];
    *o = mplh_lpa_out{};
    const mplh_lpa_step &st = steps[k];
    auto t0 = std::chrono::steady_clock::now();
    if (st.op == MPLH_OP_PLAN) {
      o->valid = planner.plan(start, goal) ? 1 : 0;
      o->cost = planner.getTrajCost();
      o->expanded = planner.getExpandedNum();
      const auto prs = planner.getTraj().getPrimitives();
      o->n_actions = o->valid ? (int)prs.size() : 0;
      for (int i = 0; i < o->n_actions && i < cap_actions; i++) {
        int found = -1;
        for (int u = 0; u < a->nU && found < 0; u++) {
          bool same = true;
          for (int d = 0; d < Dim; d++) same = same && prs[i].pr(d).coeff()(5 - order) == a->U[(size_t)u * a->udim + d];
          if (same && (a->control & 16)) same = prs[i].pr_yaw().coeff()(4) == a->U[(size_t)u * a->udim + Dim];
          if (same) found = u;
        }
        actions[(size_t)k * cap_actions + i] = found;
      }
    } else if (st.op == MPLH_OP_LINK) {
      o->n_linked = (int64_t)planner.getLinkedNodes().size();
      o->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      struct Rec {
        int64_t cell;
        uint64_t key;
        int64_t i;
      };
      std::vector<Rec> recs;
      for (const auto &it : planner.lhm_)
        for (const auto &e : it.second) {
          Rec r = {it.first, (uint64_t)hash_value(e.first), e.second};
          recs.push_back(r);
        }
      std::sort(recs.begin(), recs.end(), [](const Rec &x, const Rec &y) {
        return x.cell != y.cell ? x.cell < y.cell : (x.key != y.key ? x.key < y.key : x.i < y.i);
      });
      uint64_t h = 0xcbf29ce484222325ULL;
      for (const auto &r : recs) fnv(h, &r, sizeof r);
      o->linked_hash = h;
    } else if (st.op == MPLH_OP_BLOCK || st.op == MPLH_OP_CLEAR) {
      MPL::Tmap m = mu->getMap();
      vec_Veci<Dim> pns;
      for (int i = 0; i < st.n; i++) {
        Veci<Dim> pn;
        for (int d = 0; d < Dim; d++) pn(d) = st.cells[(size_t)i * Dim + d];
        pns.push_back(pn);
        if (!mu->isOutside(pn)) m[mu->getIndex(pn)] = st.op == MPLH_OP_BLOCK ? 100 : 0;
      }
      mu->setMap(mu->getOrigin(), mu->getDim(), m, mu->getRes());
      if (st.op == MPLH_OP_BLOCK)
        planner.updateBlockedNodes(pns);
      else
        planner.updateClearedNodes(pns);
    } else if (st.op == MPLH_OP_SUBTREE) {
      const auto &bc = planner.ss_ptr_->best_child_;
      if (st.n >= 0 && st.n < (int)bc.size()) {
        start = bc[st.n]->coord;
        planner.getSubStateSpace(st.n);
      }
    }
    if (st.op != MPLH_OP_LINK) o->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    snapshot<Dim>(planner, o);  // instrumentation, outside the timed region
  }
  return 0;
}
}  // namespace

extern "C" {
int refp_lpa_run(const mplh_plan_args *a, const mplh_lpa_step *steps, int n_steps, mplh_lpa_out *outs,
                 int32_t *actions, int cap_actions) {
  return a->dim == 2 ? lpa_run<2>(a, steps, n_steps, outs, actions, cap_actions)
                     : lpa_run<3>(a, steps, n_steps, outs, actions, cap_actions);
}
int refp_plan_trajectory(const mplh_plan_args *a, int N, mplh_plan_result *r, double *samples, double *totals,
                         double *waypoints, int cap_wp, int32_t *n_wp, double *mids) {
  *r = mplh_plan_result{};
  return a->dim == 2 ? trajectory<2>(a, N, r, samples, totals, waypoints, cap_wp, n_wp, mids)
                     : trajectory<3>(a, N, r, samples, totals, waypoints, cap_wp, n_wp, mids);
}
int refp_iterative_plan(const mplh_plan_args *a, const double *search_radius, int max_iter, mplh_plan_result *first,
                        mplh_plan_result *last, int32_t *info, uint64_t *closed_keys, int cap_closed, int32_t *actions,
                        int cap_actions) {
  *first = mplh_plan_result{};
  *last = mplh_plan_result{};
  return a->dim == 2 ? iterative<2>(a, search_radius, max_iter, first, last, info, closed_keys, cap_closed, actions, cap_actions)
                     : iterative<3>(a, search_radius, max_iter, first, last, info, closed_keys, cap_closed, actions, cap_actions);
}
int refp_plan(const mplh_plan_args *a, mplh_plan_result *r, uint64_t *closed_keys, int cap_closed, int32_t *actions,
              int cap_actions) {
  *r = mplh_plan_result{};
  return a->dim == 2 ? plan<2>(a, r, closed_keys, cap_closed, actions, cap_actions)
                     : plan<3>(a, r, closed_keys, cap_closed, actions, cap_actions);
}
int refp_update_potential_map(const mplh_plan_args *a, const double *radius, const double *range, const double *pos,
                              int8_t *out) {
  return a->dim == 2 ? potential<2>(a, radius, 1.0, range, pos, out) : potential<3>(a, radius, 1.0, range, pos, out);
}
// the same with createMask's exponent pow_ (1.0 in the reference unless a subclass assigns it)
int refp_update_potential_map_pow(const mplh_plan_args *a, const double *radius, double pow, const double *range,
                                  const double *pos, int8_t *out) {
  return a->dim == 2 ? potential<2>(a, radius, pow, range, pos, out) : potential<3>(a, radius, pow, range, pos, out);
}
int refp_set_search_region(const mplh_plan_args *a, const double *path, int n_path, const double *radius, int dense,
                           uint8_t *out) {
  return a->dim == 2 ? region<2>(a, path, n_path, radius, dense, out) : region<3>(a, path, n_path, radius, dense, out);
}
}
