// plan_capi.hpp — a flat C struct interface to one MPL::MapPlanner<Dim>::plan() call, shared by
// libmpl_host.so (GPU env) and the test harness (same planner, CPU checker env).
#pragma once
#include "mpl_host.hpp"

#include "plan_capi_types.h"

namespace mplh {
template <int Dim>
Waypoint<Dim> wp_from(const mplx_waypoint &p, int control) {
  Waypoint<Dim> w(control);
  for (int d = 0; d < Dim; d++) { w.pos(d) = p.pos[d]; w.vel(d) = p.vel[d]; w.acc(d) = p.acc[d]; w.jrk(d) = p.jrk[d]; }
  w.yaw = p.yaw; w.t = p.t;
  return w;
}
template <int Dim>
std::shared_ptr<MPL::MapUtil<Dim>> make_map(const mplh_plan_args *a) {
  auto mu = std::make_shared<MPL::MapUtil<Dim>>();
  Vecf<Dim> ori; Veci<Dim> dim; size_t n = 1;
  for (int k = 0; k < Dim; k++) { ori(k) = a->origin[k]; dim(k) = a->mdim[k]; n *= (size_t)a->mdim[k]; }
  mu->setMap(ori, dim, MPL::Tmap(a->map, a->map + n), a->res);
  return mu;
}
// Configure `planner` (whose env is already installed) from the flat args.
template <int Dim>
void configure(MPL::MapPlanner<Dim> &planner, const mplh_plan_args *a) {
  vec_E<VecDf> U;
  for (int i = 0; i < a->nU; i++) U.push_back(VecDf(a->U + (size_t)i * a->udim, a->U + (size_t)(i + 1) * a->udim));
  planner.setU(U);
  planner.setVmax(a->v_max); planner.setAmax(a->a_max); planner.setJmax(a->j_max); planner.setYawmax(a->yaw_max);
  planner.setDt(a->T); planner.setW(a->w); planner.setWyaw(a->wyaw); planner.setEpsilon(a->eps);
  planner.setTol(a->tol_pos, a->tol_vel, a->tol_acc);
  planner.setMaxNum(a->max_num);
  planner.setHeurIgnoreDynamics(a->heur_ignore_dynamics != 0);
}
// Export the state of the last plan(): cost, counts, the closed set (sorted lattice keys) and the
// trajectory's action ids.
template <int Dim>
void export_result(MPL::MapPlanner<Dim> &planner, bool valid, mplh_plan_result *r, uint64_t *closed_keys, int cap_closed,
                   int32_t *actions, int cap_actions) {
  r->valid = valid ? 1 : 0;
  r->cost = planner.getTrajCost();
  r->expanded = planner.getExpandedNum();
  std::vector<uint64_t> keys;
  if (planner.initialized())
    for (const auto *s : planner.getCloseSetStates()) keys.push_back((uint64_t)s->key);
  std::sort(keys.begin(), keys.end());
  r->n_closed = (int)keys.size();
  r->n_open = planner.initialized() ? (int)planner.getOpenSetSize() : 0;
  if (closed_keys)
    for (int i = 0; i < (int)keys.size() && i < cap_closed; i++) closed_keys[i] = keys[i];
  const auto traj = planner.getTraj();
  r->n_actions = (int)traj.size();
  if (actions)
    for (int i = 0; i < (int)traj.size() && i < cap_actions; i++) actions[i] = traj[i].action_id;
}
// One plan() call: configure, plan, export.
template <int Dim>
void run(MPL::MapPlanner<Dim> &planner, const mplh_plan_args *a, mplh_plan_result *r, uint64_t *closed_keys,
         int cap_closed, int32_t *actions, int cap_actions) {
  configure<Dim>(planner, a);
  const Waypoint<Dim> start = wp_from<Dim>(a->start, a->control), goal = wp_from<Dim>(a->goal, a->control);
  auto t0 = std::chrono::steady_clock::now();
  const bool ok = planner.plan(start, goal);
  r->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  export_result<Dim>(planner, ok, r, closed_keys, cap_closed, actions, cap_actions);
}
// plan(), then iterativePlan() from that trajectory inside a tunnel of the given radius
// (map_planner.cpp:393-433).  info[0] = plan() calls made by iterativePlan, info[1] = its return value.
// `first` describes the initial plan, `last` (+ closed set / actions) the final one.
template <int Dim>
void run_iterative(MPL::MapPlanner<Dim> &planner, const mplh_plan_args *a, const double *search_radius, int max_iter,
                   mplh_plan_result *first, mplh_plan_result *last, int32_t *info, uint64_t *closed_keys,
                   int cap_closed, int32_t *actions, int cap_actions) {
  configure<Dim>(planner, a);
  const Waypoint<Dim> start = wp_from<Dim>(a->start, a->control), goal = wp_from<Dim>(a->goal, a->control);
  auto t0 = std::chrono::steady_clock::now();
  const bool ok0 = planner.plan(start, goal);
  first->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  export_result<Dim>(planner, ok0, first, nullptr, 0, nullptr, 0);
  info[0] = info[1] = 0;
  *last = *first;
  if (!ok0) return;
  Vecf<Dim> rad;
  for (int k = 0; k < Dim; k++) rad(k) = search_radius[k];
  planner.setSearchRadius(rad);
  t0 = std::chrono::steady_clock::now();
  const bool ok = planner.iterativePlan(start, goal, planner.getWaypointPositions(), max_iter);
  last->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  info[0] = planner.iterations();
  info[1] = ok ? 1 : 0;
  export_result<Dim>(planner, ok, last, closed_keys, cap_closed, actions, cap_actions);
}

// plan(), then describe the recovered trajectory: samples = Trajectory::sample(N) as (N+1) rows of
// {pos, vel, acc, jrk (Dim each), yaw, yaw_dot, t}; totals = {getTotalTime(), J(control), Jyaw(), #segments};
// waypoints = getWaypoints() as rows of {pos, vel, acc, jrk (Dim each), yaw, t}; mids = evaluate(t) (the
// Waypoint overload) at the N+1 sample times, same row layout as waypoints.
template <int Dim>
void run_trajectory(MPL::MapPlanner<Dim> &planner, const mplh_plan_args *a, int N, mplh_plan_result *r, double *samples,
                    double *totals, double *waypoints, int cap_wp, int32_t *n_wp, double *mids) {
  run<Dim>(planner, a, r, nullptr, 0, nullptr, 0);
  *n_wp = 0;
  totals[0] = totals[1] = totals[2] = totals[3] = 0;
  if (!r->valid) return;
  const Trajectory<Dim> traj = planner.getTrajectory();
  totals[0] = traj.getTotalTime();
  totals[1] = traj.J(a->control);
  totals[2] = traj.Jyaw();
  totals[3] = (double)traj.segs.size();
  const auto cmds = traj.sample(N);
  const int W = 4 * Dim + 3;
  for (int i = 0; i <= N; i++) {
    double *o = samples + (size_t)i * W;
    for (int d = 0; d < Dim; d++) { o[d] = cmds[i].pos(d); o[Dim + d] = cmds[i].vel(d); o[2 * Dim + d] = cmds[i].acc(d); o[3 * Dim + d] = cmds[i].jrk(d); }
    o[4 * Dim] = cmds[i].yaw; o[4 * Dim + 1] = cmds[i].yaw_dot; o[4 * Dim + 2] = cmds[i].t;
  }
  const int V = 4 * Dim + 2;
  auto put = [&](double *o, const Waypoint<Dim> &w) {
    for (int d = 0; d < Dim; d++) { o[d] = w.pos(d); o[Dim + d] = w.vel(d); o[2 * Dim + d] = w.acc(d); o[3 * Dim + d] = w.jrk(d); }
    o[4 * Dim] = w.yaw; o[4 * Dim + 1] = w.t;
  };
  const auto ws = traj.getWaypoints();
  *n_wp = (int)ws.size();
  for (int i = 0; i < (int)ws.size() && i < cap_wp; i++) put(waypoints + (size_t)i * V, ws[i]);
  const decimal_t dt = traj.getTotalTime() / N;
  for (int i = 0; i <= N; i++) put(mids + (size_t)i * V, traj.evaluate(i * dt));
}

inline void fnv(uint64_t &h, const void *p, size_t n) {
  const unsigned char *b = (const unsigned char *)p;
  for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 0x100000001b3ULL; }
}

// Snapshot of the search state after a step: counts + a hash of every state's (key, g, rhs, flags).
template <int Dim>
void snapshot(MPL::MapPlanner<Dim> &planner, mplh_lpa_out *o) {
  struct Rec { uint64_t key; double g, rhs; uint64_t flags; };
  std::vector<Rec> recs;
  o->n_closed = o->n_open = 0;
  if (planner.initialized())
    for (const auto *s : planner.stateSpace()->order_) {
      recs.push_back(Rec{(uint64_t)s->key, s->g, s->rhs, (uint64_t)((s->iterationopened ? 1 : 0) | (s->iterationclosed ? 2 : 0))});
      if (s->iterationclosed) o->n_closed++;
      else if (s->iterationopened) o->n_open++;
    }
  std::sort(recs.begin(), recs.end(), [](const Rec &a, const Rec &b) { return a.key < b.key; });
  o->n_states = (int)recs.size();
  uint64_t h = 0xcbf29ce484222325ULL;
  for (const auto &r : recs) fnv(h, &r, sizeof r);
  o->state_hash = h;
}

// Run a scripted LPA* session (plan_capi_types.h) on `planner`, whose env and map_util are installed.
template <int Dim>
void run_lpa(MPL::MapPlanner<Dim> &planner, const std::shared_ptr<MPL::MapUtil<Dim>> &mu, const mplh_plan_args *a,
             const mplh_lpa_step *steps, int n_steps, mplh_lpa_out *outs, int32_t *actions, int cap_actions) {
  vec_E<VecDf> U;
  for (int i = 0; i < a->nU; i++) U.push_back(VecDf(a->U + (size_t)i * a->udim, a->U + (size_t)(i + 1) * a->udim));
  planner.setU(U);
  planner.setVmax(a->v_max); planner.setAmax(a->a_max); planner.setJmax(a->j_max); planner.setYawmax(a->yaw_max);
  planner.setDt(a->T); planner.setW(a->w); planner.setWyaw(a->wyaw); planner.setEpsilon(a->eps);
  planner.setTol(a->tol_pos, a->tol_vel, a->tol_acc);
  planner.setMaxNum(a->max_num);
  planner.setHeurIgnoreDynamics(a->heur_ignore_dynamics != 0);
  planner.setLPAstar(true);
  Waypoint<Dim> start = wp_from<Dim>(a->start, a->control);
  const Waypoint<Dim> goal = wp_from<Dim>(a->goal, a->control);
  for (int k = 0; k < n_steps; k++) {
    mplh_lpa_out *o = &outs[k];
    *o = mplh_lpa_out{};
    const mplh_lpa_step &st = steps[k];
    auto t0 = std::chrono::steady_clock::now();
    if (st.op == MPLH_OP_PLAN) {
      o->valid = planner.plan(start, goal) ? 1 : 0;
      o->cost = planner.getTrajCost();
      o->expanded = planner.getExpandedNum();
      const auto traj = planner.getTraj();
      o->n_actions = o->valid ? (int)traj.size() : 0;
      for (int i = 0; i < o->n_actions && i < cap_actions; i++) actions[(size_t)k * cap_actions + i] = traj[i].action_id;
    } else if (st.op == MPLH_OP_LINK) {
      o->n_linked = (int64_t)planner.getLinkedNodes().size();
      o->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      struct Rec { int64_t cell; uint64_t key; int64_t i; };
      std::vector<Rec> recs;
      const auto &lt = planner.linkedTable();
      for (std::size_t c = 0; c < lt.voxel.size(); c++) {
        const auto &e = lt.owner[lt.edge[c]];
        recs.push_back(Rec{lt.voxel[c], (uint64_t)e.first->key, e.second});
      }
      std::sort(recs.begin(), recs.end(), [](const Rec &x, const Rec &y) {
        return x.cell != y.cell ? x.cell < y.cell : (x.key != y.key ? x.key < y.key : x.i < y.i);
      });
      uint64_t h = 0xcbf29ce484222325ULL;
      for (const auto &r : recs) fnv(h, &r, sizeof r);
      o->linked_hash = h;
    } else if (st.op == MPLH_OP_BLOCK || st.op == MPLH_OP_CLEAR) {
      vec_E<Veci<Dim>> pns, inside;
      for (int i = 0; i < st.n; i++) {
        Veci<Dim> pn;
        for (int d = 0; d < Dim; d++) pn(d) = st.cells[(size_t)i * Dim + d];
        pns.push_back(pn);
        if (!mu->isOutside(pn)) inside.push_back(pn);
      }
      mu->setCells(inside, std::vector<int8_t>(inside.size(), st.op == MPLH_OP_BLOCK ? 100 : 0));
      if (st.op == MPLH_OP_BLOCK) planner.updateBlockedNodes(pns);
      else planner.updateClearedNodes(pns);
    } else if (st.op == MPLH_OP_SUBTREE) {
      const auto &bc = planner.stateSpace()->best_child_;
      if (st.n >= 0 && st.n < (int)bc.size()) {
        start = bc[st.n]->coord;
        planner.getSubStateSpace(st.n);
      }
    }
    if (st.op != MPLH_OP_LINK) o->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    snapshot<Dim>(planner, o);  // instrumentation, outside the timed region
  }
}
}  // namespace mplh
