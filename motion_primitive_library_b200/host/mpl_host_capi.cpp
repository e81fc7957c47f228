// libmpl_host.so — C entry point that runs MPL::MapPlanner<Dim>::plan() with the GPU env
// (env_map_gpu -> libmplx).  Used by the Python tests and tools; C++ users include mpl_host.hpp.
#include <cstdlib>

#include "plan_capi.hpp"

static thread_local std::string g_err;

namespace {
/// A MapPlanner with the GPU env on map mu (map_planner.cpp:14-18), a's control and a's speculation (0 = the
/// library default)
template <int Dim>
std::unique_ptr<MPL::MapPlanner<Dim>> gpu_planner(const mplh_plan_args *a, const std::shared_ptr<MPL::MapUtil<Dim>> &mu) {
  auto planner = std::make_unique<MPL::MapPlanner<Dim>>(false);
  planner->setMapUtil(mu, a->device);
  planner->setControl(a->control);
  if (a->speculate > 0) planner->setSpeculation(a->speculate);
  return planner;
}

/// a's potential map and its two weights, when a has one
template <int Dim>
void set_potential(MPL::MapPlanner<Dim> &planner, const mplh_plan_args *a) {
  if (!a->potential) return;
  planner.gpu_env()->set_potential_map(std::vector<int8_t>(a->potential, a->potential + mplh::n_cells<Dim>(a)));
  planner.setPotentialWeight(a->potential_weight);
  planner.setGradientWeight(a->gradient_weight);
}
}  // namespace

extern "C" {
const char *mplh_last_error(void) { return g_err.c_str(); }

int mplh_plan(const mplh_plan_args *a, mplh_plan_result *r, uint64_t *closed_keys, int cap_closed, int32_t *actions,
              int cap_actions) {
  *r = mplh_plan_result{};
  return mplh::with_dim(a->dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    auto planner = gpu_planner<Dim>(a, mplh::make_map<Dim>(a));
    set_potential(*planner, a);
    mplh::run<Dim>(*planner, a, r, closed_keys, cap_closed, actions, cap_actions);
    r->gpu_nodes = planner->gpu_env()->stats_nodes();
    r->gpu_calls = planner->gpu_env()->stats_calls();
    r->gpu_launches = planner->gpu_env()->launches();
  });
}

/* mplh_plan that also returns the nodes A* expanded, in pop order (graph_search.h:66-75): the replay
 * frontier of the benchmark.  *n_trace = nodes recorded (<= cap_trace). */
int mplh_plan_trace(const mplh_plan_args *a, mplh_plan_result *r, mplx_waypoint *trace, int cap_trace, int32_t *n_trace) {
  *r = mplh_plan_result{};
  return mplh::with_dim(a->dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    std::vector<mplx_waypoint> tr;
    auto planner = gpu_planner<Dim>(a, mplh::make_map<Dim>(a));
    planner->gpu_env()->set_trace(&tr);
    std::vector<uint64_t> closed(1);
    std::vector<int32_t> actions(1);
    mplh::run<Dim>(*planner, a, r, closed.data(), 0, actions.data(), 0);
    planner->gpu_env()->set_trace(nullptr);
    const int n = (int)std::min<std::size_t>(tr.size(), (std::size_t)cap_trace);
    std::copy(tr.begin(), tr.begin() + n, trace);
    if (n_trace) *n_trace = n;
  });
}

/* MapPlanner::plan() with the GPU env, then the recovered Trajectory (include/mpl_basis/trajectory.h):
 * sample(N), getTotalTime / J / Jyaw, getWaypoints and evaluate(t); layouts in plan_capi.hpp. */
int mplh_plan_trajectory(const mplh_plan_args *a, int N, mplh_plan_result *r, double *samples, double *totals,
                         double *waypoints, int cap_wp, int32_t *n_wp, double *mids) {
  *r = mplh_plan_result{};
  return mplh::with_dim(a->dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    auto planner = gpu_planner<Dim>(a, mplh::make_map<Dim>(a));
    mplh::run_trajectory<Dim>(*planner, a, N, r, samples, totals, waypoints, cap_wp, n_wp, mids);
  });
}

/* MapPlanner::plan() followed by MapPlanner::iterativePlan() (map_planner.cpp:393-433) with the GPU
 * env: every iteration builds the tunnel around the previous trajectory on the device
 * (mplx_set_search_region_path) and replans inside it.  info[0] = plan() calls made by
 * iterativePlan, info[1] = its return value. */
int mplh_iterative_plan(const mplh_plan_args *a, const double *search_radius, int max_iter, mplh_plan_result *first,
                        mplh_plan_result *last, int32_t *info, uint64_t *closed_keys, int cap_closed, int32_t *actions,
                        int cap_actions) {
  *first = mplh_plan_result{};
  *last = mplh_plan_result{};
  return mplh::with_dim(a->dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    auto planner = gpu_planner<Dim>(a, mplh::make_map<Dim>(a));
    set_potential(*planner, a);
    mplh::run_iterative<Dim>(*planner, a, search_radius, max_iter, first, last, info, closed_keys, cap_closed, actions,
                             cap_actions);
  });
}

/* A scripted LPA* session (plan_capi_types.h: PLAN / LINK / BLOCK / CLEAR / SUBTREE steps) on one
 * MapPlanner with the GPU env: get_succ, the getLinkedNodes voxel walk and the is_free(pr)
 * re-validation of decreaseCost all run on the device.  outs has n_steps entries; the action ids of
 * the trajectory found by PLAN step k go to actions[k*cap_actions ...]. */
int mplh_lpa_run(const mplh_plan_args *a, const mplh_lpa_step *steps, int n_steps, mplh_lpa_out *outs,
                 int32_t *actions, int cap_actions) {
  return mplh::with_dim(a->dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    auto mu = mplh::make_map<Dim>(a);
    auto planner = gpu_planner<Dim>(a, mu);
    mplh::run_lpa<Dim>(*planner, mu, a, steps, n_steps, outs, actions, cap_actions);
  });
}

/* Lock-step batched A* over many (start, goal) pairs on one map (MPL::MultiQueryPlanner) as a
 * session: open once (map upload, parameters), plan any number of query sets — the search states of a
 * set are recycled for the next one, so a steady stream of batches allocates its state memory once —
 * and close.  totals (7 doubles): [0] lock-step iterations (= device launches of the expansion
 * kernel), [1] nodes expanded over all queries, [2] wall seconds of the search, [3..5] seconds in the
 * pop / device expansion (incl. PCIe) / relax phases, [6] 0 (states are kept for the next set). */
}  // extern "C"
namespace {
struct BatchSession {
  int dim = 0;
  int control = 0;
  void *mq = nullptr;  // MPL::MultiQueryPlanner<dim>*
  // trajectories and closed sets of the last mplh_batch_plan_keep, query q's at [offset[q], offset[q+1])
  std::vector<int64_t> aoff, coff;
  std::vector<int32_t> actions;
  std::vector<uint64_t> closed;
};
/// the Dim of a MultiQueryPlanner<Dim>, for the bodies with_session runs
template <class Q>
struct mq_dim;
template <int Dim>
struct mq_dim<MPL::MultiQueryPlanner<Dim>> : std::integral_constant<int, Dim> {};

template <int Dim>
MPL::MultiQueryPlanner<Dim> *open_mq(const mplh_plan_args *a) {
  auto *mq = new MPL::MultiQueryPlanner<Dim>(mplh::make_map<Dim>(a), a->device);
  auto &e = mq->env();
  if (const char *t = std::getenv("MPLH_THREADS")) mq->setHostThreads(std::atoi(t));
  vec_E<VecDf> U;
  for (int i = 0; i < a->nU; i++) U.push_back(VecDf(a->U + (size_t)i * a->udim, a->U + (size_t)(i + 1) * a->udim));
  e.set_u(U); e.set_control(a->control);
  e.set_v_max(a->v_max); e.set_a_max(a->a_max); e.set_j_max(a->j_max); e.set_yaw_max(a->yaw_max);
  e.set_dt(a->T); e.set_w(a->w); e.set_wyaw(a->wyaw);
  e.set_tol_pos(a->tol_pos); e.set_tol_vel(a->tol_vel); e.set_tol_acc(a->tol_acc);
  if (a->potential) {
    e.set_potential_map(std::vector<int8_t>(a->potential, a->potential + mplh::n_cells<Dim>(a)));
    e.set_potential_weight(a->potential_weight);
    e.set_gradient_weight(a->gradient_weight);
  }
  return mq;
}

/// Runs f(mq, s) on the session s and its MPL::MultiQueryPlanner<Dim> mq and returns 0.  A null handle, or
/// ok == false, returns 1 with `refusal`; an exception thrown by f returns 1 with its message.
template <typename F>
int with_session(void *session, F &&f, bool ok = true, const char *refusal = "null session") {
  BatchSession *s = (BatchSession *)session;
  if (!s || !s->mq || !ok) {
    g_err = refusal;
    return 1;
  }
  return mplh::with_dim(s->dim, g_err, 1, [&](auto dimtag) {
    f(*(MPL::MultiQueryPlanner<decltype(dimtag)::value> *)s->mq, *s);
  });
}

/// mplh_batch_plan, and with keep mplh_batch_plan_keep
int batch_plan(void *session, const mplx_waypoint *starts, const mplx_waypoint *goals, int n_q, double eps, int max_num,
               bool keep, bool collect_closed, mplh_query_result *out, double *totals) {
  return with_session(session, [&](auto &mq, BatchSession &s) {
    constexpr int Dim = mq_dim<std::decay_t<decltype(mq)>>::value;
    mq.setCollectClosed(keep && collect_closed);
    // the session's later plans must not keep collecting, whatever plan() does
    struct Reset {
      decltype(mq) p;
      ~Reset() { p.setCollectClosed(false); }
    } reset{mq};
    vec_E<Waypoint<Dim>> S, G;
    for (int q = 0; q < n_q; q++) {
      S.push_back(mplh::wp_from<Dim>(starts[q], s.control));
      G.push_back(mplh::wp_from<Dim>(goals[q], s.control));
    }
    auto t0 = std::chrono::steady_clock::now();
    auto res = mq.plan(S, G, eps, max_num);
    const double secs = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    if (keep) {
      s.aoff.assign((size_t)n_q + 1, 0);
      s.coff.assign((size_t)n_q + 1, 0);
      s.actions.clear();
      s.closed.clear();
    }
    for (int q = 0; q < n_q; q++) {
      out[q].valid = res[q].valid ? 1 : 0;
      out[q].cost = res[q].cost;
      out[q].expanded = res[q].expanded;
      out[q].n_closed = (int)res[q].n_closed;
      out[q].n_actions = (int)res[q].actions.size();
      if (!keep) continue;
      s.actions.insert(s.actions.end(), res[q].actions.begin(), res[q].actions.end());
      s.closed.insert(s.closed.end(), res[q].closed_keys.begin(), res[q].closed_keys.end());
      s.aoff[q + 1] = (int64_t)s.actions.size();
      s.coff[q + 1] = (int64_t)s.closed.size();
    }
    if (totals) {
      totals[0] = (double)mq.iterations(); totals[1] = (double)mq.nodes_expanded(); totals[2] = secs;
      totals[3] = mq.t_pop(); totals[4] = mq.t_device(); totals[5] = mq.t_relax(); totals[6] = 0.0;
    }
  });
}
}  // namespace
extern "C" {

void *mplh_batch_open(const mplh_plan_args *a) {
  BatchSession *s = nullptr;
  mplh::with_dim(a->dim, g_err, 1, [&](auto dimtag) {
    s = new BatchSession{a->dim, a->control, open_mq<decltype(dimtag)::value>(a)};
  });
  return s;
}

int mplh_batch_plan(void *session, const mplx_waypoint *starts, const mplx_waypoint *goals, int n_q, double eps, int max_num,
                    mplh_query_result *out, double *totals) {
  return batch_plan(session, starts, goals, n_q, eps, max_num, false, false, out, totals);
}

/* MapUtil::setCells on the session's map: cells (n x dim cell coordinates) get values[k], a later entry
 * for the same cell winning.  The next mplh_batch_plan sends only these voxels to the device and keeps
 * the potential map.  A cell outside the map fails the call with nothing changed. */
int mplh_batch_update_cells(void *session, const int32_t *cells, const int8_t *values, int n) {
  return with_session(session, [&](auto &mq, BatchSession &) {
    constexpr int Dim = mq_dim<std::decay_t<decltype(mq)>>::value;
    if (n < 0 || (n > 0 && (!cells || !values))) throw std::runtime_error("cells/values missing");
    vec_E<Veci<Dim>> pns(n);
    for (int i = 0; i < n; i++)
      for (int d = 0; d < Dim; d++) pns[i](d) = cells[(size_t)i * Dim + d];
    mq.map_util().setCells(pns, std::vector<int8_t>(values, values + n));
  });
}

/* Grid transfers of the session's env so far: *full = whole-grid uploads, *delta = sparse updates. */
int mplh_batch_map_uploads(void *session, int64_t *full, int64_t *delta) {
  return with_session(session, [&](auto &mq, BatchSession &) {
    if (full) *full = mq.env().full_uploads();
    if (delta) *delta = mq.env().delta_uploads();
  });
}

/* Which loop the session's plans run (MultiQueryPlanner::Path): 0 = automatic (a device search once the
 * batch is large enough: for a bounded search mplx_plan_batch for occupancy planning and
 * mplx_plan_batch_cost_terms for potential-field and yaw planning, for an unbounded one
 * mplx_plan_batch_grow), 1 = always lock-step, 2 = the occupancy device search whenever the plan allows it,
 * 3 = the cost-term device search for every plan, 4 = the growing device search for every plan. */
int mplh_batch_set_path(void *session, int path) {
  return with_session(session, [&](auto &mq, BatchSession &) { mq.setPath(path); }, path >= 0 && path <= 4,
                      "null session or path not in 0..4");
}

/* Diagnostics: the first and the largest arena capacity (records) of the session's growing device searches;
 * 0 = automatic (mplx_plan_batch_grow).  Negative values fail. */
int mplh_batch_set_grow_caps(void *session, int64_t first_cap, int64_t max_cap) {
  return with_session(session, [&](auto &mq, BatchSession &) { mq.setGrowCaps(first_cap, max_cap); },
                      first_cap >= 0 && max_cap >= 0, "null session or negative capacity");
}

/* The growing device search of the session's last plan (all 0 when it ran another path): kernel launches,
 * query searches abandoned and repeated, records per arena in the first and the last round, and queries it
 * handed to the lock-step loop.  Any pointer may be NULL. */
int mplh_batch_grow_stats(void *session, int32_t *rounds, int64_t *reruns, int64_t *first_cap, int64_t *last_cap,
                          int32_t *lockstep) {
  return with_session(session, [&](const auto &mq, BatchSession &) {
    if (rounds) *rounds = mq.growRounds();
    if (reruns) *reruns = mq.growReruns();
    if (first_cap) *first_cap = mq.growFirstCap();
    if (last_cap) *last_cap = mq.growLastCap();
    if (lockstep) *lockstep = mq.growLockstep();
  });
}

/* The last plan of the session: *device = 1 when it ran the occupancy device search, 2 when it ran the
 * cost-term device search, 3 when it ran the growing device search (then *slots and *arena_bytes describe
 * its (first round's) arenas), 0 when it ran the lock-step loop. */
int mplh_batch_last_path(void *session, int32_t *device, int32_t *slots, int64_t *arena_bytes) {
  return with_session(session, [&](const auto &mq, BatchSession &) {
    if (device) *device = mq.lastDevicePath();
    if (slots) *slots = mq.searchSlots();
    if (arena_bytes) *arena_bytes = mq.searchArenaBytes();
  });
}

/* mplh_batch_plan that keeps every query's trajectory (action ids) and, with collect_closed, closed set
 * (sorted lattice keys) in the session for mplh_batch_kept; out[q].n_actions and out[q].n_closed size
 * them, whatever max_num is. */
int mplh_batch_plan_keep(void *session, const mplx_waypoint *starts, const mplx_waypoint *goals, int n_q, double eps,
                         int max_num, int collect_closed, mplh_query_result *out, double *totals) {
  return batch_plan(session, starts, goals, n_q, eps, max_num, true, collect_closed != 0, out, totals);
}

/* Copies what the last mplh_batch_plan_keep kept: query q's action ids at actions[action_offset[q],
 * action_offset[q+1]) and closed keys likewise with closed_offset (closed_keys NULL = skip).  A capacity
 * that is too small fails the call with nothing written. */
int mplh_batch_kept(void *session, int64_t *action_offset, int32_t *actions, int64_t cap_actions,
                    int64_t *closed_offset, uint64_t *closed_keys, int64_t cap_closed) {
  return with_session(session, [&](const auto &, BatchSession &s) {
    if (!action_offset || (!actions && !s.actions.empty()) || (closed_keys && !closed_offset))
      throw std::runtime_error("missing output array");
    if ((int64_t)s.actions.size() > cap_actions) throw std::runtime_error("action capacity too small");
    if (closed_keys && (int64_t)s.closed.size() > cap_closed) throw std::runtime_error("closed capacity too small");
    std::copy(s.aoff.begin(), s.aoff.end(), action_offset);
    std::copy(s.actions.begin(), s.actions.end(), actions);
    if (closed_keys) {
      std::copy(s.coff.begin(), s.coff.end(), closed_offset);
      std::copy(s.closed.begin(), s.closed.end(), closed_keys);
    }
  });
}

/* Frees the session incl. the search states it kept; seconds spent are returned in *release_seconds. */
int mplh_batch_close(void *session, double *release_seconds) {
  if (!session) return 0;
  auto t0 = std::chrono::steady_clock::now();
  with_session(session, [](auto &mq, BatchSession &) { delete &mq; });
  delete (BatchSession *)session;
  if (release_seconds) *release_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return 0;
}
}

/* ---- TrajSolver (mpl_host.hpp): one path on the host -------------------------------------------------- */

namespace {
template <int Dim>
void put_samples(const Trajectory<Dim> &traj, int n_samples, double *samples) {
  const auto cmds = traj.sample(n_samples);
  for (int i = 0; i <= n_samples; i++) mplh::put_command_row<Dim>(samples, i, cmds[i]);
}
template <int Dim>
void put_waypoints(const Trajectory<Dim> &traj, double *waypoints) {
  const auto ws = traj.getWaypoints();
  for (std::size_t i = 0; i < ws.size(); i++) mplh::put_waypoint_row<Dim>(waypoints, i, ws[i]);
}
/// Trajectory<Dim> of n_seg segments with durations seg_t and coefficients coeff (mplh_traj_solve's layout), each
/// segment with the control flag `control`
template <int Dim>
Trajectory<Dim> make_trajectory(int n_seg, const double *seg_t, const double *coeff, int control) {
  vec_E<Primitive<Dim>> prs;
  for (int j = 0; j < n_seg; j++) {
    vec_E<Vecf<6>> cs(Dim + 1);
    for (int a = 0; a <= Dim; a++)
      for (int k = 0; k < 6; k++) cs[a](k) = coeff[((size_t)j * (Dim + 1) + a) * 6 + k];
    prs.push_back(Primitive<Dim>(cs, seg_t[j], control));
  }
  return Trajectory<Dim>(prs);
}
}  // namespace

extern "C" {
/* MPL::TrajSolver<dim>(control, yaw_control) on one path of n_wp waypoints.  wp_control NULL: setPath(wps[].pos);
 * else setWaypoints(wps, waypoint i with control wp_control[i]).  dts (n_wp - 1 entries) given: setDts(dts).
 * setV(v), then solve().  Outputs (host arrays; any may be NULL except n_seg):
 *   *n_seg     segments of the solved trajectory (0 when it is empty)
 *   seg_t      [n_wp - 1] getDts(): the segment times used
 *   coeff      [n_seg * (dim + 1) * 6] segment j's Primitive1D coefficients, highest order first, axes then yaw
 *   samples    [(n_samples + 1) * (4 dim + 3)] Trajectory::sample(n_samples) as command rows (traj_rows.hpp)
 *   waypoints  [(n_seg + 1) * (4 dim + 2)] Trajectory::getWaypoints() as waypoint rows (traj_rows.hpp)
 * 1: bad argument (dim, n_wp < 0, samples with n_samples < 1, missing wps); 2: solve() threw (no segment times). */
int mplh_traj_solve(int dim, int control, int yaw_control, const mplx_waypoint *wps, const uint8_t *wp_control, int n_wp,
                    const double *dts, double v, int n_samples, int32_t *n_seg, double *seg_t, double *coeff,
                    double *samples, double *waypoints) {
  if (n_wp < 0 || (n_wp > 0 && !wps) || !n_seg || (samples && n_samples < 1)) { g_err = "bad argument"; return 1; }
  *n_seg = 0;
  return mplh::with_dim(dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    MPL::TrajSolver<Dim> solver(control, yaw_control);
    if (wp_control) {
      vec_E<Waypoint<Dim>> ws;
      for (int i = 0; i < n_wp; i++) ws.push_back(mplh::wp_from<Dim>(wps[i], wp_control[i]));
      solver.setWaypoints(ws);
    } else {
      vec_E<Vecf<Dim>> path(n_wp);
      for (int i = 0; i < n_wp; i++)
        for (int d = 0; d < Dim; d++) path[i](d) = wps[i].pos[d];
      solver.setPath(path);
    }
    if (dts && n_wp > 0) solver.setDts(std::vector<decimal_t>(dts, dts + (n_wp - 1)));
    solver.setV(v);
    const Trajectory<Dim> traj = solver.solve();
    *n_seg = (int32_t)traj.segs.size();
    const std::vector<decimal_t> used = solver.getDts();
    if (seg_t)
      for (std::size_t i = 0; i < used.size() && (int)i + 1 < n_wp; i++) seg_t[i] = used[i];
    if (coeff)
      for (std::size_t j = 0; j < traj.segs.size(); j++)
        for (int a = 0; a <= Dim; a++)
          for (int k = 0; k < 6; k++) coeff[(j * (Dim + 1) + a) * 6 + k] = (a < Dim ? traj.segs[j].pr(a) : traj.segs[j].pr_yaw()).c[k];
    if (samples) put_samples<Dim>(traj, n_samples, samples);
    if (waypoints) put_waypoints<Dim>(traj, waypoints);
  });
}

/* Trajectory<dim> of n_seg segments with durations seg_t and coefficients coeff (mplh_traj_solve's layout), each
 * segment with the control flag `control`: sample(n_samples) into samples and getWaypoints() into waypoints
 * (layouts as mplh_traj_solve's; either may be NULL). */
int mplh_traj_sample(int dim, int n_seg, const double *seg_t, const double *coeff, int control, int n_samples,
                     double *samples, double *waypoints) {
  if (n_seg < 0 || (n_seg > 0 && (!seg_t || !coeff)) || (samples && n_samples < 1)) { g_err = "bad argument"; return 1; }
  return mplh::with_dim(dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    const Trajectory<Dim> traj = make_trajectory<Dim>(n_seg, seg_t, coeff, control);
    if (samples) put_samples<Dim>(traj, n_samples, samples);
    if (waypoints) put_waypoints<Dim>(traj, waypoints);
  });
}
}

/* ---- Trajectory time scaling (mpl_host.hpp): one path on the host ------------------------------------------ */

namespace {
/// whether mplx_traj_check evaluates this path at all: at least one segment, every segment time finite and
/// > 0, every coefficient finite
template <int Dim>
bool checkable(int n_seg, const double *seg_t, const double *coeff) {
  if (n_seg < 1) return false;
  for (int j = 0; j < n_seg; j++)
    if (!(std::isfinite(seg_t[j]) && seg_t[j] > 0)) return false;
  for (size_t k = 0; k < (size_t)n_seg * (Dim + 1) * 6; k++)
    if (!std::isfinite(coeff[k])) return false;
  return true;
}

/// whether mplx_traj_scale would scale this path (status 1 or 2) rather than refuse it (status 0)
template <int Dim>
bool scalable(int n_seg, const double *seg_t, const double *coeff, int mode, double mv, double ri, double rf) {
  auto pos = [](double x) { return std::isfinite(x) && x > 0; };
  return pos(ri) && pos(rf) && (mode != MPLX_TRAJ_SCALE_DOWN || pos(mv)) && checkable<Dim>(n_seg, seg_t, coeff);
}
}  // namespace

extern "C" {
/* Trajectory<dim> of n_seg segments (mplh_traj_sample's inputs), then scale(ri, rf) (mode MPLX_TRAJ_SCALE) or
 * scale_down(mv, ri, rf) (MPLX_TRAJ_SCALE_DOWN), as mplx_traj_scale does it for one path.  Outputs (host arrays):
 *   *status    1 scaled, 2 scale_down returned false (unchanged), 0 not scaled: mplx_traj_scale's classes
 *   *total_t   getTotalTime() (0 for status 0)
 *   seg_T      [n_seg + 1] getSegmentTimes(), then 0 (all 0 for status 0)
 *   *n_lambda  lambda segments (NULL allowed)
 *   lambda     NULL or [(n_seg + 1) * 5 * dim * 7] {a3, a2, a1, a0, ti, tf, dT} per lambda segment, then zeros
 *   samples    NULL or [(n_samples + 1) * (4 dim + 3)] sample(n_samples) rows (zeros for status 0)
 * 1: bad argument (dim, mode, n_seg < 0, missing arrays, samples with n_samples < 1). */
int mplh_traj_scale(int dim, int n_seg, const double *seg_t, const double *coeff, int control, int mode, double mv,
                    double ri, double rf, int n_samples, int32_t *status, double *total_t, double *seg_T,
                    int32_t *n_lambda, double *lambda, double *samples) {
  if (n_seg < 0 || (n_seg > 0 && (!seg_t || !coeff)) || !status || !total_t || !seg_T || (samples && n_samples < 1) ||
      (mode != MPLX_TRAJ_SCALE && mode != MPLX_TRAJ_SCALE_DOWN)) {
    g_err = "bad argument";
    return 1;
  }
  return mplh::with_dim(dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    const size_t n_slot = (size_t)(n_seg + 1) * 5 * Dim;
    *status = 0;
    *total_t = 0;
    for (int j = 0; j <= n_seg; j++) seg_T[j] = 0;
    if (n_lambda) *n_lambda = 0;
    if (lambda) std::fill(lambda, lambda + n_slot * 7, 0.0);
    if (samples) std::fill(samples, samples + (size_t)(n_samples + 1) * (4 * Dim + 3), 0.0);
    if (!scalable<Dim>(n_seg, seg_t, coeff, mode, mv, ri, rf)) return;
    Trajectory<Dim> traj = make_trajectory<Dim>(n_seg, seg_t, coeff, control);
    const bool scaled = mode == MPLX_TRAJ_SCALE ? traj.scale(ri, rf) : traj.scale_down(mv, ri, rf);
    *status = scaled ? 1 : 2;
    *total_t = traj.getTotalTime();
    const std::vector<decimal_t> dts = traj.getSegmentTimes();
    for (int j = 0; j < n_seg; j++) seg_T[j] = dts[j];
    const auto &ls = traj.lambda().segs;
    if (ls.size() > n_slot) throw std::logic_error("lambda segments exceed their slots");
    if (n_lambda) *n_lambda = (int32_t)ls.size();
    if (lambda)
      for (size_t k = 0; k < ls.size(); k++) {
        double *o = lambda + k * 7;
        for (int i = 0; i < 4; i++) o[i] = ls[k].a[i];
        o[4] = ls[k].ti; o[5] = ls[k].tf; o[6] = ls[k].dT;
      }
    if (samples) put_samples<Dim>(traj, n_samples, samples);
  });
}

/* The closed-form root solver solve(a, b, c, d, e) (mpl_host.hpp): *n roots (at most 4) into roots. */
int mplh_solve(double a, double b, double c, double d, double e, int32_t *n, double *roots) {
  const std::vector<decimal_t> r = solve(a, b, c, d, e);
  *n = (int32_t)r.size();
  for (size_t k = 0; k < r.size() && k < 4; k++) roots[k] = r[k];
  return 0;
}
}

/* ---- Trajectory checks (mpl_host.hpp): env_map_host::traverse_trajectory, is_free, validate_primitive ------- */

namespace {
template <int Dim>
struct CheckEnv : MPL::env_map_host<Dim> {  // the map queries only: get_succ is never called
  using MPL::env_map_host<Dim>::env_map_host;
  void get_succ(const Waypoint<Dim> &, vec_E<Waypoint<Dim>> &, std::vector<decimal_t> &, std::vector<int> &) const override {}
};
}  // namespace

extern "C" {
/* mplx_traj_check on the host, the map and parameters given directly: the grid map[prod(mdim)] at origin with
 * resolution res, potential NULL or [prod(mdim)] with its two weights, region NULL or [prod(mdim)] search-region
 * bytes, and the limits.  The paths, control, total_t / n_lambda / lambda and the outputs are mplx_traj_check's
 * (slots as mplx_traj_out's; total_t, n_lambda and lambda all NULL or all given).  Paths are spread over
 * nthreads threads (< 1: one).  1: bad argument (dim, map, offset, missing arrays, n_lambda out of range). */
int mplh_traj_check(int dim, const int8_t *map, const int32_t *mdim, const double *origin, double res,
                    const int8_t *potential, double potential_weight, double gradient_weight, const uint8_t *region,
                    double v_max, double a_max, double j_max, double yaw_max, int n_paths, const int64_t *offset,
                    const double *seg_t, const double *coeff, const uint8_t *control, const double *total_t,
                    const int32_t *n_lambda, const double *lambda, int nthreads, int32_t *status, double *cost,
                    uint8_t *seg_free, uint8_t *seg_valid) {
  const bool scaled = lambda != nullptr;
  if (!map || !mdim || !origin || n_paths < 0 || !offset || offset[0] != 0 || !status || !cost ||
      (seg_valid && !control) || (total_t != nullptr) != scaled || (n_lambda != nullptr) != scaled) {
    g_err = "bad argument";
    return 1;
  }
  for (int p = 0; p < n_paths; p++)
    if (offset[p + 1] < offset[p] ||
        (scaled && (n_lambda[p] < 0 || n_lambda[p] > (offset[p + 1] - offset[p]) * 5 * dim))) {
      g_err = "bad argument";
      return 1;
    }
  if (offset[n_paths] > 0 && (!seg_t || !coeff)) { g_err = "bad argument"; return 1; }
  return mplh::with_dim(dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    auto mu = std::make_shared<MPL::MapUtil<Dim>>();
    Vecf<Dim> ori;
    Veci<Dim> md;
    size_t nvox = 1;
    for (int k = 0; k < Dim; k++) {
      ori(k) = origin[k];
      md(k) = mdim[k];
      nvox *= (size_t)mdim[k];
    }
    mu->setMap(ori, md, MPL::Tmap(map, map + nvox), res);
    CheckEnv<Dim> env(mu);
    env.set_v_max(v_max);
    env.set_a_max(a_max);
    env.set_j_max(j_max);
    env.set_yaw_max(yaw_max);
    if (potential) {
      env.set_potential_map(std::vector<int8_t>(potential, potential + nvox));
      env.set_potential_weight(potential_weight);
      env.set_gradient_weight(gradient_weight);
    }
    if (region) env.set_search_region(std::vector<bool>(region, region + nvox));
    const size_t NC = (size_t)5 * Dim;
    auto one = [&](int p) {
      const int64_t b = offset[p];
      const int W = (int)(offset[p + 1] - b), S = W - 1;
      status[p] = 0;
      cost[p] = 0;
      for (int j = 0; j < W; j++) {
        if (seg_free) seg_free[b + j] = 0;
        if (seg_valid) seg_valid[b + j] = 0;
      }
      if (!checkable<Dim>(S, seg_t + b, coeff + b * (Dim + 1) * 6)) return;
      Trajectory<Dim> traj =
          make_trajectory<Dim>(S, seg_t + b, coeff + b * (Dim + 1) * 6, control ? control[p] : Control::NONE);
      if (scaled && n_lambda[p] > 0) {
        Lambda lam;
        for (int k = 0; k < n_lambda[p]; k++) {
          const double *r = lambda + ((size_t)b * NC + k) * 7;
          LambdaSeg g;
          for (int i = 0; i < 4; i++) g.a[i] = r[i];
          g.ti = r[4]; g.tf = r[5]; g.dT = r[6];
          lam.segs.push_back(g);
        }
        traj.set_lambda(lam, total_t[p]);
      }
      if (env.traverse_samples(traj) > 0) {
        status[p] = 1;
        cost[p] = env.traverse_trajectory(traj);
      }
      for (int j = 0; j < S; j++) {
        if (seg_free) seg_free[b + j] = env.is_free(traj.segs[j]) ? 1 : 0;
        if (seg_valid) seg_valid[b + j] = validate_primitive(traj.segs[j], v_max, a_max, j_max, yaw_max) ? 1 : 0;
      }
    };
    const int nt = std::max(1, std::min(nthreads, n_paths));
    std::atomic<int> next{0};
    std::vector<std::thread> pool;
    for (int t = 1; t < nt; t++)
      pool.emplace_back([&] { for (int p; (p = next++) < n_paths;) one(p); });
    for (int p; (p = next++) < n_paths;) one(p);
    for (auto &th : pool) th.join();
  });
}
}
