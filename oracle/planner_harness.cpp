// planner_harness.cpp — TEST INFRASTRUCTURE.  The product's host planner (mpl_host.hpp:
// StateSpace, GraphSearch::Astar, MapPlanner::plan) driven by a CPU env whose get_succ is the
// ORACLE (orc_get_succ).  tests/test_planner_e2e_gpu.py runs the same plan through
// libmpl_host.so (GPU env) and requires identical closed sets, costs and action sequences.
#include "../motion_primitive_library_b200/host/plan_capi.hpp"
#include "mpl_oracle.h"

namespace {
template <int Dim>
class env_map_oracle : public MPL::env_map_host<Dim> {
 public:
  env_map_oracle(std::shared_ptr<MPL::MapUtil<Dim>> mu, const mplh_plan_args *a) : MPL::env_map_host<Dim>(mu), a_(a) {}
  void get_succ(const Waypoint<Dim> &curr, vec_E<Waypoint<Dim>> &succ, std::vector<decimal_t> &succ_cost,
                std::vector<int> &action_idx) const override {
    succ.clear(); succ_cost.clear(); action_idx.clear();
    this->expanded_nodes_.push_back(curr.pos);
    const auto t_in = std::chrono::steady_clock::now();
    struct Acc { double &s; std::chrono::steady_clock::time_point t0; ~Acc() { s += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); } } acc{seconds_in_get_succ, t_in};
    const orc_env e = env();
    const orc_waypoint c = pod(curr);
    std::vector<orc_waypoint> s(e.nU); std::vector<double> cost(e.nU); std::vector<int32_t> act(e.nU);
    keys_.resize(e.nU);
    const int n = orc_get_succ(&e, &c, s.data(), cost.data(), act.data(), (uint64_t *)keys_.data(), nullptr);
    for (int j = 0; j < n; j++) {
      Waypoint<Dim> w(curr.control);
      for (int d = 0; d < Dim; d++) { w.pos(d) = s[j].pos[d]; w.vel(d) = s[j].vel[d]; w.acc(d) = s[j].acc[d]; w.jrk(d) = s[j].jrk[d]; }
      w.yaw = s[j].yaw; w.t = s[j].t;
      succ.push_back(w); succ_cost.push_back(cost[j]); action_idx.push_back(act[j]);
    }
  }
  void is_free_edges(const vec_E<Waypoint<Dim>> &parents, const std::vector<int> &actions, std::vector<uint8_t> &free,
                     std::vector<decimal_t> &cost) const override {
    const orc_env e = env();
    std::vector<orc_waypoint> in(parents.size());
    for (std::size_t i = 0; i < parents.size(); i++) in[i] = pod(parents[i]);
    free.assign(parents.size(), 0);
    cost.assign(parents.size(), 0);
    orc_edges_is_free(&e, in.data(), actions.data(), (int)parents.size(), free.data(), cost.data());
  }
  void edge_cells(const vec_E<Waypoint<Dim>> &parents, const std::vector<int> &actions, std::vector<long long> &offset,
                  std::vector<int> &cells, std::vector<int> &table_voxel, std::vector<int> &table_edge) const override {
    table_voxel.clear(); table_edge.clear();  // the planner sorts on the host
    const orc_env e = env();
    std::vector<orc_waypoint> in(parents.size());
    for (std::size_t i = 0; i < parents.size(); i++) in[i] = pod(parents[i]);
    offset.assign(parents.size() + 1, 0);
    const int64_t total = orc_edges_cells(&e, in.data(), actions.data(), (int)parents.size(), (int64_t *)offset.data(), nullptr, 0);
    cells.assign((std::size_t)total * Dim, 0);
    orc_edges_cells(&e, in.data(), actions.data(), (int)parents.size(), (int64_t *)offset.data(), cells.data(), total);
  }

  /// MapPlanner::setSearchRegion (src/mpl_planner/map_planner.cpp:46-95) restated on the CPU for the checker env
  void search_region_from_path(const vec_E<Vecf<Dim>> &path, const Vecf<Dim> &radius, bool dense) override {
    auto &mu = *this->map_util_;
    vec_E<Veci<Dim>> ps;
    if (!dense) {
      for (unsigned int i = 1; i < path.size(); i++) {
        auto pns = mu.rayTrace(path[i - 1], path[i]);
        ps.insert(ps.end(), pns.begin(), pns.end());
        ps.push_back(mu.floatToInt(path[i]));
      }
    } else {
      for (const auto &pt : path) ps.push_back(mu.floatToInt(pt));
    }
    int rn[3] = {0, 0, 0};
    for (int i = 0; i < Dim; i++) rn[i] = (int)std::ceil(radius(i) / mu.getRes());
    const Veci<Dim> dim = mu.getDim();
    std::size_t nvox = 1;
    for (int i = 0; i < Dim; i++) nvox *= (std::size_t)dim(i);
    std::vector<bool> in_region(nvox, false);
    for (const auto &it : ps)
      for (int dx = -rn[0]; dx <= rn[0]; dx++)
        for (int dy = -rn[1]; dy <= rn[1]; dy++)
          for (int dz = -rn[2]; dz <= rn[2]; dz++) {
            Veci<Dim> pn = it;
            pn(0) += dx; pn(1) += dy;
            if (Dim == 3) pn(Dim - 1) += dz;
            if (mu.isOutside(pn)) continue;
            in_region[mu.getIndex(pn)] = true;
          }
    this->set_search_region(in_region);
    region_bytes_.assign(in_region.begin(), in_region.end());
  }
  /// like the GPU env, the oracle hands the successors' lattice keys back with them
  const std::size_t *last_succ_keys() const override { return keys_.data(); }
  mutable std::vector<std::size_t> keys_;
  std::vector<uint8_t> region_bytes_;  // search_region_ as one byte per voxel for orc_env
  /// wall time spent inside get_succ (the oracle), so a caller can split plan() into env and bookkeeping
  mutable double seconds_in_get_succ = 0;

 private:
  static orc_waypoint pod(const Waypoint<Dim> &w) {
    orc_waypoint c{};
    for (int d = 0; d < Dim; d++) { c.pos[d] = w.pos(d); c.vel[d] = w.vel(d); c.acc[d] = w.acc(d); c.jrk[d] = w.jrk(d); }
    c.yaw = w.yaw; c.t = w.t;
    return c;
  }
  // the env reads the planner's CURRENT map (it changes between the steps of an LPA* session)
  orc_env env() const {
    orc_env e{};
    e.dim = Dim; e.control = a_->control; e.T = this->dt_; e.w = this->w_; e.wyaw = this->wyaw_;
    e.v_max = this->v_max_; e.a_max = this->a_max_; e.j_max = this->j_max_; e.yaw_max = this->yaw_max_;
    e.nU = a_->nU; e.udim = a_->udim; e.U = a_->U;
    for (int k = 0; k < 3; k++) { e.mdim[k] = k < Dim ? a_->mdim[k] : 1; e.origin[k] = k < Dim ? a_->origin[k] : 0; }
    e.res = a_->res; e.map = (const int8_t *)this->map_util_->map().data(); e.potential = a_->potential;
    e.potential_weight = a_->potential_weight; e.gradient_weight = a_->gradient_weight;
    e.region = region_bytes_.empty() ? nullptr : region_bytes_.data();
    return e;
  }
  const mplh_plan_args *a_;
};
}  // namespace

// the message of the last failed orcp_* call, under the host library's name so the same bindings read it
static thread_local std::string g_err;
extern "C" const char *mplh_last_error(void) { return g_err.c_str(); }

extern "C" int orcp_lpa_run(const mplh_plan_args *a, const mplh_lpa_step *steps, int n_steps, mplh_lpa_out *outs,
                            int32_t *actions, int cap_actions) {
  return mplh::with_dim(a->dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    MPL::MapPlanner<Dim> planner(false);
    auto mu = mplh::make_map<Dim>(a);
    planner.setEnv(std::make_shared<env_map_oracle<Dim>>(mu, a), mu);
    mplh::run_lpa<Dim>(planner, mu, a, steps, n_steps, outs, actions, cap_actions);
  });
}

extern "C" int orcp_plan(const mplh_plan_args *a, mplh_plan_result *r, uint64_t *closed_keys, int cap_closed,
                         int32_t *actions, int cap_actions) {
  *r = mplh_plan_result{};
  return mplh::with_dim(a->dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    MPL::MapPlanner<Dim> planner(false);
    auto env = std::make_shared<env_map_oracle<Dim>>(mplh::make_map<Dim>(a), a);
    planner.setEnv(env);
    mplh::run<Dim>(planner, a, r, closed_keys, cap_closed, actions, cap_actions);
    if (std::getenv("ORCP_TRACE"))
      std::fprintf(stderr, "[orcp_plan] plan %.1f ms: get_succ (oracle) %.1f ms, host bookkeeping %.1f ms, %d expansions, %d closed + %d open states\n",
                   r->seconds * 1e3, env->seconds_in_get_succ * 1e3, (r->seconds - env->seconds_in_get_succ) * 1e3, r->expanded,
                   r->n_closed, r->n_open);
  });
}

extern "C" int orcp_iterative_plan(const mplh_plan_args *a, const double *search_radius, int max_iter,
                                   mplh_plan_result *first, mplh_plan_result *last, int32_t *info, uint64_t *closed_keys,
                                   int cap_closed, int32_t *actions, int cap_actions) {
  *first = mplh_plan_result{};
  *last = mplh_plan_result{};
  return mplh::with_dim(a->dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    MPL::MapPlanner<Dim> planner(false);
    auto mu = mplh::make_map<Dim>(a);
    planner.setEnv(std::make_shared<env_map_oracle<Dim>>(mu, a), mu);
    mplh::run_iterative<Dim>(planner, a, search_radius, max_iter, first, last, info, closed_keys, cap_closed, actions,
                             cap_actions);
  });
}

extern "C" int orcp_plan_trajectory(const mplh_plan_args *a, int N, mplh_plan_result *r, double *samples, double *totals,
                                    double *waypoints, int cap_wp, int32_t *n_wp, double *mids) {
  *r = mplh_plan_result{};
  return mplh::with_dim(a->dim, g_err, 2, [&](auto dimtag) {
    constexpr int Dim = decltype(dimtag)::value;
    MPL::MapPlanner<Dim> planner(false);
    auto mu = mplh::make_map<Dim>(a);
    planner.setEnv(std::make_shared<env_map_oracle<Dim>>(mu, a), mu);
    mplh::run_trajectory<Dim>(planner, a, N, r, samples, totals, waypoints, cap_wp, n_wp, mids);
  });
}
