// integration/env_map_b200.h — the reference-side binding of libmplx.so, as INTEGRATION.md §1 lists it.
//
// Compiled in this repository against the UNMODIFIED reference headers (oracle/Makefile, target
// _ref/libmplref_b200.so: -I /root/reference/include) and exercised by tests/test_integration_gpu.py:
// the reference's own GraphSearch::Astar / PlannerBase::plan drive this env, and the closed sets must
// equal the ones the reference's env_map produces.
#pragma once
#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <vector>

#include <mpl_planner/env/env_map.h>
#include <mplx.h>

namespace MPL {
template <int Dim>
class env_map_b200 : public env_map<Dim> {
 public:
  explicit env_map_b200(std::shared_ptr<MapUtil<Dim>> mu, int device = 0) : env_map<Dim>(mu) {
    if (mplx_create(Dim, device, &ctx_)) throw std::runtime_error(mplx_last_error());  // no CPU fallback
    upload_map();
  }
  ~env_map_b200() { mplx_destroy(ctx_); }

  // MapUtil is shared by pointer and can change behind the env (setMap, updatePotentialMap
  // overwrites it: map_planner.cpp:387): call after any change, or from plan().
  void upload_map() {
    const auto dim = this->map_util_->getDim();
    const auto ori = this->map_util_->getOrigin();
    const Tmap m = this->map_util_->getMap();
    check(mplx_set_map(ctx_, m.data(), dim.data(), ori.data(), this->map_util_->getRes()));
    if (!this->potential_map_.empty())
      check(mplx_set_potential(ctx_, this->potential_map_.data(), this->potential_weight_, this->gradient_weight_));
    if (!this->search_region_.empty()) {
      std::vector<uint8_t> r(this->search_region_.begin(), this->search_region_.end());
      check(mplx_set_search_region(ctx_, r.data()));
    }
    params_dirty_ = true;
  }

  // batched body of get_succ: the seam the speculative / multi-query drivers use
  void get_succ_batch(const vec_E<Waypoint<Dim>>& nodes, std::vector<int32_t>& count,
                      std::vector<mplx_waypoint>& succ, std::vector<double>& cost, std::vector<int32_t>& action,
                      std::vector<uint64_t>& key) const {
    sync_params(nodes.front().control);
    const int nU = (int)this->U_.size(), n = (int)nodes.size();
    std::vector<mplx_waypoint> in(n);
    for (int i = 0; i < n; i++) to_pod(nodes[i], in[i]);
    count.resize(n); succ.resize((size_t)n * nU); cost.resize((size_t)n * nU);
    action.resize((size_t)n * nU); key.resize((size_t)n * nU);
    mplx_succ_out out{count.data(), succ.data(), cost.data(), action.data(), key.data(), nullptr};
    check(mplx_expand(ctx_, in.data(), n, &out));
  }

  // the reference's virtual (env_base.h:358-362): one node, same outputs, same order
  void get_succ(const Waypoint<Dim>& curr, vec_E<Waypoint<Dim>>& succ, std::vector<decimal_t>& succ_cost,
                std::vector<int>& action_idx) const override {
    succ.clear(); succ_cost.clear(); action_idx.clear();
    this->expanded_nodes_.push_back(curr.pos);                    // env_map.h:154
    std::vector<int32_t> cnt, act; std::vector<mplx_waypoint> s; std::vector<double> c; std::vector<uint64_t> k;
    get_succ_batch({curr}, cnt, s, c, act, k);
    for (int j = 0; j < cnt[0]; j++) {
      Waypoint<Dim> tn(curr.control);                             // primitive.h:322 (flags follow curr)
      for (int d = 0; d < Dim; d++) { tn.pos(d) = s[j].pos[d]; tn.vel(d) = s[j].vel[d];
                                      tn.acc(d) = s[j].acc[d]; tn.jrk(d) = s[j].jrk[d]; }
      tn.yaw = s[j].yaw; tn.t = s[j].t;
      succ.push_back(tn); succ_cost.push_back(c[j]); action_idx.push_back(act[j]);
      if (!std::isinf(c[j])) {                                    // env_map.h:164-167, rebuilt lazily
        Primitive<Dim> pr; this->forward_action(curr, act[j], pr); this->expanded_edges_.push_back(pr);
      }
    }
  }

 private:
  void sync_params(Control::Control control) const {
    if (!params_dirty_ && control == control_) return;
    const int udim = (int)this->U_.front().size();
    std::vector<double> U; for (const auto& u : this->U_) for (int k = 0; k < udim; k++) U.push_back(u(k));
    check(mplx_set_params(ctx_, control, this->dt_, this->w_, this->wyaw_, this->v_max_, this->a_max_, this->j_max_,
                          this->yaw_max_, U.data(), (int)this->U_.size(), udim));
    control_ = control; params_dirty_ = false;
  }
  static void to_pod(const Waypoint<Dim>& w, mplx_waypoint& p) {
    p = mplx_waypoint{};
    for (int d = 0; d < Dim; d++) { p.pos[d] = w.pos(d); p.vel[d] = w.vel(d); p.acc[d] = w.acc(d); p.jrk[d] = w.jrk(d); }
    p.yaw = w.yaw; p.t = w.t;
  }
  static void check(int rc) { if (rc) throw std::runtime_error(mplx_last_error()); }
  mplx_ctx* ctx_ = nullptr;
  mutable bool params_dirty_ = true;
  mutable Control::Control control_ = Control::NONE;
};
}  // namespace MPL

namespace MPL {
/// MapPlanner whose virtual setMapUtil (map_planner.h:29, map_planner.cpp:14-18) installs the GPU env:
/// the drop-in that needs no edit of the reference's sources.
template <int Dim>
class MapPlannerB200 : public MapPlanner<Dim> {
 public:
  explicit MapPlannerB200(bool verbose, int device = 0) : MapPlanner<Dim>(verbose), device_(device) {}
  void setMapUtil(const std::shared_ptr<MapUtil<Dim>>& map_util) override {
    this->ENV_.reset(new env_map_b200<Dim>(map_util, device_));
    this->map_util_ = map_util;
  }

 private:
  int device_;
};
}  // namespace MPL
