// The device search's trace-back (motion_primitive_library_b200/csrc/mplx_search.cuh, search::finish with its
// state chain) and the host planner's recoverTraj (host/mpl_host.hpp) on the same scripted search graph, compiled
// by g++.  TEST INFRASTRUCTURE: tests/test_batch_traj_cpu.py builds it into a shared library and compares the
// chain finish yields with recoverTraj's best_child_.
#include <cmath>
#include <memory>
#include <vector>

#include "../motion_primitive_library_b200/csrc/mplx_search.cuh"
#include "../motion_primitive_library_b200/host/mpl_host.hpp"

using namespace mplx::search;

// A graph of n states (g[i], key[i]) and np predecessor records (to[k] gets the record node[k], action[k],
// cost[k], in record order).  status: kGoal, kTrivial or kFailed; cur: the state the search ended on.
// Device side: finish() with an action buffer of `cap` entries and a chain of cap + 1 (the chain's two entries
// after that must keep the sentinel -7); writes dev_cost, dev_na, dev_actions[cap], dev_chain[cap + 3].
// Host side (only for kGoal): recoverTraj from state cur; writes host_found, host_na, host_actions and
// host_chain (best_child_ as state indices, host_nchain of them).
extern "C" int btj_trace(int n, const double *g, const uint64_t *key, int np, const int32_t *to, const int32_t *node,
                         const int32_t *action, const double *cost, int status, int cur, uint64_t start_key, int cap,
                         double *dev_cost, int32_t *dev_na, int32_t *dev_actions, int32_t *dev_chain,
                         int32_t *host_found, int32_t *host_na, int32_t *host_actions, int32_t *host_chain,
                         int32_t *host_nchain) {
  const Layout L = layout_cap(std::max(n, np) + 1);
  std::vector<unsigned char> mem((size_t)L.bytes + 256, 0);
  unsigned char *base = mem.data() + ((256 - ((uintptr_t)mem.data() & 255)) & 255);
  Arena A = arena_at(base, L, 1);
  for (int i = 0; i < n; i++) {
    bool created = false;
    const int s = get_or_make(A, key[i], created);
    if (!created || s != i) return 1;
    A.st[i].g = g[i];
  }
  for (int k = 0; k < np; k++) {
    const int p = A.n_preds++;
    A.pr[p].node = node[k];
    A.pr[p].action = action[k];
    A.pr[p].cost = cost[k];
    A.pr[p].next = -1;
    SState &t = A.st[to[k]];
    if (t.pred_tail < 0) t.pred_head = p;
    else A.pr[t.pred_tail].next = p;
    t.pred_tail = p;
  }
  Query S;
  S.status = status;
  S.cur = cur;
  S.start_key = start_key;
  S.expanded = 0;
  S.max_expand = 0;
  S.eps = 1;
  for (int i = 0; i < cap + 3; i++) dev_chain[i] = -7;
  int na = 0;
  *dev_cost = finish(A, S, dev_actions, cap, &na, dev_chain);
  *dev_na = na;

  *host_found = 0;
  *host_na = 0;
  *host_nchain = 0;
  if (status != kGoal) return 0;
  using HS = MPL::State<2>;
  std::vector<std::unique_ptr<HS>> hs;
  for (int i = 0; i < n; i++) {
    hs.emplace_back(new HS(Waypoint<2>(), (std::size_t)key[i]));
    hs.back()->g = g[i];
  }
  for (int k = 0; k < np; k++) hs[to[k]]->pred.push_back(HS::Pred{hs[node[k]].get(), cost[k], action[k]});
  MPL::StateSpace<2> ss(1.0);
  std::vector<MPL::Edge<2>> traj;
  *host_found = MPL::recoverTraj<2>(hs[cur].get(), ss, (std::size_t)start_key, traj) ? 1 : 0;
  *host_na = (int32_t)traj.size();
  for (std::size_t j = 0; j < traj.size(); j++) host_actions[j] = traj[j].action_id;
  for (const HS *p : ss.best_child_) {
    int idx = -1;
    for (int i = 0; i < n; i++)
      if (hs[i].get() == p) idx = i;
    host_chain[(*host_nchain)++] = idx;
  }
  return 0;
}
