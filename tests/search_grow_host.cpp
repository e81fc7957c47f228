// The capacity check of the device search's bookkeeping (motion_primitive_library_b200/csrc/mplx_search.cuh,
// consume<true>) compiled by g++ and driven on the CPU with successors from the oracle's get_succ.  TEST
// INFRASTRUCTURE: tests/test_search_grow_cpu.py builds it into a shared library, runs each query in a large
// arena for its result and its need, and then at capacities around the need.
#include <string.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "../motion_primitive_library_b200/csrc/mplx_search.cuh"
#include "../oracle/mpl_oracle.h"

using namespace mplx::search;

static_assert(sizeof(orc_waypoint) == sizeof(mplx_waypoint), "one waypoint layout");

// One A* query (max_expand <= 0: unbounded) in an arena of `cap` states and predecessor records.
// *status receives the final status (kOverflow when the query outgrew the arena).  Only a query that did
// not overflow writes the other outputs: *need = max(states, predecessor records) it used, and its result
// (closed keys sorted, at most closed_cap; actions at most act_cap).
extern "C" int sgr_plan(const orc_env *env, const mplx_waypoint *start, const mplx_waypoint *goal, double eps,
                        int max_expand, int64_t cap, double tol_pos, double tol_vel, double tol_acc, int32_t *status,
                        int64_t *need, int32_t *valid, double *cost, int32_t *expanded, int32_t *n_closed,
                        uint64_t *closed, int64_t closed_cap, int32_t *actions, int64_t act_cap, int32_t *n_actions) {
  if (cap < 1) return 1;
  const Layout L = layout_cap(cap);
  std::vector<unsigned char> mem((size_t)L.bytes + 256, 0);
  unsigned char *base = mem.data() + ((256 - ((uintptr_t)mem.data() & 255)) & 255);
  Arena A = arena_at(base, L, 1);
  Grid G;
  G.map = env->map;
  G.dim = env->dim;
  for (int k = 0; k < 3; k++) {
    G.mdim[k] = env->mdim[k];
    G.origin[k] = env->origin[k];
  }
  G.res = env->res;
  Goal Q;
  Q.w = *goal;
  Q.key = orc_hash(env, (const orc_waypoint *)goal, nullptr, nullptr);
  Q.tol_pos = tol_pos;
  Q.tol_vel = tol_vel;
  Q.tol_acc = tol_acc;
  Q.tol_yaw = -1;
  Q.w_heur = env->w;
  Q.v_max = env->v_max;
  Query S;
  begin(A, S, G, Q, *start, orc_hash(env, (const orc_waypoint *)start, nullptr, nullptr), is_free(G, start->pos), eps,
        max_expand);
  std::vector<orc_waypoint> succ(env->nU);
  std::vector<double> c(env->nU);
  std::vector<int32_t> act(env->nU);
  std::vector<uint64_t> key(env->nU);
  while (S.status == kRunning) {
    const int cur = pop(A, S);
    orc_waypoint node;
    memcpy(&node, &A.st[cur].coord, sizeof node);
    const int n = orc_get_succ(env, &node, succ.data(), c.data(), act.data(), key.data(), nullptr);
    consume<true>(
        A, S, G, Q, n, [&](int s) { return key[s]; }, [&](int s) { return c[s]; }, [&](int s) { return (int)act[s]; },
        [&](int s, mplx_waypoint &w) { memcpy(&w, &succ[s], sizeof w); });
  }
  *status = S.status;
  if (S.status == kOverflow) return 0;
  *need = std::max(A.n_states, A.n_preds);
  int na = 0;
  *cost = finish(A, S, actions, (int)std::min<int64_t>(act_cap, 1 << 30), &na);
  *valid = std::isinf(*cost) ? 0 : 1;
  *expanded = S.expanded;
  *n_actions = na;
  std::vector<uint64_t> keys;
  if (S.status != kIdle && S.status != kTrivial)
    for (int s = 0; s < A.n_states; s++)
      if (A.st[s].flags & kClosed) keys.push_back(A.st[s].key);
  std::sort(keys.begin(), keys.end());
  std::copy(keys.begin(), keys.begin() + std::min<int64_t>((int64_t)keys.size(), closed_cap), closed);
  *n_closed = (int)keys.size();
  return 0;
}

// layout_for and layout_cap as the device computes them: {cap, tab, off_pred, off_heap, off_tab, bytes}
extern "C" void sgr_layout_for(int max_expand, int nU, int64_t *out) {
  const Layout L = layout_for(max_expand, nU);
  const int64_t v[6] = {L.cap, L.tab, L.off_pred, L.off_heap, L.off_tab, L.bytes};
  memcpy(out, v, sizeof v);
}
extern "C" void sgr_layout_cap(int64_t cap, int64_t *out) {
  const Layout L = layout_cap(cap);
  const int64_t v[6] = {L.cap, L.tab, L.off_pred, L.off_heap, L.off_tab, L.bytes};
  memcpy(out, v, sizeof v);
}
