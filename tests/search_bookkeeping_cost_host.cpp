// The device search's bookkeeping (motion_primitive_library_b200/csrc/mplx_search.cuh) compiled by g++ and
// driven on the CPU with successors from the oracle's get_succ, for the plans of mplx_plan_batch_cost_terms:
// the oracle env carries the potential map, the gradient weight, the search region and the yaw control, and
// the goal test takes tol_yaw.  TEST INFRASTRUCTURE: tests/test_device_search_cost_terms_gpu.py builds it into
// a shared library and compares every device query with it.
#include <string.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "../motion_primitive_library_b200/csrc/mplx_search.cuh"
#include "../oracle/mpl_oracle.h"

using namespace mplx::search;

static_assert(sizeof(orc_waypoint) == sizeof(mplx_waypoint), "one waypoint layout");

extern "C" int sbkc_plan(const orc_env *env, const mplx_waypoint *start, const mplx_waypoint *goal, double eps,
                         int max_expand, double tol_pos, double tol_vel, double tol_acc, double tol_yaw,
                         int32_t *valid, double *cost, int32_t *expanded, int32_t *n_closed, uint64_t *closed,
                         int32_t *actions, int32_t *n_actions) {
  if (max_expand <= 0) return 1;
  const Layout L = layout_for(max_expand, env->nU);
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
  Q.tol_yaw = tol_yaw;
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
    consume(
        A, S, G, Q, n, [&](int s) { return key[s]; }, [&](int s) { return c[s]; }, [&](int s) { return (int)act[s]; },
        [&](int s, mplx_waypoint &w) { memcpy(&w, &succ[s], sizeof w); });
  }
  int na = 0;
  *cost = finish(A, S, actions, max_expand, &na);
  *valid = std::isinf(*cost) ? 0 : 1;
  *expanded = S.expanded;
  *n_actions = na;
  int nc = 0;
  if (S.status != kIdle && S.status != kTrivial)
    for (int s = 0; s < A.n_states; s++)
      if (A.st[s].flags & kClosed) closed[nc++] = A.st[s].key;
  std::sort(closed, closed + nc);
  *n_closed = nc;
  return 0;
}
