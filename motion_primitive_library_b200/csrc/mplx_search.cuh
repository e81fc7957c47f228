// mplx_search.cuh — the bookkeeping of one A* query (the heap, the key table, the predecessor lists,
// the relax step, the goal test and the trace-back) as plain __host__ __device__ code over a flat
// arena.  The device search (mplx_search.cu) runs it in thread 0 of a CTA; g++ compiles the same
// header for the CPU test of the bookkeeping.  Every operation restates the host planner
// (host/mpl_host.hpp) step by step, so a query gives what AstarStepper gives:
//   PriorityQueue      mpl_host.hpp:1050-1102  (the same swaps and heap_idx updates)
//   AstarStepper       mpl_host.hpp:1449-1518  (start / pop / consume / finish)
//   recoverTraj        mpl_host.hpp:1392-1433 (with its best_child_ chain)
//   env_map_host       mpl_host.hpp:572-587    (is_goal with the walkRay test, is_free)
//   env_base           mpl_host.hpp:460-474    (get_heur / cal_heur)
// Plain IEEE operations only (the library builds with -fmad=false; the CPU test with
// -ffp-contract=off).  This header depends on nothing but mplx.h and <math.h>.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/mplx.h"

#ifdef __CUDACC__
#define MPLX_HD __host__ __device__ __forceinline__
#else
#define MPLX_HD inline
#endif

namespace mplx {
namespace search {

enum : uint32_t { kOpened = 1u, kClosed = 2u };
// kOverflow: the query needed more states or predecessor records than its arena holds (only with the
// capacity check, consume<true>); the search is abandoned and nothing of it is a result.
enum Status : int { kIdle = 0, kRunning = 1, kTrivial = 2, kGoal = 3, kFailed = 4, kOverflow = 5 };

// State<Dim> (mpl_host.hpp:1017-1043) without the LPA* members: rhs is never set by A*, so the
// comparator's min(g, rhs) is g.
struct SState {
  mplx_waypoint coord;
  double g, h;
  uint64_t key;
  int32_t heap_idx, pred_head, pred_tail;
  uint32_t flags;
};
// one predecessor record; the records of a state form a list in insertion order
struct SPred {
  int32_t node, action, next, pad;
  double cost;
};
struct SHeapItem {
  double f;
  int32_t state, pad;
};
// key table entry: valid only while `epoch` is the query's (no clearing between queries)
struct SSlot {
  uint64_t key;
  uint32_t state, epoch;
};

// An arena of cap states, as many predecessor records and heap entries, and a power-of-two key table
// at most half full.
struct Layout {
  int64_t cap;  // states = predecessor records = heap entries
  int64_t tab;  // key table entries (power of two >= 2*cap)
  int64_t off_pred, off_heap, off_tab, bytes;
};
MPLX_HD Layout layout_cap(int64_t cap) {
  Layout L;
  L.cap = cap;
  L.tab = 1;
  while (L.tab < 2 * L.cap) L.tab <<= 1;
  const int64_t st = (L.cap * (int64_t)sizeof(SState) + 255) & ~(int64_t)255;
  const int64_t pr = (L.cap * (int64_t)sizeof(SPred) + 255) & ~(int64_t)255;
  const int64_t hp = (L.cap * (int64_t)sizeof(SHeapItem) + 255) & ~(int64_t)255;
  L.off_pred = st;
  L.off_heap = st + pr;
  L.off_tab = st + pr + hp;
  L.bytes = L.off_tab + L.tab * (int64_t)sizeof(SSlot);
  return L;
}
// The worst case of one query: 1 + max_expand*nU states (one per finite successor and the start), so no
// query of a search capped at max_expand expansions can overflow it.
MPLX_HD Layout layout_for(int max_expand, int nU) { return layout_cap(1 + (int64_t)max_expand * nU); }

struct Arena {
  SState *st;
  SPred *pr;
  SHeapItem *hp;
  SSlot *tab;
  uint32_t tmask, epoch;
  int32_t n_states, n_preds, heap_n;
  int32_t cap;  // states = predecessor records the arena holds (read by the capacity check only)
};
MPLX_HD Arena arena_at(unsigned char *base, const Layout &L, uint32_t epoch) {
  Arena A;
  A.st = reinterpret_cast<SState *>(base);
  A.pr = reinterpret_cast<SPred *>(base + L.off_pred);
  A.hp = reinterpret_cast<SHeapItem *>(base + L.off_heap);
  A.tab = reinterpret_cast<SSlot *>(base + L.off_tab);
  A.tmask = (uint32_t)(L.tab - 1);
  A.epoch = epoch;
  A.n_states = A.n_preds = A.heap_n = 0;
  A.cap = (int32_t)L.cap;
  return A;
}

// ---- PriorityQueue (mpl_host.hpp:1050-1102) ----------------------------------------------------
// compare_pair: true when a has LOWER priority than b; key ties broken on the states' current g
MPLX_HD bool lower(const Arena &A, const SHeapItem &a, const SHeapItem &b) {
  if (a.f == b.f) return A.st[a.state].g > A.st[b.state].g;
  return a.f > b.f;
}
MPLX_HD void swap_at(Arena &A, int a, int b) {
  const SHeapItem t = A.hp[a];
  A.hp[a] = A.hp[b];
  A.hp[b] = t;
  A.st[A.hp[a].state].heap_idx = a;
  A.st[A.hp[b].state].heap_idx = b;
}
MPLX_HD void siftup(Arena &A, int i) {
  while (i != 0) {
    const int p = (i - 1) / 2;
    if (lower(A, A.hp[p], A.hp[i])) {
      swap_at(A, p, i);
      i = p;
    } else
      return;
  }
}
MPLX_HD void siftdown(Arena &A, int i) {
  const int n = A.heap_n;
  while (2 * i + 1 < n) {
    int c = 2 * i + 1;
    if (c + 1 < n && lower(A, A.hp[c], A.hp[c + 1])) c = c + 1;
    if (!lower(A, A.hp[c], A.hp[i])) {
      swap_at(A, c, i);
      i = c;
    } else
      return;
  }
}
MPLX_HD void heap_push(Arena &A, double f, int s) {
  A.st[s].heap_idx = A.heap_n;
  A.hp[A.heap_n].f = f;
  A.hp[A.heap_n].state = s;
  A.hp[A.heap_n].pad = 0;
  A.heap_n++;
  siftup(A, A.st[s].heap_idx);
}
MPLX_HD void heap_pop(Arena &A) {
  swap_at(A, 0, A.heap_n - 1);
  A.st[A.hp[A.heap_n - 1].state].heap_idx = -1;
  A.heap_n--;
  if (A.heap_n != 0) siftdown(A, 0);
}
MPLX_HD void heap_increase(Arena &A, int s, double f) {
  A.hp[A.st[s].heap_idx].f = f;
  siftup(A, A.st[s].heap_idx);
}

// ---- key table (the state space's hash map) ------------------------------------------------------
MPLX_HD uint32_t slot_of(const Arena &A, uint64_t k) {
  return (uint32_t)((k * 0x9e3779b97f4a7c15ULL) >> 20) & A.tmask;
}
// the state of key k, or a new one (coordinates left to the caller) when absent.  CHECK: -1, with
// nothing changed, when a new state would pass the arena's capacity.
template <bool CHECK = false>
MPLX_HD int get_or_make(Arena &A, uint64_t k, bool &created) {
  for (uint32_t i = slot_of(A, k);; i = (i + 1) & A.tmask) {
    SSlot &e = A.tab[i];
    if (e.epoch != A.epoch) {
      if (CHECK && A.n_states >= A.cap) return -1;
      const int s = A.n_states++;
      e.key = k;
      e.state = (uint32_t)s;
      e.epoch = A.epoch;
      SState &n = A.st[s];
      n.g = INFINITY;
      n.h = INFINITY;
      n.key = k;
      n.heap_idx = -1;
      n.pred_head = n.pred_tail = -1;
      n.flags = 0;
      created = true;
      return s;
    }
    if (e.key == k) {
      created = false;
      return (int)e.state;
    }
  }
}

// ---- env_map_host goal test, free test and heuristic ------------------------------------------
struct Grid {
  const int8_t *map;
  int dim;
  int mdim[3];
  double origin[3];
  double res;
};
struct Goal {
  mplx_waypoint w;
  uint64_t key;
  double tol_pos, tol_vel, tol_acc, tol_yaw;
  double w_heur, v_max;
};

// Vecf::lpNormInf (mpl_host.hpp:60): m = std::max(m, |d_i|) from 0
MPLX_HD double linf(int dim, const double *a, const double *b) {
  double m = 0;
  for (int i = 0; i < dim; i++) {
    const double x = fabs(a[i] - b[i]);
    m = (m < x) ? x : m;
  }
  return m;
}
// MapUtil::floatToInt (mpl_host.hpp:388-392)
MPLX_HD int float_to_int(const Grid &G, double p, int k) { return (int)round((p - G.origin[k]) / G.res - 0.5); }
MPLX_HD bool outside(const Grid &G, const int *pn) {
  for (int i = 0; i < G.dim; i++)
    if (pn[i] < 0 || pn[i] >= G.mdim[i]) return true;
  return false;
}
MPLX_HD int64_t index_of(const Grid &G, const int *pn) {
  return G.dim == 2 ? (int64_t)pn[0] + (int64_t)G.mdim[0] * pn[1]
                    : (int64_t)pn[0] + (int64_t)G.mdim[0] * pn[1] + (int64_t)G.mdim[0] * G.mdim[1] * pn[2];
}
// env_map_host::is_free (mpl_host.hpp:587) = MapUtil::isFree(floatToInt(pt)) (:338,344)
MPLX_HD bool is_free(const Grid &G, const double *pos) {
  int pn[3] = {0, 0, 0};
  for (int k = 0; k < G.dim; k++) pn[k] = float_to_int(G, pos[k], k);
  if (outside(G, pn)) return false;
  const int v = G.map[index_of(G, pn)];
  return v < 100 && v >= 0;
}
// MapUtil::walkRay (mpl_host.hpp:400-416) with the visitor of is_goal (:579-582): true when no cell
// the ray reports is occupied
MPLX_HD bool ray_clear(const Grid &G, const double *p1, const double *p2) {
  double span[3], m = 0;
  for (int k = 0; k < G.dim; k++) {
    span[k] = p2[k] - p1[k];
    const double x = fabs(span[k] / G.res);
    m = (m < x) ? x : m;
  }
  const int steps = (int)(m / 0.8);
  double inc[3];
  for (int k = 0; k < G.dim; k++) inc[k] = span[k] * (1.0 / steps);
  bool have_last = false;
  int last[3] = {0, 0, 0};
  for (int i = 1; i < steps; i++) {
    int cell[3] = {0, 0, 0};
    for (int k = 0; k < G.dim; k++) cell[k] = float_to_int(G, p1[k] + inc[k] * (double)i, k);
    if (outside(G, cell)) return true;
    bool differs = !have_last;
    for (int k = 0; k < G.dim; k++) differs = differs || cell[k] != last[k];
    if (differs && G.map[index_of(G, cell)] == 100) return false;
    for (int k = 0; k < G.dim; k++) last[k] = cell[k];
    have_last = true;
  }
  return true;
}
// One segment of MapPlanner::setSearchRegion's ray trace (map_planner.cpp:49-58, MapUtil::rayTrace map_util.h:120-137),
// the samples ray_clear walks: the cell of each sample p1 + (diff·s)·n, n = 1 .. max_diff - 1, that differs from the
// one before, up to the first outside the map, then p2's cell.  emit(i, cell) receives the i-th of them (z = 0 in
// 2-D); returns their number.  G.map is not read.  emit may be host-only where the walk runs on the host.
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <typename Emit>
MPLX_HD int segment_cells(const Grid &G, const double *p1, const double *p2, Emit emit) {
  double diff[3] = {0, 0, 0}, m = 0;
  for (int k = 0; k < G.dim; k++) {
    diff[k] = p2[k] - p1[k];
    const double x = fabs(diff[k] / G.res);
    m = (m < x) ? x : m;
  }
  const int max_diff = (int)(m / 0.8);
  const double s = 1.0 / max_diff;
  int n_out = 0;
  int prev[3] = {-1, -1, -1};
  for (int n = 1; n < max_diff; n++) {
    int pn[3] = {0, 0, 0};
    for (int k = 0; k < G.dim; k++) pn[k] = float_to_int(G, p1[k] + (diff[k] * s) * (double)n, k);
    if (outside(G, pn)) break;
    bool differs = false;
    for (int k = 0; k < G.dim; k++) differs = differs || pn[k] != prev[k];
    if (differs) emit(n_out++, pn);
    for (int k = 0; k < 3; k++) prev[k] = pn[k];
  }
  int pe[3] = {0, 0, 0};
  for (int k = 0; k < G.dim; k++) pe[k] = float_to_int(G, p2[k], k);
  emit(n_out++, pe);
  return n_out;
}
// env_map_host::is_goal (mpl_host.hpp:572-585)
MPLX_HD bool is_goal(const Grid &G, const Goal &Q, const mplx_waypoint &s) {
  bool goaled = linf(G.dim, s.pos, Q.w.pos) <= Q.tol_pos;
  if (goaled && Q.tol_vel >= 0) goaled = linf(G.dim, s.vel, Q.w.vel) <= Q.tol_vel;
  if (goaled && Q.tol_acc >= 0) goaled = linf(G.dim, s.acc, Q.w.acc) <= Q.tol_acc;
  if (goaled && Q.tol_yaw >= 0) goaled = fabs(s.yaw - Q.w.yaw) <= Q.tol_yaw;
  if (goaled) goaled = ray_clear(G, s.pos, Q.w.pos);
  return goaled;
}
// env_base::get_heur(state, key) (mpl_host.hpp:463-474): the goal's key short-circuits cal_heur
MPLX_HD double heur(const Grid &G, const Goal &Q, const mplx_waypoint &s, uint64_t key) {
  if (Q.key == key) return 0;
  if (Q.v_max > 0) return Q.w_heur * linf(G.dim, s.pos, Q.w.pos) / Q.v_max;
  return Q.w_heur * linf(G.dim, s.pos, Q.w.pos);
}

// ---- AstarStepper (mpl_host.hpp:1441-1530) -------------------------------------------------------
struct Query {
  int status, expanded, cur, max_expand;
  uint64_t start_key;
  double eps;
};

// planner_base.h:283-287 (a start that is not free is never started) + AstarStepper::start
MPLX_HD void begin(Arena &A, Query &S, const Grid &G, const Goal &Q, const mplx_waypoint &start, uint64_t start_key,
                   bool start_free, double eps, int max_expand) {
  S.status = kIdle;
  S.expanded = 0;
  S.cur = -1;
  S.max_expand = max_expand;
  S.start_key = start_key;
  S.eps = eps;
  if (!start_free) return;
  if (is_goal(G, Q, start)) {
    S.status = kTrivial;
    return;
  }
  bool created;
  const int n = get_or_make(A, start_key, created);
  A.st[n].coord = start;
  A.st[n].g = 0;
  A.st[n].h = eps == 0 ? 0 : heur(G, Q, start, start_key);
  heap_push(A, A.st[n].g + eps * A.st[n].h, n);
  A.st[n].flags = kOpened;
  S.status = kRunning;
}

// graph_search.h:64-68: the node this iteration expands
MPLX_HD int pop(Arena &A, Query &S) {
  S.expanded++;
  S.cur = A.hp[0].state;
  heap_pop(A);
  A.st[S.cur].flags |= kClosed;
  return S.cur;
}

// AstarStepper::consume (mpl_host.hpp:1479-1508) for the n successors of the popped node:
// key_at(s), cost_at(s), action_at(s), coord_at(s) describe successor s in control order.
// CHECK: a new state or predecessor record that would pass the arena's capacity ends the query with
// kOverflow.  States and records only ever grow, and the search never reads the capacity otherwise, so
// with cap >= need (the larger of the final state and record counts of the query in an unbounded arena)
// the query runs exactly as unchecked, and with cap < need it ends in kOverflow.  Heap entries never
// outnumber states.
template <bool CHECK = false, typename KeyAt, typename CostAt, typename ActAt, typename CoordAt>
MPLX_HD void consume(Arena &A, Query &S, const Grid &G, const Goal &Q, int n, KeyAt key_at, CostAt cost_at,
                     ActAt action_at, CoordAt coord_at) {
  const int cur = S.cur;
  for (int s = 0; s < n; ++s) {
    const double c = cost_at(s);
    if (isinf(c)) continue;
    const uint64_t k = key_at(s);
    bool created;
    const int sn = get_or_make<CHECK>(A, k, created);
    if (CHECK && (sn < 0 || A.n_preds >= A.cap)) {
      S.status = kOverflow;
      return;
    }
    if (created) {
      coord_at(s, A.st[sn].coord);
      A.st[sn].h = S.eps == 0 ? 0 : heur(G, Q, A.st[sn].coord, k);
    }
    // predecessor list: append
    const int p = A.n_preds++;
    A.pr[p].node = cur;
    A.pr[p].action = action_at(s);
    A.pr[p].cost = c;
    A.pr[p].next = -1;
    A.pr[p].pad = 0;
    if (A.st[sn].pred_tail < 0) A.st[sn].pred_head = p;
    else A.pr[A.st[sn].pred_tail].next = p;
    A.st[sn].pred_tail = p;
    const double tentative = A.st[cur].g + c;
    if (tentative < A.st[sn].g) {
      A.st[sn].g = tentative;
      const double fval = A.st[sn].g + S.eps * A.st[sn].h;
      const uint32_t fl = A.st[sn].flags;
      if ((fl & kOpened) && !(fl & kClosed)) {
        heap_increase(A, sn, fval);
      } else {
        heap_push(A, fval, sn);
        A.st[sn].flags = fl | kOpened;
      }
    }
  }
  if (is_goal(G, Q, A.st[cur].coord))
    S.status = kGoal;
  else if (S.max_expand > 0 && S.expanded >= S.max_expand)
    S.status = kFailed;
  else if (A.heap_n == 0)
    S.status = kFailed;
}

// AstarStepper::finish + recoverTraj (mpl_host.hpp:1392-1433, 1511-1518).  Writes the action ids
// from start to goal into actions[0, *n_actions) (at most cap; more sets *n_actions = -1) and
// returns the cost (+inf when no trajectory).  chain, when given, has room for cap + 1 state indices and
// receives the states the trace-back walked, recoverTraj's best_child_ from start to goal: *n_actions + 1
// of them when a trajectory is found (its contents are undefined otherwise).
MPLX_HD double finish(const Arena &A, const Query &S, int32_t *actions, int cap, int *n_actions,
                      int32_t *chain = nullptr) {
  *n_actions = 0;
  if (S.status == kTrivial) return 0;
  if (S.status != kGoal) return INFINITY;
  int curr = S.cur;
  int n = 0;
  bool found = false;
  if (chain) chain[0] = curr;
  for (int guard = 0; guard <= A.n_states && A.st[curr].pred_head >= 0; guard++) {
    int min_id = -1, min_node = -1;
    double min_rhs = INFINITY, min_g = INFINITY;
    for (int p = A.st[curr].pred_head; p >= 0; p = A.pr[p].next) {
      const double pg = A.st[A.pr[p].node].g;
      const double ac = A.pr[p].cost;
      if (min_rhs > pg + ac) {
        min_rhs = pg + ac;
        min_g = pg;
        min_id = p;
        min_node = A.pr[p].node;
      } else if (!isinf(ac) && min_rhs == pg + ac) {
        if (min_g < pg) {
          min_g = pg;
          min_id = p;
          min_node = A.pr[p].node;
        }
      }
    }
    if (min_id < 0) break;
    if (n < cap) actions[n] = A.pr[min_id].action;
    n++;
    curr = min_node;
    if (chain && n <= cap) chain[n] = curr;
    if (A.st[curr].key == S.start_key) {
      found = true;
      break;
    }
  }
  if (!found) return INFINITY;
  if (n > cap) {
    *n_actions = -1;
    return A.st[S.cur].g;
  }
  for (int i = 0, j = n - 1; i < j; i++, j--) {
    const int32_t t = actions[i];
    actions[i] = actions[j];
    actions[j] = t;
  }
  if (chain)
    for (int i = 0, j = n; i < j; i++, j--) {
      const int32_t t = chain[i];
      chain[i] = chain[j];
      chain[j] = t;
    }
  *n_actions = n;
  return A.st[S.cur].g;
}

}  // namespace search
}  // namespace mplx
