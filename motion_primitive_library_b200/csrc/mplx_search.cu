// mplx_search.cu — mplx_plan_batch: the A* searches of a multi-query batch run on the device.
//
// One CTA runs one query's whole A* at a time and takes its next query from a global counter when the
// current one ends (persistent CTAs, one per arena slot).  Per iteration:
//   thread 0     pops the best open state and copies its coordinates to shared memory;
//   all threads  expand it: phase A/B of the expansion kernels (phase_ab, mplx_expand.cuh) gives the
//                successors in control order with their keys, and each thread runs the sample loop of
//                its primitive (traverse_groups) for the edge cost;
//   thread 0     relaxes the successors, tests the goal and the limits (mplx_search.cuh).
// So there is no launch, no PCIe transfer and no host work per iteration.
//
// The occupancy search (no potential map, no yaw control) runs search_kernel<DIM, ORD, false, false>: the
// sample loop never evaluates velocities.  The cost-term search serves every plan, including
// potential-field, gradient and yaw planning, with search_kernel<DIM, ORD, YAW, true>: the sample loop sums
// the potential, gradient and yaw-alignment terms per sample in loop order (sample_group), as the register
// and dealing kernels do, so the edge costs equal theirs bit for bit.
//
// Every entry point searches in rounds of one launch each (run_round).  A round searches a list of queries
// in arenas of one capacity; a query that outgrows its arena ends in kOverflow (consume<true>), and one that
// finishes reserves room for its closed keys and actions in a device result pool, drained after the round.
// mplx_plan_batch and mplx_plan_batch_cost_terms run one round with worst-case arenas and a pool that holds
// every query's worst case, so none of their queries can overflow or find the pool full.  A round in
// worst-case arenas runs the kernel without the capacity check (CHECK false), which gives the same results
// and spills less.
// mplx_plan_batch_grow sizes arenas for the batch and searches overflowed queries again in larger arenas
// (include/mplx.h states its round schedule).
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "mplx_dispatch.h"
#include "mplx_expand.cuh"
#include "mplx_fx.cuh"
#include "mplx_internal.h"
#include "mplx_search.cuh"

namespace mplx {
namespace {

using namespace search;

struct Job {
  const mplx_waypoint *starts, *goals;
  const uint8_t *start_free;  // nullptr: is_free(start.pos) on the device grid
  int n_q, max_expand;
  bool closed;  // the closed keys are stored
  double eps, tol_pos, tol_vel, tol_acc, tol_yaw;
  unsigned char *arena;
  Layout L;
  uint32_t epoch0;  // the i-th query of the launch uses epoch epoch0 + i
  // per-slot successor scratch (nU entries each)
  mplx_waypoint *s_succ;
  int32_t *s_count, *s_action;
  double *s_cost;
  uint64_t *s_key;
  int *counter;
  // per-query results: the launch searches queries qlist[0, n_q); query q = qlist[i] writes state[q]
  // (kDone / kOverflowed / kPoolFull) and, when done, its results, its closed keys (with `closed`) and
  // then its actions into pool[offs[q], ...), reserved with one atomicAdd on *pool_used; when the pool is
  // full, offs[q] receives the units it needed
  const int32_t *qlist;
  int32_t *valid, *expanded, *n_closed, *n_actions, *state;
  double *cost;
  uint64_t *pool;
  unsigned long long *pool_used, *offs;
  unsigned long long pool_cap;  // in uint64 units
};
enum GrowState : int32_t { kDone = 1, kOverflowed = 2, kPoolFull = 3 };

// Samples per group of the cost-term sample loop; the result does not depend on the group size.  Groups
// of 4 spill with the cost terms (as in the dealing kernel, mplx_deal.cu).  Spill stores / loads in bytes
// under -Xptxas -v (nvcc 12.9, sm_90a) of the instantiations without the capacity check that spill at 2 or 1,
// <DIM, ORD, YAW>:
//                      groups of 2    groups of 1
//   <2, JRK, yaw>        52 /  76        0 /   0
//   <2, SNP, no yaw>    148 / 252      180 / 292
//   <2, SNP, yaw>        80 / 192       80 / 200
//   <3, ACC, no yaw>     76 / 100       52 /  76
//   <3, ACC, yaw>        32 /  56        0 /   0
//   <3, JRK, no yaw>      0 /   0      312 / 368
//   <3, JRK, yaw>       164 / 292      244 / 340
// The other 9 spill at neither.  Groups of 2: 552 B of spill stores over the 16, against 868 B at 1.  With
// the capacity check (CHECK): 760 B at 2, against 940 B at 1.
constexpr int kCostUnr = 2;

// hash_value(waypoint) (waypoint.h:93-125) as phase A computes it for `tn == curr`: the yaw lattice id
// comes last for a yaw control.  The start's and the goal's keys must be these for the search to find them.
template <int DIM, int ORD, bool YAW>
__device__ __forceinline__ uint64_t node_hash(const mplx_waypoint *w) {
  uint64_t h = curr_hash<DIM, ORD>(w);
  if (YAW) hash_combine(h, lattice_id(w->yaw, 0.1, 10.0));
  return h;
}

// COST: the sample loop sums per-sample cost terms (potential, gradient, yaw alignment); without it the
// kernel is the occupancy search, whose code does not carry the velocity coefficients.
// CHECK: the arena's capacity is checked (consume<true>).  A launch whose arenas hold every query's worst
// case (layout_for) runs without it, exactly as with it, and spills less in the sample loop.
template <int DIM, int ORD, bool YAW, bool COST, bool CHECK>
__global__ void __launch_bounds__(kThreads) search_kernel(const __grid_constant__ EnvParams P, const __grid_constant__ Job J) {
  static_assert(COST || !YAW, "a yaw control always sums cost terms");
  __shared__ mplx_waypoint s_node;
  __shared__ uint32_t vbits[9];
  __shared__ int s_q, s_status;
  const int slot = blockIdx.x;
  const int nU = P.nU;
  const int words = (nU + 31) >> 5;
  const OutPtrs o{J.s_count + slot, J.s_succ + (size_t)slot * nU, nullptr, J.s_action + (size_t)slot * nU,
                  J.s_key + (size_t)slot * nU, nullptr};
  double *s_cost = J.s_cost + (size_t)slot * nU;
  Grid G;
  G.map = P.map;
  G.dim = DIM;
  for (int k = 0; k < 3; k++) {
    G.mdim[k] = P.mdim[k];
    G.origin[k] = P.origin[k];
  }
  G.res = P.res;
  Arena A;
  Query S;
  Goal Q;
  for (;;) {
    if (threadIdx.x == 0) {
      s_q = atomicAdd(J.counter, 1);
      s_status = kIdle;
      if (s_q < J.n_q) {
        const int q = J.qlist[s_q];
        A = arena_at(J.arena + (size_t)slot * J.L.bytes, J.L, J.epoch0 + (uint32_t)s_q);
        Q.w = J.goals[q];
        Q.key = node_hash<DIM, ORD, YAW>(&J.goals[q]);
        Q.tol_pos = J.tol_pos;
        Q.tol_vel = J.tol_vel;
        Q.tol_acc = J.tol_acc;
        Q.tol_yaw = J.tol_yaw;
        Q.w_heur = P.w;
        Q.v_max = P.v_max;
        const mplx_waypoint st = J.starts[q];
        const bool free_ = J.start_free ? J.start_free[q] != 0 : is_free(G, st.pos);
        begin(A, S, G, Q, st, node_hash<DIM, ORD, YAW>(&st), free_, J.eps, J.max_expand);
        if (S.status == kRunning) s_node = A.st[pop(A, S)].coord;
        s_status = S.status;
      }
    }
    __syncthreads();
    if (s_q >= J.n_q) return;
    while (s_status == kRunning) {
      PrimState<DIM, ORD, YAW> pr;
      bool emit, same;
      double max_v;
      size_t sl;
      phase_ab<DIM, ORD, YAW, false>(P, &s_node, 1, threadIdx.x, nU, nU, 0, vbits, words, o, pr, emit, same, max_v,
                                     sl);
      if (emit) {
        double cost = 0.0;
        const double intrinsic = intrinsic_cost<DIM, ORD, YAW>(P, pr);
        if (!same) {
          // the velocity coefficients only when a cost term reads them (need_vel), as in the register kernel
          const bool vel = COST && need_vel(P, YAW);
          double cf[CoefLayout<DIM, ORD, YAW>::NCMAX];
          fill_coef<DIM, ORD, YAW>(pr, vel, cf);
          double dt;
          const int n = sample_count_n(P, max_v, dt);
          unsigned n_samples = 0;
          cost = traverse_groups<DIM, ORD, YAW, COST ? kCostUnr : 4>(P, cf, vel, dt, sample_loop_count(P, n, dt),
                                                                     n_samples);
        }
        if (!isinf(cost)) cost += intrinsic;
        s_cost[sl] = cost;
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        consume<CHECK>(
            A, S, G, Q, o.count[0], [&](int s) { return (uint64_t)o.key[s]; }, [&](int s) { return s_cost[s]; },
            [&](int s) { return (int)o.action[s]; }, [&](int s, mplx_waypoint &w) { w = o.succ[s]; });
        if (S.status == kRunning) s_node = A.st[pop(A, S)].coord;
        s_status = S.status;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      const int q = J.qlist[s_q];
      if (S.status == kOverflow) {
        J.state[q] = kOverflowed;
      } else {
        // the trace-back reads only states and predecessor records, so the dead heap (4*cap int32, more than
        // the at most n_states + 1 actions) holds the trajectory until the pool has room for it
        int32_t *traj = reinterpret_cast<int32_t *>(A.hp);
        int na = 0;
        const double c = finish(A, S, traj, 4 * A.cap, &na);
        int nc = 0;
        if (S.status != kIdle && S.status != kTrivial)
          for (int s = 0; s < A.n_states; s++) nc += (A.st[s].flags & kClosed) ? 1 : 0;
        const unsigned long long nk = J.closed ? (unsigned long long)nc : 0ull;
        const unsigned long long units = nk + (unsigned long long)(na + 1) / 2;
        const unsigned long long off = atomicAdd(J.pool_used, units);
        if (off + units > J.pool_cap) {
          J.offs[q] = units;  // the room its rerun's pool must have
          J.state[q] = kPoolFull;
        } else {
          uint64_t *keys = J.pool + off;
          if (J.closed) {
            int k = 0;
            for (int s = 0; s < A.n_states; s++)
              if (A.st[s].flags & kClosed) keys[k++] = A.st[s].key;
          }
          int32_t *acts = reinterpret_cast<int32_t *>(keys + nk);
          for (int i = 0; i < na; i++) acts[i] = traj[i];
          J.cost[q] = c;
          J.valid[q] = isinf(c) ? 0 : 1;
          J.expanded[q] = S.expanded;
          J.n_actions[q] = na;
          J.n_closed[q] = nc;
          J.offs[q] = off;
          J.state[q] = kDone;
        }
      }
    }
    __syncthreads();
  }
}

// The instantiation a plan runs: <DIM, ORD, false, false> for the occupancy search, <DIM, ORD, yaw bit,
// true> for the cost-term search, each with the capacity check or without.  f receives the kernel's address.
template <class F>
cudaError_t with_search_kernel(const EnvParams &P, bool cost_terms, bool check, F &&f) {
  return with_bool(check, [&](auto CHECK) {
    return with_dim(P.dim, [&](auto DIM) {
      return with_order(P.control, [&](auto ORD) {
        if (!cost_terms) return f(search_kernel<DIM, ORD, false, false, CHECK>);
        return with_bool(P.control & 16, [&](auto YAW) { return f(search_kernel<DIM, ORD, YAW, true, CHECK>); });
      });
    });
  });
}

int resident_ctas(const EnvParams &P, bool cost_terms, bool check, int block) {
  int per_sm = 0;
  const cudaError_t e = with_search_kernel(P, cost_terms, check, [&](auto kernel) {
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, 0);
  });
  if (e != cudaSuccess) {
    cudaGetLastError();
    per_sm = 1;
  }
  return std::max(1, per_sm) * sm_count();
}

}  // namespace
}  // namespace mplx

using namespace mplx;
using namespace mplx::search;

namespace {
// Bytes of the per-query arrays of one search call: start and goal, the start-is-free flag, valid, expanded,
// n_closed, n_actions, state and the launch's query list, the cost and the place in the result pool.
constexpr size_t kQueryBytes =
    2 * sizeof(mplx_waypoint) + 1 + 6 * sizeof(int32_t) + sizeof(double) + sizeof(unsigned long long);

// The device memory one search call may take: a quarter of the device memory free at the call, counting the
// arenas and the result pool the ctx already holds as free (they are reused or replaced), at most
// kSearchArenaBudget.
int search_budget(const SearchBufs &B, size_t &budget) {
  size_t free_b = 0, total_b = 0;
  CU(cudaMemGetInfo(&free_b, &total_b));
  const size_t held = B.arena.cap + B.closed.cap * sizeof(uint64_t);
  budget = std::min(kSearchArenaBudget, (free_b + held) / 4);
  return MPLX_OK;
}

// The result pool (uint64 units) of a call whose every query may take its worst case: max_expand closed keys
// (with_closed) and max_expand action ids, two to a unit.
int64_t worst_pool_units(int n_q, int max_expand, bool with_closed) {
  return (int64_t)n_q * ((with_closed ? max_expand : 0) + (max_expand + 1) / 2);
}

// mplx_plan_batch*'s device memory: the per-query arrays, a result pool for every query's worst case and as
// many worst-case arenas as fit next to them in the budget (search_budget).  MPLX_ERR_ALLOC, with nothing
// changed, when not even one arena fits.
int size_batch(mplx_ctx *c, const char *fn, bool cost_terms, int n_q, int max_expand, bool with_closed, Layout &L,
               int64_t &slots) {
  const int nU = c->P.nU;
  L = layout_for(max_expand, nU);
  const int block = ((nU + 31) / 32) * 32;
  size_t budget = 0;
  const int rc = search_budget(c->sb, budget);
  if (rc) return rc;
  const size_t results =
      (size_t)n_q * kQueryBytes + (size_t)worst_pool_units(n_q, max_expand, with_closed) * sizeof(uint64_t);
  slots = std::min<int64_t>(std::max(n_q, 1), (int64_t)resident_ctas(c->P, cost_terms, false, block));
  const size_t left = results < budget ? budget - results : 0;
  slots = std::min<int64_t>(slots, (int64_t)(left / (size_t)L.bytes));
  if (slots < 1)
    return fail(MPLX_ERR_ALLOC,
                "%s: one search arena (%lld bytes) and the results (%lld bytes) exceed the budget of %lld bytes", fn,
                (long long)L.bytes, (long long)results, (long long)budget);
  return MPLX_OK;
}

// The refusals of the entry points; the occupancy search (cost_terms false) also refuses the plans with
// per-sample cost terms, and all but mplx_plan_batch_grow (unbounded_ok) an unbounded search.
int check_plan(mplx_ctx *c, const char *fn, bool cost_terms, int max_expand, bool unbounded_ok = false) {
  if (!c) return fail(MPLX_ERR_ARG, "%s: null ctx", fn);
  if (!c->has_map || !c->has_params) return fail(MPLX_ERR_ARG, "%s: map or params not set", fn);
  if (!cost_terms) {
    if (c->has_pot)
      return fail(MPLX_ERR_ARG, "%s: a potential map is installed (mplx_plan_batch_cost_terms serves it)", fn);
    if (c->P.control & 16) return fail(MPLX_ERR_ARG, "%s: yaw controls take mplx_plan_batch_cost_terms", fn);
  }
  if (max_expand <= 0 && !unbounded_ok) return fail(MPLX_ERR_ARG, "%s: max_expand must be > 0", fn);
  if (c->P.nU > kThreads) return fail(MPLX_ERR_ARG, "%s: nU > %d", fn, kThreads);
  return MPLX_OK;
}

// `slots` arenas of layout L for a launch that takes n_epochs fresh epochs.
int prepare_arenas(mplx_ctx *c, const Layout &L, int64_t slots, int64_t n_epochs) {
  SearchBufs &B = c->sb;
  const size_t need = (size_t)slots * (size_t)L.bytes;
  if (B.arena.cap < need) {
    B.arena.release();  // freed before the larger one is taken: the budget counted it as free
    B.cleared = 0;
    CU(B.arena.reserve(need));
  }
  // key-table entries of earlier queries must not look valid: the bytes this call uses start cleared
  // after a new layout, past what was cleared for this layout, or when the epochs run out
  if (B.layout_bytes != L.bytes || B.cleared < need ||
      (uint64_t)B.next_epoch + (uint64_t)n_epochs >= 0xffffffffull) {
    CU(cudaMemsetAsync(B.arena.p, 0, need, c->stream));
    B.layout_bytes = L.bytes;
    B.cleared = need;
    B.next_epoch = 1;
  }
  return MPLX_OK;
}

// One search call's queries and parameters.
struct Batch {
  int n_q, max_expand;
  bool cost_terms, with_closed, start_free;
  double eps, tol_pos, tol_vel, tol_acc, tol_yaw;
};

// The per-query arrays of a call, with the queries uploaded.
int upload(mplx_ctx *c, const mplx_waypoint *starts, const mplx_waypoint *goals, const uint8_t *start_free, int n_q) {
  SearchBufs &B = c->sb;
  CU(B.queries.reserve(2 * (size_t)n_q));
  CU(B.free_.reserve((size_t)n_q));
  CU(B.ires.reserve(6 * (size_t)n_q));
  CU(B.dres.reserve((size_t)n_q));
  CU(B.offs.reserve((size_t)n_q + 1));
  CU(cudaMemcpyAsync(B.queries.p, starts, sizeof(mplx_waypoint) * n_q, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemcpyAsync(B.queries.p + n_q, goals, sizeof(mplx_waypoint) * n_q, cudaMemcpyHostToDevice, c->stream));
  if (start_free) CU(cudaMemcpyAsync(B.free_.p, start_free, n_q, cudaMemcpyHostToDevice, c->stream));
  return MPLX_OK;
}

// What a round gives back, indexed by query id; only the round's queries' entries are from it.
enum RoundField { kValid = 0, kExpanded = 1, kNClosed = 2, kNActions = 3, kState = 4 };
struct Round {
  std::vector<int32_t> ires;  // the RoundFields, n_q of each
  std::vector<double> cost;
  std::vector<unsigned long long> offs;  // kDone: the query's place in pool; kPoolFull: the units it needed
  std::vector<uint64_t> pool;            // the result pool, drained
  double seconds = 0;  // device time of the round's launch
  int32_t at(RoundField f, int q) const { return ires[(size_t)f * cost.size() + q]; }
};

// One launch over the queries `qlist` in `slots` arenas of layout L with a result pool of pool_units
// uint64: reserves the per-slot scratch and the pool, launches, and copies the results and the pool back.
int run_round(mplx_ctx *c, const Batch &b, const std::vector<int32_t> &qlist, const Layout &L, int64_t slots,
              int64_t pool_units, Round &R) {
  SearchBufs &B = c->sb;
  const int nU = c->P.nU;
  const int n_q = b.n_q;
  const int64_t n = (int64_t)qlist.size();
  int rc = prepare_arenas(c, L, slots, n);
  if (rc) return rc;
  CU(B.succ.reserve((size_t)slots * nU));
  CU(B.cost.reserve((size_t)slots * nU));
  CU(B.key.reserve((size_t)slots * nU));
  CU(B.action.reserve((size_t)slots * nU));
  CU(B.count.reserve((size_t)slots + 1));
  CU(B.closed.reserve((size_t)pool_units));
  int32_t *ql = B.ires.p + 5 * (size_t)n_q;
  CU(cudaMemcpyAsync(ql, qlist.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemsetAsync(B.count.p + slots, 0, sizeof(int32_t), c->stream));
  CU(cudaMemsetAsync(B.offs.p + n_q, 0, sizeof(unsigned long long), c->stream));

  Job J{};
  J.starts = B.queries.p;
  J.goals = B.queries.p + n_q;
  J.start_free = b.start_free ? B.free_.p : nullptr;
  J.n_q = (int)n;
  J.max_expand = b.max_expand;
  J.closed = b.with_closed;
  J.eps = b.eps;
  J.tol_pos = b.tol_pos;
  J.tol_vel = b.tol_vel;
  J.tol_acc = b.tol_acc;
  J.tol_yaw = b.tol_yaw;
  J.arena = B.arena.p;
  J.L = L;
  J.epoch0 = B.next_epoch;
  J.s_succ = B.succ.p;
  J.s_count = B.count.p;
  J.s_action = B.action.p;
  J.s_cost = B.cost.p;
  J.s_key = B.key.p;
  J.counter = B.count.p + slots;
  J.qlist = ql;
  J.valid = B.ires.p;
  J.expanded = B.ires.p + n_q;
  J.n_closed = B.ires.p + 2 * (size_t)n_q;
  J.n_actions = B.ires.p + 3 * (size_t)n_q;
  J.state = B.ires.p + 4 * (size_t)n_q;
  J.cost = B.dres.p;
  J.pool = B.closed.p;
  J.pool_used = B.offs.p + n_q;
  J.offs = B.offs.p;
  J.pool_cap = (unsigned long long)pool_units;
  B.next_epoch += (uint32_t)n;

  EnvParams P = c->P;
  P.stats = nullptr;
  const int block = ((nU + 31) / 32) * 32;
  // worst-case arenas cannot overflow: the capacity check would change nothing
  const bool check = b.max_expand <= 0 || L.cap < 1 + (int64_t)b.max_expand * nU;
  TimedRun timed;
  const cudaError_t le = timed.run(c->stream, c->launches, [&](int *launches) {
    return with_search_kernel(P, b.cost_terms, check, [&](auto kernel) {
      kernel<<<(int)slots, block, 0, c->stream>>>(P, J);
      const cudaError_t e = cudaGetLastError();
      if (e == cudaSuccess) *launches += 1;
      return e;
    });
  });
  if (le != cudaSuccess) {
    cudaGetLastError();
    return fail(MPLX_ERR_CUDA, "search kernel launch failed: %s", cudaGetErrorString(le));
  }
  R.ires.resize(5 * (size_t)n_q);
  R.cost.resize(n_q);
  R.offs.resize(n_q);
  unsigned long long used = 0;
  CU(cudaMemcpyAsync(R.ires.data(), B.ires.p, sizeof(int32_t) * R.ires.size(), cudaMemcpyDeviceToHost, c->stream));
  CU(cudaMemcpyAsync(R.cost.data(), B.dres.p, sizeof(double) * n_q, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaMemcpyAsync(R.offs.data(), B.offs.p, sizeof(unsigned long long) * n_q, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaMemcpyAsync(&used, B.offs.p + n_q, sizeof used, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  CU(timed.seconds(&R.seconds));
  // the pool is drained before the next round reuses it
  R.pool.resize((size_t)std::min<unsigned long long>(used, (unsigned long long)pool_units));
  if (!R.pool.empty())
    CU(cudaMemcpy(R.pool.data(), B.closed.p, sizeof(uint64_t) * R.pool.size(), cudaMemcpyDeviceToHost));
  return MPLX_OK;
}

int plan_batch_fits(mplx_ctx *c, const char *fn, bool cost_terms, int n_q, int max_expand, int with_closed,
                    int32_t *slots, int64_t *arena_bytes) {
  int rc = check_plan(c, fn, cost_terms, max_expand);
  if (rc) return rc;
  if (n_q < 0) return fail(MPLX_ERR_ARG, "%s: n_q < 0", fn);
  rc = mplx_bind(c);
  if (rc) return rc;
  Layout L;
  int64_t s = 0;
  rc = size_batch(c, fn, cost_terms, n_q, max_expand, with_closed != 0, L, s);
  if (rc) return rc;
  if (slots) *slots = (int32_t)s;
  if (arena_bytes) *arena_bytes = L.bytes;
  return MPLX_OK;
}

int plan_batch(mplx_ctx *c, const char *fn, bool cost_terms, const mplx_waypoint *starts, const mplx_waypoint *goals,
               const uint8_t *start_free, int n_q, double eps, int max_expand, double tol_pos, double tol_vel,
               double tol_acc, double tol_yaw, mplx_batch_out *out) {
  int rc = check_plan(c, fn, cost_terms, max_expand);
  if (rc) return rc;
  if (!out) return fail(MPLX_ERR_ARG, "%s: null out", fn);
  if (n_q < 0 || (n_q > 0 && (!starts || !goals))) return fail(MPLX_ERR_ARG, "%s: bad query arrays", fn);
  if (!out->valid || !out->cost || !out->expanded || !out->n_closed || !out->action_offset || !out->actions)
    return fail(MPLX_ERR_ARG, "%s: missing output array", fn);
  if (out->closed_keys && !out->closed_offset) return fail(MPLX_ERR_ARG, "%s: closed_offset missing", fn);
  if (out->action_capacity < (int64_t)n_q * max_expand ||
      (out->closed_keys && out->closed_capacity < (int64_t)n_q * max_expand))
    return fail(MPLX_ERR_ARG, "%s: capacities below n_q*max_expand", fn);
  rc = mplx_bind(c);
  if (rc) return rc;
  const bool with_closed = out->closed_keys != nullptr;
  Layout L;
  int64_t slots = 0;
  rc = size_batch(c, fn, cost_terms, n_q, max_expand, with_closed, L, slots);
  if (rc) return rc;
  out->slots = 0;
  out->arena_bytes = 0;
  out->seconds = 0;
  out->action_offset[0] = 0;
  if (out->closed_offset) out->closed_offset[0] = 0;
  if (n_q == 0) return MPLX_OK;

  rc = upload(c, starts, goals, start_free, n_q);
  if (rc) return rc;
  const Batch b{n_q, max_expand, cost_terms, with_closed, start_free != nullptr, eps, tol_pos, tol_vel, tol_acc, tol_yaw};
  std::vector<int32_t> all(n_q);
  std::iota(all.begin(), all.end(), 0);
  Round R;
  rc = run_round(c, b, all, L, slots, worst_pool_units(n_q, max_expand, with_closed), R);
  if (rc) return rc;
  int64_t ao = 0, co = 0;
  for (int q = 0; q < n_q; q++) {
    // worst-case arenas and pool: no query can overflow or find the pool full
    if (R.at(kState, q) != kDone)
      return fail(MPLX_ERR_CUDA, "%s: query %d did not fit its worst-case arena and result pool", fn, q);
    out->valid[q] = R.at(kValid, q);
    out->cost[q] = R.cost[q];
    out->expanded[q] = R.at(kExpanded, q);
    const int nc = R.at(kNClosed, q);
    out->n_closed[q] = nc;
    const int na = R.at(kNActions, q);
    if (na > max_expand) return fail(MPLX_ERR_ARG, "%s: query %d: trajectory longer than max_expand", fn, q);
    // nc = expanded <= max_expand and na <= max_expand, so the compacted outputs stay within n_q*max_expand
    const uint64_t *keys = R.pool.data() + R.offs[q];
    const int nk = with_closed ? nc : 0;
    const int32_t *a = reinterpret_cast<const int32_t *>(keys + nk);
    std::copy(a, a + na, out->actions + ao);
    ao += na;
    out->action_offset[q + 1] = ao;
    if (with_closed) {
      // the closed set's keys sorted ascending, as mplh_plan returns them (plan_capi.hpp export_result)
      std::copy(keys, keys + nk, out->closed_keys + co);
      std::sort(out->closed_keys + co, out->closed_keys + co + nk);
      co += nk;
      out->closed_offset[q + 1] = co;
    }
  }
  out->slots = (int32_t)slots;
  out->arena_bytes = L.bytes;
  out->seconds = R.seconds;
  return MPLX_OK;
}

// ---- mplx_plan_batch_grow ------------------------------------------------------------------------------

// the capacity of a query's next arena after it outgrew one (include/mplx.h, the round schedule)
constexpr int64_t kGrowFactor = 4;

// The largest capacity at which `slots` arenas fit `avail` bytes (0 when not even capacity 1 does).
int64_t cap_fitting(int64_t slots, size_t avail) {
  int64_t lo = 0, hi = (int64_t)INT32_MAX / 4;  // 4*cap int32 of trajectory scratch stay addressable by int
  while (lo < hi) {
    const int64_t mid = lo + (hi - lo + 1) / 2;
    if ((size_t)slots * (size_t)layout_cap(mid).bytes <= avail) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

int plan_batch_grow(mplx_ctx *c, int cost_terms, const mplx_waypoint *starts, const mplx_waypoint *goals,
                    const uint8_t *start_free, int n_q, double eps, int max_expand, double tol_pos, double tol_vel,
                    double tol_acc, double tol_yaw, int with_closed, int64_t first_cap, int64_t max_cap,
                    int64_t pool_bytes, mplx_grow_out *out) {
  const char *fn = "mplx_plan_batch_grow";
  if (cost_terms != 0 && cost_terms != 1) return fail(MPLX_ERR_ARG, "%s: cost_terms must be 0 or 1", fn);
  int rc = check_plan(c, fn, cost_terms != 0, max_expand, true);
  if (rc) return rc;
  if (!out) return fail(MPLX_ERR_ARG, "%s: null out", fn);
  if (n_q < 0 || (n_q > 0 && (!starts || !goals))) return fail(MPLX_ERR_ARG, "%s: bad query arrays", fn);
  if (!out->valid || !out->cost || !out->expanded || !out->n_closed || !out->n_actions || !out->searched)
    return fail(MPLX_ERR_ARG, "%s: missing output array", fn);
  if (first_cap < 0 || max_cap < 0 || pool_bytes < 0)
    return fail(MPLX_ERR_ARG, "%s: first_cap, max_cap and pool_bytes must be >= 0", fn);
  rc = mplx_bind(c);
  if (rc) return rc;
  const int nU = c->P.nU;
  const int block = ((nU + 31) / 32) * 32;
  const bool ct = cost_terms != 0;

  // the per-query arrays and the pool's automatic size come off the budget first
  size_t budget = 0;
  rc = search_budget(c->sb, budget);
  if (rc) return rc;
  SearchBufs &B = c->sb;
  const size_t results = (size_t)n_q * kQueryBytes;
  const size_t pool_auto = budget / 8;
  const size_t avail = results + pool_auto < budget ? budget - results - pool_auto : 0;
  const int64_t resident = resident_ctas(c->P, ct, true, block);
  int64_t cap_max = cap_fitting(1, avail);
  if (cap_max < 1)
    return fail(MPLX_ERR_ALLOC, "%s: one search arena and the results (%lld bytes) exceed the budget of %lld bytes",
                fn, (long long)results, (long long)budget);
  if (max_expand > 0) cap_max = std::min<int64_t>(cap_max, 1 + (int64_t)max_expand * nU);
  if (max_cap > 0) cap_max = std::min(cap_max, max_cap);
  int64_t cap = first_cap > 0 ? first_cap : cap_fitting(std::min<int64_t>(std::max(n_q, 1), resident), avail);
  cap = std::max<int64_t>(1, std::min(cap, cap_max));
  const int64_t pool_units =
      std::max<int64_t>(1, pool_bytes > 0 ? pool_bytes / (int64_t)sizeof(uint64_t) : (int64_t)(pool_auto / 8));

  memset(out->valid, 0, sizeof(int32_t) * n_q);
  memset(out->expanded, 0, sizeof(int32_t) * n_q);
  memset(out->n_closed, 0, sizeof(int32_t) * n_q);
  memset(out->n_actions, 0, sizeof(int32_t) * n_q);
  memset(out->searched, 0, sizeof(int32_t) * n_q);
  for (int q = 0; q < n_q; q++) out->cost[q] = INFINITY;
  out->rounds = 0;
  out->slots = 0;
  out->first_cap = cap;
  out->last_cap = 0;
  out->arena_bytes = 0;
  out->reruns = 0;
  out->seconds = 0;
  std::vector<std::vector<int32_t>> acts(n_q);
  std::vector<std::vector<uint64_t>> keys(n_q);
  auto publish = [&]() {
    B.grow_aoff.assign((size_t)n_q + 1, 0);
    B.grow_coff.assign((size_t)n_q + 1, 0);
    B.grow_actions.clear();
    B.grow_closed.clear();
    for (int q = 0; q < n_q; q++) {
      B.grow_actions.insert(B.grow_actions.end(), acts[q].begin(), acts[q].end());
      std::sort(keys[q].begin(), keys[q].end());
      B.grow_closed.insert(B.grow_closed.end(), keys[q].begin(), keys[q].end());
      B.grow_aoff[q + 1] = (int64_t)B.grow_actions.size();
      B.grow_coff[q + 1] = (int64_t)B.grow_closed.size();
    }
  };
  if (n_q == 0) {
    publish();
    return MPLX_OK;
  }

  rc = upload(c, starts, goals, start_free, n_q);
  if (rc) return rc;
  const Batch b{n_q, max_expand, ct, with_closed != 0, start_free != nullptr, eps, tol_pos, tol_vel, tol_acc, tol_yaw};
  std::vector<int32_t> cur(n_q), next;
  std::iota(cur.begin(), cur.end(), 0);
  Round R;
  double seconds = 0;
  int32_t rounds = 0;
  int64_t reruns = 0;
  int64_t again_units = 0;  // the most pool units a query of this round's list found no room for
  for (;;) {
    const Layout L = layout_cap(cap);
    const int64_t n = (int64_t)cur.size();
    const int64_t slots = std::max<int64_t>(1, std::min({n, resident, (int64_t)(avail / (size_t)L.bytes)}));
    // a pool that holds the largest query that found it full: the first of them to reserve fits, so every
    // round completes at least one query
    rc = run_round(c, b, cur, L, slots, std::max(pool_units, again_units), R);
    if (rc) return rc;
    seconds += R.seconds;
    if (rounds == 0) {
      out->slots = (int32_t)slots;
      out->arena_bytes = L.bytes;
    }
    rounds++;
    out->last_cap = cap;

    std::vector<int32_t> again;  // the result pool was full: the same capacity again
    again_units = 0;
    for (const int32_t q : cur) {
      const int32_t st = R.at(kState, q);
      if (st == kDone) {
        out->valid[q] = R.at(kValid, q);
        out->expanded[q] = R.at(kExpanded, q);
        out->n_closed[q] = R.at(kNClosed, q);
        out->n_actions[q] = R.at(kNActions, q);
        out->cost[q] = R.cost[q];
        out->searched[q] = 1;
        const uint64_t *k = R.pool.data() + R.offs[q];
        const size_t nk = with_closed ? (size_t)out->n_closed[q] : 0;
        keys[q].assign(k, k + nk);
        const int32_t *a = reinterpret_cast<const int32_t *>(k + nk);
        acts[q].assign(a, a + out->n_actions[q]);
      } else if (st == kPoolFull) {
        again.push_back(q);
        again_units = std::max(again_units, (int64_t)R.offs[q]);
      } else if (cap < cap_max) {
        next.push_back(q);
      }  // overflowed at the largest capacity: searched stays 0
    }
    reruns += (int64_t)again.size();
    if (!again.empty()) {
      cur.swap(again);
    } else if (!next.empty()) {
      reruns += (int64_t)next.size();
      cur.swap(next);
      next.clear();
      cap = std::min(cap * kGrowFactor, cap_max);
    } else {
      break;
    }
  }
  out->rounds = rounds;
  out->reruns = reruns;
  out->seconds = seconds;
  publish();
  return MPLX_OK;
}
}  // namespace

extern "C" int mplx_plan_batch_fits(mplx_ctx *c, int n_q, int max_expand, int with_closed, int32_t *slots,
                                    int64_t *arena_bytes) {
  return plan_batch_fits(c, "mplx_plan_batch_fits", false, n_q, max_expand, with_closed, slots, arena_bytes);
}

extern "C" int mplx_plan_batch(mplx_ctx *c, const mplx_waypoint *starts, const mplx_waypoint *goals,
                               const uint8_t *start_free, int n_q, double eps, int max_expand, double tol_pos,
                               double tol_vel, double tol_acc, double tol_yaw, mplx_batch_out *out) {
  return plan_batch(c, "mplx_plan_batch", false, starts, goals, start_free, n_q, eps, max_expand, tol_pos, tol_vel,
                    tol_acc, tol_yaw, out);
}

extern "C" int mplx_plan_batch_cost_terms_fits(mplx_ctx *c, int n_q, int max_expand, int with_closed, int32_t *slots,
                                               int64_t *arena_bytes) {
  return plan_batch_fits(c, "mplx_plan_batch_cost_terms_fits", true, n_q, max_expand, with_closed, slots,
                         arena_bytes);
}

extern "C" int mplx_plan_batch_cost_terms(mplx_ctx *c, const mplx_waypoint *starts, const mplx_waypoint *goals,
                                          const uint8_t *start_free, int n_q, double eps, int max_expand,
                                          double tol_pos, double tol_vel, double tol_acc, double tol_yaw,
                                          mplx_batch_out *out) {
  return plan_batch(c, "mplx_plan_batch_cost_terms", true, starts, goals, start_free, n_q, eps, max_expand, tol_pos,
                    tol_vel, tol_acc, tol_yaw, out);
}

extern "C" int mplx_plan_batch_grow(mplx_ctx *c, int cost_terms, const mplx_waypoint *starts,
                                    const mplx_waypoint *goals, const uint8_t *start_free, int n_q, double eps,
                                    int max_expand, double tol_pos, double tol_vel, double tol_acc, double tol_yaw,
                                    int with_closed, int64_t first_cap, int64_t max_cap, int64_t pool_bytes,
                                    mplx_grow_out *out) {
  return plan_batch_grow(c, cost_terms, starts, goals, start_free, n_q, eps, max_expand, tol_pos, tol_vel, tol_acc,
                         tol_yaw, with_closed, first_cap, max_cap, pool_bytes, out);
}

extern "C" int mplx_plan_batch_grow_results(mplx_ctx *c, int64_t *action_offset, int32_t *actions,
                                            int64_t action_capacity, int64_t *closed_offset, uint64_t *closed_keys,
                                            int64_t closed_capacity) {
  const char *fn = "mplx_plan_batch_grow_results";
  if (!c) return fail(MPLX_ERR_ARG, "%s: null ctx", fn);
  const SearchBufs &B = c->sb;
  if (B.grow_aoff.empty()) return fail(MPLX_ERR_ARG, "%s: no mplx_plan_batch_grow call yet", fn);
  if (!action_offset || (B.grow_actions.size() && !actions) || (closed_keys && !closed_offset))
    return fail(MPLX_ERR_ARG, "%s: missing output array", fn);
  if (action_capacity < (int64_t)B.grow_actions.size() ||
      (closed_keys && closed_capacity < (int64_t)B.grow_closed.size()))
    return fail(MPLX_ERR_ARG, "%s: capacities below %lld actions / %lld closed keys", fn,
                (long long)B.grow_actions.size(), (long long)B.grow_closed.size());
  memcpy(action_offset, B.grow_aoff.data(), sizeof(int64_t) * B.grow_aoff.size());
  if (!B.grow_actions.empty()) memcpy(actions, B.grow_actions.data(), sizeof(int32_t) * B.grow_actions.size());
  if (closed_keys) {
    memcpy(closed_offset, B.grow_coff.data(), sizeof(int64_t) * B.grow_coff.size());
    if (!B.grow_closed.empty()) memcpy(closed_keys, B.grow_closed.data(), sizeof(uint64_t) * B.grow_closed.size());
  }
  return MPLX_OK;
}
