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
// Two entry points share the kernel.  mplx_plan_batch serves occupancy planning only (no potential map,
// no yaw control) with search_kernel<DIM, ORD, false, false>: the sample loop never evaluates
// velocities.  mplx_plan_batch_cost_terms serves every plan, including potential-field, gradient and
// yaw planning, with search_kernel<DIM, ORD, YAW, true>: the sample loop sums the potential, gradient
// and yaw-alignment terms per sample in loop order (sample_group), as the register and dealing kernels
// do, so the edge costs equal theirs bit for bit.
//
// mplx_plan_batch_grow runs either instantiation with GROW: arenas sized for the batch rather than the worst
// case, a query that outgrows its arena abandoned (kOverflow) and searched again in a larger one in the next
// round, and results gathered in a device pool that is drained between rounds (include/mplx.h).
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>
#include <chrono>
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
  int n_q, max_expand, act_stride;
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
  // per-query results
  int32_t *valid, *expanded, *n_closed, *n_actions, *actions;
  double *cost;
  uint64_t *closed;  // nullptr: skip
  // mplx_plan_batch_grow only: the round searches queries qlist[0, n_q); query qlist[i] writes
  // state[qlist[i]] (kDone / kOverflowed / kPoolFull) and, when done, its closed keys (with `closed` set)
  // and then its actions into pool[offs[q], ...), reserved with one atomicAdd on *pool_used; when the pool
  // is full, offs[q] receives the units it needed
  const int32_t *qlist;
  int32_t *state;
  uint64_t *pool;
  unsigned long long *pool_used, *offs;
  unsigned long long pool_cap;  // in uint64 units
};
enum GrowState : int32_t { kDone = 1, kOverflowed = 2, kPoolFull = 3 };

// Samples per group of the cost-term sample loop; the result does not depend on the group size.  Groups
// of 4 spill with the cost terms (as in the dealing kernel, mplx_deal.cu).  Spill stores / loads in bytes
// under -Xptxas -v (nvcc 12.9, sm_90a) of the instantiations that spill at 2 or 1, <DIM, ORD, YAW>:
//                      groups of 2    groups of 1
//   <2, JRK, yaw>        52 /  76        0 /   0
//   <2, SNP, no yaw>    164 / 260      212 / 324
//   <2, SNP, yaw>        84 / 196       84 / 204
//   <3, ACC, no yaw>     76 / 100       52 /  76
//   <3, ACC, yaw>        32 /  56        0 /   0
//   <3, JRK, no yaw>      0 /   0      308 / 364
//   <3, JRK, yaw>       196 / 316      244 / 364
// The other 9 spill at neither.  Groups of 2: 604 B of spill stores over the 16, against 900 B at 1.
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
// GROW: mplx_plan_batch_grow's kernel: the arena's capacity is checked (consume<true>), the queries come
// from J.qlist, and results go to the result pool; without it the code is mplx_plan_batch's.
template <int DIM, int ORD, bool YAW, bool COST, bool GROW>
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
        const int q = GROW ? J.qlist[s_q] : s_q;
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
        consume<GROW>(
            A, S, G, Q, o.count[0], [&](int s) { return (uint64_t)o.key[s]; }, [&](int s) { return s_cost[s]; },
            [&](int s) { return (int)o.action[s]; }, [&](int s, mplx_waypoint &w) { w = o.succ[s]; });
        if (S.status == kRunning) s_node = A.st[pop(A, S)].coord;
        s_status = S.status;
      }
      __syncthreads();
    }
    if (GROW && threadIdx.x == 0) {
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
    if (!GROW && threadIdx.x == 0) {
      const int q = s_q;
      int na = 0;
      const double c = finish(A, S, J.actions + (size_t)q * J.act_stride, J.act_stride, &na);
      J.cost[q] = c;
      J.valid[q] = isinf(c) ? 0 : 1;
      J.expanded[q] = S.expanded;
      J.n_actions[q] = na;
      int nc = 0;
      if (S.status != kIdle && S.status != kTrivial) {
        for (int s = 0; s < A.n_states; s++)
          if (A.st[s].flags & kClosed) {
            if (J.closed && nc < J.max_expand) J.closed[(size_t)q * J.max_expand + nc] = A.st[s].key;
            nc++;
          }
      }
      J.n_closed[q] = nc;
    }
    __syncthreads();
  }
}

// The instantiation a plan runs: <DIM, ORD, false, false> for mplx_plan_batch, <DIM, ORD, yaw bit, true>
// for mplx_plan_batch_cost_terms, each with GROW for mplx_plan_batch_grow.  f receives the kernel's address.
template <bool GROW = false, class F>
cudaError_t with_search_kernel(const EnvParams &P, bool cost_terms, F &&f) {
  return with_dim(P.dim, [&](auto DIM) {
    return with_order(P.control, [&](auto ORD) {
      if (!cost_terms) return f(search_kernel<DIM, ORD, false, false, GROW>);
      return with_bool(P.control & 16, [&](auto YAW) { return f(search_kernel<DIM, ORD, YAW, true, GROW>); });
    });
  });
}

template <bool GROW = false>
int resident_ctas(const EnvParams &P, bool cost_terms, int block) {
  int per_sm = 0;
  const cudaError_t e = with_search_kernel<GROW>(P, cost_terms, [&](auto kernel) {
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
// The device memory of one search call: per-query results (n_q*max_expand action ids, and as many
// closed keys when asked for; the queries and the per-query counters) and as many worst-case arenas as fit
// next to them.  The budget is a quarter of the device memory free at the call, counting the search
// buffers the ctx already holds as free (they are reused or replaced), at most kSearchArenaBudget.
// MPLX_ERR_ALLOC, with nothing changed, when not even one arena fits.
int size_batch(mplx_ctx *c, const char *fn, bool cost_terms, int n_q, int max_expand, bool with_closed, Layout &L,
               int64_t &slots) {
  const int nU = c->P.nU;
  L = layout_for(max_expand, nU);
  const int block = ((nU + 31) / 32) * 32;
  size_t free_b = 0, total_b = 0;
  CU(cudaMemGetInfo(&free_b, &total_b));
  const SearchBufs &B = c->sb;
  const size_t held = B.arena.cap + B.actions.cap * sizeof(int32_t) + B.closed.cap * sizeof(uint64_t);
  const size_t budget = std::min(kSearchArenaBudget, (free_b + held) / 4);
  const size_t per_q = (size_t)max_expand * (sizeof(int32_t) + (with_closed ? sizeof(uint64_t) : 0));
  const size_t results = (size_t)n_q * (per_q + 2 * sizeof(mplx_waypoint) + 1 + 4 * sizeof(int32_t) + sizeof(double));
  slots = std::min<int64_t>(std::max(n_q, 1), (int64_t)resident_ctas(c->P, cost_terms, block));
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
  const int nU = c->P.nU;
  Layout L;
  int64_t slots = 0;
  rc = size_batch(c, fn, cost_terms, n_q, max_expand, out->closed_keys != nullptr, L, slots);
  if (rc) return rc;
  const int block = ((nU + 31) / 32) * 32;
  out->slots = 0;
  out->arena_bytes = 0;
  out->seconds = 0;
  out->action_offset[0] = 0;
  if (out->closed_offset) out->closed_offset[0] = 0;
  if (n_q == 0) return MPLX_OK;

  SearchBufs &B = c->sb;
  rc = prepare_arenas(c, L, slots, n_q);
  if (rc) return rc;
  CU(B.succ.reserve((size_t)slots * nU));
  CU(B.cost.reserve((size_t)slots * nU));
  CU(B.key.reserve((size_t)slots * nU));
  CU(B.action.reserve((size_t)slots * nU));
  CU(B.count.reserve((size_t)slots + 1));
  CU(B.queries.reserve(2 * (size_t)n_q));
  CU(B.free_.reserve((size_t)n_q));
  CU(B.ires.reserve(4 * (size_t)n_q));
  CU(B.dres.reserve((size_t)n_q));
  CU(B.actions.reserve((size_t)n_q * max_expand));
  if (out->closed_keys) CU(B.closed.reserve((size_t)n_q * max_expand));
  CU(cudaMemcpyAsync(B.queries.p, starts, sizeof(mplx_waypoint) * n_q, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemcpyAsync(B.queries.p + n_q, goals, sizeof(mplx_waypoint) * n_q, cudaMemcpyHostToDevice, c->stream));
  if (start_free) CU(cudaMemcpyAsync(B.free_.p, start_free, n_q, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemsetAsync(B.count.p + slots, 0, sizeof(int32_t), c->stream));

  Job J{};
  J.starts = B.queries.p;
  J.goals = B.queries.p + n_q;
  J.start_free = start_free ? B.free_.p : nullptr;
  J.n_q = n_q;
  J.max_expand = max_expand;
  J.act_stride = max_expand;
  J.eps = eps;
  J.tol_pos = tol_pos;
  J.tol_vel = tol_vel;
  J.tol_acc = tol_acc;
  J.tol_yaw = tol_yaw;
  J.arena = B.arena.p;
  J.L = L;
  J.epoch0 = B.next_epoch;
  J.s_succ = B.succ.p;
  J.s_count = B.count.p;
  J.s_action = B.action.p;
  J.s_cost = B.cost.p;
  J.s_key = B.key.p;
  J.counter = B.count.p + slots;
  J.valid = B.ires.p;
  J.expanded = B.ires.p + n_q;
  J.n_closed = B.ires.p + 2 * n_q;
  J.n_actions = B.ires.p + 3 * n_q;
  J.actions = B.actions.p;
  J.cost = B.dres.p;
  J.closed = out->closed_keys ? B.closed.p : nullptr;
  B.next_epoch += (uint32_t)n_q;

  EnvParams P = c->P;
  P.stats = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  CU(cudaEventCreate(&e0));
  CU(cudaEventCreate(&e1));
  cudaEventRecord(e0, c->stream);
  cudaError_t le = with_search_kernel(P, cost_terms, [&](auto kernel) {
    kernel<<<(int)slots, block, 0, c->stream>>>(P, J);
    return cudaGetLastError();
  });
  cudaEventRecord(e1, c->stream);
  if (le != cudaSuccess) {
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaGetLastError();
    return fail(MPLX_ERR_CUDA, "search kernel launch failed: %s", cudaGetErrorString(le));
  }
  c->launches++;
  std::vector<int32_t> ires(4 * (size_t)n_q);
  std::vector<int32_t> acts((size_t)n_q * max_expand);
  cudaError_t ce = cudaMemcpyAsync(ires.data(), B.ires.p, sizeof(int32_t) * 4 * n_q, cudaMemcpyDeviceToHost, c->stream);
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(out->cost, B.dres.p, sizeof(double) * n_q, cudaMemcpyDeviceToHost, c->stream);
  if (ce == cudaSuccess)
    ce = cudaMemcpyAsync(acts.data(), B.actions.p, sizeof(int32_t) * acts.size(), cudaMemcpyDeviceToHost, c->stream);
  if (ce == cudaSuccess && out->closed_keys)
    ce = cudaMemcpyAsync(out->closed_keys, B.closed.p, sizeof(uint64_t) * (size_t)n_q * max_expand,
                         cudaMemcpyDeviceToHost, c->stream);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(c->stream);
  float ms = 0;
  if (ce == cudaSuccess) ce = cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  CU(ce);
  int64_t ao = 0;
  for (int q = 0; q < n_q; q++) {
    out->valid[q] = ires[q];
    out->expanded[q] = ires[n_q + q];
    out->n_closed[q] = ires[2 * n_q + q];
    const int na = ires[3 * n_q + q];
    if (na < 0) return fail(MPLX_ERR_ARG, "%s: query %d: trajectory longer than max_expand", fn, q);
    // out->actions holds at least n_q*max_expand entries and ao <= q*max_expand, so compaction is in bounds
    memcpy(out->actions + ao, acts.data() + (size_t)q * max_expand, sizeof(int32_t) * na);
    ao += na;
    out->action_offset[q + 1] = ao;
  }
  if (out->closed_keys) {
    // the closed set's keys sorted ascending, as mplh_plan returns them (plan_capi.hpp export_result)
    int64_t co = 0;
    for (int q = 0; q < n_q; q++) {
      uint64_t *src = out->closed_keys + (size_t)q * max_expand;
      const int nc = out->n_closed[q];
      std::sort(src, src + nc);
      memmove(out->closed_keys + co, src, sizeof(uint64_t) * nc);
      co += nc;
      out->closed_offset[q + 1] = co;
    }
  }
  out->slots = (int32_t)slots;
  out->arena_bytes = L.bytes;
  out->seconds = ms * 1e-3;
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

  // the budget of size_batch; the per-query arrays and the pool's automatic size come off it first
  size_t free_b = 0, total_b = 0;
  CU(cudaMemGetInfo(&free_b, &total_b));
  SearchBufs &B = c->sb;
  const size_t held = B.arena.cap + B.actions.cap * sizeof(int32_t) + B.closed.cap * sizeof(uint64_t);
  const size_t budget = std::min(kSearchArenaBudget, (free_b + held) / 4);
  const size_t results = (size_t)n_q * (2 * sizeof(mplx_waypoint) + 1 + 6 * sizeof(int32_t) + sizeof(double) +
                                        sizeof(unsigned long long));
  const size_t pool_auto = budget / 8;
  const size_t avail = results + pool_auto < budget ? budget - results - pool_auto : 0;
  const int64_t resident = resident_ctas<true>(c->P, ct, block);
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

  CU(B.queries.reserve(2 * (size_t)n_q));
  CU(B.free_.reserve((size_t)n_q));
  CU(B.ires.reserve(6 * (size_t)n_q));
  CU(B.dres.reserve((size_t)n_q));
  CU(B.offs.reserve((size_t)n_q + 1));
  CU(cudaMemcpyAsync(B.queries.p, starts, sizeof(mplx_waypoint) * n_q, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemcpyAsync(B.queries.p + n_q, goals, sizeof(mplx_waypoint) * n_q, cudaMemcpyHostToDevice, c->stream));
  if (start_free) CU(cudaMemcpyAsync(B.free_.p, start_free, n_q, cudaMemcpyHostToDevice, c->stream));

  EnvParams P = c->P;
  P.stats = nullptr;
  std::vector<int32_t> cur(n_q), next, ires(6 * (size_t)n_q);
  for (int q = 0; q < n_q; q++) cur[q] = q;
  std::vector<double> dres(n_q);
  std::vector<unsigned long long> offs(n_q);
  std::vector<uint64_t> pool;
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
    const int64_t units = std::max(pool_units, again_units);
    rc = prepare_arenas(c, L, slots, n);
    if (rc) return rc;
    CU(B.succ.reserve((size_t)slots * nU));
    CU(B.cost.reserve((size_t)slots * nU));
    CU(B.key.reserve((size_t)slots * nU));
    CU(B.action.reserve((size_t)slots * nU));
    CU(B.count.reserve((size_t)slots + 1));
    CU(B.closed.reserve((size_t)units));
    int32_t *qlist = B.ires.p + 5 * (size_t)n_q;
    CU(cudaMemcpyAsync(qlist, cur.data(), sizeof(int32_t) * n, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemsetAsync(B.count.p + slots, 0, sizeof(int32_t), c->stream));
    CU(cudaMemsetAsync(B.offs.p + n_q, 0, sizeof(unsigned long long), c->stream));

    Job J{};
    J.starts = B.queries.p;
    J.goals = B.queries.p + n_q;
    J.start_free = start_free ? B.free_.p : nullptr;
    J.n_q = (int)n;
    J.max_expand = max_expand;
    J.eps = eps;
    J.tol_pos = tol_pos;
    J.tol_vel = tol_vel;
    J.tol_acc = tol_acc;
    J.tol_yaw = tol_yaw;
    J.arena = B.arena.p;
    J.L = L;
    J.epoch0 = B.next_epoch;
    J.s_succ = B.succ.p;
    J.s_count = B.count.p;
    J.s_action = B.action.p;
    J.s_cost = B.cost.p;
    J.s_key = B.key.p;
    J.counter = B.count.p + slots;
    J.valid = B.ires.p;
    J.expanded = B.ires.p + n_q;
    J.n_closed = B.ires.p + 2 * (size_t)n_q;
    J.n_actions = B.ires.p + 3 * (size_t)n_q;
    J.state = B.ires.p + 4 * (size_t)n_q;
    J.cost = B.dres.p;
    J.closed = with_closed ? B.closed.p : nullptr;  // only read as a flag here: keys go to the pool
    J.qlist = qlist;
    J.pool = B.closed.p;
    J.pool_used = B.offs.p + n_q;
    J.offs = B.offs.p;
    J.pool_cap = (unsigned long long)units;
    B.next_epoch += (uint32_t)n;

    cudaEvent_t e0 = nullptr, e1 = nullptr;
    CU(cudaEventCreate(&e0));
    CU(cudaEventCreate(&e1));
    cudaEventRecord(e0, c->stream);
    cudaError_t le = with_search_kernel<true>(P, ct, [&](auto kernel) {
      kernel<<<(int)slots, block, 0, c->stream>>>(P, J);
      return cudaGetLastError();
    });
    cudaEventRecord(e1, c->stream);
    if (le != cudaSuccess) {
      cudaEventDestroy(e0);
      cudaEventDestroy(e1);
      cudaGetLastError();
      return fail(MPLX_ERR_CUDA, "search kernel launch failed: %s", cudaGetErrorString(le));
    }
    c->launches++;
    unsigned long long used = 0;
    cudaError_t ce = cudaMemcpyAsync(ires.data(), B.ires.p, sizeof(int32_t) * 5 * n_q, cudaMemcpyDeviceToHost, c->stream);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(dres.data(), B.dres.p, sizeof(double) * n_q, cudaMemcpyDeviceToHost, c->stream);
    if (ce == cudaSuccess)
      ce = cudaMemcpyAsync(offs.data(), B.offs.p, sizeof(unsigned long long) * n_q, cudaMemcpyDeviceToHost, c->stream);
    if (ce == cudaSuccess)
      ce = cudaMemcpyAsync(&used, B.offs.p + n_q, sizeof used, cudaMemcpyDeviceToHost, c->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(c->stream);
    float ms = 0;
    if (ce == cudaSuccess) ce = cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    CU(ce);
    // the pool is drained before the next round reuses it
    pool.resize((size_t)std::min<unsigned long long>(used, (unsigned long long)units));
    if (!pool.empty())
      CU(cudaMemcpy(pool.data(), B.closed.p, sizeof(uint64_t) * pool.size(), cudaMemcpyDeviceToHost));
    seconds += ms * 1e-3;
    if (rounds == 0) {
      out->slots = (int32_t)slots;
      out->arena_bytes = L.bytes;
    }
    rounds++;
    out->last_cap = cap;

    std::vector<int32_t> again;  // the result pool was full: the same capacity again
    again_units = 0;
    for (const int32_t q : cur) {
      const int32_t st = ires[4 * (size_t)n_q + q];
      if (st == kDone) {
        out->valid[q] = ires[q];
        out->expanded[q] = ires[(size_t)n_q + q];
        out->n_closed[q] = ires[2 * (size_t)n_q + q];
        out->n_actions[q] = ires[3 * (size_t)n_q + q];
        out->cost[q] = dres[q];
        out->searched[q] = 1;
        const uint64_t *k = pool.data() + offs[q];
        const size_t nk = with_closed ? (size_t)out->n_closed[q] : 0;
        keys[q].assign(k, k + nk);
        const int32_t *a = reinterpret_cast<const int32_t *>(k + nk);
        acts[q].assign(a, a + out->n_actions[q]);
      } else if (st == kPoolFull) {
        again.push_back(q);
        again_units = std::max(again_units, (int64_t)offs[q]);
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
