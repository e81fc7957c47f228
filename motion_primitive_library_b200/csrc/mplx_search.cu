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
  uint32_t epoch0;  // query q uses epoch epoch0 + q
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
};

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
template <int DIM, int ORD, bool YAW, bool COST>
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
        const int q = s_q;
        A = arena_at(J.arena + (size_t)slot * J.L.bytes, J.L, J.epoch0 + (uint32_t)q);
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
        consume(
            A, S, G, Q, o.count[0], [&](int s) { return (uint64_t)o.key[s]; }, [&](int s) { return s_cost[s]; },
            [&](int s) { return (int)o.action[s]; }, [&](int s, mplx_waypoint &w) { w = o.succ[s]; });
        if (S.status == kRunning) s_node = A.st[pop(A, S)].coord;
        s_status = S.status;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
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
// for mplx_plan_batch_cost_terms.  f receives the kernel's address.
template <class F>
cudaError_t with_search_kernel(const EnvParams &P, bool cost_terms, F &&f) {
  return with_dim(P.dim, [&](auto DIM) {
    return with_order(P.control, [&](auto ORD) {
      if (!cost_terms) return f(search_kernel<DIM, ORD, false, false>);
      return with_bool(P.control & 16, [&](auto YAW) { return f(search_kernel<DIM, ORD, YAW, true>); });
    });
  });
}

int resident_ctas(const EnvParams &P, bool cost_terms, int block) {
  int per_sm = 0;
  const cudaError_t e = with_search_kernel(P, cost_terms, [&](auto kernel) {
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

// The refusals of both entry points; mplx_plan_batch also refuses the plans with per-sample cost terms.
int check_plan(mplx_ctx *c, const char *fn, bool cost_terms, int max_expand) {
  if (!c) return fail(MPLX_ERR_ARG, "%s: null ctx", fn);
  if (!c->has_map || !c->has_params) return fail(MPLX_ERR_ARG, "%s: map or params not set", fn);
  if (!cost_terms) {
    if (c->has_pot)
      return fail(MPLX_ERR_ARG, "%s: a potential map is installed (mplx_plan_batch_cost_terms serves it)", fn);
    if (c->P.control & 16) return fail(MPLX_ERR_ARG, "%s: yaw controls take mplx_plan_batch_cost_terms", fn);
  }
  if (max_expand <= 0) return fail(MPLX_ERR_ARG, "%s: max_expand must be > 0", fn);
  if (c->P.nU > kThreads) return fail(MPLX_ERR_ARG, "%s: nU > %d", fn, kThreads);
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
  const size_t need = (size_t)slots * (size_t)L.bytes;
  if (B.arena.cap < need) {
    B.arena.release();  // freed before the larger one is taken: the budget counted it as free
    B.cleared = 0;
    CU(B.arena.reserve(need));
  }
  // key-table entries of earlier queries must not look valid: the bytes this call uses start cleared
  // after a new layout, past what was cleared for this layout, or when the epochs run out
  if (B.layout_bytes != L.bytes || B.cleared < need || (uint64_t)B.next_epoch + (uint64_t)n_q >= 0xffffffffull) {
    CU(cudaMemsetAsync(B.arena.p, 0, need, c->stream));
    B.layout_bytes = L.bytes;
    B.cleared = need;
    B.next_epoch = 1;
  }
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

  Job J;
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
