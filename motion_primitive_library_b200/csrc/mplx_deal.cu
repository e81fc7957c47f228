// mplx_deal.cu — expand_deal_kernel: the expansion with phase C dealt from a CTA-wide queue.
//
// In the register kernel (mplx_kernels.cu) a thread keeps the primitive it built through the
// sample loop, so a warp runs until its longest primitive is done while lanes whose primitive was
// rejected, is short or hit an obstacle early idle: on the 512^3 ACC-27 workload only ~54 % of the
// lane-steps of the sample loop do work, ~37 % with JRK-125 where half the primitives fail the
// dynamic limits.  Here a CTA runs phases A/B for `rounds` batches of 256 (node, control) items
// first; every primitive that needs sampling leaves a 16-byte ticket {slot, node, action, n} in a
// shared-memory queue (long loops at the front, short ones at the back).  Then all 256 lanes pull tickets: a lane rebuilds the primitive's quotients
// from the node (L1/L2 hit) and U[action] — the same code path as phase A, so the same bits —
// walks the reference's loop four samples at a time (sample_group), writes the cost, and pulls the next ticket
// while its neighbours are still busy.  Results are identical to the other kernels (the order in
// which primitives are sampled does not enter any result).
#include <stdlib.h>

#include "mplx_expand.cuh"

namespace mplx {

struct Ticket {
  unsigned slot;  // output slot of the successor: node * nU + rank  (< 2^31, mplx_check_ready)
  int node;       // frontier index
  int action;     // control index
  int n;          // max(5, ceil(max_v*T/res)): env_map.h:95
};

template <int DIM, int ORD, bool YAW, bool VEL, int UNR, int MINB, bool LAT>
__global__ void __launch_bounds__(kThreads, MINB)
expand_deal_kernel(const __grid_constant__ EnvParams P, const mplx_waypoint *__restrict__ nodes, int n_nodes,
                   int npb, const __grid_constant__ OutPtrs o, int rounds) {
  extern __shared__ __align__(16) unsigned char dsm[];
  Ticket *queue = reinterpret_cast<Ticket *>(dsm);  // rounds * kThreads tickets
  __shared__ uint32_t vbits[9];
  __shared__ unsigned long long s_stats[2];
  __shared__ int q_long, q_short, q_head;
  const int nU = P.nU;
  const int items = npb * nU;  // <= 256
  const int words = (items + 31) >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x < 2) s_stats[threadIdx.x] = 0;
  if (threadIdx.x == 0) q_long = q_short = q_head = 0;
  const int cap = rounds * kThreads;
  // longest-first dealing in two classes: tickets of long loops fill the queue from the front,
  // short ones from the back, and the queue is pulled front to back, so the primitives that are
  // still running when the queue dries up are short ones
  const int n_long = (5 + P.maxn) / 2;
  __syncthreads();
  unsigned n_emitted = 0;

  // ---- phases A/B for `rounds` batches of npb nodes; tickets for what needs sampling ----
  for (int r = 0; r < rounds; r++) {
    const int node0 = (blockIdx.x * rounds + r) * npb;
    PrimState<DIM, ORD, YAW> pr;
    bool emit, same;
    double max_v;
    size_t slot;
    phase_ab<DIM, ORD, YAW, LAT>(P, nodes, n_nodes, threadIdx.x, items, nU, node0, vbits, words, o, pr, emit, same,
                                 max_v, slot);
    const bool push = emit && !same;
    if (emit) {
      n_emitted++;
      // curr.pos == tn.pos: no collision check, cost 0 + intrinsic (env_map.h:163-165)
      if (same && o.cost) o.cost[slot] = 0.0 + intrinsic_cost<DIM, ORD, YAW>(P, pr);
    }
    double dt_unused;
    const int n = push ? sample_count_n(P, max_v, dt_unused) : 0;
    const bool is_long = push && n >= n_long;
    const unsigned ml = __ballot_sync(0xffffffffu, is_long);
    const unsigned ms = __ballot_sync(0xffffffffu, push && !is_long);
    if (ml | ms) {
      int base_l = 0, base_s = 0;
      if (ml) {
        const int leader = __ffs(ml) - 1;
        if (lane == leader) base_l = atomicAdd(&q_long, __popc(ml));
        base_l = __shfl_sync(0xffffffffu, base_l, leader);
      }
      if (ms) {
        const int leader = __ffs(ms) - 1;
        if (lane == leader) base_s = atomicAdd(&q_short, __popc(ms));
        base_s = __shfl_sync(0xffffffffu, base_s, leader);
      }
      if (push) {
        Ticket tk;
        tk.slot = (unsigned)slot;
        const int nl = threadIdx.x / nU;
        tk.node = node0 + nl;
        tk.action = threadIdx.x - nl * nU;
        tk.n = n;
        const unsigned below = (1u << lane) - 1u;
        const int qi = is_long ? base_l + __popc(ml & below) : cap - 1 - (base_s + __popc(ms & below));
        queue[qi] = tk;
      }
    }
    __syncthreads();  // vbits is reused by the next round; the queue is read after the last one
  }

  // ---- phase C: every lane pulls tickets until the queue is dry ----
  const int n_front = q_long;
  const int total = n_front + q_short;
  double cf[CoefLayout<DIM, ORD, YAW>::NCMAX];
  double dt = 0.0, t = 0.0, c = 0.0, intrinsic = 0.0;
  YawRot yr;
  unsigned slot = 0, n_samples = 0;
  int left = 0;  // iterations of the reference's sample loop still to visit
  bool have = false, dry = false;
  for (;;) {
    const unsigned need = dry ? 0u : __ballot_sync(0xffffffffu, !have);
    if (need) {
      int base = 0;
      const int leader = __ffs(need) - 1;
      if (lane == leader) base = atomicAdd(&q_head, __popc(need));
      base = __shfl_sync(0xffffffffu, base, leader);
      dry = base + __popc(need) > total;  // warp-uniform: this pull reached the end of the queue
      if (!have) {
        const int qi = base + __popc(need & ((1u << lane) - 1u));
        if (qi < total) {
          const Ticket tk = queue[qi < n_front ? qi : cap - 1 - (qi - n_front)];
          // Primitive(curr, U[action], dt): primitive.h:220-256, as phase A builds it
          PrimState<DIM, ORD, YAW> pr;
          const mplx_waypoint *cp = nodes + tk.node;
          const double *u = P.U + (size_t)tk.action * P.udim;
#pragma unroll
          for (int k = 0; k < DIM; k++) pr.ax[k].build(__ldg(u + k), cp->pos[k], cp->vel[k], cp->acc[k], cp->jrk[k]);
          if (YAW) {
            pr.yaw_u = __ldg(u + DIM);
            pr.yaw0 = cp->yaw;
          }
          fill_coef<DIM, ORD, YAW>(pr, VEL, cf);
          intrinsic = intrinsic_cost<DIM, ORD, YAW>(P, pr);
          dt = tk.n <= kNMax ? __ldg(P.tdt + tk.n) : P.T / tk.n;  // T/n (env_map.h:98)
          left = sample_loop_count(P, tk.n, dt);
          slot = tk.slot;
          t = 0.0;
          c = 0.0;
          if (YAW) yr.init(pr.yaw_u, pr.yaw0, dt);
          have = true;
        }
      }
    }
    if (!__any_sync(0xffffffffu, have)) break;
    if (have) {
      const int st = sample_group<DIM, ORD, YAW, UNR>(P, cf, VEL, dt, left, t, c, n_samples, yr);
      left -= UNR;
      if (st != 0) {
        if (o.cost) o.cost[slot] = st == 2 ? (double)INFINITY : c + intrinsic;
        have = false;
      }
    }
  }
  if (P.stats) {
    atomicAdd(&s_stats[0], (unsigned long long)n_samples);
    atomicAdd(&s_stats[1], (unsigned long long)n_emitted);
    __syncthreads();
    if (threadIdx.x < 2) atomicAdd(&P.stats[threadIdx.x], s_stats[threadIdx.x]);
  }
}

template <int DIM, int ORD, bool YAW>
static cudaError_t launch_deal_t(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes, const mplx_succ_out &so,
                                 cudaStream_t st, int rounds) {
  const OutPtrs o{so.count, so.succ, so.cost, so.action, so.key, so.lattice};
  const int npb = kThreads / P.nU;
  const int per_cta = npb * rounds;
  const int grid = (n_nodes + per_cta - 1) / per_cta;
  const size_t smem = (size_t)rounds * kThreads * sizeof(Ticket);
  const bool nv = YAW || (P.pot != nullptr && P.grad_w != 0.0);
  static const int unr_env = [] { const char *v = getenv("MPLX_DEAL_UNR"); return v ? atoi(v) : 0; }();  // tuning
  // groups of 2 samples when per-sample cost terms are summed (yaw alignment, gradient): groups of 4 spill
  // ~220 B per thread there (cfg4: 2.00 -> 1.68 ms per 262 144 nodes), and for short loops
  const bool short_loops = unr_env ? unr_env == 2 : (P.maxn <= 15 || nv);
  const bool lat = o.lattice != nullptr;
#define MPLX_LAUNCH_DEAL(VEL, UNR, LAT) \
  expand_deal_kernel<DIM, ORD, YAW, VEL, UNR, 4, LAT><<<grid, kThreads, smem, st>>>(P, d_nodes, n_nodes, npb, o, rounds)
  if (nv) {
    if (short_loops) { if (lat) MPLX_LAUNCH_DEAL(true, 2, true); else MPLX_LAUNCH_DEAL(true, 2, false); }
    else { if (lat) MPLX_LAUNCH_DEAL(true, 4, true); else MPLX_LAUNCH_DEAL(true, 4, false); }
  } else {
    if (short_loops) { if (lat) MPLX_LAUNCH_DEAL(YAW, 2, true); else MPLX_LAUNCH_DEAL(YAW, 2, false); }
    else { if (lat) MPLX_LAUNCH_DEAL(YAW, 4, true); else MPLX_LAUNCH_DEAL(YAW, 4, false); }
  }
#undef MPLX_LAUNCH_DEAL
  return cudaGetLastError();
}

template <int DIM>
static cudaError_t launch_deal_d(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes, const mplx_succ_out &o,
                                 cudaStream_t st, int rounds) {
  const bool yaw = (P.control & 16) != 0;
  switch (P.control & 15) {
    case MPLX_VEL: return yaw ? launch_deal_t<DIM, 1, true>(P, d_nodes, n_nodes, o, st, rounds) : launch_deal_t<DIM, 1, false>(P, d_nodes, n_nodes, o, st, rounds);
    case MPLX_ACC: return yaw ? launch_deal_t<DIM, 2, true>(P, d_nodes, n_nodes, o, st, rounds) : launch_deal_t<DIM, 2, false>(P, d_nodes, n_nodes, o, st, rounds);
    case MPLX_JRK: return yaw ? launch_deal_t<DIM, 3, true>(P, d_nodes, n_nodes, o, st, rounds) : launch_deal_t<DIM, 3, false>(P, d_nodes, n_nodes, o, st, rounds);
    case MPLX_SNP: return yaw ? launch_deal_t<DIM, 4, true>(P, d_nodes, n_nodes, o, st, rounds) : launch_deal_t<DIM, 4, false>(P, d_nodes, n_nodes, o, st, rounds);
  }
  return cudaErrorInvalidValue;
}

// rounds: batches of 256 items per CTA.  More rounds = better lane use in phase C but fewer,
// longer CTAs; keep at least ~8 CTAs per resident slot (SMs x 4 CTAs) so the grid tail stays small.
cudaError_t launch_expand_deal(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes, const mplx_succ_out &o,
                               cudaStream_t st, int rounds) {
  if (n_nodes <= 0) return cudaSuccess;
  const int npb = kThreads / P.nU;
  if (rounds <= 0) {
    const long ctas1 = ((long)n_nodes + npb - 1) / npb;  // CTAs at one round each
    rounds = (int)(ctas1 / (sm_count() * 4 * 8));
    rounds = rounds < 1 ? 1 : (rounds > kDealMaxRounds ? kDealMaxRounds : rounds);
  }
  if (rounds > kDealMaxRounds) rounds = kDealMaxRounds;
  return P.dim == 2 ? launch_deal_d<2>(P, d_nodes, n_nodes, o, st, rounds) : launch_deal_d<3>(P, d_nodes, n_nodes, o, st, rounds);
}

}  // namespace mplx
