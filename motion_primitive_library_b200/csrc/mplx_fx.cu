// mplx_fx.cu — expand_fx_kernel: the expansion for occupancy planning (no potential field, no yaw
// term) with the sample loop of traverse_primitive (env_map.h:90-132) decided in fixed point.
//
// Why.  With the cost terms absent, traverse_primitive returns 0 unless SOME sample of the loop is
// blocked (outside the map, occupied, outside the tunnel), in which case it returns inf whatever the
// other samples say.  What a sample needs is therefore only its cell, and the reference's cell
//     floor(y_ref),  y_ref = RN((P_ref(t) - origin)/res),  P_ref = the rounded polynomial chain
// costs ~10 FP64 instructions per axis when reproduced operation by operation (mplx_expand.cuh).
// Here each axis is ONE Horner chain of ORD fused multiply-adds in cell units whose last addend
// carries the constant 1.5*2^20 + 2^-26: the result's low mantissa word is the fraction of
// y_fx + 2^-26 in units of 2^-32 and its high word is 0x41380000 + floor(y_fx + 2^-26) — the cell
// costs one integer subtraction, no conversion, no division.  |y_fx - y_ref| < 2^-30 for every
// coordinate below 2^18 cells (bound in DESIGN.md §4.2, checked against the literal chain in
// tests/arith_identities.cpp), so
//   fraction word >= 128  (y_fx + eps at least 2 eps = 2^-25 above a cell boundary)
//       => floor(y_ref) = floor(y_fx + eps): the sample is CERTAIN and its verdict is the voxel bit;
//   fraction word <  128  => the sample is UNCERTAIN: y_ref lies within 2^-25 of the boundary below
//       cell c' = floor(y_fx + eps), its true cell is c' or c'-1 on that axis.  A second bitmap (the
//       summary half of occ2, apart from the occupancy half the certain samples read) holds,
//       per voxel, the OR of the occupancy of the <= 2^Dim cells {c', c'-1}^Dim (out of map = 1): if
//       that bit is clear every candidate is free and the sample is free whichever the reference
//       picks; otherwise the sample is AMBIGUOUS and is re-evaluated with the exact FP64 chain.
// Lattice-aligned states put ~3 % of the samples exactly on a boundary (e.g. v = +-1, u = 0 on an axis
// while n = 20), so "uncertain" is common, but "ambiguous" needs an obstacle surface next to it:
// ~0.4 % of the samples.  They are not evaluated by the lane that found them (its warp would wait):
// the lane leaves a 64-bit mask of its ambiguous samples in shared memory, and after a CTA barrier
// the queued primitives are dealt to the first lanes of the CTA, which rebuild the exact quotients
// from (node, action) with the code phase A uses and run sample_cell on exactly those samples.
//
// Results are bit-identical to the other kernels: every decision is either proven equal to the
// reference's (certain), independent of it (all candidates free), or made by the exact chain.
#include "mplx_dispatch.h"
#include "mplx_fx.cuh"
#include "mplx_pack.cuh"

namespace mplx {

constexpr int kFxThreads = kThreads + 32;  // 256 primitive threads + one helper warp

struct FxShared {
  unsigned long long amask[kThreads];  // ambiguous samples k < 64 of the thread's primitive
  uint64_t hcurr[kThreads];            // hash_value(curr) of the CTA's nodes (waypoint.h:93-125)
  double intrinsic[kThreads];          // J + w*T of a queued primitive
  unsigned slot[kThreads];             // its output slot
  uint32_t vbits[9];
  int q_n;
  unsigned char q[kThreads];     // owners (thread ids) with ambiguous samples
  unsigned char n[kThreads];     // their n (<= kNMax)
  unsigned char full[kThreads];  // 1: re-evaluate every sample (an ambiguous one lies beyond bit 63)
};

// The helper warp's second job: exact re-evaluation of the queued ambiguous samples.  A lane takes a
// queued primitive, rebuilds its exact quotients from (node, action) with the code phase A uses,
// walks the ambiguous samples with eval_pos + sample_cell at the loop's own times (sample-time table)
// and writes the primitive's cost.
template <int DIM, int ORD, bool REGION>
__device__ __forceinline__ void fx_resolve(const EnvParams &P, const mplx_waypoint *__restrict__ nodes, int node0,
                                           int nU, int inv_nU, const FxShared &S, int lane, double *__restrict__ cost) {
  const int qn = S.q_n;
  for (int i = lane; i < qn; i += 32) {
    const int owner = S.q[i];
    const int nl = (owner * inv_nU) >> 20;
    const int ci = owner - nl * nU;
    const mplx_waypoint *cp = nodes + node0 + nl;
    const double *u = P.U + (size_t)ci * P.udim;
    PrimState<DIM, ORD, false> q;  // Primitive(curr, U[action], dt) as phase A builds it
#pragma unroll
    for (int k = 0; k < DIM; k++) q.ax[k].build(__ldg(u + k), cp->pos[k], cp->vel[k], cp->acc[k], cp->jrk[k]);
    double cf[CoefLayout<DIM, ORD, false>::NCMAX];
    fill_coef<DIM, ORD, false>(q, false, cf);
    const int n = S.n[owner];
    const double *tt = P.ttab + (size_t)n * kTStride;
    unsigned long long m = S.amask[owner];
    const int count = __ldg(P.tcount + n);
    const bool full = S.full[owner] != 0;
    bool blocked = false;
    for (int k = 0; !blocked; k++) {
      if (full) {
        if (k >= count) break;
      } else {
        if (m == 0) break;
        k = __ffsll((long long)m) - 1;
        m &= m - 1;
      }
      double pk[DIM];
      eval_pos<DIM, ORD>(cf, __ldg(tt + k), pk);
      int idx;
      blocked = !sample_cell<DIM>(P, pk, idx);
      if (!blocked) {
        blocked = (__ldg(P.occ_bits + (idx >> 5)) >> (idx & 31)) & 1u;
        if (REGION) blocked = blocked || !((__ldg(P.region_bits + (idx >> 5)) >> (idx & 31)) & 1u);
      }
    }
    if (cost) cost[S.slot[owner]] = blocked ? (double)INFINITY : 0.0 + S.intrinsic[owner];
  }
}

// Threads 0..255: one (node, control) primitive each through phases A, B and the fixed-point phase C.
// Threads 256..287 (the helper warp): hash_value(curr) of the CTA's nodes while the others run phase
// A, then the exact re-evaluation of whatever phase C queued.  Barriers: B1 publishes the node
// hashes (the self-loop test `tn == curr`, env_map.h:158, is the last step of phase A), B2 the
// validity ballots of phase B, B3 the queue.  CHECK: the sample loop tests every sample against the map
// (fx_issue); without it a primitive that may leave the guard band of occ2 (fx_band) takes the literal loop.
template <int DIM, int ORD, int UNR, int MINB, bool LAT, bool REGION, bool CHECK>
__global__ void __launch_bounds__(kFxThreads, MINB)
expand_fx_kernel(const __grid_constant__ EnvParams P, const mplx_waypoint *__restrict__ nodes, int n_nodes, int npb,
                 int inv_nU, const __grid_constant__ OutPtrs o) {
  __shared__ FxShared S;
  const int nU = P.nU;
  const int items = npb * nU;  // <= 256
  const int node0 = blockIdx.x * npb;
  if (threadIdx.x >= kThreads) {
    const int lane = threadIdx.x - kThreads;
    if (lane == 0) S.q_n = 0;
    for (int j = lane; j < npb; j += 32)
      if (node0 + j < n_nodes) S.hcurr[j] = node_hash<DIM, ORD, false>(nodes + node0 + j);
    __syncthreads();  // B1
    __syncthreads();  // B2
    __syncthreads();  // B3
    fx_resolve<DIM, ORD, REGION>(P, nodes, node0, nU, inv_nU, S, lane, o.cost);
    return;
  }

  // ---- phase A (thread = primitive): as phase_ab (mplx_expand.cuh), hash_value(curr) from the helper ----
  const int item = threadIdx.x;
  const int nl = (item * inv_nU) >> 20;  // item / nU  (inv_nU = ceil(2^20 / nU), exact for item < 256)
  const int ci = item - nl * nU;
  const int ni = node0 + nl;
  const bool active = item < items && ni < n_nodes;
  PrimState<DIM, ORD, false> pr;
  bool ok = false, same = true;
  double max_v = 0;
  mplx_waypoint tn;
  int lat[LAT ? MPLX_LATTICE_MAX : 1];
  uint64_t key = 0;
  if (active) {
    const mplx_waypoint *cp = nodes + ni;
    const double *u = P.U + (size_t)ci * P.udim;
#pragma unroll
    for (int k = 0; k < DIM; k++) pr.ax[k].build(__ldg(u + k), cp->pos[k], cp->vel[k], cp->acc[k], cp->jrk[k]);
    const double T = P.T;
    const double pw3T = (T * T) * T, pw4T = pw3T * T;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      if (k < DIM) {
        tn.pos[k] = pr.ax[k].template p<true>(T, pw3T, pw4T);
        tn.vel[k] = pr.ax[k].v(T, pw3T);
        tn.acc[k] = pr.ax[k].a(T);
        tn.jrk[k] = pr.ax[k].j(T);
        same = same && (pr.ax[k].c5 == tn.pos[k]);  // curr.pos == tn.pos (env_map.h:163)
      } else {
        tn.pos[k] = tn.vel[k] = tn.acc[k] = tn.jrk[k] = 0.0;
      }
    }
    tn.yaw = 0.0;
    tn.t = cp->t + T;  // env_map.h:161
    ok = true;
#pragma unroll
    for (int k = 0; k < DIM; k++) {
      const double mv = pr.ax[k].max_vel(T);
      if (ORD >= 2 && P.v_max > 0) ok = ok && !(mv > P.v_max);
      if (mv > max_v) max_v = mv;
    }
    if (ok && ORD >= 3 && P.a_max > 0) {
#pragma unroll
      for (int k = 0; k < DIM; k++) ok = ok && !(pr.ax[k].max_acc(T) > P.a_max);
    }
    if (ok && ORD >= 4 && P.j_max > 0) {
#pragma unroll
      for (int k = 0; k < DIM; k++) ok = ok && !(pr.ax[k].max_jrk(T) > P.j_max);
    }
    if (ok) {
      int nl_ = 0;
#pragma unroll
      for (int k = 0; k < DIM; k++) {
        int id = lattice_id(tn.pos[k], 0.01, 100.0);
        hash_combine(key, id);
        if (LAT) lat[nl_++] = id;
        if (ORD >= 2) { id = lattice_id(tn.vel[k], 0.1, 10.0); hash_combine(key, id); if (LAT) lat[nl_++] = id; }
        if (ORD >= 3) { id = lattice_id(tn.acc[k], 0.1, 10.0); hash_combine(key, id); if (LAT) lat[nl_++] = id; }
        if (ORD >= 4) { id = lattice_id(tn.jrk[k], 0.1, 10.0); hash_combine(key, id); if (LAT) lat[nl_++] = id; }
      }
      if (LAT) {
#pragma unroll
        for (int q = 0; q < MPLX_LATTICE_MAX; q++)
          if (q >= nl_) lat[q] = 0;
      }
    }
  }
  __syncthreads();  // B1: node hashes are in shared memory
  // tn == curr  <=>  hash_value(tn) == hash_value(curr)  (waypoint.h:133-135)
  const bool emit = ok && key != S.hcurr[nl];

  // ---- phase B: stable per-node compaction (control order) ----
  const unsigned bal = __ballot_sync(0xffffffffu, emit);
  if ((threadIdx.x & 31) == 0) S.vbits[item >> 5] = bal;
  __syncthreads();  // B2
  size_t slot = 0;
  if (active) {
    const int s = nl * nU;  // first item of my node
    int rank = 0;
    for (int wd = s >> 5; wd <= (item >> 5); wd++) {
      uint32_t m = S.vbits[wd];
      const int lo = wd << 5;
      if (s > lo) m &= ~0u << (s - lo);
      if (item < lo + 32) m &= (1u << (item - lo)) - 1u;
      rank += __popc(m);
    }
    if (ci == nU - 1) o.count[ni] = rank + (emit ? 1 : 0);
    if (emit) {
      slot = (size_t)ni * nU + rank;
      if (o.succ) store_waypoint(o.succ + slot, tn);
      if (o.action) __stcs(o.action + slot, ci);
      if (o.key) __stcs(reinterpret_cast<unsigned long long *>(o.key + slot), (unsigned long long)key);
      if (LAT && o.lattice) {
#pragma unroll
        for (int q = 0; q < MPLX_LATTICE_MAX; q++) o.lattice[slot * MPLX_LATTICE_MAX + q] = lat[q];
      }
    }
  }

  // ---- phase C: 0 free, 1 blocked, 2 ambiguous (queued for the helper warp) ----
  if (emit) {
    int verdict = 0;
    const double intrinsic = intrinsic_cost<DIM, ORD, false>(P, pr);
    if (!same) {
      double dt;
      const int n = sample_count_n(P, max_v, dt);
      // Range the error bound covers: every sample lies within max_v*T <= n*res of the start, so the
      // start decides (DESIGN.md §4.2): (|p0| + |origin|)/res < 2^17 on every axis, n <= kNMax.
      double reach = 0.0;
#pragma unroll
      for (int a = 0; a < DIM; a++) reach = fmax(reach, (fabs(pr.ax[a].c5) + fabs(P.origin[a])) * P.rinv);
      double C[DIM][ORD + 1];
      bool band = true;
#pragma unroll
      for (int a = 0; a < DIM; a++) {
        fx_axis<ORD>(pr.ax[a], P.origin[a], P.rinv, C[a]);
        if (!REGION && !CHECK) band = band && fx_band<ORD>(C[a], P.T, P.mdim[a]);
      }
      if (n > kNMax || !(reach < kFxRange) || !band) {
        // beyond the sample-time table, the range of the fixed-point bound or (unchecked loop) able to leave
        // the guard band: the literal loop
        double cf[CoefLayout<DIM, ORD, false>::NCMAX];
        fill_coef<DIM, ORD, false>(pr, false, cf);
        unsigned ns = 0;
        verdict = isinf(traverse_loop<DIM, ORD, false>(P, cf, false, max_v, ns)) ? 1 : 0;
      } else {
        const unsigned *__restrict__ occ_words = P.occ2;
        unsigned long long amask = 0;
        bool full = false;
        double t = 0;
        int base = 0;
        for (int left = __ldg(P.tcount + n);; left -= UNR, base += UNR) {
          unsigned amb;
          const int st = fx_group<DIM, ORD, UNR, REGION, CHECK>(P, occ_words, C, dt, left, t, amb);
          if (st == 2) {
            verdict = 1;
            break;
          }
          if (amb) {
            if (base + UNR <= 64)
              amask |= (unsigned long long)amb << base;
            else
              full = true;
          }
          if (st == 1) break;
        }
        if (verdict == 0 && (amask != 0 || full)) {
          verdict = 2;
          const int qi = atomicAdd(&S.q_n, 1);
          S.q[qi] = (unsigned char)threadIdx.x;
          S.amask[threadIdx.x] = amask;
          S.n[threadIdx.x] = (unsigned char)n;
          S.full[threadIdx.x] = full ? 1 : 0;
          S.slot[threadIdx.x] = (unsigned)slot;
          S.intrinsic[threadIdx.x] = intrinsic;
        }
      }
    }
    if (verdict != 2 && o.cost) o.cost[slot] = verdict == 1 ? (double)INFINITY : 0.0 + intrinsic;
  }
  __syncthreads();  // B3: the queue is complete; the helper warp takes it from here
}

// Occupancy planning only (no potential map, no yaw control), |U| <= 128 (hcurr slots), stats off.
bool fx_supported(const EnvParams &P) {
  // occ2_sep_k counts the padded map's cells in 32 bits
  return P.occ2 != nullptr && P.occ2_sum <= (1u << 27) && P.pot == nullptr && (P.control & 16) == 0 && P.nU <= kThreads &&
         P.stats == nullptr;
}

cudaError_t launch_expand_fx(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes, const OutPtrs &o,
                             cudaStream_t st) {
  static const int unr_env = [] {
    const char *e = getenv("MPLX_FX_UNR");  // tuning override: 4 or 8 samples per group
    return e ? atoi(e) : 0;
  }();
  static const int minb_env = [] {
    const char *e = getenv("MPLX_FX_MINB");  // tuning: resident CTAs per SM the register budget is cut for
    return e ? atoi(e) : 0;
  }();
  const int unr = unr_env == 4 || unr_env == 8 ? unr_env : (P.maxn <= 15 ? 4 : 8);
  const int npb = kThreads / P.nU;
  const int grid = (n_nodes + npb - 1) / npb;
  const int inv_nU = ((1 << 20) + P.nU - 1) / P.nU;
  return with_dim(P.dim, [&](auto DIM) {
    return with_order(P.control, [&](auto ORD) {
      return with_bool(unr == 8, [&](auto UNR8) {
        return with_bool(o.lattice != nullptr, [&](auto LAT) {
          // the REGION loop tests every sample; otherwise CHECK as in launch_expand_fxn
          return with_bool(P.region_bits != nullptr || P.maxn + 2 > kOcc2Guard, [&](auto CHECK) {
            auto launch = [&](auto MINB, auto REGION) {
              expand_fx_kernel<DIM, ORD, UNR8 ? 8 : 4, MINB, LAT, REGION, CHECK>
                  <<<grid, kFxThreads, 0, st>>>(P, d_nodes, n_nodes, npb, inv_nU, o);
              return cudaGetLastError();
            };
            if constexpr (CHECK) {
              if (P.region_bits != nullptr) return launch(Int<4>(), std::true_type{});
            }
            // MPLX_FX_MINB = 5 or 6 is for the plain 3-D ACC plan
            if constexpr (DIM == 3 && ORD == 2 && !LAT) {
              if (minb_env == 5) return launch(Int<5>(), std::false_type{});
              if (minb_env == 6) return launch(Int<6>(), std::false_type{});
            }
            return launch(Int<4>(), std::false_type{});
          });
        });
      });
    });
  });
}

// The {occupancy word, candidate-summary word} pairs in bricks of the padded map (layout and bits:
// occ2_guard_brick_pair), each half of the buffer holding one word of every pair.
__global__ void pack_occ2_kernel(const uint32_t *__restrict__ occ, size_t nvox, int dim, int nx, int ny, int nz,
                                 uint32_t *__restrict__ out) {
  const size_t npairs = occ2_guard_pair_count(dim, nx, ny, nz);
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < npairs; p += (size_t)gridDim.x * blockDim.x) {
    uint32_t o, s;
    occ2_guard_brick_pair(occ, p, nvox, dim, nx, ny, nz, o, s);
    out[p] = o;
    out[npairs + p] = s;
  }
}

cudaError_t launch_pack_occ2(const uint32_t *d_occ, size_t nvox, int dim, int nx, int ny, int nz, uint32_t *d_out,
                             cudaStream_t st) {
  const size_t npairs = occ2_guard_pair_count(dim, nx, ny, nz);
  int grid = (int)((npairs + 255) / 256);
  if (grid > sm_count() * 16) grid = sm_count() * 16;
  if (grid < 1) grid = 1;
  pack_occ2_kernel<<<grid, 256, 0, st>>>(d_occ, nvox, dim, nx, ny, nz, d_out);
  return cudaGetLastError();
}

}  // namespace mplx
