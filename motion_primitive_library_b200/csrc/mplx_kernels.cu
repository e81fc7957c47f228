// mplx_kernels.cu — expand(frontier x U): the batched body of env_map<Dim>::get_succ
// (include/mpl_planner/env/env_map.h:147-172) for sm_90a.
//
// Work decomposition.  A CTA of 256 threads covers NPB = 256/|U| whole frontier nodes, one
// thread per (node, control) primitive:
//   phase A  build the primitive (primitive.h:220-256), evaluate the end state tn
//            (:321-331), the dynamic validity (primitive.h:449-525) and, for the survivors, the
//            lattice key (waypoint.h:93-125) in registers;
//   phase B  stable, control-ordered compaction of each node's successors with warp ballots
//            (the push_back order of env_map.h:155-170) and write-out of tn/key/action;
//   phase C  traverse_primitive (env_map.h:90-132), three interchangeable implementations:
//     expand_reg_kernel  (default) thread = primitive, quotients in registers, the reference's
//                        t += dt loop in groups of 4 samples with group-level control flow;
//     expand_flat_kernel the samples of a warp's 32 primitives laid end to end and dealt to the
//                        lanes (quotients staged in shared memory, sample times from the table
//                        that reproduces the running sum, atomicMin of the first blocking sample);
//     expand_seq_kernel  the literal per-primitive loop; serves |U| > 256.
// The occupancy grid is read as 1 bit/voxel (16 MiB at 512^3: L2-resident); potential-field
// planning reads the int8 grid.  No tensor cores: there is no dense contraction on this path.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false  (see mplx_device.cuh).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/mplx.h"
#include "mplx_device.cuh"
#include "mplx_expand.cuh"

namespace mplx {

// ---- sequential kernel (any |U| <= kMaxU) ---------------------------------------------------
template <int DIM, int ORD, bool YAW>
__global__ void __launch_bounds__(kThreads)
expand_seq_kernel(const __grid_constant__ EnvParams P, const mplx_waypoint *__restrict__ nodes, int n_nodes,
                  int npb, const __grid_constant__ OutPtrs o) {
  const bool need_vel = YAW || (P.pot != nullptr && P.grad_w != 0.0);
  __shared__ uint32_t vbits[kMaxU / 32 + 9];
  __shared__ unsigned long long s_stats[2];
  const int nU = P.nU;
  const int items = npb * nU;
  const int node0 = blockIdx.x * npb;
  const int words = (items + 31) >> 5;
  if (threadIdx.x < 2) s_stats[threadIdx.x] = 0;
  for (int base = 0; base < items; base += kThreads) {
    PrimState<DIM, ORD, YAW> pr;
    bool emit, same;
    double max_v;
    size_t slot;
    phase_ab<DIM, ORD, YAW, true>(P, nodes, n_nodes, base + threadIdx.x, items, nU, node0, vbits, words, o, pr, emit,
                            same, max_v, slot);
    unsigned n_samples = 0;
    if (emit) {
      double cf[CoefLayout<DIM, ORD, YAW>::NCMAX];
      fill_coef<DIM, ORD, YAW>(pr, need_vel, cf);
      double cost = same ? 0.0 : traverse_loop<DIM, ORD, YAW>(P, cf, need_vel, max_v, n_samples);
      if (!isinf(cost)) cost += intrinsic_cost<DIM, ORD, YAW>(P, pr);
      if (o.cost) o.cost[slot] = cost;
    }
    if (P.stats) {
      atomicAdd(&s_stats[0], (unsigned long long)n_samples);
      if (emit) atomicAdd(&s_stats[1], 1ull);
    }
    __syncthreads();
  }
  if (threadIdx.x < 2 && P.stats) atomicAdd(&P.stats[threadIdx.x], s_stats[threadIdx.x]);
}

// ---- register kernel (|U| <= 256): thread = primitive through all three phases ----------------
// Phase C keeps the primitive's quotients in registers and walks the reference's own loop
// `for (t = 0; t < T; t += dt)` (env_map.h:99) four samples at a time: the four cell indices are
// computed and their voxel loads issued back to back, then the samples are classified IN ORDER,
// so the first blocking sample ends the primitive exactly where the reference returns inf, the
// potential / yaw sums accumulate in the reference's order, and up to three samples past a block
// are computed for nothing (they are bounds-checked like any other).  No shared-memory staging,
// no atomics; lanes whose primitive is invalid or short idle while the longest one finishes.
// Phase C of the register kernel: the reference's loop `for (t = 0; t < T; t += dt)`
// (env_map.h:99) in groups of UNR samples with group-level control flow only (sample_group,
// mplx_expand.cuh).  count = iterations of that loop (sample_loop_count).
template <int DIM, int ORD, bool YAW, int UNR>
__device__ __forceinline__ double traverse_groups(const EnvParams &P, const double (&cf)[CoefLayout<DIM, ORD, YAW>::NCMAX],
                                                 bool need_vel, double dt, int count, unsigned &n_samples) {
  double c = 0;
  double t = 0;
  YawRot yr;
  if (YAW) yr.init(cf[CoefLayout<DIM, ORD, YAW>::ncoef(need_vel) - 2], cf[CoefLayout<DIM, ORD, YAW>::ncoef(need_vel) - 1], dt);
  for (int left = count;; left -= UNR) {
    const int st = sample_group<DIM, ORD, YAW, UNR>(P, cf, need_vel, dt, left, t, c, n_samples, yr);
    if (st == 2) return INFINITY;
    if (st == 1) return c;
  }
}

template <int DIM, int ORD, bool YAW, bool VEL, int UNR, int MINB, bool LAT>
__global__ void __launch_bounds__(kThreads, MINB)
expand_reg_kernel(const __grid_constant__ EnvParams P, const mplx_waypoint *__restrict__ nodes, int n_nodes,
                  int npb, const __grid_constant__ OutPtrs o) {
  __shared__ uint32_t vbits[9];
  __shared__ unsigned long long s_stats[2];
  const int nU = P.nU;
  const int items = npb * nU;  // <= 256
  const int node0 = blockIdx.x * npb;
  const int words = (items + 31) >> 5;
  if (threadIdx.x < 2) s_stats[threadIdx.x] = 0;
  PrimState<DIM, ORD, YAW> pr;
  bool emit, same;
  double max_v;
  size_t slot;
  phase_ab<DIM, ORD, YAW, LAT>(P, nodes, n_nodes, threadIdx.x, items, nU, node0, vbits, words, o, pr, emit, same,
                               max_v, slot);
  unsigned n_samples = 0;
  if (emit) {
    double cost = 0.0;
    const double intrinsic = intrinsic_cost<DIM, ORD, YAW>(P, pr);  // before the loop: pr dies here
    if (!same) {
      double cf[CoefLayout<DIM, ORD, YAW>::NCMAX];
      fill_coef<DIM, ORD, YAW>(pr, VEL, cf);
      double dt;
      const int n = sample_count_n(P, max_v, dt);
      cost = traverse_groups<DIM, ORD, YAW, UNR>(P, cf, VEL, dt, sample_loop_count(P, n, dt), n_samples);
    }
    if (!isinf(cost)) cost += intrinsic;
    if (o.cost) o.cost[slot] = cost;
  }
  if (P.stats) {
    atomicAdd(&s_stats[0], (unsigned long long)n_samples);
    if (emit) atomicAdd(&s_stats[1], 1ull);
    __syncthreads();
    if (threadIdx.x < 2) atomicAdd(&P.stats[threadIdx.x], s_stats[threadIdx.x]);
  }
}

// ---- flat kernel (|U| <= 256) -----------------------------------------------------------------
// Per-warp shared-memory slab (doubles first so everything stays 8-byte aligned):
//   coef [32][NC]  loop-invariant polynomial quotients of each lane's primitive
//   cost [32]      accumulated potential / yaw cost        dt [32]  T/n
//   n[32] first[32]  (int)        owner[32*maxns] (uint16: lane<<8 | sample k; k <= kNMax < 256)
template <int DIM, int ORD, bool YAW>
struct FlatLayout : CoefLayout<DIM, ORD, YAW> {
  using CoefLayout<DIM, ORD, YAW>::ncoef;
  __host__ __device__ static size_t warp_bytes(bool need_vel, int maxns) {
    size_t b = (size_t)32 * ncoef(need_vel) * 8 + 32 * 8 * 2 + 32 * 4 * 2 + (size_t)32 * maxns * 2;
    return (b + 15) & ~(size_t)15;
  }
};

template <int DIM, int ORD, bool YAW>
__global__ void __launch_bounds__(kThreads, 4)
expand_flat_kernel(const __grid_constant__ EnvParams P, const mplx_waypoint *__restrict__ nodes, int n_nodes,
                   int npb, const __grid_constant__ OutPtrs o, int maxns, int need_vel_i) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ uint32_t vbits[9];
  __shared__ unsigned long long s_stats[2];
  using L = FlatLayout<DIM, ORD, YAW>;
  const bool need_vel = need_vel_i != 0;
  const int NC = L::ncoef(need_vel);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned char *wb = smem + (size_t)warp * L::warp_bytes(need_vel, maxns);
  double *w_coef = reinterpret_cast<double *>(wb);
  double *w_cost = w_coef + 32 * NC;
  double *w_dt = w_cost + 32;
  int *w_n = reinterpret_cast<int *>(w_dt + 32);
  int *w_first = w_n + 32;
  unsigned short *w_owner = reinterpret_cast<unsigned short *>(w_first + 32);

  const int nU = P.nU;
  const int items = npb * nU;  // <= 256
  const int node0 = blockIdx.x * npb;
  const int words = (items + 31) >> 5;
  if (threadIdx.x < 2) s_stats[threadIdx.x] = 0;

  PrimState<DIM, ORD, YAW> pr;
  bool emit, same;
  double max_v;
  size_t slot;
  phase_ab<DIM, ORD, YAW, true>(P, nodes, n_nodes, threadIdx.x, items, nU, node0, vbits, words, o, pr, emit, same,
                                max_v, slot);

  // ---- phase C set-up: coefficient slot, n, sample count ----
  const double T = P.T;
  fill_coef<DIM, ORD, YAW>(pr, need_vel, w_coef + lane * NC);
  int n = 0, ns = 0;
  bool seq = false;
  double cost_seq = 0.0;
  unsigned seq_samples = 0;
  if (emit && !same) {
    // n = max(5, (int)ceil(max_v*T/res))  (env_map.h:95), exact quotient and ceiling
    const double nd = ceil_exact(div_exact(max_v * T, P.res, P.rinv));
    if (nd <= (double)P.maxn) {
      n = max(5, (int)nd);
      ns = __ldg(P.tcount + n);
    } else {
      seq = true;  // beyond the table: literal loop in this lane, coefficients from its smem slot
      cost_seq = traverse_loop_cold<DIM, ORD, YAW>(&P, w_coef + lane * NC, need_vel, max_v, &seq_samples);
    }
  }
  int incl = ns;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  const int start = incl - ns;
  const int S = __shfl_sync(0xffffffffu, incl, 31);
  w_cost[lane] = 0.0;
  w_dt[lane] = __ldg(P.tdt + n);  // T/n, env_map.h:98
  w_n[lane] = n;
  w_first[lane] = kNoBlock;
  for (int k = 0; k < ns; k++) w_owner[start + k] = (unsigned short)((lane << 8) | k);
  __syncwarp();

  // ---- phase C: the warp's samples, dealt round-robin to its lanes, two per lane per trip ----
  // prep: owner/time/coefficients -> cell index (or -1 outside, -2 nothing to do);
  // then the voxel loads of both samples are issued before either is consumed.
  struct Prep {
    int i, k, idx;
    double t;
  };
  auto prep = [&](int s, bool valid) {
    Prep r;
    const unsigned ow = valid ? (unsigned)w_owner[s] : 0u;
    r.i = (int)(ow >> 8);
    r.k = (int)(ow & 255u);
    r.idx = -2;
    r.t = 0.0;
    // an earlier sample of this primitive already blocks: the result is inf whatever this one says
    if (!valid || *(volatile int *)(w_first + r.i) < r.k) return r;
    r.t = __ldg(P.ttab + w_n[r.i] * kTStride + r.k);
    double pk[DIM];
    eval_pos<DIM, ORD>(w_coef + r.i * NC, r.t, pk);
    r.idx = sample_index<DIM>(P, pk);
    return r;
  };
  auto finish = [&](const Prep &r, VoxelRaw raw) {
    if (r.idx == -2) return;
    if (r.idx < 0) {
      atomicMin(w_first + r.i, r.k);
      return;
    }
    const double *cf = w_coef + r.i * NC;
    double vel[DIM];
    double gterm = 0.0;
    if (need_vel) {
      eval_vel<DIM, ORD>(cf + L::NCP, r.t, vel);
      gterm = grad_term<DIM>(P, vel);
    }
    const double dt = w_dt[r.i];
    double term = 0.0;
    if (voxel_classify(P, raw, dt, gterm, term)) {
      atomicMin(w_first + r.i, r.k);
      return;
    }
    if (YAW) {
      if (P.wyaw > 0) term += yaw_term(P, vel[0], vel[1], normalize_angle(cf[NC - 2] * r.t + cf[NC - 1]), dt);
    }
    if (term != 0.0) atomicAdd(w_cost + r.i, term);
  };
  for (int s = lane; s < S; s += 64) {
    const Prep a = prep(s, true);
    const Prep b = prep(s + 32, s + 32 < S);
    VoxelRaw ra = kVoxelNone, rb = kVoxelNone;
    if (a.idx >= 0) ra = voxel_fetch(P, a.idx);
    if (b.idx >= 0) rb = voxel_fetch(P, b.idx);
    finish(a, ra);
    finish(b, rb);
  }
  __syncwarp();

  if (emit) {
    const int fb = w_first[lane];
    double cost = same ? 0.0 : seq ? cost_seq : (fb != kNoBlock ? (double)INFINITY : w_cost[lane]);
    if (!isinf(cost)) cost += intrinsic_cost<DIM, ORD, YAW>(P, pr);
    if (o.cost) o.cost[slot] = cost;
    if (P.stats) {
      // samples the reference loop visits: up to and including the first blocking one
      const unsigned visited = seq ? seq_samples : (fb != kNoBlock ? (unsigned)fb + 1u : (unsigned)ns);
      atomicAdd(&s_stats[0], (unsigned long long)visited);
      atomicAdd(&s_stats[1], 1ull);
    }
  }
  if (P.stats) {
    __syncthreads();
    if (threadIdx.x < 2) atomicAdd(&P.stats[threadIdx.x], s_stats[threadIdx.x]);
  }
}

template <int DIM, int ORD, bool YAW>
static cudaError_t launch_t(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes,
                            const mplx_succ_out &so, cudaStream_t st, int force_seq) {
  const OutPtrs o{so.count, so.succ, so.cost, so.action, so.key, so.lattice};
  const int npb = P.nU >= kThreads ? 1 : kThreads / P.nU;
  const int grid = (n_nodes + npb - 1) / npb;
  if (P.nU > kThreads || force_seq == 1) {
    expand_seq_kernel<DIM, ORD, YAW><<<grid, kThreads, 0, st>>>(P, d_nodes, n_nodes, npb, o);
    return cudaGetLastError();
  }
  const bool nv = YAW || (P.pot != nullptr && P.grad_w != 0.0);
  if (force_seq != 3) {  // register kernel (default)
    // samples in flight per lane: 4, or 2 when every primitive of the plan has a short loop
    // (n <= 15: a group of 4 would mostly run past the end of the loop)
    const bool short_loops = P.maxn <= 15;
    const bool lat = o.lattice != nullptr;
    // groups of 8 samples for plain long-loop planning (measured 0.810 vs 0.828 ms on 512^3 ACC-27, no
    // change on 256^3); MPLX_UNR4=1 restores groups of 4
    static const bool unr8 = getenv("MPLX_UNR4") == nullptr;
#define MPLX_LAUNCH_REG(VEL, UNR, LAT) \
  expand_reg_kernel<DIM, ORD, YAW, VEL, UNR, 4, LAT><<<grid, kThreads, 0, st>>>(P, d_nodes, n_nodes, npb, o)
    if (nv) {
      if (short_loops) { if (lat) MPLX_LAUNCH_REG(true, 2, true); else MPLX_LAUNCH_REG(true, 2, false); }
      else { if (lat) MPLX_LAUNCH_REG(true, 4, true); else MPLX_LAUNCH_REG(true, 4, false); }
    } else {
      if (short_loops) { if (lat) MPLX_LAUNCH_REG(YAW, 2, true); else MPLX_LAUNCH_REG(YAW, 2, false); }
      else { if (lat) MPLX_LAUNCH_REG(YAW, 4, true); else if (unr8) MPLX_LAUNCH_REG(YAW, 8, false); else MPLX_LAUNCH_REG(YAW, 4, false); }
    }
#undef MPLX_LAUNCH_REG
    return cudaGetLastError();
  }
  using L = FlatLayout<DIM, ORD, YAW>;
  const bool need_vel = YAW || (P.pot != nullptr && P.grad_w != 0.0);
  const int maxns = P.maxn + 1;
  const size_t smem = kWarps * L::warp_bytes(need_vel, maxns);
  if (smem > 48 * 1024) {  // the attribute is per device: set it on every such launch (a host-side call)
    cudaError_t e = cudaFuncSetAttribute(expand_flat_kernel<DIM, ORD, YAW>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  expand_flat_kernel<DIM, ORD, YAW><<<grid, kThreads, smem, st>>>(P, d_nodes, n_nodes, npb, o, maxns,
                                                                   need_vel ? 1 : 0);
  return cudaGetLastError();
}

template <int DIM>
static cudaError_t launch_d(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes,
                            const mplx_succ_out &o, cudaStream_t st, int fs) {
  const bool yaw = (P.control & 16) != 0;
  switch (P.control & 15) {
    case MPLX_VEL: return yaw ? launch_t<DIM, 1, true>(P, d_nodes, n_nodes, o, st, fs) : launch_t<DIM, 1, false>(P, d_nodes, n_nodes, o, st, fs);
    case MPLX_ACC: return yaw ? launch_t<DIM, 2, true>(P, d_nodes, n_nodes, o, st, fs) : launch_t<DIM, 2, false>(P, d_nodes, n_nodes, o, st, fs);
    case MPLX_JRK: return yaw ? launch_t<DIM, 3, true>(P, d_nodes, n_nodes, o, st, fs) : launch_t<DIM, 3, false>(P, d_nodes, n_nodes, o, st, fs);
    case MPLX_SNP: return yaw ? launch_t<DIM, 4, true>(P, d_nodes, n_nodes, o, st, fs) : launch_t<DIM, 4, false>(P, d_nodes, n_nodes, o, st, fs);
  }
  return cudaErrorInvalidValue;
}

cudaError_t launch_expand(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes,
                          const mplx_succ_out &o, cudaStream_t st, int force_seq, const FxScratch *fs) {
  if (n_nodes <= 0) return cudaSuccess;
  // large occupancy-planning batches: node-cooperative rows + flat sample items (mplx_fxn.cu)
  static const bool fxn_off = getenv("MPLX_FX_NOROWS") != nullptr;
  if (force_seq == 0 && !fxn_off && fs && fs->q && fxn_supported(P, n_nodes))
    return launch_expand_fxn(P, d_nodes, n_nodes, o, st, fs->q, fs->n, fs->cap);
  // auto (0): the dealing kernel where lanes of the register kernel idle most — controls whose
  // dynamic limits reject many primitives (JRK/SNP) and sample loops with per-sample work beyond the
  // voxel bit (potential field, yaw) — once the batch is large enough for multi-round CTAs; the register kernel otherwise
  // (measured: 512^3 JRK-125 +21 %, ACCxYAW-81 with potential +35 %, plain ACC-27 -3 %).
  // occupancy planning (no potential field, no yaw): the fixed-point kernel (mplx_fx.cu)
  if ((force_seq == 0 || force_seq == 5) && fx_supported(P)) return launch_expand_fx(P, d_nodes, n_nodes, o, st);
  if (force_seq == 5) force_seq = 0;  // not applicable to this plan: the auto rule below
  const bool heavy = (P.control & 15) >= MPLX_JRK || (P.control & 16) != 0 || P.pot != nullptr;
  // (at one round per CTA the dealing kernel only adds overhead: 4096-node JRK launches of the lock-step
  // multi-query driver run 0.37 ms faster on the register kernel, so auto needs >= 2 rounds' worth of CTAs)
  const bool deal = force_seq == 4 || (force_seq == 0 && heavy && (long)n_nodes * P.nU >= 2L * 256 * sm_count() * 4 * 8);
  if (deal && P.nU <= kThreads) {
    static const int rounds_env = [] {
      const char *e = getenv("MPLX_DEAL_ROUNDS");  // tuning override
      return e ? atoi(e) : 0;
    }();
    return launch_expand_deal(P, d_nodes, n_nodes, o, st, rounds_env);
  }
  return P.dim == 2 ? launch_d<2>(P, d_nodes, n_nodes, o, st, force_seq)
                    : launch_d<3>(P, d_nodes, n_nodes, o, st, force_seq);
}

int sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
    cudaGetLastError();  // the launch that follows reports the device error
    return 1;
  }
  return n;
}

// ---- set-up kernels -------------------------------------------------------------------------

// std::vector<bool> search_region_ (env_base.h:400) arrives as one byte per voxel; the grid
// arrives as int8.  Both are packed to 1 bit per voxel (OCC: bit = (map == 100), isOccupied
// map_util.h:48) so the per-sample test is a 4-byte read-only load from an L2-resident array.
template <bool OCC>
__global__ void pack_bits_kernel(const int8_t *__restrict__ bytes, size_t nvox, uint32_t *__restrict__ bits) {
  const size_t nwords = (nvox + 31) >> 5;
  for (size_t wd = (size_t)blockIdx.x * blockDim.x + threadIdx.x; wd < nwords;
       wd += (size_t)gridDim.x * blockDim.x) {
    uint32_t m = 0;
    const size_t b0 = wd << 5;
#pragma unroll 8
    for (int b = 0; b < 32; b++) {
      const size_t i = b0 + b;
      if (i < nvox && (OCC ? bytes[i] == 100 : bytes[i] != 0)) m |= 1u << b;
    }
    bits[wd] = m;
  }
}

cudaError_t launch_pack_bits(const int8_t *d_bytes, size_t nvox, uint32_t *d_bits, bool occ, cudaStream_t st) {
  const size_t nwords = (nvox + 31) >> 5;
  int grid = (int)((nwords + 255) / 256);
  if (grid > sm_count() * 16) grid = sm_count() * 16;
  if (grid < 1) grid = 1;
  if (occ)
    pack_bits_kernel<true><<<grid, 256, 0, st>>>(d_bytes, nvox, d_bits);
  else
    pack_bits_kernel<false><<<grid, 256, 0, st>>>(d_bytes, nvox, d_bits);
  return cudaGetLastError();
}

// Sample-time table: thread n runs the reference loop `for (t = 0; t < T; t += T/n)`
// (env_map.h:98-99) once and records every t_k and the iteration count.
__global__ void build_ttab_kernel(double T, double *__restrict__ ttab, int *__restrict__ tcount,
                                  double *__restrict__ tdt) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n > kNMax) return;
  if (n < 1) {
    tcount[n] = 0;
    tdt[n] = 0.0;
    return;
  }
  const double dt = T / n;
  tdt[n] = dt;
  int k = 0;
  for (double t = 0; t < T; t += dt) {
    if (k < kTStride) ttab[n * kTStride + k] = t;
    k++;
  }
  tcount[n] = k;
}

cudaError_t launch_build_ttab(double T, double *d_ttab, int *d_tcount, double *d_tdt, cudaStream_t st) {
  build_ttab_kernel<<<(kNMax + 1 + 127) / 128, 128, 0, st>>>(T, d_ttab, d_tcount, d_tdt);
  return cudaGetLastError();
}

}  // namespace mplx
