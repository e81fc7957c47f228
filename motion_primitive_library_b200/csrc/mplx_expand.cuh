// mplx_expand.cuh — device code shared by the expansion kernels (mplx_kernels.cu: register, flat and
// sequential kernels; mplx_deal.cu: the dealing kernel): voxel classification, the cell rule,
// the literal sample loop, phases A/B, intrinsic cost, sample count.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/mplx.h"
#include "mplx_device.cuh"
#include "mplx_kernels.h"
#include "mplx_prim.cuh"
#include "mplx_tunnel.cuh"

namespace mplx {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kNoBlock = 0x7fffffff;

// ---- voxel classification shared by all sample loops ---------------------------------------
// Two steps so that a caller can issue the loads of several samples before consuming any.
// voxel_fetch returns one packed word for a valid in-map index:
//   bits 0..7  the potential value (int8) when a potential map is set, else the occupancy bit
//   bit  8     1 = inside the tunnel (search_region_ empty counts as inside)
// voxel_classify applies env_map.h:104-121 to it: true = the sample blocks the primitive,
// otherwise the potential term is added to `term`.
typedef unsigned int VoxelRaw;
constexpr VoxelRaw kVoxelNone = 0x100u;  // in-region, free
__device__ __forceinline__ VoxelRaw voxel_fetch(const EnvParams &P, int idx) {
  unsigned r = 0x100u;
  if (P.region_bits != nullptr) r = ((__ldg(P.region_bits + (idx >> 5)) >> (idx & 31)) & 1u) << 8;
  if (P.pot != nullptr)
    r |= (unsigned)(unsigned char)__ldg(P.pot + idx);
  else
    r |= (__ldg(P.occ_bits + (idx >> 5)) >> (idx & 31)) & 1u;
  return r;
}
// voxel_fetch with the tunnel bit read from one query's tunnel (mplx_set_batch_regions) in place of
// P.region_bits, which a tunnelled query ignores
__device__ __forceinline__ VoxelRaw voxel_fetch_tunnel(const EnvParams &P, const TunnelView &tv, int idx) {
  const int x = idx % P.mdim[0], yz = idx / P.mdim[0];
  unsigned r = (unsigned)tunnel_has(tv, P.dim, P.mdim, x, yz % P.mdim[1], yz / P.mdim[1]) << 8;
  if (P.pot != nullptr)
    r |= (unsigned)(unsigned char)__ldg(P.pot + idx);
  else
    r |= (__ldg(P.occ_bits + (idx >> 5)) >> (idx & 31)) & 1u;
  return r;
}
__device__ __forceinline__ bool voxel_classify(const EnvParams &P, VoxelRaw r, double dt, double vnorm_w,
                                               double &term) {
  if (!(r & 0x100u)) return true;  // outside the tunnel (env_map.h:104-106)
  if (P.pot != nullptr) {
    const int pv = (int)(signed char)(r & 0xffu);
    if (pv < 100 && pv > 0)
      term += dt * (P.pot_w * pv + vnorm_w);
    else if (pv >= 100)
      return true;
    return false;
  }
  return r & 1u;
}
__device__ __forceinline__ bool voxel_blocks(const EnvParams &P, int idx, double dt, double vnorm_w,
                                             double &term) {
  return voxel_classify(P, voxel_fetch(P, idx), dt, vnorm_w, term);
}

// floatToInt + isOutside + getIndex (map_util.h:103-108, 51-55, 34-41) for one sample.
// pk[] are the sample's position coordinates.  Returns the cell index or -1 when outside.
//
// With the exact quotient y = RN((p - origin)/res) the reference's
//     pn = (int)std::round(RN(y - 0.5));   inside <=> 0 <= pn < dim
// is equivalent to
//     inside <=> 2^-55 < y < dim;          pn = floor(y)
// because y - 0.5 is exact for y >= 0.5, rounds into (-0.5, 0) for 2^-55 < y < 0.5 and to
// exactly -0.5 (-> -1, half away from zero) for 0 <= y <= 2^-55; a tie x = J - 0.5 with J >= 1
// rounds up to J = floor(y).  (tests/arith_identities.cpp: check_cell_rule.)
template <int DIM>
__device__ __forceinline__ int sample_index(const EnvParams &P, const double (&pk)[DIM]) {
  int pn[DIM];
  bool inside = true;
#pragma unroll
  for (int k = 0; k < DIM; k++) {
    const double y = div_exact(pk[k] - P.origin[k], P.res, P.rinv);
    // floor(y) on the (otherwise idle) conversion pipe: saturates for |y| >= 2^31 and gives 0
    // for NaN, both of which the two tests below classify as outside
    pn[k] = __double2int_rd(y);
    inside = inside && (y > 0x1p-55) && ((unsigned)pn[k] < (unsigned)P.mdim[k]);
  }
  if (!inside) return -1;
  int idx = pn[0] + P.mdim[0] * pn[1];
  if (DIM == 3) idx += P.mdim[0] * P.mdim[1] * pn[DIM - 1];
  return idx;
}

// The yaw-alignment term of env_map.h:122-129.
__device__ __forceinline__ double yaw_term(const EnvParams &P, double v0, double v1, double yaw, double dt) {
  if (sqrt(v0 * v0 + v1 * v1) > 1e-5) {
    double sn, cs;
    sincos(yaw, &sn, &cs);
    const double v_value = 1 - dot2_normalized(v0, v1, cs, sn);
    return P.wyaw * v_value * dt;
  }
  return 0.0;
}

// The yaw angle of a primitive is linear in t (pr_yaw_ = [0,0,0,0,u,yaw]: primitive.h:235-248) and the
// sample loop advances t by the same dt every step, so (cos yaw, sin yaw) of consecutive samples differ
// by one fixed rotation: cs/sn hold the current sample's values, dc/ds = cos/sin(yaw_u * dt).  The
// alignment cost is compared at 1e-6 relative (north_star), the recurrence drifts by ~1e-16 per step
// over <= 129 steps; the reference's sincos per sample (~100 instructions in FP64) becomes 6.
struct YawRot {
  double cs, sn, dc, ds;
  __device__ __forceinline__ void init(double yaw_u, double yaw0, double dt) {
    sincos(yaw0, &sn, &cs);
    sincos(yaw_u * dt, &ds, &dc);
  }
  __device__ __forceinline__ void step() {
    const double c2 = cs * dc - sn * ds;
    sn = sn * dc + cs * ds;
    cs = c2;
  }
};
// env_map.h:122-129 with the sample's (cos, sin) given: wyaw * (1 - v_hat . (cos, sin)) * dt when |v| > 1e-5
__device__ __forceinline__ double yaw_term_cs(const EnvParams &P, double v0, double v1, double cs, double sn, double dt) {
  const double nn = sqrt(v0 * v0 + v1 * v1);
  if (nn > 1e-5) return P.wyaw * (1 - (v0 * cs + v1 * sn) / nn) * dt;
  return 0.0;
}

// pt.vel.norm() scaled by gradient_weight_ (env_map.h:115-116); Eigen's unrolled reduction
// associates a 3-vector sum as a0 + (a1 + a2).
template <int DIM>
__device__ __forceinline__ double grad_term(const EnvParams &P, const double (&vel)[DIM]) {
  if (P.grad_w == 0.0) return 0.0;  // gradient_weight_(0) * norm == +0 for a finite norm
  const double n2 = DIM == 2 ? vel[0] * vel[0] + vel[1] * vel[1]
                             : vel[0] * vel[0] + (vel[1] * vel[1] + vel[DIM - 1] * vel[DIM - 1]);
  return P.grad_w * sqrt(n2);
}

// Whether the sample loop evaluates velocities: the yaw term and the gradient term read them.
__host__ __device__ __forceinline__ bool need_vel(const EnvParams &P, bool yaw) {
  return yaw || (P.pot != nullptr && P.grad_w != 0.0);
}

// traverse_primitive, literal per-primitive loop: include/mpl_planner/env/env_map.h:90-132.
// max_v is the caller's max_i pr.max_vel(i) (the reference recomputes it at :91-94).
template <int DIM, int ORD, bool YAW>
__device__ __forceinline__ double traverse_loop(const EnvParams &P, const double *cf, bool need_vel,
                                                double max_v, unsigned &n_samples) {
  using CL = CoefLayout<DIM, ORD, YAW>;
  const double T = P.T;
  const int n = max(5, (int)ceil(max_v * T / P.res));
  double c = 0;
  const double dt = T / n;
  const int NC = CL::ncoef(need_vel);
  for (double t = 0; t < T; t += dt) {
    n_samples++;
    double pk[DIM], vel[DIM];
    eval_pos<DIM, ORD>(cf, t, pk);
    const int idx = sample_index<DIM>(P, pk);
    if (idx < 0) return INFINITY;
    double gterm = 0.0;
    if (need_vel) {
      eval_vel<DIM, ORD>(cf + CL::NCP, t, vel);
      gterm = grad_term<DIM>(P, vel);
    }
    double term = 0.0;
    if (voxel_blocks(P, idx, dt, gterm, term)) return INFINITY;
    c += term;
    if (YAW) {
      if (P.wyaw > 0) c += yaw_term(P, vel[0], vel[1], normalize_angle(cf[NC - 2] * t + cf[NC - 1]), dt);
    }
  }
  return c;
}

// Out-of-line copy for the flat kernel's rare fallback (cf lives in shared memory there).
template <int DIM, int ORD, bool YAW>
__device__ __noinline__ double traverse_loop_cold(const EnvParams *P, const double *cf, bool need_vel,
                                                  double max_v, unsigned *n_samples) {
  unsigned ns = 0;
  const double c = traverse_loop<DIM, ORD, YAW>(*P, cf, need_vel, max_v, ns);
  *n_samples = ns;
  return c;
}

// validate_yaw: include/mpl_basis/primitive.h:503-525
template <int DIM, int ORD, bool YAW>
__device__ __forceinline__ bool validate_yaw(const EnvParams &P, const PrimState<DIM, ORD, YAW> &pr) {
  if (P.yaw_max <= 0) return true;
  const double T = P.T;
  const double pw3T = (T * T) * T;
#pragma unroll
  for (int e = 0; e < 2; e++) {
    const double t = e == 0 ? 0.0 : T;
    const double v0 = pr.ax[0].v(t, e == 0 ? 0.0 : pw3T);
    const double v1 = pr.ax[1].v(t, e == 0 ? 0.0 : pw3T);
    if (v0 != 0 || v1 != 0) {
      const double yaw = normalize_angle(0.0 + pr.yaw_u * t + pr.yaw0);
      double sn, cs;
      sincos(yaw, &sn, &cs);
      const double d = dot2_normalized(v0, v1, cs, sn);
      if (d < P.cos_yaw_max) return false;
    }
  }
  return true;
}

// One successor Waypoint (112 bytes = 7 x 16) to global memory as seven 16-byte stores, the widest
// store sm_90 has, when the destination allows it (cudaMalloc'ed arrays always do): half the store
// instructions and half the partial-sector writes of fourteen 8-byte stores at a 112-byte stride between lanes.
// The stores are streaming (st.global.cs): the 132-byte records are written once and never read by the
// kernel, and at ~0.9 GB per launch they would otherwise sweep the voxel bitmaps out of the L2.
__device__ __forceinline__ void store_waypoint(mplx_waypoint *dst, const mplx_waypoint &w) {
  if ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
    double2 *d = reinterpret_cast<double2 *>(dst);
    __stcs(d + 0, make_double2(w.pos[0], w.pos[1]));
    __stcs(d + 1, make_double2(w.pos[2], w.vel[0]));
    __stcs(d + 2, make_double2(w.vel[1], w.vel[2]));
    __stcs(d + 3, make_double2(w.acc[0], w.acc[1]));
    __stcs(d + 4, make_double2(w.acc[2], w.jrk[0]));
    __stcs(d + 5, make_double2(w.jrk[1], w.jrk[2]));
    __stcs(d + 6, make_double2(w.yaw, w.t));
  } else {
    *dst = w;
  }
}
struct OutPtrs {
  int32_t *count;
  mplx_waypoint *succ;
  double *cost;
  int32_t *action;
  uint64_t *key;
  int32_t *lattice;
};

// hash_value(waypoint) (waypoint.h:93-125) as phase_ab folds it into hcurr: once per node in the fixed-point
// kernels, and the device search's start and goal keys.
template <int DIM, int ORD, bool YAW>
__device__ __forceinline__ uint64_t node_hash(const mplx_waypoint *w) {
  uint64_t h = 0;
#pragma unroll
  for (int k = 0; k < DIM; k++) {
    hash_combine(h, lattice_id(w->pos[k], 0.01, 100.0));
    if (ORD >= 2) hash_combine(h, lattice_id(w->vel[k], 0.1, 10.0));
    if (ORD >= 3) hash_combine(h, lattice_id(w->acc[k], 0.1, 10.0));
    if (ORD >= 4) hash_combine(h, lattice_id(w->jrk[k], 0.1, 10.0));
  }
  if (YAW) hash_combine(h, lattice_id(w->yaw, 0.1, 10.0));
  return h;
}

// Phases A and B for one item (all threads of the CTA must call it: it contains a barrier).
// LAT: the caller asked for the lattice ints (mplx_succ_out.lattice); without it the 13-entry
// array never exists (it would cost 13 registers through phase A).
template <int DIM, int ORD, bool YAW, bool LAT>
__device__ __forceinline__ void phase_ab(const EnvParams &P, const mplx_waypoint *__restrict__ nodes,
                                         int n_nodes, int item, int items, int nU, int node0,
                                         uint32_t *vbits, int words, const OutPtrs &o,
                                         PrimState<DIM, ORD, YAW> &pr, bool &emit, bool &same,
                                         double &max_v, size_t &slot, const uint64_t *s_hcurr = nullptr) {
  const int nl = item / nU;
  const int ci = item - nl * nU;
  const int ni = node0 + nl;
  const bool active = item < items && ni < n_nodes;
  emit = false;
  same = true;
  max_v = 0;
  slot = 0;

  mplx_waypoint tn;
  int lat[LAT ? MPLX_LATTICE_MAX : 1];
  uint64_t key = 0;
  if (active) {
    const mplx_waypoint *cp = nodes + ni;
    const double *u = P.U + (size_t)ci * P.udim;
    // Primitive(curr, U[i], dt): primitive.h:220-256
#pragma unroll
    for (int k = 0; k < DIM; k++) pr.ax[k].build(__ldg(u + k), cp->pos[k], cp->vel[k], cp->acc[k], cp->jrk[k]);
    if (YAW) {
      pr.yaw_u = __ldg(u + DIM);
      pr.yaw0 = cp->yaw;
    }
    // tn = pr.evaluate(dt): primitive.h:321-331 (all four derivative vectors are filled)
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
    // pr_yaw_.p(t) = 0/120*.. + c4*t + c5 with the leading +0 sum (primitive.h:128-131,328)
    if (YAW) tn.yaw = normalize_angle(0.0 + pr.yaw_u * T + pr.yaw0);
    tn.t = cp->t + T;  // env_map.h:161

    // !validate_primitive (primitive.h:449-475) first: the test is pure, and a primitive that fails
    // it is dropped whatever its key, so the lattice key is only computed for the survivors
    bool ok = true;
    if (YAW) ok = validate_yaw<DIM, ORD, YAW>(P, pr);
    // max_vel per axis serves validate_xxx(VEL) (primitive.h:482-496) and traverse (env_map.h:91-94)
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
      // tn == curr  <=>  hash_value(tn) == hash_value(curr)  (waypoint.h:133-135, 93-125)
      // hash_value(curr): per thread, or once per node by the caller (s_hcurr[node in CTA]).  Per thread it is
      // node_hash folded in here axis by axis beside the key: calling node_hash after the key loop instead
      // changes the compiled code of the register, dealing and search kernels.
      uint64_t hcurr = s_hcurr ? s_hcurr[nl] : 0;
      int nl_ = 0;
#pragma unroll
      for (int k = 0; k < DIM; k++) {
        if (!s_hcurr) {
          hash_combine(hcurr, lattice_id(cp->pos[k], 0.01, 100.0));
          if (ORD >= 2) hash_combine(hcurr, lattice_id(cp->vel[k], 0.1, 10.0));
          if (ORD >= 3) hash_combine(hcurr, lattice_id(cp->acc[k], 0.1, 10.0));
          if (ORD >= 4) hash_combine(hcurr, lattice_id(cp->jrk[k], 0.1, 10.0));
        }
        int id = lattice_id(tn.pos[k], 0.01, 100.0);
        hash_combine(key, id);
        if (LAT) lat[nl_++] = id;
        if (ORD >= 2) { id = lattice_id(tn.vel[k], 0.1, 10.0); hash_combine(key, id); if (LAT) lat[nl_++] = id; }
        if (ORD >= 3) { id = lattice_id(tn.acc[k], 0.1, 10.0); hash_combine(key, id); if (LAT) lat[nl_++] = id; }
        if (ORD >= 4) { id = lattice_id(tn.jrk[k], 0.1, 10.0); hash_combine(key, id); if (LAT) lat[nl_++] = id; }
      }
      if (YAW) {
        if (!s_hcurr) hash_combine(hcurr, lattice_id(cp->yaw, 0.1, 10.0));
        const int id = lattice_id(tn.yaw, 0.1, 10.0);
        hash_combine(key, id);
        if (LAT) lat[nl_++] = id;
      }
      if (LAT) {
#pragma unroll
        for (int q = 0; q < MPLX_LATTICE_MAX; q++)
          if (q >= nl_) lat[q] = 0;
      }
      ok = key != hcurr;
    }
    emit = ok;
  }

  // ---- phase B: stable per-node compaction (control order) ----
  const unsigned bal = __ballot_sync(0xffffffffu, emit);
  if ((threadIdx.x & 31) == 0 && (item >> 5) < words) vbits[item >> 5] = bal;
  __syncthreads();
  if (active) {
    const int s = nl * nU;  // first item of my node
    int rank = 0;
    for (int wd = s >> 5; wd <= (item >> 5); wd++) {
      uint32_t m = vbits[wd];
      const int lo = wd << 5;
      if (s > lo) m &= ~0u << (s - lo);
      if (item < lo + 32) m &= (item - lo) ? (~0u >> (32 - (item - lo))) : 0u;
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
}

// calculate_intrinsic_cost: env_base.h:343-345 ; Primitive::J: primitive.h:403-407
template <int DIM, int ORD, bool YAW>
__device__ __forceinline__ double intrinsic_cost(const EnvParams &P, const PrimState<DIM, ORD, YAW> &pr) {
  double J = pr.ax[0].J(P.T);
#pragma unroll
  for (int k = 1; k < DIM; k++) J += pr.ax[k].J(P.T);
  return J + P.w * P.T;
}

// n = max(5, (int)ceil(max_v*T/res)), dt = T/n  (env_map.h:95,98): exact quotient + ceiling;
// T/n from the table for n <= kNMax, a true division beyond it.
__device__ __forceinline__ int sample_count_n(const EnvParams &P, double max_v, double &dt) {
  const double nd = ceil_exact(div_exact(max_v * P.T, P.res, P.rinv));
  const int n = nd < 5.0 ? 5 : (nd < 2.0e9 ? (int)nd : 2000000000);
  dt = n <= kNMax ? __ldg(P.tdt + n) : P.T / n;
  return n;
}

// The cell of one sample as (inside, index): the same rule as sample_index, with the verdict kept
// as a predicate (the six comparisons chain into one predicate register; no index is forced to -1).
template <int DIM>
__device__ __forceinline__ bool sample_cell(const EnvParams &P, const double (&pk)[DIM], int &idx) {
  int pn[DIM];
  bool inside = true;
#pragma unroll
  for (int k = 0; k < DIM; k++) {
    const double y = div_exact(pk[k] - P.origin[k], P.res, P.rinv);
    pn[k] = __double2int_rd(y);  // floor; saturates for |y| >= 2^31, 0 for NaN: both fail a test below
    inside = inside && (y > 0x1p-55) && ((unsigned)pn[k] < (unsigned)P.mdim[k]);
  }
  idx = pn[0] + P.mdim[0] * pn[1];
  if (DIM == 3) idx += P.mdim[0] * P.mdim[1] * pn[DIM - 1];
  return inside;
}

// Iterations of `for (t = 0; t < T; t += dt)` with dt = T/n (env_map.h:98-99): n or n+1 depending on
// how the running sum rounds.  From the table (built by running that very loop, build_ttab_kernel)
// for n <= kNMax, by running the loop beyond it.
__device__ __forceinline__ int sample_loop_count(const EnvParams &P, int n, double dt) {
  if (n <= kNMax) return __ldg(P.tcount + n);
  int k = 0;
  for (double t = 0; t < P.T; t += dt) k++;
  return k;
}

// One group of UNR samples of the reference's loop `for (t = 0; t < T; t += dt)` (env_map.h:99).
// `left` = iterations of that loop not yet visited (sample j of the group exists iff j < left: the
// loop's own `t < T` test, counted instead of re-compared in FP64).  All UNR samples are evaluated
// unconditionally (one past the end or outside the map just gets no load), their voxel loads are
// issued back to back, and two decisions close the group:
//   some existing sample blocks -> 2: the primitive's cost is inf (the reference returns at the
//                                   first such sample; later ones cannot change an inf);
//   the group held the loop's end -> 1: the accumulated cost is in c;
// otherwise the terms of the group were added to c in sample order -> 0, call again with left - UNR.
// n_samples counts what the reference's loop visits (up to and including the first blocking
// sample) and is only maintained when the stats counters are on.
// TUN: the tunnel bit comes from the query's tunnel *tv (voxel_fetch_tunnel) rather than P.region_bits.
template <int DIM, int ORD, bool YAW, int UNR, bool TUN = false>
__device__ __forceinline__ int sample_group(const EnvParams &P, const double (&cf)[CoefLayout<DIM, ORD, YAW>::NCMAX],
                                            bool need_vel, double dt, int left, double &t, double &c,
                                            unsigned &n_samples, YawRot &yr, const TunnelView *tv = nullptr) {
  using CL = CoefLayout<DIM, ORD, YAW>;
  const int NC = CL::ncoef(need_vel);
  const bool plain = !TUN && P.pot == nullptr && P.region_bits == nullptr && !YAW;
  double ts[UNR];
  int idx[UNR];
  bool in[UNR];
  double ycs[YAW ? UNR : 1], ysn[YAW ? UNR : 1];
#pragma unroll
  for (int j = 0; j < UNR; j++) {
    ts[j] = t;
    if (YAW) {
      ycs[j] = yr.cs;
      ysn[j] = yr.sn;
      yr.step();
    }
    double pk[DIM];
    eval_pos<DIM, ORD>(cf, t, pk);
    in[j] = sample_cell<DIM>(P, pk, idx[j]);
    t += dt;  // the reference's running sum
  }
  if (plain) {
    // occupancy planning: the only question per sample is the voxel bit
    unsigned word[UNR];
#pragma unroll
    for (int j = 0; j < UNR; j++) {
      word[j] = 0;
      if (j < left && in[j]) word[j] = __ldg(P.occ_bits + (idx[j] >> 5));
    }
    bool any_blocked = false;
#pragma unroll
    for (int j = 0; j < UNR; j++)
      any_blocked = any_blocked || (j < left && (!in[j] || ((word[j] >> (idx[j] & 31)) & 1u)));
    if (P.stats) {
      bool open = true;  // still before the first blocking sample
#pragma unroll
      for (int j = 0; j < UNR; j++) {
        if (open && j < left) n_samples++;
        open = open && !(j < left && (!in[j] || ((word[j] >> (idx[j] & 31)) & 1u)));
      }
    }
    if (any_blocked) return 2;
    return left <= UNR ? 1 : 0;
  }
  VoxelRaw raw[UNR];
#pragma unroll
  for (int j = 0; j < UNR; j++) {
    raw[j] = kVoxelNone;
    if (j < left && in[j]) raw[j] = TUN ? voxel_fetch_tunnel(P, *tv, idx[j]) : voxel_fetch(P, idx[j]);
  }
  bool blocked[UNR];
  double term[UNR];
#pragma unroll
  for (int j = 0; j < UNR; j++) {
    term[j] = 0.0;
    blocked[j] = !in[j];
    if (j < left && in[j]) {
      double vel[DIM];
      double gterm = 0.0;
      if (need_vel) {
        eval_vel<DIM, ORD>(cf + CL::NCP, ts[j], vel);
        gterm = grad_term<DIM>(P, vel);
      }
      blocked[j] = voxel_classify(P, raw[j], dt, gterm, term[j]);
      if (YAW) {
        if (!blocked[j] && P.wyaw > 0) term[j] += yaw_term_cs(P, vel[0], vel[1], ycs[j], ysn[j], dt);
      }
    }
  }
  bool any_blocked = false;
#pragma unroll
  for (int j = 0; j < UNR; j++) any_blocked = any_blocked || (j < left && blocked[j]);
  if (P.stats) {
    bool open = true;
#pragma unroll
    for (int j = 0; j < UNR; j++) {
      if (open && j < left) n_samples++;
      open = open && !(j < left && blocked[j]);
    }
  }
  if (any_blocked) return 2;
#pragma unroll
  for (int j = 0; j < UNR; j++)
    if (j < left) c += term[j];
  return left <= UNR ? 1 : 0;
}

// Phase C of the register kernel (mplx_kernels.cu) and the edge cost of the device search
// (mplx_search.cu): the reference's loop `for (t = 0; t < T; t += dt)` (env_map.h:99) in groups of UNR
// samples with group-level control flow only (sample_group).  count = iterations of that loop
// (sample_loop_count).  TUN and tv: as sample_group.
template <int DIM, int ORD, bool YAW, int UNR, bool TUN = false>
__device__ __forceinline__ double traverse_groups(const EnvParams &P, const double (&cf)[CoefLayout<DIM, ORD, YAW>::NCMAX],
                                                 bool need_vel, double dt, int count, unsigned &n_samples,
                                                 const TunnelView *tv = nullptr) {
  double c = 0;
  double t = 0;
  YawRot yr;
  if (YAW) yr.init(cf[CoefLayout<DIM, ORD, YAW>::ncoef(need_vel) - 2], cf[CoefLayout<DIM, ORD, YAW>::ncoef(need_vel) - 1], dt);
  for (int left = count;; left -= UNR) {
    const int st = sample_group<DIM, ORD, YAW, UNR, TUN>(P, cf, need_vel, dt, left, t, c, n_samples, yr, tv);
    if (st == 2) return INFINITY;
    if (st == 1) return c;
  }
}

}  // namespace mplx
