// mplx_fxn.cu — expand_fxn_kernel: the occupancy-planning expansion for large batches, built on the
// fixed-point cell rule of mplx_fx.cuh with two further ideas.
//
// 1. Node-cooperative phase A.  A primitive is Dim independent Primitive1D polynomials
//    (primitive.h:220-256) and the control sets the reference's users build are products of a few
//    values per axis (nested loops, test/test_planner_2d.cpp:49-53), so everything phase A computes
//    per axis — end state, max |vel|/|acc|/|jrk|, lattice ids, the fixed-point coefficients — depends
//    only on (node, axis, value of u on that axis): 9 distinct evaluations per node for U = {-1,0,1}^3
//    instead of 81.  mplx_set_params lists the distinct values of every axis (bitwise) as "rows"; the
//    CTA first fills one shared-memory row per (node, row) — split in three parts over three threads,
//    each calling exactly the functions the per-thread phase A calls, so the same bits — while 9 more
//    threads hash the nodes themselves (hash_value(curr), waypoint.h:93-125).  A primitive thread then
//    only gathers its Dim rows: validity = AND of the row flags, max_v = max of the row maxima,
//    key = hash over the row ids, tn = the row end states.
// 2. A software-pipelined sample loop (fx_traverse, mplx_fx.cuh): the voxel words of group g+1 are
//    requested before group g is decided, so their L2 latency — the top stall of the plain loop — is
//    covered by the next group's arithmetic.
// Ambiguous primitives (an uncertain sample next to an obstacle surface, ~5 %) are appended to a queue
// in global memory and re-evaluated with the exact FP64 chain by fx_resolve_kernel afterwards.
#include <string.h>

#include "mplx_fx.cuh"

namespace mplx {

template <int ORD>
struct FxnRow {
  double st[4];       // Primitive1D::p/v/a/j at T (primitive.h:128-145)
  double C[ORD + 1];  // fixed-point coefficients (fx_axis)
  double mv;          // max_vel (primitive.h:353-363)
  double J;           // Primitive1D::J (primitive.h:92-122)
  int id[4];          // lattice ids of pos, vel, acc, jrk (waypoint.h:96-110)
  uint64_t km[ORD];   // their value-only hash parts (hash_premix), folded into a key per primitive
  unsigned char f0, f1, f2, pad[5];  // flags written by part 0 / 1 / 2
};
// part 0: kSame (c5 == pos, env_map.h:163), kReach (range of the fixed-point bound)
// part 1: kVel within v_max; part 2: kAcc, kJrk within a_max, j_max (primitive.h:482-496)
constexpr unsigned char kSame = 1, kReach = 2, kVel = 1, kAcc = 1, kJrk = 2;


struct FxnWork {
  unsigned rows_n;  // the primitive's three rows (bytes 0..2) and n (byte 3)
  unsigned slot;    // output slot of the successor
};

constexpr int kMaxNpb = kThreads / 9;  // a position control set has >= 3^2 members
struct FxnShared {
  uint64_t hcurr[kMaxNpb];         // hash_value(curr) of the CTA's nodes
  uint64_t ckm[kMaxNpb * 3 * 4];   // hash_premix of their own lattice ids, [node][axis*ORD + field]
  double tcurr[kMaxNpb];           // curr.t
  FxnWork work[kThreads];      // primitives that need sampling, longest loops first
  unsigned char owner[kThreads];  // their phase-A threads (node, control)
  uint32_t vbits[8];
  // stable counting sort by number of sample groups (clamped to 32): members per (warp, bin) and the
  // first sorted position of each (warp, bin)
  unsigned short cnt[kWarps][33], start[kWarps][33];
};
constexpr unsigned kNoWork = 0xffffffffu;
constexpr int kStageBytes = 32 * (int)sizeof(mplx_waypoint);  // one warp's successor records

template <int DIM, int ORD, int UNR, int MINB, bool LAT, bool REGION, bool SORT>
__global__ void __launch_bounds__(kThreads, MINB)
expand_fxn_kernel(const __grid_constant__ EnvParams P, const mplx_waypoint *__restrict__ nodes, int n_nodes, int npb,
                  int inv_nU, int inv_rows, FxAmbRec *__restrict__ amb_q, unsigned *__restrict__ amb_n,
                  unsigned amb_cap, const __grid_constant__ OutPtrs o, int pf_ahead, int stage_off) {
  extern __shared__ __align__(16) unsigned char fx_dyn[];
  FxnRow<ORD> *rows = reinterpret_cast<FxnRow<ORD> *>(fx_dyn);
  __shared__ FxnShared S;
  const int nU = P.nU;
  const int items = npb * nU;  // <= 256
  const int node0 = blockIdx.x * npb;
  const int n_rows = P.n_rows;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  if (SORT) {
    for (int b = threadIdx.x; b < kWarps * 33; b += kThreads) (&S.cnt[0][0])[b] = 0;
    S.work[threadIdx.x].slot = kNoWork;
  }
  // The nodes are read once, from DRAM, at the head of every CTA's dependency chain: ask the L2 for the block
  // of the CTA that starts two waves from now.
  if (pf_ahead > 0 && threadIdx.x < 16) {
    const long long first = ((long long)blockIdx.x + pf_ahead) * npb;
    const char *pfp = reinterpret_cast<const char *>(nodes + first) + 128 * threadIdx.x;
    if (first < n_nodes && pfp < reinterpret_cast<const char *>(nodes + min((long long)n_nodes, first + npb)))
      asm volatile("prefetch.global.L2 [%0];" ::"l"(pfp));
  }

  // ---- phase A0: rows (three parts each) and node hashes ----
  {
    const double T = P.T;
    const int R = npb * n_rows;
    // The warp with the fewest row items also hashes the nodes themselves; its loads go out first so that they
    // overlap the row work (mplx_waypoint = pos[3], vel[3], acc[3], jrk[3], yaw, t: field f of axis a is double 3f+a).
    // (a warp without row items when there is one)
    const int tail = (3 * R) & (kThreads - 1);
    const bool hash_warp = warp == (tail <= kThreads - 32 ? kWarps - 1 : tail >> 5);
    double cx[2] = {0.0, 0.0}, ct = 0.0;
    auto load_ids = [&] {
      constexpr int F = DIM * ORD;
#pragma unroll
      for (int k = 0; k < 2; k++) {
        const int q = lane + 32 * k;
        const int j = q / F, af = q - j * F;
        if (q < npb * F && node0 + j < n_nodes)
          cx[k] = reinterpret_cast<const double *>(nodes + node0 + j)[(af % ORD) * 3 + af / ORD];
      }
      if (lane < npb && node0 + lane < n_nodes) ct = nodes[node0 + lane].t;
    };
    if (hash_warp) load_ids();
    for (int it = threadIdx.x; it < 3 * R; it += kThreads) {
      const int part = it >= 2 * R ? 2 : (it >= R ? 1 : 0);
      const int r = it - part * R;
      const int nl = (r * inv_rows) >> 20;  // r / n_rows
      const int rr = r - nl * n_rows;
      if (node0 + nl >= n_nodes) continue;
      const mplx_waypoint *cp = nodes + node0 + nl;
      const int a = __ldg(P.row_axis + rr);
      Axis<ORD> ax;
      ax.build(__ldg(P.row_u + rr), cp->pos[a], cp->vel[a], cp->acc[a], cp->jrk[a]);
      FxnRow<ORD> &Rw = rows[r];
      if (part == 0) {
        const double origin = a == 0 ? P.origin[0] : (a == 1 ? P.origin[1] : P.origin[2]);
        const double pw3T = (T * T) * T, pw4T = pw3T * T;
        const double pos = ax.template p<true>(T, pw3T, pw4T);
        Rw.st[0] = pos;
        const int id = lattice_id(pos, 0.01, 100.0);
        Rw.id[0] = id;
        Rw.km[0] = hash_premix(id);
        unsigned char f = 0;
        if (ax.c5 == pos) f |= kSame;
        if ((fabs(ax.c5) + fabs(origin)) * P.rinv < kFxRange) f |= kReach;
        Rw.f0 = f;
        Rw.J = ax.J(T);
      } else if (part == 1) {
        const double pw3T = (T * T) * T;
        const double vel = ax.v(T, pw3T);
        Rw.st[1] = vel;
        const int id = ORD >= 2 ? lattice_id(vel, 0.1, 10.0) : 0;
        Rw.id[1] = id;
        if (ORD >= 2) Rw.km[ORD >= 2 ? 1 : 0] = hash_premix(id);
        const double mv = ax.max_vel(T);
        Rw.mv = mv;
        // validate_xxx (primitive.h:482-496): a limit <= 0 passes
        Rw.f1 = (ORD >= 2 && P.v_max > 0 && mv > P.v_max) ? 0 : kVel;
      } else {
        const double origin = a == 0 ? P.origin[0] : (a == 1 ? P.origin[1] : P.origin[2]);
        fx_axis<ORD>(ax, origin, P.rinv, Rw.C);
        const double acc = ax.a(T), jrk = ax.j(T);
        Rw.st[2] = acc;
        Rw.st[3] = jrk;
        Rw.id[2] = ORD >= 3 ? lattice_id(acc, 0.1, 10.0) : 0;
        Rw.id[3] = ORD >= 4 ? lattice_id(jrk, 0.1, 10.0) : 0;
        if (ORD >= 3) Rw.km[ORD >= 3 ? 2 : 0] = hash_premix(Rw.id[2]);
        if (ORD >= 4) Rw.km[ORD >= 4 ? 3 : 0] = hash_premix(Rw.id[3]);
        unsigned char f = kAcc | kJrk;
        if (ORD >= 3 && P.a_max > 0 && ax.max_acc(T) > P.a_max) f &= ~kAcc;
        if (ORD >= 4 && P.j_max > 0 && ax.max_jrk(T) > P.j_max) f &= ~kJrk;
        Rw.f2 = f;
      }
    }
    // hash_value(curr) of the CTA's nodes (waypoint.h:93-125): the lattice ids were loaded above; one exact
    // quotient + premix per lane and round, then one lane per node folds them.
    if (hash_warp) {
      constexpr int F = DIM * ORD;
#pragma unroll
      for (int k = 0; k < 2; k++) {
        const int q = lane + 32 * k;
        if (q < npb * F) {
          const bool is_pos = (q % F) % ORD == 0;
          S.ckm[q] = hash_premix(lattice_id(cx[k], is_pos ? 0.01 : 0.1, is_pos ? 100.0 : 10.0));
        }
      }
      for (int q = lane + 64; q < npb * F; q += 32) {
        const int j = q / F, af = q - j * F;
        const bool is_pos = af % ORD == 0;
        const double x = node0 + j < n_nodes ? reinterpret_cast<const double *>(nodes + node0 + j)[(af % ORD) * 3 + af / ORD] : 0.0;
        S.ckm[q] = hash_premix(lattice_id(x, is_pos ? 0.01 : 0.1, is_pos ? 100.0 : 10.0));
      }
      __syncwarp();
      for (int j = lane; j < npb; j += 32) {
        uint64_t h = 0;
#pragma unroll
        for (int af = 0; af < F; af++) hash_fold(h, S.ckm[j * F + af]);
        S.hcurr[j] = h;
        if (j == lane) S.tcurr[j] = ct;
        else if (node0 + j < n_nodes) S.tcurr[j] = nodes[node0 + j].t;
      }
    }
  }
  __syncthreads();  // B1: rows and node hashes are in shared memory

  // ---- phase A1 (thread = primitive): gather the Dim rows ----
  const int item = threadIdx.x;
  const int nl = (item * inv_nU) >> 20;  // item / nU
  const int ci = item - nl * nU;
  const int ni = node0 + nl;
  const bool active = item < items && ni < n_nodes;
  bool ok = false, same = true, reach = true;
  double max_v = 0;
  uint64_t key = 0;
  int ra[DIM];
#pragma unroll
  for (int a = 0; a < DIM; a++) ra[a] = 0;
  if (active) {
    unsigned f0 = kSame | kReach, f1 = kVel, f2 = kAcc | kJrk;
#pragma unroll
    for (int a = 0; a < DIM; a++) {
      ra[a] = nl * n_rows + __ldg(P.prow + ci * 3 + a);
      const FxnRow<ORD> &Rw = rows[ra[a]];
      f0 &= Rw.f0;
      f1 &= Rw.f1;
      f2 &= Rw.f2;
      if (Rw.mv > max_v) max_v = Rw.mv;
    }
    ok = f1 == kVel && f2 == (kAcc | kJrk);
    same = (f0 & kSame) != 0;
    reach = (f0 & kReach) != 0;
    if (ok) {
#pragma unroll
      for (int a = 0; a < DIM; a++) {
        const FxnRow<ORD> &Rw = rows[ra[a]];
#pragma unroll
        for (int f = 0; f < ORD; f++) hash_fold(key, Rw.km[f]);
      }
    }
  }
  // tn == curr  <=>  hash_value(tn) == hash_value(curr)  (waypoint.h:133-135)
  const bool emit = ok && key != S.hcurr[nl];

  // sample loop of this primitive: n and its iteration count
  int n = 0, count = 0;
  double dt = 0.0;
  const bool literal = emit && !same && !reach;  // outside the range of the fixed-point bound (rare)
  bool beyond = false;                           // beyond the sample-time table (rare)
  if (emit && !same) {
    n = sample_count_n(P, max_v, dt);
    beyond = n > kNMax;
    if (!beyond && !literal) count = __ldg(P.tcount + n);
  }
  // CTA-wide counting sort of the primitives that need sampling by their number of sample groups,
  // longest first: the lanes of a warp then run loops of (nearly) the same length instead of idling
  // until the warp's longest one ends.  Which lane samples a primitive does not enter any result.
  // The sort is stable (thread order kept inside a bin), so the lanes of a warp still hold primitives
  // of the same few nodes and their voxel words share sectors.
  // SORT pays where many lanes would idle (JRK/SNP: half the primitives fail the dynamic limits, cfg3
  // 2.16 -> 1.85 ms); for ACC-27 the exchange and its barrier cost more than the idle lanes.
  const int g = (count + UNR - 1) / UNR;
  const int gk = g > 32 ? 32 : g;
  int bin_rank = 0;
  if (SORT) {
    const unsigned peers = __match_any_sync(0xffffffffu, gk);
    bin_rank = __popc(peers & ((1u << lane) - 1u));
    if (gk > 0 && bin_rank == 0) S.cnt[warp][gk] = (unsigned short)__popc(peers);
  }

  // ---- phase B: stable per-node compaction (control order) ----
  const unsigned bal = __ballot_sync(0xffffffffu, emit);
  if (lane == 0) S.vbits[warp] = bal;
  __syncthreads();  // B2
  if (SORT) {
    if (warp == 0) {
      // lane l owns bin l+1: members per warp, bins sorted descending
      unsigned c[kWarps], tot = 0;
#pragma unroll
      for (int w = 0; w < kWarps; w++) {
        c[w] = S.cnt[w][lane + 1];
        tot += c[w];
      }
      unsigned above = tot;  // inclusive suffix sum over the bins >= mine
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const unsigned v = __shfl_down_sync(0xffffffffu, above, d);
        if (lane + d < 32) above += v;
      }
      unsigned at = above - tot;
#pragma unroll
      for (int w = 0; w < kWarps; w++) {
        S.start[w][lane + 1] = (unsigned short)at;
        at += c[w];
      }
    }
    __syncthreads();  // B2b: sorted positions are known
  }
  size_t slot = 0;
  double intrinsic = 0.0;
  if (active) {
    const int s = nl * nU;  // first item of my node
    int rank = 0;
    if (nU <= 32) {
      // the node's items sit in this warp and at most the one before it
      const unsigned below = (1u << lane) - 1u;
      if ((s >> 5) == warp) {
        rank = __popc(bal & below & (~0u << (s & 31)));
      } else {
        rank = __popc(bal & below) + __popc(S.vbits[warp - 1] >> (s & 31));
      }
    } else {
      for (int wd = s >> 5; wd <= (item >> 5); wd++) {
        uint32_t m = S.vbits[wd];
        const int lo = wd << 5;
        if (s > lo) m &= ~0u << (s - lo);
        if (item < lo + 32) m &= (1u << (item - lo)) - 1u;
        rank += __popc(m);
      }
    }
    if (ci == nU - 1) o.count[ni] = rank + (emit ? 1 : 0);
    if (o.succ && emit) {
      mplx_waypoint tn;
#pragma unroll
      for (int k = 0; k < 3; k++) {
        if (k < DIM) {
          const FxnRow<ORD> &Rw = rows[ra[k < DIM ? k : 0]];
          tn.pos[k] = Rw.st[0];
          tn.vel[k] = Rw.st[1];
          tn.acc[k] = Rw.st[2];
          tn.jrk[k] = Rw.st[3];
        } else {
          tn.pos[k] = tn.vel[k] = tn.acc[k] = tn.jrk[k] = 0.0;
        }
      }
      tn.yaw = 0.0;
      tn.t = S.tcurr[nl] + P.T;  // env_map.h:161
      if (stage_off >= 0) {
        // the warp's records, compacted in lane order (= slot order), wait in shared memory for the bulk copies below
        double2 *sp = reinterpret_cast<double2 *>(fx_dyn + stage_off + warp * kStageBytes +
                                                  __popc(bal & ((1u << lane) - 1u)) * (int)sizeof(mplx_waypoint));
        sp[0] = make_double2(tn.pos[0], tn.pos[1]);
        sp[1] = make_double2(tn.pos[2], tn.vel[0]);
        sp[2] = make_double2(tn.vel[1], tn.vel[2]);
        sp[3] = make_double2(tn.acc[0], tn.acc[1]);
        sp[4] = make_double2(tn.acc[2], tn.jrk[0]);
        sp[5] = make_double2(tn.jrk[1], tn.jrk[2]);
        sp[6] = make_double2(tn.yaw, tn.t);
      } else {
        // 128-bit stores (store_waypoint).  (Staging the CTA's records in shared memory for a coalesced copy-out
        // by the threads themselves was measured: slower — the extra pass and barrier cost more than it saves.)
        store_waypoint(o.succ + (size_t)ni * nU + rank, tn);
      }
    }
    if (emit) {
      slot = (size_t)ni * nU + rank;
      if (o.action) __stcs(o.action + slot, ci);
      if (o.key) __stcs(reinterpret_cast<unsigned long long *>(o.key + slot), (unsigned long long)key);
      if (LAT && o.lattice) {
        int q = 0;
#pragma unroll
        for (int a = 0; a < DIM; a++) {
          const FxnRow<ORD> &Rw = rows[ra[a]];
#pragma unroll
          for (int f = 0; f < ORD; f++) o.lattice[slot * MPLX_LATTICE_MAX + q++] = Rw.id[f];
        }
        for (; q < MPLX_LATTICE_MAX; q++) o.lattice[slot * MPLX_LATTICE_MAX + q] = 0;
      }
      // calculate_intrinsic_cost (env_base.h:343-345): the axes' J in axis order, + w*T
      double J = rows[ra[0]].J;
#pragma unroll
      for (int a = 1; a < DIM; a++) J += rows[ra[a]].J;
      intrinsic = J + P.w * P.T;
    }
  }

  // The records leave through the bulk-copy engine (cp.async.bulk, shared -> global): the emitting lanes of one
  // node hold consecutive slots, so each node's part of the warp is ONE contiguous copy issued by its first
  // lane, and the 112-byte records never pass the L1's tag stage (as per-lane stores they cost it as many
  // look-ups as all voxel loads of the kernel).
  bool bulk_issued = false;
  if (stage_off >= 0 && o.succ) {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // my generic-proxy writes, before the async reads
    __syncwarp();
    const unsigned peers = __match_any_sync(0xffffffffu, nl) & bal;  // emitting lanes of my node in this warp
    if (emit && lane == __ffs(peers) - 1) {
      const unsigned bytes = (unsigned)__popc(peers) * (unsigned)sizeof(mplx_waypoint);
      const unsigned src = (unsigned)__cvta_generic_to_shared(
          fx_dyn + stage_off + warp * kStageBytes + __popc(bal & ((1u << lane) - 1u)) * (int)sizeof(mplx_waypoint));
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(o.succ + slot), "r"(src), "r"(bytes)
                   : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      bulk_issued = true;
    }
  }

  // my work record: published at its sorted position, or kept
  FxnWork wk;
  wk.rows_n = (unsigned)ra[0] | ((unsigned)ra[1] << 8) | ((unsigned)(DIM == 3 ? ra[DIM - 1] : 0) << 16) | ((unsigned)n << 24);
  wk.slot = g > 0 ? (unsigned)slot : kNoWork;
  int wowner = threadIdx.x;
  if (SORT && g > 0) {
    const int pos = (int)S.start[warp][gk] + bin_rank;
    S.work[pos] = wk;
    S.owner[pos] = (unsigned char)threadIdx.x;
  }
  // primitives that are not sampled: curr.pos == tn.pos (cost 0 + intrinsic, env_map.h:163-165) or the
  // rare literal-loop cases
  if (emit && g == 0) {
    int v = 0;
    if (literal || beyond) {
      PrimState<DIM, ORD, false> pr;
      const mplx_waypoint *cp = nodes + ni;
      const double *u = P.U + (size_t)ci * P.udim;
#pragma unroll
      for (int k = 0; k < DIM; k++) pr.ax[k].build(__ldg(u + k), cp->pos[k], cp->vel[k], cp->acc[k], cp->jrk[k]);
      double cf[CoefLayout<DIM, ORD, false>::NCMAX];
      fill_coef<DIM, ORD, false>(pr, false, cf);
      unsigned ns = 0;
      v = isinf(traverse_loop<DIM, ORD, false>(P, cf, false, max_v, ns)) ? 1 : 0;
    }
    if (o.cost) o.cost[slot] = v == 1 ? (double)INFINITY : 0.0 + intrinsic;
  }
  if (SORT) {
    __syncthreads();  // B3: the sorted work list is complete
    wk = S.work[threadIdx.x];
    wowner = S.owner[threadIdx.x];
  }

  // ---- phase C (thread = work item): the fixed-point sample loop, two groups in flight ----
  int verdict = -1;  // 0 free, 1 blocked, 2 ambiguous, 3 literal loop (queue full)
  unsigned long long amask = 0;
  bool full = false;
  unsigned wslot = 0;
  int wn = 0;
  double wintr = 0.0;
  if (wk.slot != kNoWork) {
    wslot = wk.slot;
    wn = (int)(wk.rows_n >> 24);
    int wr[DIM];
    wr[0] = wk.rows_n & 255u;
    wr[1] = (wk.rows_n >> 8) & 255u;
    if (DIM == 3) wr[DIM - 1] = (wk.rows_n >> 16) & 255u;
    double C[DIM][ORD + 1];
#pragma unroll
    for (int a = 0; a < DIM; a++) {
      const FxnRow<ORD> &Rw = rows[wr[a]];
#pragma unroll
      for (int i = 0; i <= ORD; i++) C[a][i] = Rw.C[i];
    }
    // calculate_intrinsic_cost (env_base.h:343-345) again from the rows: the same sum as the owner's
    double J = rows[wr[0]].J;
#pragma unroll
    for (int a = 1; a < DIM; a++) J += rows[wr[a]].J;
    wintr = J + P.w * P.T;
    verdict = fx_traverse<DIM, ORD, UNR, REGION>(P, C, __ldg(P.tdt + wn), __ldg(P.tcount + wn), amask, full);
    if (verdict == 0 && (amask != 0 || full)) verdict = 2;
  }
  // warp-aggregated append to this CTA's segment of the global queue
  const unsigned am = __ballot_sync(0xffffffffu, verdict == 2);
  if (am) {
    const unsigned seg = blockIdx.x & (kFxSegments - 1);
    const unsigned segcap = amb_cap / kFxSegments;
    unsigned base = 0;
    const int leader = __ffs(am) - 1;
    if (lane == leader) base = atomicAdd(amb_n + seg, (unsigned)__popc(am));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (verdict == 2) {
      const unsigned pos = base + __popc(am & ((1u << lane) - 1u));
      if (pos < segcap) {
        FxAmbRec rec;
        const int onl = (wowner * inv_nU) >> 20;
        rec.slot = wslot;
        rec.node = node0 + onl;
        rec.action = (unsigned short)(wowner - onl * nU);
        rec.n = (unsigned char)wn;
        rec.full = full ? 1 : 0;
        rec.amask = amask;
        amb_q[(size_t)seg * segcap + pos] = rec;
      } else {
        verdict = 3;  // segment full: decide here with the literal loop
      }
    }
  }
  if (verdict == 3) {
    const int onl = (wowner * inv_nU) >> 20;
    PrimState<DIM, ORD, false> pr;
    const mplx_waypoint *cp = nodes + node0 + onl;
    const double *u = P.U + (size_t)(wowner - onl * nU) * P.udim;
    double mv = 0;
#pragma unroll
    for (int k = 0; k < DIM; k++) {
      pr.ax[k].build(__ldg(u + k), cp->pos[k], cp->vel[k], cp->acc[k], cp->jrk[k]);
      const double m1 = pr.ax[k].max_vel(P.T);
      if (m1 > mv) mv = m1;
    }
    double cf[CoefLayout<DIM, ORD, false>::NCMAX];
    fill_coef<DIM, ORD, false>(pr, false, cf);
    unsigned ns = 0;
    verdict = isinf(traverse_loop<DIM, ORD, false>(P, cf, false, mv, ns)) ? 1 : 0;
  }
  if ((verdict == 0 || verdict == 1) && o.cost) __stcs(o.cost + wslot, verdict == 1 ? (double)INFINITY : 0.0 + wintr);
  // the staging buffer must outlive the copies that read it
  if (bulk_issued) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// Exact re-evaluation of the queued primitives: a thread rebuilds the exact quotients from (node,
// action) with the code phase A uses, walks the ambiguous samples with eval_pos + sample_cell at the
// loop's own times (sample-time table), and writes the primitive's cost.
template <int DIM, int ORD, bool REGION>
__global__ void __launch_bounds__(128)
fx_resolve_kernel(const __grid_constant__ EnvParams P, const mplx_waypoint *__restrict__ nodes,
                  const FxAmbRec *__restrict__ amb_q, const unsigned *__restrict__ amb_n, unsigned amb_cap,
                  double *__restrict__ cost) {
  // grid = kFxSegments * k CTAs: CTA b walks segment b % kFxSegments with its k-1 siblings
  const unsigned seg = blockIdx.x & (kFxSegments - 1);
  const unsigned segcap = amb_cap / kFxSegments;
  unsigned total = amb_n[seg];
  if (total > segcap) total = segcap;
  const unsigned sib = blockIdx.x / kFxSegments, nsib = gridDim.x / kFxSegments;
  for (unsigned i = sib * blockDim.x + threadIdx.x; i < total; i += nsib * blockDim.x) {
    const FxAmbRec rec = amb_q[(size_t)seg * segcap + i];
    const mplx_waypoint *cp = nodes + rec.node;
    const double *u = P.U + (size_t)rec.action * P.udim;
    PrimState<DIM, ORD, false> pr;  // Primitive(curr, U[action], dt): primitive.h:220-256
#pragma unroll
    for (int k = 0; k < DIM; k++) pr.ax[k].build(__ldg(u + k), cp->pos[k], cp->vel[k], cp->acc[k], cp->jrk[k]);
    double cf[CoefLayout<DIM, ORD, false>::NCMAX];
    fill_coef<DIM, ORD, false>(pr, false, cf);
    const int n = rec.n;
    const double *tt = P.ttab + (size_t)n * kTStride;
    unsigned long long m = rec.amask;
    const int count = __ldg(P.tcount + n);
    const bool full = rec.full != 0;
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
    if (cost) cost[rec.slot] = blocked ? (double)INFINITY : 0.0 + intrinsic_cost<DIM, ORD, false>(P, pr);
  }
}

template <int DIM, int ORD>
static cudaError_t launch_fxn_t(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes, const mplx_succ_out &so,
                                cudaStream_t st, FxAmbRec *amb_q, unsigned *amb_n, unsigned amb_cap) {
  const OutPtrs o{so.count, so.succ, so.cost, so.action, so.key, so.lattice};
  const int npb = kThreads / P.nU;
  const int grid = (n_nodes + npb - 1) / npb;
  const bool lat = o.lattice != nullptr;
  const bool region = P.region_bits != nullptr;
  const int inv_nU = ((1 << 20) + P.nU - 1) / P.nU;
  const int inv_rows = ((1 << 20) + P.n_rows - 1) / P.n_rows;
  const int rows_bytes = (int)(((size_t)npb * P.n_rows * sizeof(FxnRow<ORD>) + 15) & ~(size_t)15);
  static const int sort_env = [] { const char *v = getenv("MPLX_FXN_SORT"); return v ? atoi(v) : -1; }();  // tuning
  const bool sort = sort_env >= 0 ? sort_env != 0 : ORD >= 3;
  // staging of the successor records for the bulk copies (expand_fxn_kernel): destination 16-byte aligned
  // The sorted path (JRK-125 with the CTA sort) keeps the per-lane stores: on that workload the bulk copies
  // were measured slower.
  static const int bulk_env = [] { const char *v = getenv("MPLX_FXN_BULK"); return v ? atoi(v) : -1; }();  // tuning / A-B
  const bool bulk = (bulk_env >= 0 ? bulk_env != 0 : !sort) && o.succ != nullptr &&
                    (reinterpret_cast<uintptr_t>(o.succ) & 15u) == 0;
  const int stage_off = bulk ? rows_bytes : -1;
  const size_t smem = (size_t)rows_bytes + (bulk ? (size_t)kWarps * kStageBytes : 0);
  cudaError_t e = cudaMemsetAsync(amb_n, 0, sizeof(unsigned) * kFxSegments, st);
  if (e != cudaSuccess) return e;
  // Keep the voxel bitmaps in the L2's persisting carve-out: every CTA of every launch re-reads them while
  // ~0.9 GB of successor records stream through the same cache (mplx_set_map sized the carve-out).
  static const bool no_window = getenv("MPLX_NO_L2_WINDOW") != nullptr;  // tuning / A-B
  if (!no_window && P.occ2_bytes > 0) {
    cudaStreamAttrValue av;
    memset(&av, 0, sizeof av);
    av.accessPolicyWindow.base_ptr = const_cast<uint2 *>(P.occ2);
    av.accessPolicyWindow.num_bytes = P.occ2_bytes;
    av.accessPolicyWindow.hitRatio = 1.0f;
    av.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    av.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    if (cudaStreamSetAttribute(st, cudaStreamAttributeAccessPolicyWindow, &av) != cudaSuccess) cudaGetLastError();
  }
  static const int carve = [] { const char *v = getenv("MPLX_FXN_CARVE"); return v ? atoi(v) : -1; }();  // tuning: % of 228 KB
  // CTAs ahead (0 = off); default: two waves of 4 CTAs per SM
  static const int pf_env = [] { const char *v = getenv("MPLX_FXN_PREFETCH"); return v ? atoi(v) : -1; }();
  const int pf_ahead = pf_env >= 0 ? pf_env : 2 * 4 * sm_count();
  static const int unr_env = [] { const char *v = getenv("MPLX_FXN_UNR"); return v ? atoi(v) : 0; }();    // tuning
  static const int minb_env = [] { const char *v = getenv("MPLX_FXN_MINB"); return v ? atoi(v) : 0; }();  // tuning
#define MPLX_LAUNCH_FXN_S(UNR, MINB, LAT, REGION, SORT)                                                         \
  do {                                                                                                          \
    if (smem > 32 * 1024) { /* static + dynamic may pass the 48 KB default */                                   \
      e = cudaFuncSetAttribute(expand_fxn_kernel<DIM, ORD, UNR, MINB, LAT, REGION, SORT>,                       \
                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);                         \
      if (e != cudaSuccess) return e;                                                                           \
    }                                                                                                           \
    if (carve >= 0) {                                                                                           \
      e = cudaFuncSetAttribute(expand_fxn_kernel<DIM, ORD, UNR, MINB, LAT, REGION, SORT>,                       \
                               cudaFuncAttributePreferredSharedMemoryCarveout, carve);                          \
      if (e != cudaSuccess) return e;                                                                           \
    }                                                                                                           \
    expand_fxn_kernel<DIM, ORD, UNR, MINB, LAT, REGION, SORT><<<grid, kThreads, smem, st>>>(                    \
        P, d_nodes, n_nodes, npb, inv_nU, inv_rows, amb_q, amb_n, amb_cap, o, pf_ahead, stage_off);                        \
  } while (0)
#define MPLX_LAUNCH_FXN(UNR, MINB, LAT, REGION)                     \
  do {                                                              \
    if (sort) MPLX_LAUNCH_FXN_S(UNR, MINB, LAT, REGION, true);      \
    else MPLX_LAUNCH_FXN_S(UNR, MINB, LAT, REGION, false);          \
  } while (0)
  if (region) { if (lat) MPLX_LAUNCH_FXN(4, 4, true, true); else MPLX_LAUNCH_FXN(4, 4, false, true); }
  else if (lat) MPLX_LAUNCH_FXN(4, 4, true, false);
  else if (unr_env == 8 && minb_env == 3) MPLX_LAUNCH_FXN(8, 3, false, false);
  else if (unr_env == 4 && minb_env == 3) MPLX_LAUNCH_FXN(4, 3, false, false);
  else if (unr_env == 8) MPLX_LAUNCH_FXN(8, 4, false, false);
  else if (minb_env == 5) MPLX_LAUNCH_FXN(4, 5, false, false);
  else MPLX_LAUNCH_FXN(4, 4, false, false);
#undef MPLX_LAUNCH_FXN
#undef MPLX_LAUNCH_FXN_S
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int rgrid = kFxSegments * 8;
  if (region)
    fx_resolve_kernel<DIM, ORD, true><<<rgrid, 128, 0, st>>>(P, d_nodes, amb_q, amb_n, amb_cap, o.cost);
  else
    fx_resolve_kernel<DIM, ORD, false><<<rgrid, 128, 0, st>>>(P, d_nodes, amb_q, amb_n, amb_cap, o.cost);
  return cudaGetLastError();
}

// The rows must pay against Dim evaluations per control, everything must fit shared memory, and the
// batch must be worth two launches.
bool fxn_supported(const EnvParams &P, int n_nodes) {
  if (!fx_supported(P) || P.n_rows <= 0 || P.nU > kThreads) return false;
  if (P.n_rows * 2 > P.dim * P.nU) return false;
  const int npb = kThreads / P.nU;
  if (npb * P.n_rows > 255 || npb > kMaxNpb) return false;  // row indices are bytes; node tables of FxnShared
  const size_t smem = (size_t)npb * P.n_rows * 128;
  if (smem > 64 * 1024) return false;
  return (long)n_nodes * P.nU >= 64L * kThreads;
}

cudaError_t launch_expand_fxn(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes, const mplx_succ_out &o,
                              cudaStream_t st, void *amb_q, unsigned *amb_n, unsigned amb_cap) {
  if (n_nodes <= 0) return cudaSuccess;
  FxAmbRec *q = static_cast<FxAmbRec *>(amb_q);
#define MPLX_FXN_ORD(DIM)                                                                         \
  switch (P.control & 15) {                                                                       \
    case MPLX_VEL: return launch_fxn_t<DIM, 1>(P, d_nodes, n_nodes, o, st, q, amb_n, amb_cap);     \
    case MPLX_ACC: return launch_fxn_t<DIM, 2>(P, d_nodes, n_nodes, o, st, q, amb_n, amb_cap);     \
    case MPLX_JRK: return launch_fxn_t<DIM, 3>(P, d_nodes, n_nodes, o, st, q, amb_n, amb_cap);     \
    case MPLX_SNP: return launch_fxn_t<DIM, 4>(P, d_nodes, n_nodes, o, st, q, amb_n, amb_cap);     \
  }
  if (P.dim == 2) {
    MPLX_FXN_ORD(2)
  } else {
    MPLX_FXN_ORD(3)
  }
#undef MPLX_FXN_ORD
  return cudaErrorInvalidValue;
}

size_t fx_amb_record_bytes() { return sizeof(FxAmbRec); }

}  // namespace mplx
