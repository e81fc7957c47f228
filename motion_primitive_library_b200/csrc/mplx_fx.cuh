// mplx_fx.cuh — the fixed-point cell evaluation shared by the occupancy-planning kernels
// (mplx_fx.cu: per-thread phase A with a helper warp; mplx_fxn.cu: node-cooperative rows + flat
// sample items).  See mplx_fx.cu for the derivation and the certainty rule.
#pragma once
#include "mplx_expand.cuh"
#include "mplx_pack.cuh"

namespace mplx {

constexpr double kFxEps = 0x1p-26;       // certainty margin in cells (error bound 2^-30)
constexpr unsigned kFxUnc = 128u;        // 2*eps in units of 2^-32
constexpr double kFxRange = 131072.0;    // 2^17: start coordinates (cells) the error bound covers (see the kernel)

// Cell-unit coefficients of one axis: y(t) = C[ORD] t^ORD + .. + C[1] t + C[0], C[0] carrying
// -origin/res + eps + magic.
template <int ORD>
__device__ __forceinline__ void fx_axis(const Axis<ORD> &ax, double origin, double rinv, double (&C)[ORD + 1]) {
  // position quotients as Primitive1D::p uses them (primitive.h:128-131): c1/24 c2/6 c3/2 c4 c5
  double q[5];
  q[0] = ax.c5;
  q[1] = ax.c4;
  q[2] = ax.c3 / 2;
  q[3] = ax.c2 / 6;
  q[4] = ax.c1 / 24;
#pragma unroll
  for (int i = 1; i <= ORD; i++) C[i] = q[i] * rinv;
  C[0] = (q[0] - origin) * rinv + (kFxMagic + kFxEps);
}

// Whether every sample of one axis stays inside the guard band of occ2 (mplx_pack.cuh): the start cell
// floor(y(0) + eps) lies in the map, [0, mdim), and the displacement y(t) - y(0) over the loop's times
// t in [0, T) is at most G - 2 cells (occ2_band_reach).  The bound is taken from the coefficients alone and
// not from max_vel, whose root filter (primitive.h:353-363) may miss an extremum.  Every sample cell then
// lies in [-G + 1, mdim + G - 1), whatever the rounding of the chain (< 2^-25 cells).
template <int ORD>
__device__ __forceinline__ bool fx_band(const double (&C)[ORD + 1], double T, int mdim) {
  if ((unsigned)(__double2hiint(C[0]) - kFxHiBase) >= (unsigned)mdim) return false;
  return occ2_band_reach<ORD>(C, T) + 2.0 <= (double)kOcc2Guard;
}

// One group of UNR samples, in two halves for a software-pipelined loop: fx_issue evaluates the UNR cells
// starting at time t and issues their word loads; fx_decide consumes the words.  A caller that issues
// group g+1 before deciding group g hides the L2 latency of the voxel words behind the next group's
// arithmetic.  `left` (>= 1) is the number of loop samples from the group's first; samples past it are
// masked.  fx_decide returns 2 when a CERTAIN sample blocks, else 1 when the group held the loop's end,
// else 0; bit j of `amb` = sample j is ambiguous.
// Per sample one 32-bit word is loaded: the occupancy word of the cell when the sample is certain, the
// candidate-summary word when it is uncertain (the two halves of occ2, mplx_pack.cuh).  The word is rotated
// so that the cell's bit lands on bit j, and the group is decided on the OR of those bits.  A cell outside
// the map reads blocked when certain and ambiguous when uncertain: its bit in the guard band is 1 in both
// halves (occ2) or its word stays all-ones (CHECK, REGION).
//   CHECK = false: the primitive's rows passed fx_band, so every loop sample lies in the guard band and its
//                  bit index comes from the high words alone (occ2_sep_k).  Samples past the loop's end
//                  may not, and are not loaded (their word is 0).
//   CHECK = true:  each sample is tested against the map (the same index otherwise).
//   REGION:        the voxel-order occupancy and search-region bitmaps, tested against the map.
__device__ __forceinline__ unsigned rotr_wrap(unsigned x, unsigned s) {
  unsigned r;
  asm("shf.r.wrap.b32 %0, %1, %1, %2;" : "=r"(r) : "r"(x), "r"(s));  // only the low 5 bits of s count
  return r;
}

template <int UNR>
struct FxWords {
  unsigned w[UNR], rot[UNR];
  unsigned uncm;
};

template <int DIM, int ORD, int UNR, bool REGION, bool CHECK>
__device__ __forceinline__ void fx_issue(const EnvParams &P, const unsigned *__restrict__ base,
                                         const double (&C)[DIM][ORD + 1], double dt, int left, double &t,
                                         FxWords<UNR> &G) {
  G.uncm = 0;
#pragma unroll
  for (int j = 0; j < UNR; j++) {
    int hi[DIM];
    unsigned lo[DIM];
    bool inside = true;
#pragma unroll
    for (int a = 0; a < DIM; a++) {
      double h = C[a][ORD];
#pragma unroll
      for (int i = ORD - 1; i >= 1; i--) h = __fma_rn(h, t, C[a][i]);
      const double m = __fma_rn(h, t, C[a][0]);
      hi[a] = __double2hiint(m);  // kFxHiBase + cell
      lo[a] = (unsigned)__double2loint(m);
      if (REGION || CHECK) inside = inside && ((unsigned)(hi[a] - kFxHiBase) < (unsigned)P.mdim[a]);
    }
    const unsigned fr = DIM == 3 ? min(min(lo[0], lo[1]), lo[DIM - 1]) : min(lo[0], lo[1]);
    const unsigned ub = fr < kFxUnc ? 1u : 0u;
    G.uncm += ub << j;
    if (REGION) {
      // no candidate summary for the tunnel: an uncertain sample is ambiguous (word stays all-ones);
      // a certain one is blocked when occupied or outside the tunnel (env_map.h:104-106).  Both bitmaps
      // are in voxel order.
      int idx = (hi[0] - kFxHiBase) + P.mdim[0] * (hi[1] - kFxHiBase);
      if (DIM == 3) idx += P.mdim[0] * P.mdim[1] * (hi[DIM - 1] - kFxHiBase);
      G.rot[j] = (unsigned)(idx - j);  // rotate right by it: the cell's bit lands on bit j
      G.w[j] = 0xffffffffu;
      if (inside && !ub) {
        const unsigned wi = (unsigned)idx >> 5;
        G.w[j] = __ldg(P.occ_bits + wi) | ~__ldg(P.region_bits + wi);
      }
    } else {
      // occ2: the padded pair of the cell, its occupancy (certain) or summary word
      const unsigned k = occ2_sep_k<DIM>(hi, P.occ2_e, P.occ2_k0);
      G.rot[j] = k - j;
      const unsigned *wp = base + ((k >> 5) + (ub ? P.occ2_sum : 0u));
      if (CHECK) {
        G.w[j] = 0xffffffffu;  // a sample past the loop's end may be loaded too: its bit is masked
        if (inside) G.w[j] = __ldg(wp);
      } else {
        G.w[j] = 0u;
        if (j == 0 || j < left) G.w[j] = __ldg(wp);
      }
    }
    t += dt;  // the reference's running sum (env_map.h:99)
  }
}

template <int UNR, bool MASK>
__device__ __forceinline__ int fx_decide(const FxWords<UNR> &G, int left, unsigned &amb) {
  unsigned r = 0;
#pragma unroll
  for (int j = 0; j < UNR; j++) r |= rotr_wrap(G.w[j], G.rot[j]) & (1u << j);
  if (MASK && left < UNR) r &= (1u << left) - 1u;
  amb = r & G.uncm;
  if (r & ~G.uncm) return 2;
  return left <= UNR ? 1 : 0;
}

template <int DIM, int ORD, int UNR, bool REGION, bool CHECK>
__device__ __forceinline__ int fx_group(const EnvParams &P, const unsigned *__restrict__ base,
                                        const double (&C)[DIM][ORD + 1], double dt, int left, double &t, unsigned &amb) {
  FxWords<UNR> G;
  fx_issue<DIM, ORD, UNR, REGION, CHECK>(P, base, C, dt, left, t, G);
  return fx_decide<UNR, REGION || CHECK>(G, left, amb);
}

// The whole sample loop of one primitive, software-pipelined two groups deep.  Returns 1 when a
// certain sample blocks, else 0 with the ambiguous samples in amask (k < 64) / full (some k >= 64).
template <int DIM, int ORD, int UNR, bool REGION, bool CHECK>
__device__ __forceinline__ int fx_traverse(const EnvParams &P, const double (&C)[DIM][ORD + 1], double dt, int count,
                                           unsigned long long &amask, bool &full) {
  constexpr bool MASK = REGION || CHECK;
  const unsigned *__restrict__ base = P.occ2;
  amask = 0;
  full = false;
  double t = 0;
  int left = count, k0 = 0;
  FxWords<UNR> A, B;
  fx_issue<DIM, ORD, UNR, REGION, CHECK>(P, base, C, dt, left, t, A);
  for (;;) {
    unsigned amb;
    int st;
    // ---- group in A; group after it goes to B ----
    if (left > UNR) fx_issue<DIM, ORD, UNR, REGION, CHECK>(P, base, C, dt, left - UNR, t, B);
    st = fx_decide<UNR, MASK>(A, left, amb);
    if (st == 2) return 1;
    if (amb) {
      if (k0 + UNR <= 64) amask |= (unsigned long long)amb << k0; else full = true;
    }
    if (st == 1) return 0;
    left -= UNR;
    k0 += UNR;
    // ---- group in B; group after it goes to A ----
    if (left > UNR) fx_issue<DIM, ORD, UNR, REGION, CHECK>(P, base, C, dt, left - UNR, t, A);
    st = fx_decide<UNR, MASK>(B, left, amb);
    if (st == 2) return 1;
    if (amb) {
      if (k0 + UNR <= 64) amask |= (unsigned long long)amb << k0; else full = true;
    }
    if (st == 1) return 0;
    left -= UNR;
    k0 += UNR;
  }
}

constexpr unsigned kFxSegments = 64;  // the global queue is cut in segments (one counter each) to spread the atomics

// One ambiguous primitive handed to the exact re-evaluation kernel (mplx_fxn.cu).
struct FxAmbRec {
  unsigned slot;             // output slot of the successor
  int node;                  // frontier index
  unsigned short action;     // control index
  unsigned char n;           // max(5, ceil(max_v*T/res)) <= kNMax
  unsigned char full;        // 1: every sample of the loop, 0: the samples of `amask`
  unsigned long long amask;  // ambiguous samples k < 64
};

}  // namespace mplx
