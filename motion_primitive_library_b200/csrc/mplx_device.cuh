// mplx_device.cuh — device-side arithmetic of the node-expansion path (sm_90a).
//
// Everything here must reproduce the reference's IEEE-754 double results bit for bit where
// they feed a lattice key, so this translation unit is compiled with -fmad=false (no FMA
// contraction: the reference build has none, CMakeLists.txt:8) and uses true divisions,
// round-half-away (round()), and the reference's operand association.  Citations are
// path:line relative to the reference checkout.
#pragma once
#include <limits.h>
#include <stdint.h>

namespace mplx {

// Kernel-visible copy of the env state (env_base.h:368-400, env_map.h:288-296,
// map_util.h:300-313).  Passed by value as a kernel parameter.
struct EnvParams {
  int dim, control, nU, udim;
  double T, w, wyaw;
  double v_max, a_max, j_max, yaw_max;
  double cos_yaw_max;  // cos(yaw_max) evaluated on the host (primitive.h:521 calls libm cos)
  int mdim[3];
  double origin[3];
  double res;
  double rinv;     // RN(1/res), host-computed (exact-quotient correction, see div_exact)
  double dimd[3];  // (double)mdim[k]
  double pot_w, grad_w;
  const int8_t *map;           // x-fastest int8 grid in HBM
  const int8_t *pot;           // potential grid or nullptr
  const uint32_t *region_bits; // 1 bit / voxel (bit i of word i>>5) or nullptr
  const double *U;             // nU*udim
  unsigned long long *stats;   // [0]=samples visited, [1]=successors emitted; or nullptr
  const uint32_t *occ_bits;    // 1 bit / voxel: map[idx] == 100 (isOccupied, map_util.h:48)
  // Sample-time table of `for (t = 0; t < T; t += T/n)` (env_map.h:98-99): row n holds the
  // running-sum times t_k, tcount[n] their number (n or n+1).  Depends on T only.
  const double *ttab;          // [(kNMax+1) * kTStride]
  const int *tcount;           // [kNMax+1]
  const double *tdt;           // [kNMax+1]  T/n (env_map.h:98)
  int maxn;                    // largest n the flat sample phase accepts (<= kNMax)
  // {occupancy word, candidate-summary word} pairs of the fixed-point kernels (mplx_fx.cu), in bricks of
  // the map padded by a guard band, occupancy half first (layout: mplx_pack.cuh)
  const uint32_t *occ2;
  unsigned occ2_sum;  // words of each half: the summary word of pair p is occ2[occ2_sum + p]
  size_t occ2_bytes;  // bytes of occ2 (from its start) an L2 persisting carve-out was granted for, else 0
  // the per-axis terms of a cell's bit index from the high words of the fixed-point sample loop
  // (occ2_sep_k, occ2_sep_terms with H = kFxHiBase)
  unsigned occ2_e[3], occ2_k0;
  // Per-axis value tables of U for the node-cooperative kernel (mplx_fx.cu): the distinct values of
  // U[.][a] (bitwise) of all axes listed one after the other as "rows"; U[i][a] == row_u[prow[3*i+a]].
  const unsigned char *prow;      // [nU*3]
  const double *row_u;            // [n_rows]
  const unsigned char *row_axis;  // [n_rows]
  int n_rows;                     // 0: tables not available (more than 255 rows)
};

// the fixed-point cell rule of mplx_fx.cu: y + kFxMagic has the high word kFxHiBase + floor(y)
constexpr double kFxMagic = 1572864.0;   // 1.5 * 2^20: ulp(2^20..2^21) = 2^-32
constexpr int kFxHiBase = 0x41380000;    // high word of kFxMagic; + floor(y) for |y| < 2^19

constexpr int kNMax = 128;          // rows of the sample-time table
constexpr int kTStride = kNMax + 2; // doubles per row

#define MPLX_PI 3.14159265358979323846 /* M_PI */

// normalize_angle: include/mpl_basis/math.h:15-19
__device__ __forceinline__ double normalize_angle(double a) {
  while (a > MPLX_PI) a -= 2.0 * MPLX_PI;
  while (a < -MPLX_PI) a += 2.0 * MPLX_PI;
  return a;
}

// boost::hash_combine, 64-bit size_t, Boost 1.56-1.80 (hash_combine_impl(uint64&,uint64));
// boost::hash<int> = sign-extending cast.  waypoint.h:98..121 call sites.
// Split in the part that depends on the value alone (two of the three 64-bit multiplications; computed once
// per lattice id and shared by every key the id enters) and the part that folds it into the running hash.
__device__ __forceinline__ uint64_t hash_premix(int v) {
  uint64_t k = (uint64_t)(int64_t)v;
  const uint64_t m = 0xc6a4a7935bd1e995ULL;
  k *= m;
  k ^= k >> 47;
  k *= m;
  return k;
}
__device__ __forceinline__ void hash_fold(uint64_t &h, uint64_t k) {
  const uint64_t m = 0xc6a4a7935bd1e995ULL;
  h ^= k;
  h *= m;
  h += 0xe6546b64ULL;
}
__device__ __forceinline__ void hash_combine(uint64_t &h, int v) { hash_fold(h, hash_premix(v)); }

// ---- exact IEEE quotients and roundings without DDIV / round() / F2I ----------------------
// The reference computes  k = (int)std::round(RN(x / r) [- 0.5])  (waypoint.h:97-121,
// map_util.h:106) and n = ceil(RN(RN(max_v*T) / res)) (env_map.h:95).  A generic IEEE double
// division is ~25 instructions incl. MUFU.RCP64H, and round()/ceil()/F2I run on the
// quarter-rate XU pipe, which saturated in the first kernel.  All divisors on this path are
// per-plan constants (0.01, 0.1, res), so their correctly rounded reciprocals binv = RN(1/b)
// are precomputed and the quotient is finished with one Markstein correction:
//     q0 = RN(a*binv);  r = fma(-b, q0, a)  (exact);  q = fma(r, binv, q0) = RN(a/b)
// — the same tail nvcc's own IEEE division ends with.  tests/test_arith_identities.py checks
// the identity on >1e9 structured and random operands (the only exceptions are subnormal
// numerators, for which every use below yields 0 either way).
// Rounding to nearest uses the 1.5*2^52 magic constant (two FP64 adds); std::round's
// half-away-from-zero rule is restored exactly by looking at the (exact) remainder.
#define MPLX_MAGIC 6755399441055744.0 /* 1.5 * 2^52 */

__device__ __forceinline__ double div_exact(double a, double b, double binv) {
  const double q0 = a * binv;
  const double r = __fma_rn(-b, q0, a);
  return __fma_rn(r, binv, q0);
}

// std::round(x) as a double, |x| < 2^51 (beyond that the value is astronomically far from any
// grid or lattice the int conversion could represent).
__device__ __forceinline__ double round_haz(double x, int &k) {
  const double m = x + MPLX_MAGIC;  // RN-even integer in the low mantissa bits
  double kd = m - MPLX_MAGIC;
  const double f = x - kd;  // exact, in [-0.5, 0.5]
  k = __double2loint(m);
  if (fabs(f) == 0.5) {  // an exact tie (uncommon): RN-even may have gone toward zero
    if (f > 0.0 && x > 0.0) { kd += 1.0; k += 1; }  // rounded down to even: away from zero is up
    if (f < 0.0 && x < 0.0) { kd -= 1.0; k -= 1; }  // rounded up to even: away from zero is down
  }
  return kd;
}

// floatToInt (map_util.h:103-108): (int)std::round((p - origin)/res - 0.5), true division.
// NaN / out-of-int-range inputs convert to INT_MIN, the x86-64 cvttsd2si result the reference
// build produces for them (a sample there is outside every map).
__device__ __forceinline__ int float_to_int(double p, double origin, double res) {
  const double x = (p - origin) / res - 0.5;
  if (!(fabs(x) < 2147483648.0)) return INT_MIN;
  int k;
  round_haz(x, k);
  return k;
}

// `int id = std::round(x / res)` (waypoint.h:97,101,105,109,115); rinv = RN(1/res)
__device__ __forceinline__ int lattice_id(double x, double res, double rinv) {
  int k;
  round_haz(div_exact(x, res, rinv), k);
  return k;
}

// std::ceil(x) for |x| < 2^51 as a double
__device__ __forceinline__ double ceil_exact(double x) {
  const double kd = (x + MPLX_MAGIC) - MPLX_MAGIC;
  return kd < x ? kd + 1.0 : kd;
}

// One axis of a primitive built by the state+control constructor (primitive.h:220-256):
// ORD = number of state derivatives carried (VEL 1, ACC 2, JRK 3, SNP 4); the leading
// 6-1-ORD coefficients are the literal +0 of the comma initialisers (primitive.h:34-50).
// We keep the four pre-divided quotients the evaluators use (c1/24, c2/6, c3/2, ...).
template <int ORD>
struct Axis {
  double c1, c2, c3, c4, c5;  // c0 is always the literal 0

  __device__ __forceinline__ void build(double u, double p, double v, double a, double j) {
    c1 = c2 = c3 = 0.0;
    if (ORD == 1) { c4 = u; c5 = p; }
    if (ORD == 2) { c3 = u; c4 = v; c5 = p; }
    if (ORD == 3) { c2 = u; c3 = a; c4 = v; c5 = p; }
    if (ORD == 4) { c1 = u; c2 = j; c3 = a; c4 = v; c5 = p; }
  }

  // Primitive1D::p (primitive.h:128-131).  power(t,n) = ((1*t)*t).. = t*t*..*t (math.h:197-205)
  // so pw3=(t*t)*t etc. are shared by the caller.  Terms whose coefficient is the literal 0
  // contribute exactly +0 (t finite) and the running sum starts at +0.
  // EXACT_ZERO=false drops the leading `(+0) +`: identical value except that a -0 first term
  // stays -0 (irrelevant for the cell index, used only inside the sample loop).
  template <bool EXACT_ZERO>
  __device__ __forceinline__ double p(double t, double pw3, double pw4) const {
    if (EXACT_ZERO) {
      double s = 0.0;
      if (ORD >= 4) s = s + c1 / 24 * pw4;
      if (ORD >= 3) s = s + c2 / 6 * pw3;
      if (ORD >= 2) s = s + c3 / 2 * t * t;
      s = s + c4 * t;
      return s + c5;
    }
    if (ORD == 1) return c4 * t + c5;
    if (ORD == 2) return c3 / 2 * t * t + c4 * t + c5;
    if (ORD == 3) return c2 / 6 * pw3 + c3 / 2 * t * t + c4 * t + c5;
    return c1 / 24 * pw4 + c2 / 6 * pw3 + c3 / 2 * t * t + c4 * t + c5;
  }
  // Primitive1D::v (primitive.h:134-137)
  __device__ __forceinline__ double v(double t, double pw3) const {
    double s = 0.0;
    if (ORD >= 4) s = s + c1 / 6 * pw3;
    if (ORD >= 3) s = s + c2 / 2 * t * t;
    if (ORD >= 2) s = s + c3 * t;
    return s + c4;
  }
  // Primitive1D::a (primitive.h:140-142)
  __device__ __forceinline__ double a(double t) const {
    double s = 0.0;
    if (ORD >= 4) s = s + c1 / 2 * t * t;
    if (ORD >= 3) s = s + c2 * t;
    return s + c3;
  }
  // Primitive1D::j (primitive.h:145): c0/2*t*t + c1*t + c2
  __device__ __forceinline__ double j(double t) const {
    double s = 0.0;
    if (ORD >= 4) s = s + c1 * t;
    return s + c2;
  }

  // max_vel (primitive.h:353-363) with extrema_v (:152-162) and solve (math.h:117-131).
  // solve(0, c0/6, c1/2, c2, c3): with c0 = 0 the cubic branch is unreachable;
  //   c1 != 0 -> quad(c1/2, c2, c3) (math.h:22-32);  else c2 != 0 -> linear root -c3/c2.
  __device__ __forceinline__ double max_vel(double T) const {
    // v(0) = 0+..+c4 ; |v(0)| = |c4|
    double pw3T = (T * T) * T;
    double m = fmax(fabs(v(0.0, 0.0)), fabs(v(T, pw3T)));
    if (ORD >= 4 && c1 / 2 != 0) {
      double b = c1 / 2, c = c2, d = c3;
      double disc = c * c - 4 * b * d;
      if (!(disc < 0)) {
        double r0 = (-c - sqrt(disc)) / (2 * b);
        double r1 = (-c + sqrt(disc)) / (2 * b);
        // filter with the unsorted early break (primitive.h:155-160)
        bool brk = false;
        if (r0 > 0 && r0 < T) {
          double vv = fabs(v(r0, (r0 * r0) * r0));
          m = vv > m ? vv : m;
        } else if (r0 >= T)
          brk = true;
        if (!brk && r1 > 0 && r1 < T) {
          double vv = fabs(v(r1, (r1 * r1) * r1));
          m = vv > m ? vv : m;
        }
      }
    } else if (ORD >= 3 && c2 != 0) {
      double r = -c3 / c2;
      if (r > 0 && r < T) {
        double vv = fabs(v(r, (r * r) * r));
        m = vv > m ? vv : m;
      }
    }
    return m;
  }
  // max_acc (primitive.h:369-379), extrema_a (:169-179): solve(0,0,c0/2,c1,c2):
  //   c0/2 == 0 -> c1 != 0 -> linear root -c2/c1.
  __device__ __forceinline__ double max_acc(double T) const {
    double m = fmax(fabs(a(0.0)), fabs(a(T)));
    if (ORD >= 4 && c1 != 0) {
      double r = -c2 / c1;
      if (r > 0 && r < T) {
        double aa = fabs(a(r));
        m = aa > m ? aa : m;
      }
    }
    return m;
  }
  // max_jrk (primitive.h:384-394), extrema_j (:186-193): c0 == 0 -> no interior root.
  __device__ __forceinline__ double max_jrk(double T) const { return fmax(fabs(j(0.0)), fabs(j(T))); }

  // Primitive1D::J (primitive.h:92-122) for a ctor-built primitive: every term but the last
  // has a literal-0 factor and sums to +0, leaving (u*u)*T with u the control coefficient.
  __device__ __forceinline__ double J(double T) const {
    double u = ORD == 1 ? c4 : ORD == 2 ? c3 : ORD == 3 ? c2 : c1;
    return u * u * T;  // (+0) + x == x for x >= +0
  }
};

// v.normalized().dot((cos yaw, sin yaw)) with Eigen's definitions (normalized(): divide by
// sqrt(squaredNorm) when squaredNorm > 0).  primitive.h:520, env_map.h:124-125.
__device__ __forceinline__ double dot2_normalized(double v0, double v1, double c, double s) {
  double z = v0 * v0 + v1 * v1;
  double n0 = v0, n1 = v1;
  if (z > 0) {
    double nn = sqrt(z);
    n0 = v0 / nn;
    n1 = v1 / nn;
  }
  return n0 * c + n1 * s;
}

}  // namespace mplx
