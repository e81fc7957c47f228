// mplx_pack.cuh — the per-word rules of the two packed views of the grid, and the brick layout of
// the second (occ2).  The full packs of mplx_set_map (pack_bits_kernel, pack_occ2_kernel) and the
// sparse re-packs of mplx_update_cells both call these, so a word recomputed after an edit is
// bit-identical to a full re-pack.  No other file restates the layout.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

namespace mplx {

// bits b of word wd: voxel i = 32*wd + b; OCC ? (byte == 100) (isOccupied, map_util.h:48) : (byte != 0).
// Bits at i >= nvox are 0.
template <bool OCC>
__host__ __device__ inline uint32_t pack_word(const int8_t *bytes, size_t wd, size_t nvox) {
  uint32_t m = 0;
  const size_t b0 = wd << 5;
#pragma unroll 8
  for (int b = 0; b < 32; b++) {
    const size_t i = b0 + b;
    if (i < nvox && (OCC ? bytes[i] == 100 : bytes[i] != 0)) m |= 1u << b;
  }
  return m;
}

// bits b with 32*wd + b in [lo, hi)
__host__ __device__ inline uint32_t range_bits(size_t wd, size_t lo, size_t hi) {
  const size_t b0 = wd << 5;
  const size_t a = lo > b0 ? lo - b0 : 0, c = hi < b0 + 32 ? (hi > b0 ? hi - b0 : 0) : 32;
  if (a >= c) return 0;
  return (c - a == 32 ? ~0u : ((1u << (c - a)) - 1u)) << a;
}

// 32 occupancy bits starting at voxel s (s may be negative; bits before voxel 0 or past the last word are 0)
__host__ __device__ inline uint32_t occ_window(const uint32_t *occ, size_t nwords, long long s) {
  const long long w = s >> 5;  // floor
  const int r = (int)(s & 31);
  const uint32_t lo = w >= 0 && (size_t)w < nwords ? occ[w] : 0u;
  const uint32_t hi = w + 1 >= 0 && (size_t)(w + 1) < nwords ? occ[w + 1] : 0u;
  return r ? (lo >> r) | (hi << (32 - r)) : lo;
}

// Candidate-summary word wd.  Summary bit of voxel (x,y,z) = OR of the occupancy of the cells
// {x-1,x} x {y-1,y} (x {z-1,z}), a cell outside the map counting as occupied; bits at i >= nvox are 1.
// A voxel with x == 0, y == 0 or (3-D) z == 0 has an outside cell in its box, so its bit is 1; every
// other voxel's box lies inside the map, and its bit is the OR of the occupancy stream shifted by
// each box offset, word-parallel.
__host__ __device__ inline uint32_t occ2_summary_word(const uint32_t *occ, size_t wd, size_t nvox, int dim, int nx, int ny) {
  const size_t nwords = (nvox + 31) >> 5, sxy = (size_t)nx * ny, b0 = wd << 5;
  uint32_t d = range_bits(wd, nvox, ~(size_t)0);
  for (size_t i = b0 + (nx - b0 % nx) % nx; i < b0 + 32; i += nx) d |= 1u << (i - b0);  // x == 0
  for (size_t p = b0 / sxy; p * sxy < b0 + 32; p++) d |= range_bits(wd, p * sxy, p * sxy + nx);  // y == 0
  if (dim == 3) d |= range_bits(wd, 0, sxy);  // z == 0
  for (int dz = 0; dz <= (dim == 3 ? 1 : 0); dz++)
    for (int dy = 0; dy <= 1; dy++)
      for (int dx = 0; dx <= 1; dx++)
        d |= occ_window(occ, nwords, (long long)b0 - dx - (long long)dy * nx - (long long)dz * (long long)sxy);
  return d;
}

// ---- occ2: the {occupancy, candidate-summary} pairs of the fixed-point sample loop, in bricks ----
// The words above are in voxel order; occ2 stores the same bits in bricks so that a primitive's
// consecutive samples, and the 27 primitives of a node, fall on few cache lines.
//   3-D: bricks of 8x8x8 voxels, x fastest.  Inside a brick local = x&7 | (y&7)<<3 | (z&7)<<6; the
//        cell's pair is local>>5 and its bit local&31.
//   2-D: bricks of 32x16 voxels, x fastest; pair y&15, bit x&31.
// A brick is 16 words = 64 bytes in each half.  The brick layout of a map of nx x ny (x nz) cells counts
// ceil(nx/8) x ceil(ny/8) x ceil(nz/8) bricks (2-D: ceil(nx/32) x ceil(ny/16)): occ2_bricks_x/y,
// occ2_pair_count, occ2_pair, occ2_bit, occ2_brick_pair.
//
// The device buffer stores the bricks of the map padded by a guard band of kOcc2Guard cells on every
// side (every axis of the map's dimension): cell (x, y, z) of the map is cell (x+G, y+G, z+G) of the
// padded map, x, y, z in [-G, dim+G).  Every bit of a cell outside the map — the guard band and the
// padding past the last brick — is 1 in both words: such a cell reads blocked when certain and
// ambiguous when uncertain, as the sample loop decides a cell outside the map.  The band lets the loop
// address a sample that may leave the map without testing whether it did (mplx_fx.cuh).  The buffer
// holds the two halves of the pairs apart: word p (p < occ2_guard_pair_count) is the occupancy word of
// padded pair p and word occ2_guard_pair_count + p its summary word.  Only uncertain samples (~3 %) read
// the summary half, so the occupancy half alone is what the sample loop keeps hot: 72^3 bricks = 22.8 MB
// at 512^3, which the H100's persisting L2 carve-out (31.2 MiB) holds whole.
constexpr int kOcc2BrickPairs = 16;
constexpr int kOcc2Guard = 32;  // a multiple of the brick edges (8; 32 x 16)

__host__ __device__ inline int occ2_bricks_x(int dim, int nx) { return dim == 3 ? (nx + 7) >> 3 : (nx + 31) >> 5; }
__host__ __device__ inline int occ2_bricks_y(int dim, int ny) { return dim == 3 ? (ny + 7) >> 3 : (ny + 15) >> 4; }

// pairs of the whole buffer (nz = 1 in 2-D): the words of each half
__host__ __device__ inline size_t occ2_pair_count(int dim, int nx, int ny, int nz) {
  const size_t bz = dim == 3 ? (size_t)((nz + 7) >> 3) : 1;
  return (size_t)occ2_bricks_x(dim, nx) * occ2_bricks_y(dim, ny) * bz * kOcc2BrickPairs;
}

// brick of cell (x, y, z); nbx, nby from occ2_bricks_x / occ2_bricks_y
template <int DIM>
__host__ __device__ inline unsigned occ2_brick(int x, int y, int z, int nbx, int nby) {
  return DIM == 3 ? (unsigned)(x >> 3) + (unsigned)nbx * ((unsigned)(y >> 3) + (unsigned)nby * (unsigned)(z >> 3))
                  : (unsigned)(x >> 5) + (unsigned)nbx * (unsigned)(y >> 4);
}

// pair of cell (x, y, z) in the buffer
template <int DIM>
__host__ __device__ inline unsigned occ2_pair(int x, int y, int z, int nbx, int nby) {
  const unsigned in_brick = DIM == 3 ? (unsigned)(((y >> 2) & 1) | ((z & 7) << 1)) : (unsigned)(y & 15);
  return occ2_brick<DIM>(x, y, z, nbx, nby) * kOcc2BrickPairs + in_brick;
}

// bit of cell (x, y) in both words of its pair
template <int DIM>
__host__ __device__ inline unsigned occ2_bit(int x, int y) {
  return DIM == 3 ? (unsigned)((x & 7) | ((y & 3) << 3)) : (unsigned)(x & 31);
}

// Candidate-summary bits of the voxels [s, s + len) (len <= 32) in bits 0..len-1; higher bits undefined.
__host__ __device__ inline uint32_t occ2_summary_run(const uint32_t *occ, size_t s, int len, size_t nvox, int dim, int nx,
                                                     int ny) {
  const size_t w = s >> 5;
  const int r = (int)(s & 31);
  uint32_t v = occ2_summary_word(occ, w, nvox, dim, nx, ny) >> r;
  if (r + len > 32) v |= occ2_summary_word(occ, w + 1, nvox, dim, nx, ny) << (32 - r);
  return v;
}

// Pair q of the brick whose first cell, in map coordinates, is (bx0, by0, bz0) (o: occupancy word, s:
// summary word): each cell of the map has its bits in the voxel-order occupancy words (pack_word, in
// `occ`) and summary words (occ2_summary_word); every other bit is 1.  A 3-D pair holds 4 runs of 8 cells
// along x (rows y..y+3 of one z), a 2-D pair one run of 32.  bx0 is a multiple of the run.
__host__ __device__ inline void occ2_pair_words(const uint32_t *occ, int bx0, int by0, int bz0, int q, size_t nvox,
                                                int dim, int nx, int ny, int nz, uint32_t &o, uint32_t &s) {
  const size_t nwords = (nvox + 31) >> 5;
  int y0, z, run, rows;
  if (dim == 3) {
    y0 = by0 + (q & 1) * 4;
    z = bz0 + (q >> 1);
    run = 8;
    rows = 4;
  } else {
    y0 = by0 + q;
    z = 0;
    run = 32;
    rows = 1;
  }
  o = s = ~0u;
  if (bx0 < 0 || bx0 >= nx || z < 0 || z >= nz) return;
  const int len = nx - bx0 < run ? nx - bx0 : run;
  const uint32_t m = len == 32 ? ~0u : (1u << len) - 1u;
  for (int r = 0; r < rows; r++) {
    const int y = y0 + r;
    if (y < 0 || y >= ny) continue;
    const size_t i = (size_t)bx0 + (size_t)nx * ((size_t)y + (size_t)ny * z);
    const int sh = r * run;
    o = (o & ~(m << sh)) | ((occ_window(occ, nwords, (long long)i) & m) << sh);
    s = (s & ~(m << sh)) | ((occ2_summary_run(occ, i, len, nvox, dim, nx, ny) & m) << sh);
  }
}

// Pair p of the brick layout of the map itself (no guard band).
__host__ __device__ inline void occ2_brick_pair(const uint32_t *occ, size_t p, size_t nvox, int dim, int nx, int ny, int nz,
                                                uint32_t &o, uint32_t &s) {
  const size_t brick = p / kOcc2BrickPairs;
  const int nbx = occ2_bricks_x(dim, nx), nby = occ2_bricks_y(dim, ny);
  const int bx = (int)(brick % nbx);
  const size_t byz = brick / nbx;
  const int q = (int)(p % kOcc2BrickPairs);
  if (dim == 3)
    occ2_pair_words(occ, bx * 8, (int)(byz % nby) * 8, (int)(byz / nby) * 8, q, nvox, dim, nx, ny, nz, o, s);
  else
    occ2_pair_words(occ, bx * 32, (int)byz * 16, 0, q, nvox, dim, nx, ny, nz, o, s);
}

// ---- the padded map of the device buffer ----
// bricks along x / y / z and pairs of each half
__host__ __device__ inline int occ2_guard_bricks_x(int dim, int nx) { return occ2_bricks_x(dim, nx + 2 * kOcc2Guard); }
__host__ __device__ inline int occ2_guard_bricks_y(int dim, int ny) { return occ2_bricks_y(dim, ny + 2 * kOcc2Guard); }
__host__ __device__ inline int occ2_guard_bricks_z(int dim, int nz) { return dim == 3 ? (nz + 2 * kOcc2Guard + 7) >> 3 : 1; }
__host__ __device__ inline size_t occ2_guard_pair_count(int dim, int nx, int ny, int nz) {
  return (size_t)occ2_guard_bricks_x(dim, nx) * occ2_guard_bricks_y(dim, ny) * occ2_guard_bricks_z(dim, nz) * kOcc2BrickPairs;
}

// padded pair of cell (x, y, z) of the map, x, y, z in [-G, dim+G); pbx, pby from occ2_guard_bricks_x/y.  Its
// bit is occ2_bit<DIM>(x, y): G is a multiple of the brick edges.
template <int DIM>
__host__ __device__ inline unsigned occ2_guard_pair(int x, int y, int z, int pbx, int pby) {
  return occ2_pair<DIM>(x + kOcc2Guard, y + kOcc2Guard, DIM == 3 ? z + kOcc2Guard : 0, pbx, pby);
}

// Padded pair p of the device buffer.
__host__ __device__ inline void occ2_guard_brick_pair(const uint32_t *occ, size_t p, size_t nvox, int dim, int nx, int ny,
                                                      int nz, uint32_t &o, uint32_t &s) {
  const size_t brick = p / kOcc2BrickPairs;
  const int pbx = occ2_guard_bricks_x(dim, nx), pby = occ2_guard_bricks_y(dim, ny);
  const int bx = (int)(brick % pbx);
  const size_t byz = brick / pbx;
  const int q = (int)(p % kOcc2BrickPairs), G = kOcc2Guard;
  if (dim == 3)
    occ2_pair_words(occ, bx * 8 - G, (int)(byz % pby) * 8 - G, (int)(byz / pby) * 8 - G, q, nvox, dim, nx, ny, nz, o, s);
  else
    occ2_pair_words(occ, bx * 32 - G, (int)byz * 16 - G, 0, q, nvox, dim, nx, ny, nz, o, s);
}

// The padded pair and bit of a cell as one bit index K = 512 * brick + local: word K >> 5 of a half, bit
// K & 31.  K is a sum of per-axis terms of the cell's padded coordinates X_a = c_a + G:
//     K = sum_a  S_a * (X_a & (2^s_a - 1)) + (X_a >> s_a) * D_a
// (3-D: S = 1, 8, 64, s = 3, D = 512, 512 pbx, 512 pbx pby; 2-D: S = 1, 32, s = 5, 4, D = 512, 512 pbx), and
// with X & (2^s - 1) = X - ((X >> s) << s) it is sum_a S_a X_a + (X_a >> s_a) (D_a - S_a 2^s_a).  A caller
// that holds h_a = c_a + H, H - G a multiple of 2^s_a (the fixed-point sample loop: H = its high-word base),
// needs no c_a: K = sum_a S_a h_a + (h_a >> s_a) e_a + k0 in 32-bit arithmetic, e and k0 from
// occ2_sep_terms.  Exact while the padded map has fewer than 2^32 cells (occ2_guard_pair_count <= 2^27).
template <int DIM>
__host__ __device__ constexpr unsigned occ2_sep_scale(int a) { return DIM == 3 ? 1u << (3 * a) : (a == 0 ? 1u : 32u); }
template <int DIM>
__host__ __device__ constexpr int occ2_sep_shift(int a) { return DIM == 3 ? 3 : (a == 0 ? 5 : 4); }

template <int DIM>
__host__ __device__ inline unsigned occ2_sep_k(const int (&h)[DIM], const unsigned (&e)[3], unsigned k0) {
  unsigned k = k0;
#pragma unroll
  for (int a = 0; a < DIM; a++) k += occ2_sep_scale<DIM>(a) * (unsigned)h[a] + (unsigned)(h[a] >> occ2_sep_shift<DIM>(a)) * e[a];
  return k;
}

// A bound on |y(t) - y(0)| over t in [0, T] for y(t) = C[ORD] t^ORD + .. + C[1] t + C[0]: the largest
// Bernstein coefficient of y - y(0) on [0, T] in magnitude (y - y(0) is a convex combination of them there).
// A sample loop whose start cell lies in the map and whose reach + 2 <= kOcc2Guard never leaves the guard band.
template <int ORD>
__host__ __device__ inline double occ2_band_reach(const double (&C)[ORD + 1], double T) {
  double a[ORD + 1], p = T;
  for (int i = 1; i <= ORD; i++) {
    a[i] = C[i] * p;  // y - y(0) = sum_i a_i s^i, s = t/T
    p *= T;
  }
  double m = 0.0;
  for (int k = 1; k <= ORD; k++) {  // b_k = sum_{i=1..k} binom(k, i) / binom(ORD, i) a_i  (b_0 = 0)
    double b = 0.0, ck = 1.0, cn = 1.0;
    for (int i = 1; i <= k; i++) {
      ck = ck * (k - i + 1) / i;
      cn = cn * (ORD - i + 1) / i;
      b += ck / cn * a[i];
    }
    m = fmax(m, fabs(b));
  }
  return m;
}

template <int DIM>
inline void occ2_sep_terms_dim(int pbx, int pby, int H, unsigned (&e)[3], unsigned &k0) {
  const unsigned D[3] = {512u, 512u * (unsigned)pbx, 512u * (unsigned)pbx * (unsigned)pby};
  const int B = H - kOcc2Guard;
  k0 = 0;
  e[0] = e[1] = e[2] = 0;
  for (int a = 0; a < DIM; a++) {
    e[a] = D[a] - (occ2_sep_scale<DIM>(a) << occ2_sep_shift<DIM>(a));
    k0 -= occ2_sep_scale<DIM>(a) * (unsigned)B + (unsigned)(B >> occ2_sep_shift<DIM>(a)) * e[a];
  }
}

// e and k0 of occ2_sep_k for a map of nx x ny (x nz) cells and the coordinate base H
inline void occ2_sep_terms(int dim, int nx, int ny, int H, unsigned (&e)[3], unsigned &k0) {
  const int pbx = occ2_guard_bricks_x(dim, nx), pby = occ2_guard_bricks_y(dim, ny);
  if (dim == 3) occ2_sep_terms_dim<3>(pbx, pby, H, e, k0);
  else occ2_sep_terms_dim<2>(pbx, pby, H, e, k0);
}

}  // namespace mplx
