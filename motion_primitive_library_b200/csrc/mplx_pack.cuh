// mplx_pack.cuh — the per-word rules of the two packed views of the grid, and the brick layout of
// the second (occ2).  The full packs of mplx_set_map (pack_bits_kernel, pack_occ2_kernel) and the
// sparse re-packs of mplx_update_cells both call these, so a word recomputed after an edit is
// bit-identical to a full re-pack.  No other file restates the layout.
#pragma once
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
// consecutive samples, and the 27 primitives of a node, fall on few cache lines.  The buffer holds the
// two halves of the pairs apart: word p (p < occ2_pair_count) is the occupancy word of pair p and word
// occ2_pair_count + p its summary word.  Only uncertain samples (~3 %) read the summary half, so the
// occupancy half alone is what the sample loop keeps hot: 16 MiB at 512^3, which the H100's persisting
// L2 carve-out (31.2 MiB) holds whole, where the interleaved 32 MiB did not fit.
//   3-D: bricks of 8x8x8 voxels, counted ceil(nx/8) x ceil(ny/8) x ceil(nz/8), x fastest.  Inside a
//        brick local = x&7 | (y&7)<<3 | (z&7)<<6; the cell's pair is local>>5 and its bit local&31.
//   2-D: bricks of 32x16 voxels, counted ceil(nx/32) x ceil(ny/16); pair y&15, bit x&31.
// A brick is 16 words = 64 bytes in each half.  Padding bits (cells past the map's edge) are 1 in both
// words: such a cell can never look free.
constexpr int kOcc2BrickPairs = 16;

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

// Pair p of the brick buffer (o: occupancy word, s: summary word): each cell's bits are its bits in
// the voxel-order occupancy words (pack_word, in `occ`) and summary words (occ2_summary_word); padding
// bits are 1.  A 3-D pair holds 4 runs of 8 cells along x (rows y..y+3 of one z), a 2-D pair one run of 32.
__host__ __device__ inline void occ2_brick_pair(const uint32_t *occ, size_t p, size_t nvox, int dim, int nx, int ny, int nz,
                                                uint32_t &o, uint32_t &s) {
  const size_t nwords = (nvox + 31) >> 5;
  const size_t brick = p / kOcc2BrickPairs;
  const int q = (int)(p % kOcc2BrickPairs);
  const int nbx = occ2_bricks_x(dim, nx), nby = occ2_bricks_y(dim, ny);
  const int bx = (int)(brick % nbx);
  const size_t byz = brick / nbx;
  int x0, y0, z, run, rows;
  if (dim == 3) {
    x0 = bx * 8;
    y0 = (int)(byz % nby) * 8 + (q & 1) * 4;
    z = (int)(byz / nby) * 8 + (q >> 1);
    run = 8;
    rows = 4;
  } else {
    x0 = bx * 32;
    y0 = (int)byz * 16 + q;
    z = 0;
    run = 32;
    rows = 1;
  }
  o = s = ~0u;
  const int len = nx - x0 < run ? nx - x0 : run;  // x0 < nx: bx < nbx
  const uint32_t m = len == 32 ? ~0u : (1u << len) - 1u;
  for (int r = 0; r < rows; r++) {
    const int y = y0 + r;
    if (y >= ny || z >= nz) continue;
    const size_t i = (size_t)x0 + (size_t)nx * ((size_t)y + (size_t)ny * z);
    const int sh = r * run;
    o = (o & ~(m << sh)) | ((occ_window(occ, nwords, (long long)i) & m) << sh);
    s = (s & ~(m << sh)) | ((occ2_summary_run(occ, i, len, nvox, dim, nx, ny) & m) << sh);
  }
}

}  // namespace mplx
