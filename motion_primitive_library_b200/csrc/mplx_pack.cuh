// mplx_pack.cuh — the per-word rules of the two packed views of the grid.  The full packs of
// mplx_set_map (pack_bits_kernel, pack_occ2_kernel) and the sparse re-packs of mplx_update_cells
// both call these, so a word recomputed after an edit is bit-identical to a full re-pack.
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

}  // namespace mplx
