// mplx_tunnel.cuh — the per-query tunnels of the batched searches (mplx_set_batch_regions): the brick geometry
// shared by the device build (mplx_tunnel.cu), the sample loop's lookup (mplx_expand.cuh) and the CPU restatement
// (tests/tunnel_bricks_host.cpp).
//
// A tunnel is stored as the 8x8x8 bricks (8x8 tiles in 2-D) it touches, each with one bit per cell.  Every query
// owns a run of bricks sorted by key, key = (query << 32) | brick id, brick id = bx + nbx * (by + nby * bz); a
// cell's bit in its brick is (x & 7) | (y & 7) << 3 | (z & 7) << 6.  Plain integer work only, so host and device
// agree.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define MPLX_TUN_HD __host__ __device__ __forceinline__
#else
#define MPLX_TUN_HD inline
#endif

namespace mplx {

constexpr int kBrickShift = 3;  // 8 cells per brick axis

// mask words per brick: 512 bits in 3-D, 64 in 2-D
MPLX_TUN_HD int tunnel_words(int dim) { return dim == 3 ? 16 : 2; }
MPLX_TUN_HD uint32_t tunnel_brick_id(const int *mdim, int bx, int by, int bz) {
  const uint32_t nbx = (uint32_t)((mdim[0] + 7) >> kBrickShift), nby = (uint32_t)((mdim[1] + 7) >> kBrickShift);
  return (uint32_t)bx + nbx * ((uint32_t)by + nby * (uint32_t)bz);
}
MPLX_TUN_HD uint64_t tunnel_key(int q, uint32_t brick) { return ((uint64_t)(uint32_t)q << 32) | brick; }

// The bricks of one path cell's box: per axis k the cells [lo[k], hi[k]] = [cell - r, cell + r] clipped to the map
// (isOutside, map_planner.cpp:86) and the bricks blo[k] .. bhi[k] they cover; false when the box misses the map.
MPLX_TUN_HD bool tunnel_box(int dim, const int *mdim, const int *cell, const int *r, int *lo, int *hi, int *blo,
                            int *bhi) {
  for (int k = 0; k < 3; k++) {
    const int d = k < dim ? mdim[k] : 1;
    const int rk = k < dim ? r[k] : 0;
    const int c = k < dim ? cell[k] : 0;
    lo[k] = c - rk < 0 ? 0 : c - rk;
    hi[k] = c + rk > d - 1 ? d - 1 : c + rk;
    if (lo[k] > hi[k]) return false;
    blo[k] = lo[k] >> kBrickShift;
    bhi[k] = hi[k] >> kBrickShift;
  }
  return true;
}

// The most bricks one box can touch (the stamp kernel's slots per path cell).
MPLX_TUN_HD int tunnel_box_bricks(int dim, const int *r) {
  int n = 1;
  for (int k = 0; k < dim; k++) n *= ((2 * r[k] + 1 + 6) >> kBrickShift) + 1;
  return n;
}

// Mask word w of brick (bx, by, bz) intersected with the box [lo, hi]: word w holds the four rows
// y & 7 = 4 * (w & 1) + i, i = 0..3, of the layer z & 7 = w >> 1, 8 bits of x each.
MPLX_TUN_HD uint32_t tunnel_box_word(int dim, const int *lo, const int *hi, int bx, int by, int bz, int w) {
  const int z = dim == 3 ? (bz << kBrickShift) + (w >> 1) : 0;
  if (z < lo[2] || z > hi[2]) return 0u;
  const int x0 = bx << kBrickShift;
  const int xa = lo[0] > x0 ? lo[0] - x0 : 0, xb = hi[0] < x0 + 7 ? hi[0] - x0 : 7;
  if (xa > xb) return 0u;
  const uint32_t row = ((0xffu >> (7 - xb)) & (0xffu << xa)) & 0xffu;
  uint32_t m = 0;
  for (int i = 0; i < 4; i++) {
    const int y = (by << kBrickShift) + ((w & 1) << 2) + i;
    if (y >= lo[1] && y <= hi[1]) m |= row << (8 * i);
  }
  return m;
}

// One query's tunnel as the sample loop reads it: n bricks, keys ascending, tunnel_words(dim) mask words each.
struct TunnelView {
  const uint64_t *key;
  const uint32_t *bits;
  int n, q;
};

// Whether cell (x, y, z) lies in the tunnel: a binary search for its brick, then the cell's bit.
MPLX_TUN_HD bool tunnel_has(const TunnelView &t, int dim, const int *mdim, int x, int y, int z) {
  const uint64_t k = tunnel_key(t.q, tunnel_brick_id(mdim, x >> kBrickShift, y >> kBrickShift, z >> kBrickShift));
  int lo = 0, hi = t.n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (t.key[mid] < k) lo = mid + 1;
    else hi = mid;
  }
  if (lo >= t.n || t.key[lo] != k) return false;
  const int bit = (x & 7) | (y & 7) << 3 | (z & 7) << 6;
  return (t.bits[(size_t)lo * tunnel_words(dim) + (bit >> 5)] >> (bit & 31)) & 1u;
}

}  // namespace mplx
