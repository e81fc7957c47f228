// The brick build of mplx_set_batch_regions (csrc/mplx_tunnel.cu) restated on the CPU with the same geometry
// (csrc/mplx_tunnel.cuh): stamp one (query, brick) key per (path cell, brick slot), sort, de-duplicate, take each
// query's first brick by lower bound, OR each box into its bricks' mask words, then read every voxel back through
// tunnel_has, the sample loop's lookup.  tests/test_tunnel_bricks_cpu.py compares the voxels with a dense stamp.
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "../motion_primitive_library_b200/csrc/mplx_tunnel.cuh"

using namespace mplx;

extern "C" int tb_build(int dim, const int *mdim3, int n_q, const int64_t *cell_off, const int *cells, const int *r3,
                        int64_t *n_bricks, uint8_t *out) {
  const int mdim[3] = {mdim3[0], mdim3[1], dim == 3 ? mdim3[2] : 1};
  const int r[3] = {r3[0], r3[1], dim == 3 ? r3[2] : 0};
  const int per = tunnel_box_bricks(dim, r);
  const uint64_t sentinel = tunnel_key(n_q, 0);
  auto slot = [&](int c, int s, int &bx, int &by, int &bz, int *lo, int *hi) {
    int blo[3], bhi[3];
    if (!tunnel_box(dim, mdim, cells + 3 * c, r, lo, hi, blo, bhi)) return false;
    const int nbx = bhi[0] - blo[0] + 1, nby = bhi[1] - blo[1] + 1, nbz = bhi[2] - blo[2] + 1;
    if (s >= nbx * nby * nbz) return false;
    bx = blo[0] + s % nbx;
    by = blo[1] + (s / nbx) % nby;
    bz = blo[2] + s / (nbx * nby);
    return true;
  };
  const int n_cells = (int)cell_off[n_q];
  std::vector<int> owner(n_cells);
  for (int q = 0; q < n_q; q++)
    for (int64_t c = cell_off[q]; c < cell_off[q + 1]; c++) owner[c] = q;
  std::vector<uint64_t> keys;
  for (int c = 0; c < n_cells; c++)
    for (int s = 0; s < per; s++) {
      int bx, by, bz, lo[3], hi[3];
      keys.push_back(slot(c, s, bx, by, bz, lo, hi) ? tunnel_key(owner[c], tunnel_brick_id(mdim, bx, by, bz))
                                                    : sentinel);
    }
  std::sort(keys.begin(), keys.end());
  keys.erase(std::unique(keys.begin(), keys.end()), keys.end());
  std::vector<int64_t> off(n_q + 1);
  for (int q = 0; q <= n_q; q++)
    off[q] = std::lower_bound(keys.begin(), keys.end(), tunnel_key(q, 0)) - keys.begin();
  *n_bricks = off[n_q];
  const int W = tunnel_words(dim);
  std::vector<uint32_t> bits((size_t)off[n_q] * W, 0u);
  for (int c = 0; c < n_cells; c++)
    for (int s = 0; s < per; s++) {
      int bx, by, bz, lo[3], hi[3];
      if (!slot(c, s, bx, by, bz, lo, hi)) continue;
      const int q = owner[c];
      const uint64_t k = tunnel_key(q, tunnel_brick_id(mdim, bx, by, bz));
      const int64_t i = std::lower_bound(keys.begin() + off[q], keys.begin() + off[q + 1], k) - keys.begin();
      if (i >= off[q + 1] || keys[i] != k) return 1;  // every stamped brick must have been kept
      for (int w = 0; w < W; w++) bits[(size_t)i * W + w] |= tunnel_box_word(dim, lo, hi, bx, by, bz, w);
    }
  const size_t nvox = (size_t)mdim[0] * mdim[1] * mdim[2];
  for (int q = 0; q < n_q; q++) {
    const TunnelView tv{keys.data() + off[q], bits.data() + (size_t)off[q] * W, (int)(off[q + 1] - off[q]), q};
    size_t i = 0;
    for (int z = 0; z < mdim[2]; z++)
      for (int y = 0; y < mdim[1]; y++)
        for (int x = 0; x < mdim[0]; x++) out[(size_t)q * nvox + i++] = tunnel_has(tv, dim, mdim, x, y, z) ? 1 : 0;
  }
  return 0;
}
