// The word rules and brick layout of csrc/mplx_pack.cuh on the host, as a small shared library that
// tests/test_update_restatement_cpu.py loads with ctypes (no device needed): for a grid, the occupancy
// words (pack_word), the full brick buffer (occ2_brick_pair for every pair), and the brick buffer read
// back in voxel order through occ2_pair / occ2_bit the way mplx_read_map's unbrick_occ2_kernel does
// (bits past nvox: occupancy 0, summary 1), plus each voxel's (pair, bit).
#include <cstddef>
#include <cstdint>
#include <vector>

#define __host__
#define __device__
#include "../motion_primitive_library_b200/csrc/mplx_pack.cuh"

extern "C" size_t uv_pair_count(int dim, int nx, int ny, int nz) { return mplx::occ2_pair_count(dim, nx, ny, nz); }

// occ[nw], bricks[npairs * 2], pairs[nw * 2], pair_of[nvox], bit_of[nvox]
extern "C" void uv_views(const int8_t *g, int dim, int nx, int ny, int nz, uint32_t *occ, uint32_t *bricks,
                         uint32_t *pairs, uint32_t *pair_of, uint8_t *bit_of) {
  const size_t nvox = (size_t)nx * ny * nz, nw = (nvox + 31) / 32, sxy = (size_t)nx * ny;
  const size_t npairs = mplx::occ2_pair_count(dim, nx, ny, nz);
  const int nbx = mplx::occ2_bricks_x(dim, nx), nby = mplx::occ2_bricks_y(dim, ny);
  for (size_t w = 0; w < nw; w++) occ[w] = mplx::pack_word<true>(g, w, nvox);
  for (size_t p = 0; p < npairs; p++) mplx::occ2_brick_pair(occ, p, nvox, dim, nx, ny, nz, bricks[2 * p], bricks[2 * p + 1]);
  for (size_t w = 0; w < nw; w++) {
    uint32_t o = 0, s = 0;
    for (int b = 0; b < 32; b++) {
      const size_t i = (w << 5) + b;
      if (i >= nvox) {
        s |= 1u << b;
        continue;
      }
      const int x = (int)(i % nx), y = (int)(i / nx % ny), z = (int)(i / sxy);
      const unsigned p = dim == 3 ? mplx::occ2_pair<3>(x, y, z, nbx, nby) : mplx::occ2_pair<2>(x, y, 0, nbx, nby);
      const unsigned bit = dim == 3 ? mplx::occ2_bit<3>(x, y) : mplx::occ2_bit<2>(x, y);
      pair_of[i] = p;
      bit_of[i] = (uint8_t)bit;
      o |= ((bricks[2 * p] >> bit) & 1u) << b;
      s |= ((bricks[2 * p + 1] >> bit) & 1u) << b;
    }
    pairs[2 * w] = o;
    pairs[2 * w + 1] = s;
  }
}
