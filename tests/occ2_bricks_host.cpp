// Host-side checks of the occ2 brick layout of csrc/mplx_pack.cuh, run by tests/test_occ2_bricks_cpu.py (no
// device needed): on random grids with dims that are not multiples of the brick, the pairs that the full
// pack (occ2_brick_pair) builds and the addressing the sample loop uses (occ2_pair, occ2_bit) against a
// literal per-voxel statement — every voxel has a distinct (pair, bit), its bits are its occupancy and its
// candidate summary, and every bit no voxel owns (padding) is 1 in both words.
#include <cstdio>
#include <random>
#include <vector>

#define __host__
#define __device__
#include "../motion_primitive_library_b200/csrc/mplx_pack.cuh"

static int fails = 0;
#define CHECK(c)                                              \
  do {                                                        \
    if (!(c)) {                                               \
      std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); \
      fails++;                                                \
    }                                                         \
  } while (0)

// summary bit of voxel (x,y,z): OR over the box {x-1,x} x {y-1,y} (x {z-1,z}), outside = occupied
static bool summary_literal(const std::vector<int8_t> &g, int dim, int nx, int ny, int x, int y, int z) {
  for (int dz = 0; dz <= (dim == 3 ? 1 : 0); dz++)
    for (int dy = 0; dy <= 1; dy++)
      for (int dx = 0; dx <= 1; dx++) {
        const int a = x - dx, b = y - dy, c = z - dz;
        if (a < 0 || b < 0 || c < 0) return true;
        if (g[(size_t)a + (size_t)nx * ((size_t)b + (size_t)ny * c)] == 100) return true;
      }
  return false;
}

int main() {
  std::mt19937 rng(11);
  long voxels = 0, padding = 0;
  for (int t = 0; t < 600; t++) {
    const int dim = 2 + (t & 1);
    // dims around and across brick sizes (8 per axis in 3-D; 32 x 16 in 2-D), mostly not multiples
    const int nx = 1 + rng() % (dim == 3 ? 41 : 100), ny = 1 + rng() % (dim == 3 ? 27 : 50);
    const int nz = dim == 3 ? 1 + (int)(rng() % 19) : 1;
    const size_t nvox = (size_t)nx * ny * nz, nw = (nvox + 31) / 32;
    const unsigned pct = rng() % 60;
    std::vector<int8_t> g(nvox);
    for (auto &v : g) v = rng() % 100 < pct ? 100 : (int8_t)((int)(rng() % 3) - 1) * 50;
    std::vector<uint32_t> occ(nw);
    for (size_t w = 0; w < nw; w++) occ[w] = mplx::pack_word<true>(g.data(), w, nvox);

    // literal brick geometry
    const int bx = dim == 3 ? 8 : 32, by = dim == 3 ? 8 : 16, bz = dim == 3 ? 8 : 1;
    const int nbx = (nx + bx - 1) / bx, nby = (ny + by - 1) / by, nbz = (nz + bz - 1) / bz;
    const size_t npairs = (size_t)nbx * nby * nbz * 16;
    CHECK(mplx::occ2_pair_count(dim, nx, ny, nz) == npairs);
    CHECK(mplx::occ2_bricks_x(dim, nx) == nbx && mplx::occ2_bricks_y(dim, ny) == nby);
    std::vector<uint32_t> po(npairs), ps(npairs);
    for (size_t p = 0; p < npairs; p++) mplx::occ2_brick_pair(occ.data(), p, nvox, dim, nx, ny, nz, po[p], ps[p]);

    std::vector<uint32_t> owned(npairs, 0);  // bits some voxel maps to
    for (int z = 0; z < nz; z++)
      for (int y = 0; y < ny; y++)
        for (int x = 0; x < nx; x++, voxels++) {
          const size_t brick = (size_t)(x / bx) + (size_t)nbx * ((size_t)(y / by) + (size_t)nby * (z / bz));
          const int local = dim == 3 ? x % 8 + 8 * (y % 8) + 64 * (z % 8) : x % 32 + 32 * (y % 16);
          const size_t pair = brick * 16 + local / 32;
          const unsigned bit = local % 32;
          const unsigned p = dim == 3 ? mplx::occ2_pair<3>(x, y, z, nbx, nby) : mplx::occ2_pair<2>(x, y, 0, nbx, nby);
          const unsigned b = dim == 3 ? mplx::occ2_bit<3>(x, y) : mplx::occ2_bit<2>(x, y);
          CHECK(p == pair && b == bit);
          if (p != pair || b != bit) continue;
          CHECK(((owned[pair] >> bit) & 1u) == 0);  // distinct
          owned[pair] |= 1u << bit;
          const size_t i = (size_t)x + (size_t)nx * ((size_t)y + (size_t)ny * z);
          CHECK(((po[pair] >> bit) & 1u) == (g[i] == 100 ? 1u : 0u));
          CHECK(((ps[pair] >> bit) & 1u) == (summary_literal(g, dim, nx, ny, x, y, z) ? 1u : 0u));
        }
    for (size_t p = 0; p < npairs; p++) {
      CHECK((po[p] | owned[p]) == ~0u && (ps[p] | owned[p]) == ~0u);  // padding reads occupied, summary set
      padding += __builtin_popcount(~owned[p]);
    }
  }
  std::printf("occ2 bricks: %ld voxels, %ld padding bits checked\n", voxels, padding);
  std::printf("occ2_bricks_host fails %d\n", fails);
  return fails ? 1 : 0;
}
