// Host-side checks of the guard-banded occ2 buffer of csrc/mplx_pack.cuh, run by tests/test_occ2_guard_cpu.py
// (no device needed), against a literal per-cell statement on random grids with dims that are not multiples
// of the brick:
//   1. every padded pair the full pack builds (occ2_guard_brick_pair), guard band included: a map cell's bits
//      are its occupancy and candidate summary, every other bit is 1 in both words;
//   2. occ2_guard_pair / occ2_bit and the separable bit index occ2_sep_k (for the plain coordinates and for
//      the high words of the fixed-point loop) name the same pair and bit for every cell in [-G, dim+G);
//   3. the reach bound occ2_band_reach covers every sample of random primitives, evaluated with the loop's
//      own running-sum times and with the fixed-point chain of the sample loop: where the start cell is in the
//      map and reach + 2 <= G, every sample cell lies in the guard band.
#include <cmath>
#include <cstdio>
#include <cstring>
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

constexpr int G = mplx::kOcc2Guard;
constexpr int kHiBase = 0x41380000;         // high word of 1.5 * 2^20, the fixed-point loop's base (kFxHiBase)
constexpr double kMagic = 1572864.0;        // 1.5 * 2^20 (kFxMagic)
constexpr double kEps = 0x1p-26;            // kFxEps

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

template <int DIM>
static unsigned sep_k(int x, int y, int z, int H, const unsigned (&e)[3], unsigned k0) {
  int h[DIM];
  h[0] = x + H;
  h[1] = y + H;
  if (DIM == 3) h[DIM - 1] = z + H;
  return mplx::occ2_sep_k<DIM>(h, e, k0);
}

static long layout_cells = 0, guard_bits = 0;

static void check_layout(std::mt19937 &rng, int dim, int nx, int ny, int nz) {
  const size_t nvox = (size_t)nx * ny * nz, nw = (nvox + 31) / 32;
  const unsigned pct = rng() % 60;
  std::vector<int8_t> g(nvox);
  for (auto &v : g) v = rng() % 100 < pct ? 100 : (int8_t)((int)(rng() % 3) - 1) * 50;
  std::vector<uint32_t> occ(nw);
  for (size_t w = 0; w < nw; w++) occ[w] = mplx::pack_word<true>(g.data(), w, nvox);

  // literal padded geometry: the map shifted by G on every axis of its dimension, then bricked
  const int bx = dim == 3 ? 8 : 32, by = dim == 3 ? 8 : 16, bz = dim == 3 ? 8 : 1;
  const int PX = nx + 2 * G, PY = ny + 2 * G, PZ = dim == 3 ? nz + 2 * G : 1;
  const int pbx = (PX + bx - 1) / bx, pby = (PY + by - 1) / by, pbz = (PZ + bz - 1) / bz;
  const size_t npairs = (size_t)pbx * pby * pbz * 16;
  CHECK(mplx::occ2_guard_pair_count(dim, nx, ny, nz) == npairs);
  CHECK(mplx::occ2_guard_bricks_x(dim, nx) == pbx && mplx::occ2_guard_bricks_y(dim, ny) == pby &&
        mplx::occ2_guard_bricks_z(dim, nz) == pbz);
  std::vector<uint32_t> po(npairs), ps(npairs);
  for (size_t p = 0; p < npairs; p++) mplx::occ2_guard_brick_pair(occ.data(), p, nvox, dim, nx, ny, nz, po[p], ps[p]);
  unsigned e0[3], k00, eh[3], k0h;
  mplx::occ2_sep_terms(dim, nx, ny, 0, e0, k00);
  mplx::occ2_sep_terms(dim, nx, ny, kHiBase, eh, k0h);

  std::vector<uint32_t> owned(npairs, 0);  // bits some map cell owns
  const int zlo = dim == 3 ? -G : 0, zhi = dim == 3 ? nz + G : 1;
  for (int z = zlo; z < zhi; z++)
    for (int y = -G; y < ny + G; y++)
      for (int x = -G; x < nx + G; x++, layout_cells++) {
        const int X = x + G, Y = y + G, Z = dim == 3 ? z + G : 0;
        const size_t brick = (size_t)(X / bx) + (size_t)pbx * ((size_t)(Y / by) + (size_t)pby * (Z / bz));
        const int local = dim == 3 ? X % 8 + 8 * (Y % 8) + 64 * (Z % 8) : X % 32 + 32 * (Y % 16);
        const size_t pair = brick * 16 + local / 32;
        const unsigned bit = local % 32;
        const unsigned p = dim == 3 ? mplx::occ2_guard_pair<3>(x, y, z, pbx, pby) : mplx::occ2_guard_pair<2>(x, y, 0, pbx, pby);
        const unsigned b = dim == 3 ? mplx::occ2_bit<3>(x, y) : mplx::occ2_bit<2>(x, y);
        CHECK(p == pair && b == bit);
        const unsigned K = (unsigned)(pair * 32 + bit);
        for (int H : {0, kHiBase}) {
          const unsigned k = dim == 3 ? sep_k<3>(x, y, z, H, H ? eh : e0, H ? k0h : k00)
                                      : sep_k<2>(x, y, 0, H, H ? eh : e0, H ? k0h : k00);
          CHECK(k == K);
        }
        const bool in_map = x >= 0 && x < nx && y >= 0 && y < ny && z >= 0 && z < nz;
        if (!in_map) {
          CHECK(((po[pair] >> bit) & 1u) == 1u && ((ps[pair] >> bit) & 1u) == 1u);
          guard_bits++;
          continue;
        }
        CHECK(((owned[pair] >> bit) & 1u) == 0);  // distinct
        owned[pair] |= 1u << bit;
        const size_t i = (size_t)x + (size_t)nx * ((size_t)y + (size_t)ny * z);
        CHECK(((po[pair] >> bit) & 1u) == (g[i] == 100 ? 1u : 0u));
        CHECK(((ps[pair] >> bit) & 1u) == (summary_literal(g, dim, nx, ny, x, y, z) ? 1u : 0u));
      }
  for (size_t p = 0; p < npairs; p++) CHECK((po[p] | owned[p]) == ~0u && (ps[p] | owned[p]) == ~0u);
}

static int hi_word(double v) {
  uint64_t u;
  std::memcpy(&u, &v, 8);
  return (int)(u >> 32);
}

static long reach_samples = 0, reach_in_band = 0;

// One axis of a random primitive of order ORD in cell units, its start anywhere from just outside the map
// to just inside either edge.  Every loop sample (the reference's running sum t += T/n while t < T) is within
// the bound of its start, and where the rows would pass fx_band every fixed-point cell lies in [-G, dim+G).
template <int ORD>
static void check_reach(std::mt19937 &rng) {
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  const int dim = 1 + (int)(rng() % 200);
  const double T = rng() % 3 == 0 ? 1.0 : 0.25 + 2.0 * (U(rng) + 1.0);
  const double scale = (double)(1 + rng() % 40) / T;  // cells per unit time of the leading terms
  double C[ORD + 1];
  double y0;
  switch (rng() % 3) {
    case 0: y0 = U(rng) * 6.0; break;                 // near the low edge
    case 1: y0 = dim + U(rng) * 6.0; break;           // near the high edge
    default: y0 = (U(rng) + 1.0) * 0.5 * dim; break;  // anywhere
  }
  C[0] = y0 + (kMagic + kEps);
  for (int i = 1; i <= ORD; i++) C[i] = U(rng) * scale / std::pow(T, i - 1) * (rng() % 4 == 0 ? 0.0 : 1.0);
  if (rng() % 5 == 0) C[1] = std::round(C[1]);  // lattice-like values
  const double reach = mplx::occ2_band_reach<ORD>(C, T);
  const int c0 = hi_word(C[0]) - kHiBase;
  const bool band = c0 >= 0 && c0 < dim && reach + 2.0 <= (double)G;
  const int n = 5 + (int)(rng() % 60);
  const double dt = T / n;
  for (double t = 0; t < T; t += dt) {
    // the sample loop's chain: Horner in fused multiply-adds, C[0] last
    double h = C[ORD];
    for (int i = ORD - 1; i >= 1; i--) h = std::fma(h, t, C[i]);
    const double m = std::fma(h, t, C[0]);
    long double d = 0;
    for (int i = ORD; i >= 1; i--) d = (d + C[i]) * t;  // exact displacement, long double
    CHECK(std::fabs((double)d) <= reach * (1 + 1e-12) + 1e-12);
    reach_samples++;
    if (band) {
      const int c = hi_word(m) - kHiBase;
      CHECK(c >= -G && c < dim + G);
      reach_in_band++;
    }
  }
}

int main() {
  std::mt19937 rng(12);
  for (int t = 0; t < 200; t++) {
    const int dim = 2 + (t & 1);
    const int nx = 1 + rng() % (dim == 3 ? 41 : 100), ny = 1 + rng() % (dim == 3 ? 27 : 50);
    const int nz = dim == 3 ? 1 + (int)(rng() % 19) : 1;
    check_layout(rng, dim, nx, ny, nz);
  }
  std::printf("occ2 guard layout: %ld cells in [-G, dim+G), %ld guard-band bits checked\n", layout_cells, guard_bits);
  for (int t = 0; t < 40000; t++) {
    switch (t & 3) {
      case 0: check_reach<1>(rng); break;
      case 1: check_reach<2>(rng); break;
      case 2: check_reach<3>(rng); break;
      default: check_reach<4>(rng); break;
    }
  }
  std::printf("occ2 band reach: %ld samples, %ld of primitives inside the band\n", reach_samples, reach_in_band);
  std::printf("occ2_guard_host fails %d\n", fails);
  return fails ? 1 : 0;
}
