// Host-side checks of the sparse map updates, run by tests/test_map_update_cpu.py (no device needed):
//   MapUtil::setCells and its change journal (mpl_host.hpp): version bumps, last write wins, resets on
//   setMap / freeUnknown, truncation past journalLimit(), outside cells rejected with nothing changed;
//   the word rules of csrc/mplx_pack.cuh, which mplx_set_map and mplx_update_cells both use, against
//   the literal per-voxel statement of the occupancy and candidate-summary bits on random grids.
#include <cstdio>
#include <random>

#define __host__
#define __device__
#include "../motion_primitive_library_b200/csrc/mplx_pack.cuh"
#include "../motion_primitive_library_b200/host/mpl_host.hpp"

static int fails = 0;
#define CHECK(c)                                              \
  do {                                                        \
    if (!(c)) {                                               \
      std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); \
      fails++;                                                \
    }                                                         \
  } while (0)

// summary bit of voxel i: OR over the box {x-1,x} x {y-1,y} (x {z-1,z}), outside = occupied; 1 past nvox
static uint32_t summary_per_voxel(const std::vector<int8_t> &g, size_t wd, int dim, int nx, int ny, int nz) {
  const size_t nvox = g.size(), sxy = (size_t)nx * ny;
  uint32_t d = 0;
  for (int b = 0; b < 32; b++) {
    const size_t i = (wd << 5) + b;
    if (i >= nvox) { d |= 1u << b; continue; }
    const int x = (int)(i % nx), y = (int)((i / nx) % ny), z = (int)(i / sxy);
    bool any = false;
    for (int dz = 0; dz <= (dim == 3 ? 1 : 0); dz++)
      for (int dy = 0; dy <= 1; dy++)
        for (int dx = 0; dx <= 1; dx++)
          any = any || x - dx < 0 || y - dy < 0 || z - dz < 0 || g[i - dx - (size_t)dy * nx - (size_t)dz * sxy] == 100;
    if (any) d |= 1u << b;
  }
  (void)nz;
  return d;
}

int main() {
  std::mt19937 rng(5);
  {  // the word rules
    long words = 0;
    for (int t = 0; t < 2000; t++) {
      const int dim = 2 + (t & 1);
      const int nx = 1 + rng() % 70, ny = 1 + rng() % 40, nz = dim == 3 ? 1 + rng() % 12 : 1;
      const size_t nvox = (size_t)nx * ny * nz, nw = (nvox + 31) / 32;
      const unsigned pct = rng() % 101;
      std::vector<int8_t> g(nvox);
      for (auto &v : g) v = rng() % 100 < pct ? 100 : (int8_t)((int)(rng() % 3) - 1) * 50;  // 100 / -50 / 0 / 50
      std::vector<uint32_t> occ(nw);
      for (size_t w = 0; w < nw; w++) {
        occ[w] = mplx::pack_word<true>(g.data(), w, nvox);
        for (int b = 0; b < 32; b++) {
          const size_t i = (w << 5) + b;
          CHECK(((occ[w] >> b) & 1u) == (i < nvox && g[i] == 100 ? 1u : 0u));
        }
      }
      for (size_t w = 0; w < nw; w++, words++)
        CHECK(mplx::occ2_summary_word(occ.data(), w, nvox, dim, nx, ny) == summary_per_voxel(g, w, dim, nx, ny, nz));
    }
    std::printf("pack rules: %ld words checked\n", words);
  }
  {  // MapUtil::setCells and the journal
    MPL::MapUtil<3> mu;
    Veci<3> dim;
    dim(0) = 37; dim(1) = 29; dim(2) = 23;
    Vecf<3> ori;
    ori(0) = ori(1) = ori(2) = 0;
    const size_t nvox = 37 * 29 * 23;
    mu.setMap(ori, dim, MPL::Tmap(nvox, 0), 0.1);
    const unsigned long v0 = mu.version();
    std::size_t first = 99;
    CHECK(mu.changesSince(v0, first) && first == 0);      // nothing to apply
    CHECK(!mu.changesSince(v0 - 1, first));               // before the setMap: full copy
    CHECK(!mu.changesSince(~0ul, first));                 // a consumer that never copied the grid
    auto cell = [](int x, int y, int z) { Veci<3> c; c(0) = x; c(1) = y; c(2) = z; return c; };
    // last write wins within a call
    mu.setCells({cell(1, 2, 3), cell(36, 28, 22), cell(1, 2, 3)}, {100, -1, 7});
    CHECK(mu.version() == v0 + 1);
    CHECK(mu.map()[mu.getIndex(cell(1, 2, 3))] == 7 && mu.map()[nvox - 1] == -1);
    CHECK(mu.changesSince(v0, first) && first == 0 && mu.journalIndex().size() == 3);
    // ... and across calls; a consumer at v0+1 sees only the second call's entries
    mu.setCells({cell(1, 2, 3)}, {100});
    CHECK(mu.version() == v0 + 2 && mu.map()[mu.getIndex(cell(1, 2, 3))] == 100);
    CHECK(mu.changesSince(v0 + 1, first) && first == 3);
    CHECK(mu.journalIndex()[first] == mu.getIndex(cell(1, 2, 3)) && mu.journalValue()[first] == 100);
    {  // replaying the journal from v0 on the v0 grid gives the current grid
      MPL::Tmap g(nvox, 0);
      CHECK(mu.changesSince(v0, first));
      for (std::size_t k = first; k < mu.journalIndex().size(); k++) g[mu.journalIndex()[k]] = mu.journalValue()[k];
      CHECK(g == mu.map());
    }
    // an empty call still bumps the version and is covered
    mu.setCells({}, {});
    CHECK(mu.version() == v0 + 3 && mu.changesSince(v0 + 2, first) && first == mu.journalIndex().size());
    // outside cells throw with nothing changed
    const MPL::Tmap before = mu.map();
    const unsigned long vb = mu.version();
    for (const auto &bad : {cell(-1, 0, 0), cell(37, 0, 0), cell(0, 29, 0), cell(0, 0, 23)}) {
      bool threw = false;
      try {
        mu.setCells({cell(5, 5, 5), bad}, {100, 100});
      } catch (const std::out_of_range &) {
        threw = true;
      }
      CHECK(threw);
    }
    CHECK(mu.map() == before && mu.version() == vb);
    // freeUnknown and setMap reset the journal: an older consumer needs a full copy
    mu.freeUnknown();
    CHECK(mu.map()[nvox - 1] == 0 && !mu.changesSince(vb, first) && mu.changesSince(mu.version(), first));
    CHECK(mu.journalIndex().empty());
    mu.setCells({cell(2, 2, 2)}, {100});
    const unsigned long vs = mu.version();
    mu.setMap(ori, dim, mu.map(), 0.1);
    CHECK(!mu.changesSince(vs, first) && mu.journalIndex().empty());
    // truncation: more than journalLimit() entries since a version -> that version needs a full copy
    const unsigned long vt = mu.version();
    const std::size_t lim = mu.journalLimit();
    CHECK(lim == nvox / MPL::MapUtil<3>::kJournalFraction && lim > 0);
    vec_E<Veci<3>> cells;
    std::vector<int8_t> vals;
    for (std::size_t k = 0; k < lim; k++) {
      cells.push_back(cell((int)(k % 37), (int)(k / 37 % 29), (int)(k / (37 * 29))));
      vals.push_back(100);
    }
    mu.setCells(cells, vals);  // exactly at the limit: kept
    CHECK(mu.changesSince(vt, first) && mu.journalIndex().size() - first == lim);
    mu.setCells({cell(3, 3, 3)}, {0});  // one past: truncated
    CHECK(!mu.changesSince(vt, first) && !mu.changesSince(vt + 1, first));
    CHECK(mu.changesSince(mu.version(), first) && mu.journalIndex().empty());
    CHECK(mu.map()[mu.getIndex(cell(3, 3, 3))] == 0);
  }
  std::printf("map_update_host fails %d\n", fails);
  return fails ? 1 : 0;
}
