// The ray trace of MapPlanner::setSearchRegion on the CPU, two ways, for tests/test_segment_cells_cpu.py:
//   sc_walk  search::segment_cells (csrc/mplx_search.cuh), the walk mplx_set_search_region_path runs on the host and
//            the batch tunnel build runs on the device, compiled here by g++;
//   sc_loop  the per-segment loop region_path_cells (csrc/mplx_maps.cu) ran before it called that walk, restated.
// Both append (x, y, z) per cell, every point's cell with `dense`.
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include "../motion_primitive_library_b200/csrc/mplx_search.cuh"

using namespace mplx;

namespace {

search::Grid grid_of(int dim, const int *mdim, const double *origin, double res) {
  search::Grid G{};
  G.map = nullptr;
  G.dim = dim;
  G.res = res;
  for (int k = 0; k < 3; k++) {
    G.mdim[k] = mdim[k];
    G.origin[k] = origin[k];
  }
  return G;
}

int copy_out(const std::vector<int> &cells, int *out, int cap) {
  const int n = (int)(cells.size() / 3);
  if (n > cap) return -1;
  std::copy(cells.begin(), cells.end(), out);
  return n;
}

}  // namespace

extern "C" int sc_walk(int dim, const int *mdim, const double *origin, double res, const double *path, int n_pts,
                       int dense, int *out, int cap) {
  const search::Grid G = grid_of(dim, mdim, origin, res);
  std::vector<int> cells;
  auto push = [&](int, const int *pn) { cells.insert(cells.end(), pn, pn + 3); };
  if (!dense) {
    for (int i = 1; i < n_pts; i++) search::segment_cells(G, path + (size_t)(i - 1) * dim, path + (size_t)i * dim, push);
  } else {
    for (int i = 0; i < n_pts; i++) {
      int pn[3] = {0, 0, 0};
      for (int k = 0; k < dim; k++) pn[k] = search::float_to_int(G, path[(size_t)i * dim + k], k);
      push(i, pn);
    }
  }
  return copy_out(cells, out, cap);
}

extern "C" int sc_loop(int dim, const int *mdim, const double *origin, double res, const double *path, int n_pts,
                       int dense, int *out, int cap) {
  std::vector<int> cells;
  auto float_to_int = [&](const double *pt, int *pn) {
    for (int k = 0; k < 3; k++) pn[k] = k < dim ? (int)std::round((pt[k] - origin[k]) / res - 0.5) : 0;
  };
  auto push = [&](const int *pn) { cells.insert(cells.end(), pn, pn + 3); };
  auto outside = [&](const int *pn) {
    for (int k = 0; k < dim; k++)
      if (pn[k] < 0 || pn[k] >= mdim[k]) return true;
    return false;
  };
  if (!dense) {
    for (int i = 1; i < n_pts; i++) {
      const double *p1 = path + (size_t)(i - 1) * dim, *p2 = path + (size_t)i * dim;
      double diff[3] = {0, 0, 0}, linf = 0;
      for (int k = 0; k < dim; k++) {
        diff[k] = p2[k] - p1[k];
        linf = std::max(linf, std::abs(diff[k] / res));
      }
      const double kk = 0.8;
      const int max_diff = linf / kk;
      const double s = 1.0 / max_diff;
      int prev[3] = {-1, -1, -1};
      for (int n = 1; n < max_diff; n++) {
        double pt[3] = {0, 0, 0};
        for (int k = 0; k < dim; k++) pt[k] = p1[k] + (diff[k] * s) * n;
        int pn[3];
        float_to_int(pt, pn);
        if (outside(pn)) break;
        bool diffc = false;
        for (int k = 0; k < dim; k++) diffc = diffc || pn[k] != prev[k];
        if (diffc) push(pn);
        for (int k = 0; k < 3; k++) prev[k] = pn[k];
      }
      int pe[3];
      double q[3] = {0, 0, 0};
      for (int k = 0; k < dim; k++) q[k] = p2[k];
      float_to_int(q, pe);
      push(pe);
    }
  } else {
    for (int i = 0; i < n_pts; i++) {
      double q[3] = {0, 0, 0};
      for (int k = 0; k < dim; k++) q[k] = path[(size_t)i * dim + k];
      int pn[3];
      float_to_int(q, pn);
      push(pn);
    }
  }
  return copy_out(cells, out, cap);
}
