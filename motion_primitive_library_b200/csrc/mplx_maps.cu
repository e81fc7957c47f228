// mplx_maps.cu — the two map transforms that sit right before the expansion path in the
// distance-map planner (SURVEY.md §8f row 2), on the device grids:
//   mplx_update_potential_map  = MapPlanner<Dim>::createMask + updatePotentialMap
//                                (src/mpl_planner/map_planner.cpp:286-391)
//   mplx_set_search_region_path = MapPlanner<Dim>::setSearchRegion (src/mpl_planner/map_planner.cpp:46-95)
//
// Potential field.  The reference stamps, around every cell with map > 0 (inside the optional
// source range), max() of the stencil  (int8)(100 * pow((1 - hypot(dx,dy)/rn) * (1 - |dz|/hn), pow))
// (2-D: without the dz factor), kept when > 1e-3 and hypot <= rn.  For a fixed dz the value is
// monotone in a = 1 - hypot(dx,dy)/rn, so the maximum over the sources of one z-layer is attained at
// the source with the largest a.  All floating point is done ON THE HOST with the same libm calls
// as the reference (std::hypot, std::pow): the host builds
//   pair_rank[|dx|][|dy|]  rank of a among the distinct values, 0 = largest (255 = outside rn)
//   htab[rank][|dz|]       the int8 stencil value (-128 = not in the mask: h <= 1e-3)
// and the device only does integer work: kernel 1 finds, per cell and layer, the best rank among
// the occupied cells of its (2rn+1)^2 window by scanning the occupancy bits; kernel 2 takes the max
// of htab over the 2hn+1 neighbouring layers.  O(voxels * window-words) instead of the reference's
// O(occupied * stencil) scatter with max(), and bit-exact with it (tests/test_maps_gpu.py).
#include <cuda_runtime.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "mplx_internal.h"
#include "mplx_search.cuh"

namespace mplx {

constexpr int kNoRank = 255;

// source mask: 1 bit per voxel, set when map > 0 and the cell lies inside [lo, hi) per axis
__global__ void source_bits_kernel(const int8_t *__restrict__ map, int nx, int ny, int nz, int lo0, int lo1, int lo2,
                                   int hi0, int hi1, int hi2, uint32_t *__restrict__ bits) {
  const size_t nvox = (size_t)nx * ny * nz;
  const size_t nwords = (nvox + 31) >> 5;
  for (size_t wd = (size_t)blockIdx.x * blockDim.x + threadIdx.x; wd < nwords; wd += (size_t)gridDim.x * blockDim.x) {
    uint32_t m = 0;
    for (int b = 0; b < 32; b++) {
      const size_t i = (wd << 5) + b;
      if (i >= nvox) break;
      const int x = (int)(i % nx), y = (int)((i / nx) % ny), z = (int)(i / ((size_t)nx * ny));
      if (map[i] > 0 && x >= lo0 && x < hi0 && y >= lo1 && y < hi1 && z >= lo2 && z < hi2) m |= 1u << b;
    }
    bits[wd] = m;
  }
}

// kernel 1: best (smallest) rank of an occupied source cell in the cell's own z-layer window
__global__ void layer_rank_kernel(const uint32_t *__restrict__ src, int nx, int ny, int nz, int rn,
                                  const uint8_t *__restrict__ pair_rank, uint8_t *__restrict__ rank) {
  const size_t nvox = (size_t)nx * ny * nz;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvox; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % nx), y = (int)((i / nx) % ny), z = (int)(i / ((size_t)nx * ny));
    int best = kNoRank;
    const int x0 = max(0, x - rn), x1 = min(nx - 1, x + rn);
    for (int yy = max(0, y - rn); yy <= min(ny - 1, y + rn); yy++) {
      const size_t row = ((size_t)z * ny + yy) * nx;
      const uint8_t *pr = pair_rank + (size_t)abs(yy - y) * (rn + 1);
      const size_t b0 = row + x0, b1 = row + x1;
      for (size_t wd = b0 >> 5; wd <= (b1 >> 5); wd++) {
        uint32_t m = __ldg(src + wd);
        const size_t base = wd << 5;
        if (base < b0) m &= ~0u << (b0 - base);
        if (base + 31 > b1) m &= ~0u >> (base + 31 - b1);
        while (m) {
          const int b = __ffs(m) - 1;
          m &= m - 1;
          const int xx = (int)(base + b - row);
          best = min(best, (int)pr[abs(xx - x)]);
        }
      }
    }
    rank[i] = (uint8_t)best;
  }
}

// kernel 2: dmap = copy of the grid; source cells become 100; max over the neighbouring layers
__global__ void potential_combine_kernel(const int8_t *__restrict__ map, const uint32_t *__restrict__ src,
                                         const uint8_t *__restrict__ rank, int nx, int ny, int nz, int hn,
                                         const int8_t *__restrict__ htab, int8_t *__restrict__ out) {
  const size_t nvox = (size_t)nx * ny * nz, layer = (size_t)nx * ny;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvox; i += (size_t)gridDim.x * blockDim.x) {
    const int z = (int)(i / layer);
    int v = map[i];
    if ((src[i >> 5] >> (i & 31)) & 1u) v = 100;  // dmap[idx] = H_MAX (map_planner.cpp:354,372)
    for (int dz = -hn; dz <= hn; dz++) {
      const int zs = z - dz;  // a source at layer zs stamps offset n(2) = dz onto this cell
      if (zs < 0 || zs >= nz) continue;
      const int r = rank[i - (size_t)dz * layer];
      if (r != kNoRank) v = max(v, (int)htab[r * (hn + 1) + abs(dz)]);
    }
    out[i] = (int8_t)v;
  }
}

// search region: every (path cell, box offset) sets one bit
__global__ void region_stamp_kernel(const int *__restrict__ cells, int n_cells, int dim, int nx, int ny, int nz, int r0,
                                    int r1, int r2, uint32_t *__restrict__ bits) {
  const int w0 = 2 * r0 + 1, w1 = 2 * r1 + 1, w2 = dim == 3 ? 2 * r2 + 1 : 1;
  const size_t per = (size_t)w0 * w1 * w2, total = per * n_cells;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t / per);
    size_t o = t % per;
    const int dx = (int)(o % w0) - r0;
    o /= w0;
    const int dy = (int)(o % w1) - r1;
    o /= w1;
    const int dz = dim == 3 ? (int)o - r2 : 0;
    const int x = cells[c * 3] + dx, y = cells[c * 3 + 1] + dy, z = cells[c * 3 + 2] + dz;
    if (x < 0 || x >= nx || y < 0 || y >= ny || z < 0 || z >= nz) continue;  // isOutside (map_planner.cpp:86)
    const size_t idx = (size_t)x + (size_t)nx * y + (size_t)nx * ny * z;
    atomicOr(bits + (idx >> 5), 1u << (idx & 31));
  }
}

static int grid_for(size_t n) {
  size_t g = (n + 255) / 256;
  const size_t cap = (size_t)sm_count() * 32;
  if (g > cap) g = cap;
  return g < 1 ? 1 : (int)g;
}

}  // namespace mplx

using namespace mplx;

// floatToInt on the host, map_util.h:103-108
static void float_to_int(const mplx_ctx *c, const double *pt, int *pn) {
  for (int k = 0; k < 3; k++) pn[k] = k < c->dim ? (int)std::round((pt[k] - c->P.origin[k]) / c->P.res - 0.5) : 0;
}

extern "C" int mplx_update_potential_map(mplx_ctx *c, const double *radius, double pow_, const double *range,
                                         const double *pos, double potential_weight, double gradient_weight,
                                         int8_t *out_map) {
  if (int r = mplx_bind(c)) return r;
  if (!c->has_map) return fail(MPLX_ERR_ARG, "mplx_set_map must be called first");
  if (!radius) return fail(MPLX_ERR_ARG, "radius is null");
  if (!(pow_ > 0)) return fail(MPLX_ERR_ARG, "pow must be > 0 (the stencil must decrease with distance)");
  const int dim = c->dim;
  const int nx = c->P.mdim[0], ny = c->P.mdim[1], nz = dim == 3 ? c->P.mdim[2] : 1;
  const double res = c->P.res;
  // createMask: map_planner.cpp:286-320
  const int rn = (int)std::ceil(radius[0] / res);
  const int hn = dim == 3 ? (int)std::ceil(radius[2] / res) : 0;
  if (rn < 1 || (dim == 3 && hn < 1)) return fail(MPLX_ERR_ARG, "potential radius smaller than one cell");
  const double h_max = 100;  // H_MAX, map_planner.h:104
  std::vector<double> avals;
  for (int i = 0; i <= rn; i++)
    for (int j = 0; j <= rn; j++)
      if (!(std::hypot(i, j) > rn)) avals.push_back(1 - (double)std::hypot(i, j) / rn);
  std::sort(avals.begin(), avals.end(), [](double a, double b) { return a > b; });
  avals.erase(std::unique(avals.begin(), avals.end()), avals.end());
  if (avals.size() >= (size_t)kNoRank) return fail(MPLX_ERR_ARG, "potential radius of %d cells is too large (rank table)", rn);
  std::vector<uint8_t> pair_rank((size_t)(rn + 1) * (rn + 1), (uint8_t)kNoRank);
  for (int i = 0; i <= rn; i++)
    for (int j = 0; j <= rn; j++) {
      if (std::hypot(i, j) > rn) continue;
      const double a = 1 - (double)std::hypot(i, j) / rn;
      const size_t rk = std::find(avals.begin(), avals.end(), a) - avals.begin();
      pair_rank[(size_t)j * (rn + 1) + i] = (uint8_t)rk;  // indexed [|dy|][|dx|]
    }
  std::vector<int8_t> htab(avals.size() * (hn + 1), (int8_t)-128);  // -128: offset not in the mask
  for (size_t rk = 0; rk < avals.size(); rk++)
    for (int z = 0; z <= hn; z++) {
      const double h = dim == 3 ? h_max * std::pow(avals[rk] * (1 - (double)z / hn), pow_) : h_max * std::pow(avals[rk], pow_);
      if (h > 1e-3) htab[rk * (hn + 1) + z] = (int8_t)h;
    }
  // source range: updatePotentialMap, map_planner.cpp:326-346
  int lo[3] = {0, 0, 0}, hi[3] = {nx, ny, nz};
  double rnorm = 0;
  if (range)
    for (int k = 0; k < dim; k++) rnorm += range[k] * range[k];
  if (rnorm > 0) {
    if (!pos) return fail(MPLX_ERR_ARG, "pos is required with a potential map range");
    double a[3] = {0, 0, 0}, b[3] = {0, 0, 0};
    for (int k = 0; k < dim; k++) a[k] = pos[k] - range[k], b[k] = pos[k] + range[k];
    int c1[3], c2[3];
    float_to_int(c, a, c1);
    float_to_int(c, b, c2);
    for (int k = 0; k < dim; k++) {
      const int d = c->P.mdim[k];
      lo[k] = c1[k] < 0 ? 0 : (c1[k] >= d ? d - 1 : c1[k]);
      hi[k] = c2[k] < 0 ? 0 : (c2[k] >= d ? d - 1 : c2[k]);
    }
  }
  cudaStream_t st = c->stream;
  const size_t nvox = c->nvox;
  ScopedDevBuf<uint32_t> src;
  ScopedDevBuf<uint8_t> rank, d_pair;
  ScopedDevBuf<int8_t> d_htab;
  int rc = MPLX_OK;
  cudaError_t e = src.reserve((nvox + 31) / 32);
  if (e == cudaSuccess) e = rank.reserve(nvox);
  if (e == cudaSuccess) e = d_pair.reserve(pair_rank.size());
  if (e == cudaSuccess) e = d_htab.reserve(htab.size());
  if (e == cudaSuccess) e = c->pot.reserve(nvox);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_pair.p, pair_rank.data(), pair_rank.size(), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_htab.p, htab.data(), htab.size(), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) {
    source_bits_kernel<<<grid_for((nvox + 31) / 32), 256, 0, st>>>(c->map.p, nx, ny, nz, lo[0], lo[1], lo[2], hi[0], hi[1],
                                                                   hi[2], src.p);
    layer_rank_kernel<<<grid_for(nvox), 256, 0, st>>>(src.p, nx, ny, nz, rn, d_pair.p, rank.p);
    potential_combine_kernel<<<grid_for(nvox), 256, 0, st>>>(c->map.p, src.p, rank.p, nx, ny, nz, hn, d_htab.p, c->pot.p);
    e = cudaGetLastError();
    c->launches += 3;
  }
  // map_util_->setMap(.., dmap, ..) and ENV_->set_potential_map(dmap): map_planner.cpp:387-388
  if (e == cudaSuccess) e = cudaMemcpyAsync(c->map.p, c->pot.p, nvox, cudaMemcpyDeviceToDevice, st);
  if (e == cudaSuccess) e = launch_pack_bits(c->map.p, nvox, c->occ.p, true, st);
  if (e == cudaSuccess) e = launch_pack_occ2(c->occ.p, nvox, c->dim, nx, ny, nz, c->occ2.p, st);
  if (e == cudaSuccess && out_map) e = cudaMemcpyAsync(out_map, c->pot.p, nvox, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  src.release();
  rank.release();
  d_pair.release();
  d_htab.release();
  if (e != cudaSuccess) {
    cudaGetLastError();
    rc = fail(e == cudaErrorMemoryAllocation ? MPLX_ERR_ALLOC : MPLX_ERR_CUDA, "mplx_update_potential_map: %s",
              cudaGetErrorString(e));
    return rc;
  }
  c->launches++;
  c->has_pot = true;
  c->P.pot_w = potential_weight;
  c->P.grad_w = gradient_weight;
  c->P.pot = c->pot.p;
  size_l2_window(c);  // no occ2 carve-out beside a potential field
  c->P.occ2_bytes = c->occ2_window;
  return MPLX_OK;
}

// The grid geometry the ray trace of MapPlanner::setSearchRegion reads (search::segment_cells): no map values.
search::Grid mplx::region_grid(const mplx_ctx *c) {
  search::Grid G{};
  G.map = nullptr;
  G.dim = c->dim;
  G.res = c->P.res;
  for (int k = 0; k < 3; k++) {
    G.mdim[k] = c->P.mdim[k];
    G.origin[k] = c->P.origin[k];
  }
  return G;
}

// The path cells of MapPlanner::setSearchRegion (map_planner.cpp:49-58, MapUtil::rayTrace map_util.h:120-137),
// appended to `cells` as (x, y, z) triples (z = 0 in 2-D): every point's cell with `dense`, else each segment's
// cells as search::segment_cells walks them (the device build of mplx_set_batch_regions walks the same).
namespace {
struct PushCells {  // a plain host functor: segment_cells is __host__ __device__, so no (constexpr) lambda
  std::vector<int> *cells;
  void operator()(int, const int *pn) const { cells->insert(cells->end(), pn, pn + 3); }
};
}  // namespace

static void region_path_cells(const mplx_ctx *c, const double *path, int n_pts, int dense, std::vector<int> &cells) {
  const int dim = c->dim;
  const search::Grid G = region_grid(c);
  const PushCells push{&cells};
  if (!dense) {
    for (int i = 1; i < n_pts; i++) search::segment_cells(G, path + (size_t)(i - 1) * dim, path + (size_t)i * dim, push);
  } else {
    for (int i = 0; i < n_pts; i++) {
      int pn[3] = {0, 0, 0};
      for (int k = 0; k < dim; k++) pn[k] = search::float_to_int(G, path[(size_t)i * dim + k], k);
      push(i, pn);
    }
  }
}

// The tunnel's half-width in cells per axis, ceil(radius/res) (map_planner.cpp:61-63); 0 beyond ctx-dim.
void mplx::region_radius_cells(const mplx_ctx *c, const double *radius, int *rn) {
  for (int k = 0; k < 3; k++) rn[k] = k < c->dim ? (int)std::ceil(radius[k] / c->P.res) : 0;
}

extern "C" int mplx_set_search_region_path(mplx_ctx *c, const double *path, int n_pts, const double *radius, int dense,
                                           uint8_t *out_region) {
  if (int r = mplx_bind(c)) return r;
  if (!c->has_map) return fail(MPLX_ERR_ARG, "mplx_set_map must be called first");
  if (!path || n_pts < 1 || !radius) return fail(MPLX_ERR_ARG, "path/radius missing");
  const int dim = c->dim;
  const int nx = c->P.mdim[0], ny = c->P.mdim[1], nz = dim == 3 ? c->P.mdim[2] : 1;
  std::vector<int> cells;
  region_path_cells(c, path, n_pts, dense, cells);
  int rn[3];
  region_radius_cells(c, radius, rn);
  cudaStream_t st = c->stream;
  const size_t nvox = c->nvox, nwords = (nvox + 31) / 32;
  const int ncell = (int)(cells.size() / 3);
  ScopedDevBuf<int> d_cells;
  CU(c->region.reserve(nwords));
  CU(cudaMemsetAsync(c->region.p, 0, nwords * sizeof(uint32_t), st));
  if (ncell > 0) {
    CU(d_cells.reserve(cells.size()));
    CU(cudaMemcpyAsync(d_cells.p, cells.data(), cells.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    const size_t total = (size_t)ncell * (2 * rn[0] + 1) * (2 * rn[1] + 1) * (dim == 3 ? 2 * rn[2] + 1 : 1);
    region_stamp_kernel<<<grid_for(total), 256, 0, st>>>(d_cells.p, ncell, dim, nx, ny, nz, rn[0], rn[1], rn[2], c->region.p);
    CU(cudaGetLastError());
    c->launches++;
  }
  if (out_region) {
    // one byte per voxel for the host copy of env_base::search_region_
    std::vector<uint32_t> bits(nwords);
    CU(cudaMemcpyAsync(bits.data(), c->region.p, nwords * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (size_t i = 0; i < nvox; i++) out_region[i] = (bits[i >> 5] >> (i & 31)) & 1u;
  } else {
    CU(cudaStreamSynchronize(st));
  }
  d_cells.release();
  c->has_region = true;
  c->P.region_bits = c->region.p;
  return MPLX_OK;
}
