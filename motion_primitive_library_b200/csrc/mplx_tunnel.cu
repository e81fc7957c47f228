// mplx_tunnel.cu — mplx_set_batch_regions and mplx_set_batch_regions_recorded: one tunnel per query of the batched
// searches, stored as the bricks it touches (mplx_tunnel.cuh), so that its memory follows the tunnel's size rather
// than the map's.
//
// A query's points come from the host (pts) or from the path the last search call recorded for some query
// (SearchBufs::traj); the device traces them with search::segment_cells, the walk mplx_set_search_region_path runs on
// the host, so a query's tunnel is exactly the region that call builds from the same points.  The build is a fixed
// sequence of launches whatever the query count:
//   gather     one thread per point: its position, from the recorded states or the uploaded points;
//   count      one thread per point: the cells of the segment that ends there (dense: the point's own cell);
//   scan       cub::DeviceScan::ExclusiveSum: each point's first cell;
//   emit       one thread per point: its (cell, owner) pairs;
//   stamp      one slot per (path cell, brick the cell's box may touch): the (query, brick) key, or a sentinel;
//   sort       cub::DeviceRadixSort on the keys;
//   unique     cub::DeviceSelect::Unique;
//   offsets    each query's first brick (a lower bound per query; the one past the last query counts the bricks);
//   or         one thread per (path cell, brick) ORs the box's cells into the brick's mask words.
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <vector>

#include "mplx_internal.h"
#include "mplx_search.cuh"
#include "mplx_tunnel.cuh"

namespace mplx {
namespace {

// The points of every query, one after the other: point i belongs to query owner[i]; src[i] >= 0 is the recorded
// state traj[src[i]], src[i] < 0 the uploaded point pts[-1 - src[i]] (ctx-dim doubles each).
struct PathArgs {
  const int64_t *src;
  const int *owner;
  const mplx_waypoint *traj;
  const double *pts;
  double *pos;  // gathered: 3 doubles per point, 0 beyond ctx-dim
  int n_pts, dense;
  search::Grid G;
};

__global__ void tunnel_gather_kernel(PathArgs P) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n_pts; i += gridDim.x * blockDim.x) {
    const int64_t s = P.src[i];
    const double *p = s >= 0 ? P.traj[s].pos : P.pts + (-1 - s) * P.G.dim;
    for (int k = 0; k < 3; k++) P.pos[3 * (size_t)i + k] = k < P.G.dim ? p[k] : 0.0;
  }
}

// The cells point i contributes, emit(j, cell) for each: its own cell (dense), else those of the segment from the
// query's previous point (none for a query's first point).
template <typename Emit>
__device__ __forceinline__ int point_cells(const PathArgs &P, int i, Emit emit) {
  const double *p = P.pos + 3 * (size_t)i;
  if (P.dense) {
    int pn[3] = {0, 0, 0};
    for (int k = 0; k < P.G.dim; k++) pn[k] = search::float_to_int(P.G, p[k], k);
    emit(0, pn);
    return 1;
  }
  if (i == 0 || P.owner[i - 1] != P.owner[i]) return 0;
  return search::segment_cells(P.G, p - 3, p, emit);
}

// count[i] = the cells of point i, count[n_pts] = 0, so that the exclusive scan ends in the total
__global__ void tunnel_count_kernel(PathArgs P, int64_t *count) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= P.n_pts; i += gridDim.x * blockDim.x)
    count[i] = i < P.n_pts ? point_cells(P, i, [](int, const int *) {}) : 0;
}

__global__ void tunnel_emit_kernel(PathArgs P, const int64_t *first, int *cells, int *owner) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n_pts; i += gridDim.x * blockDim.x) {
    const int64_t o = first[i];
    const int q = P.owner[i];
    point_cells(P, i, [&](int j, const int *pn) {
      for (int k = 0; k < 3; k++) cells[3 * (o + j) + k] = pn[k];
      owner[o + j] = q;
    });
  }
}

struct StampArgs {
  const int *cells;  // (x, y, z) per path cell
  const int *owner;  // the query of each path cell
  int n_cells, dim, per_cell;
  int mdim[3], r[3];
};

// slot s of path cell c: the s-th brick of the cell's brick box, or the sentinel key (n_q, 0) beyond it
__device__ __forceinline__ bool stamp_slot(const StampArgs &A, int c, int s, int &bx, int &by, int &bz, int *lo,
                                           int *hi) {
  int blo[3], bhi[3];
  if (!tunnel_box(A.dim, A.mdim, A.cells + 3 * c, A.r, lo, hi, blo, bhi)) return false;
  const int nbx = bhi[0] - blo[0] + 1, nby = bhi[1] - blo[1] + 1, nbz = bhi[2] - blo[2] + 1;
  if (s >= nbx * nby * nbz) return false;
  bx = blo[0] + s % nbx;
  by = blo[1] + (s / nbx) % nby;
  bz = blo[2] + s / (nbx * nby);
  return true;
}

__global__ void tunnel_stamp_kernel(StampArgs A, uint64_t sentinel, uint64_t *keys) {
  const size_t total = (size_t)A.n_cells * A.per_cell;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t / A.per_cell), s = (int)(t % A.per_cell);
    int bx, by, bz, lo[3], hi[3];
    keys[t] = stamp_slot(A, c, s, bx, by, bz, lo, hi) ? tunnel_key(A.owner[c], tunnel_brick_id(A.mdim, bx, by, bz))
                                                      : sentinel;
  }
}

// off[q] = the first unique key >= (q, 0), for q in [0, n_q]; off[n_q] is the brick count
__global__ void tunnel_offsets_kernel(const uint64_t *ukeys, const int *n_unique, int n_q, int64_t *off) {
  const int n = *n_unique;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q <= n_q; q += gridDim.x * blockDim.x) {
    const uint64_t k = tunnel_key(q, 0);
    int lo = 0, hi = n;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ukeys[mid] < k) lo = mid + 1;
      else hi = mid;
    }
    off[q] = lo;
  }
}

__global__ void tunnel_or_kernel(StampArgs A, const uint64_t *ukeys, const int64_t *off, uint32_t *bits) {
  const size_t total = (size_t)A.n_cells * A.per_cell;
  const int W = tunnel_words(A.dim);
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t / A.per_cell), s = (int)(t % A.per_cell);
    int bx, by, bz, lo[3], hi[3];
    if (!stamp_slot(A, c, s, bx, by, bz, lo, hi)) continue;
    const int q = A.owner[c];
    const TunnelView tv{ukeys + off[q], nullptr, (int)(off[q + 1] - off[q]), q};
    const uint64_t k = tunnel_key(q, tunnel_brick_id(A.mdim, bx, by, bz));
    int a = 0, b = tv.n;
    while (a < b) {
      const int mid = (a + b) >> 1;
      if (tv.key[mid] < k) a = mid + 1;
      else b = mid;
    }
    uint32_t *m = bits + (size_t)(off[q] + a) * W;
    for (int w = 0; w < W; w++) {
      const uint32_t v = tunnel_box_word(A.dim, lo, hi, bx, by, bz, w);
      if (v) atomicOr(m + w, v);
    }
  }
}

int grid_for(size_t n) {
  size_t g = (n + 255) / 256;
  const size_t cap = (size_t)sm_count() * 32;
  if (g > cap) g = cap;
  return g < 1 ? 1 : (int)g;
}

int bits_for(uint64_t v) {
  int b = 0;
  while (b < 64 && (v >> b) != 0) b++;
  return b;
}

// The tunnels of n_q queries: query q's points are the recorded path of query from[q] of the last search call (from
// given and from[q] >= 0) or pts[pt_offset[q] .. pt_offset[q+1]).  Built aside; the ctx keeps its tunnels until the
// new ones are complete.
int set_regions(mplx_ctx *c, const char *fn, int n_q, const int32_t *from, bool recorded, const int64_t *pt_offset,
                const double *pts, const double *radius, int dense) {
  if (!c) return fail(MPLX_ERR_ARG, "%s: null ctx", fn);
  if (!c->has_map) return fail(MPLX_ERR_ARG, "%s: mplx_set_map must be called first", fn);
  if (n_q < 0) return fail(MPLX_ERR_ARG, "%s: n_q < 0", fn);
  if (int r = mplx_bind(c)) return r;
  if (n_q == 0) {
    c->tun.release();
    return MPLX_OK;
  }
  const SearchBufs &B = c->sb;
  bool with_pts = !recorded;
  if (recorded) {
    if (!from || !radius) return fail(MPLX_ERR_ARG, "%s: from or radius missing", fn);
    if (B.traj_state == kTrajNone) return fail(MPLX_ERR_ARG, "%s: no completed search call on this ctx", fn);
    if (B.traj_state == kTrajOff)
      return fail(MPLX_ERR_ARG, "%s: the last search call ran without recording (mplx_set_batch_trajectories)", fn);
    const int n_last = (int)B.traj_off.size() - 1;
    for (int q = 0; q < n_q; q++) {
      const int f = from[q];
      if (f >= n_last) return fail(MPLX_ERR_ARG, "%s: from[%d] = %d outside the last call's %d queries", fn, q, f, n_last);
      if (f >= 0 && B.traj_off[f + 1] == B.traj_off[f])
        return fail(MPLX_ERR_ARG, "%s: query %d of the last call has no recorded path", fn, f);
      with_pts = with_pts || f < 0;
    }
  }
  if (with_pts) {
    if (!pt_offset || !pts || !radius) return fail(MPLX_ERR_ARG, "%s: pt_offset, pts or radius missing", fn);
    if (pt_offset[0] != 0) return fail(MPLX_ERR_ARG, "%s: pt_offset[0] must be 0", fn);
    for (int q = 0; q < n_q; q++) {
      const bool own = !recorded || from[q] < 0;
      if (own ? pt_offset[q + 1] <= pt_offset[q] : pt_offset[q + 1] < pt_offset[q])
        return fail(MPLX_ERR_ARG, "%s: query %d has no points (pt_offset must increase)", fn, q);
    }
  }
  const int dim = c->dim;

  // every query's points: where each comes from and whose it is
  std::vector<int64_t> src;
  std::vector<int> owner_pt;
  for (int q = 0; q < n_q; q++) {
    const size_t before = src.size();
    if (recorded && from[q] >= 0) {
      for (int64_t s = B.traj_off[from[q]]; s < B.traj_off[from[q] + 1]; s++) src.push_back(B.slot_src[s]);
    } else {
      for (int64_t k = pt_offset[q]; k < pt_offset[q + 1]; k++) src.push_back(-1 - k);
    }
    owner_pt.insert(owner_pt.end(), src.size() - before, q);
  }
  if (src.size() > (size_t)INT32_MAX - 1) return fail(MPLX_ERR_ARG, "%s: %zu points exceed 2^31 - 2", fn, src.size());
  const int n_pts = (int)src.size();
  const int64_t n_up = with_pts ? pt_offset[n_q] : 0;  // uploaded points
  cudaStream_t st = c->stream;

  // the trace's scratch: sources, owners, positions, cell counts and their scan, and the uploaded points
  ScopedDevBuf<int64_t> d_src, d_count, d_first;
  ScopedDevBuf<int> d_owner_pt;
  ScopedDevBuf<double> d_pos, d_pts;
  ScopedDevBuf<unsigned char> scan_tmp;
  size_t scan_bytes = 0;
  CU(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int64_t *)nullptr, (int64_t *)nullptr, n_pts + 1, st));
  CU(d_src.reserve(n_pts));
  CU(d_owner_pt.reserve(n_pts));
  CU(d_pos.reserve((size_t)n_pts * 3));
  CU(d_count.reserve((size_t)n_pts + 1));
  CU(d_first.reserve((size_t)n_pts + 1));
  CU(d_pts.reserve(std::max<size_t>((size_t)n_up * dim, 1)));
  CU(scan_tmp.reserve(std::max<size_t>(scan_bytes, 1)));
  CU(cudaMemcpyAsync(d_src.p, src.data(), src.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(d_owner_pt.p, owner_pt.data(), owner_pt.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  if (n_up > 0)
    CU(cudaMemcpyAsync(d_pts.p, pts, (size_t)n_up * dim * sizeof(double), cudaMemcpyHostToDevice, st));
  const PathArgs P{d_src.p, d_owner_pt.p, B.traj.p, d_pts.p, d_pos.p, n_pts, dense ? 1 : 0, region_grid(c)};
  tunnel_gather_kernel<<<grid_for(n_pts), 256, 0, st>>>(P);
  CU(cudaGetLastError());
  tunnel_count_kernel<<<grid_for((size_t)n_pts + 1), 256, 0, st>>>(P, d_count.p);
  CU(cudaGetLastError());
  CU(cub::DeviceScan::ExclusiveSum(scan_tmp.p, scan_bytes, d_count.p, d_first.p, n_pts + 1, st));
  c->launches += 3;
  int64_t total_cells = 0;
  CU(cudaMemcpyAsync(&total_cells, d_first.p + n_pts, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));

  StampArgs A{};
  A.dim = dim;
  for (int k = 0; k < 3; k++) A.mdim[k] = c->P.mdim[k];
  region_radius_cells(c, radius, A.r);
  A.per_cell = tunnel_box_bricks(dim, A.r);
  const size_t n_slots = (size_t)total_cells * (size_t)A.per_cell;
  if (n_slots > (size_t)INT32_MAX)  // the unique count and the brick offsets are int
    return fail(MPLX_ERR_ARG, "%s: %zu (path cell, brick) pairs exceed 2^31 - 1", fn, n_slots);
  A.n_cells = (int)total_cells;
  const uint64_t sentinel = tunnel_key(n_q, 0);
  const int end_bit = 32 + bits_for((uint64_t)n_q);

  // the build's scratch: cells, owners, keys twice, the unique count and cub's temporary storage
  ScopedDevBuf<int> d_cells, d_owner, d_nu;
  ScopedDevBuf<uint64_t> k0, k1;
  ScopedDevBuf<unsigned char> tmp;
  size_t sort_tmp = 0, uniq_tmp = 0;
  CU(cub::DeviceRadixSort::SortKeys(nullptr, sort_tmp, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                    (int64_t)n_slots, 0, end_bit, st));
  CU(cub::DeviceSelect::Unique(nullptr, uniq_tmp, (const uint64_t *)nullptr, (uint64_t *)nullptr, (int *)nullptr,
                               (int64_t)n_slots, st));
  CU(d_cells.reserve(std::max<size_t>((size_t)A.n_cells * 3, 1)));
  CU(d_owner.reserve(std::max<size_t>((size_t)A.n_cells, 1)));
  CU(d_nu.reserve(1));
  CU(k0.reserve(std::max<size_t>(n_slots, 1)));
  CU(k1.reserve(std::max<size_t>(n_slots, 1)));
  CU(tmp.reserve(std::max<size_t>(std::max(sort_tmp, uniq_tmp), 1)));
  CU(cudaMemsetAsync(d_nu.p, 0, sizeof(int), st));
  if (A.n_cells > 0) {
    tunnel_emit_kernel<<<grid_for(n_pts), 256, 0, st>>>(P, d_first.p, d_cells.p, d_owner.p);
    CU(cudaGetLastError());
    c->launches++;
  }
  A.cells = d_cells.p;
  A.owner = d_owner.p;

  TunnelStore T;
  T.n_q = n_q;
  auto build = [&]() -> int {
    CU(T.off.reserve((size_t)n_q + 1));
    int n = 0;
    if (n_slots > 0) {
      tunnel_stamp_kernel<<<grid_for(n_slots), 256, 0, st>>>(A, sentinel, k0.p);
      CU(cudaGetLastError());
      CU(cub::DeviceRadixSort::SortKeys(tmp.p, sort_tmp, k0.p, k1.p, (int64_t)n_slots, 0, end_bit, st));
      CU(cub::DeviceSelect::Unique(tmp.p, uniq_tmp, k1.p, k0.p, d_nu.p, (int64_t)n_slots, st));
      n += 3;
    }
    tunnel_offsets_kernel<<<grid_for((size_t)n_q + 1), 256, 0, st>>>(k0.p, d_nu.p, n_q, T.off.p);
    CU(cudaGetLastError());
    n++;
    CU(cudaMemcpyAsync(&T.n_bricks, T.off.p + n_q, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    c->launches += n;
    // the store comes off the search budget, counting the tunnels it replaces as free
    size_t budget = 0;
    const int rc = search_budget(c, budget);
    if (rc) return rc;
    const size_t need = (size_t)T.n_bricks * (sizeof(uint64_t) + tunnel_words(dim) * sizeof(uint32_t)) +
                        ((size_t)n_q + 1) * sizeof(int64_t);
    if (need > budget)
      return fail(MPLX_ERR_ALLOC, "%s: the tunnels take %lld bytes, more than the search budget of %lld bytes", fn,
                  (long long)need, (long long)budget);
    CU(T.key.reserve(std::max<int64_t>(T.n_bricks, 1)));
    CU(T.bits.reserve(std::max<int64_t>(T.n_bricks, 1) * tunnel_words(dim)));
    if (T.n_bricks > 0) {
      CU(cudaMemcpyAsync(T.key.p, k0.p, T.n_bricks * sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
      CU(cudaMemsetAsync(T.bits.p, 0, T.n_bricks * tunnel_words(dim) * sizeof(uint32_t), st));
      tunnel_or_kernel<<<grid_for(n_slots), 256, 0, st>>>(A, T.key.p, T.off.p, T.bits.p);
      CU(cudaGetLastError());
      c->launches++;
    }
    CU(cudaStreamSynchronize(st));
    return MPLX_OK;
  };
  const int rc = build();
  if (rc) {
    T.release();
    return rc;
  }
  c->tun.release();
  c->tun = T;
  return MPLX_OK;
}

}  // namespace
}  // namespace mplx

using namespace mplx;

extern "C" int mplx_set_batch_regions(mplx_ctx *c, int n_q, const int64_t *pt_offset, const double *pts,
                                      const double *radius, int dense) {
  return set_regions(c, "mplx_set_batch_regions", n_q, nullptr, false, pt_offset, pts, radius, dense);
}

extern "C" int mplx_set_batch_regions_recorded(mplx_ctx *c, int n_q, const int32_t *from, const int64_t *pt_offset,
                                               const double *pts, const double *radius, int dense) {
  return set_regions(c, "mplx_set_batch_regions_recorded", n_q, from, true, pt_offset, pts, radius, dense);
}

extern "C" int mplx_batch_regions_info(mplx_ctx *c, int32_t *n_q, int64_t *n_bricks, int64_t *bytes) {
  if (!c) return fail(MPLX_ERR_ARG, "mplx_batch_regions_info: null ctx");
  if (n_q) *n_q = c->tun.n_q;
  if (n_bricks) *n_bricks = c->tun.n_bricks;
  if (bytes) *bytes = c->tun.n_q > 0 ? (int64_t)c->tun.bytes() : 0;
  return MPLX_OK;
}

extern "C" int mplx_read_batch_region(mplx_ctx *c, int q, uint8_t *out) {
  const char *fn = "mplx_read_batch_region";
  if (!c) return fail(MPLX_ERR_ARG, "%s: null ctx", fn);
  if (c->tun.n_q == 0) return fail(MPLX_ERR_ARG, "%s: no tunnels set (mplx_set_batch_regions)", fn);
  if (q < 0 || q >= c->tun.n_q) return fail(MPLX_ERR_ARG, "%s: query %d outside [0, %d)", fn, q, c->tun.n_q);
  if (!out) return fail(MPLX_ERR_ARG, "%s: null out", fn);
  if (int r = mplx_bind(c)) return r;
  const int dim = c->dim, W = tunnel_words(dim);
  int64_t off[2];
  CU(cudaMemcpy(off, c->tun.off.p + q, sizeof off, cudaMemcpyDeviceToHost));
  const int n = (int)(off[1] - off[0]);
  std::vector<uint64_t> key(n);
  std::vector<uint32_t> bits((size_t)n * W);
  if (n > 0) {
    CU(cudaMemcpy(key.data(), c->tun.key.p + off[0], n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(bits.data(), c->tun.bits.p + off[0] * W, bits.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  }
  const TunnelView tv{key.data(), bits.data(), n, q};
  const int *md = c->P.mdim;
  const int nz = dim == 3 ? md[2] : 1;
  size_t i = 0;
  for (int z = 0; z < nz; z++)
    for (int y = 0; y < md[1]; y++)
      for (int x = 0; x < md[0]; x++) out[i++] = tunnel_has(tv, dim, md, x, y, z) ? 1 : 0;
  return MPLX_OK;
}
