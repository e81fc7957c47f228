// mplx_tunnel.cu — mplx_set_batch_regions: one tunnel per query of the batched searches, stored as the bricks it
// touches (mplx_tunnel.cuh), so that its memory follows the tunnel's size rather than the map's.
//
// The cells of each query's path come from the host ray trace that mplx_set_search_region_path runs
// (region_path_cells), so a query's tunnel is exactly the region that call builds from the same points.  The build
// is a fixed sequence of launches whatever the query count:
//   stamp      one slot per (path cell, brick the cell's box may touch): the (query, brick) key, or a sentinel;
//   sort       cub::DeviceRadixSort on the keys;
//   unique     cub::DeviceSelect::Unique;
//   offsets    each query's first brick (a lower bound per query; the one past the last query counts the bricks);
//   or         one thread per (path cell, brick) ORs the box's cells into the brick's mask words.
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <vector>

#include "mplx_internal.h"
#include "mplx_tunnel.cuh"

namespace mplx {
namespace {

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

}  // namespace
}  // namespace mplx

using namespace mplx;

extern "C" int mplx_set_batch_regions(mplx_ctx *c, int n_q, const int64_t *pt_offset, const double *pts,
                                      const double *radius, int dense) {
  const char *fn = "mplx_set_batch_regions";
  if (!c) return fail(MPLX_ERR_ARG, "%s: null ctx", fn);
  if (!c->has_map) return fail(MPLX_ERR_ARG, "%s: mplx_set_map must be called first", fn);
  if (n_q < 0) return fail(MPLX_ERR_ARG, "%s: n_q < 0", fn);
  if (int r = mplx_bind(c)) return r;
  if (n_q == 0) {
    c->tun.release();
    return MPLX_OK;
  }
  if (!pt_offset || !pts || !radius) return fail(MPLX_ERR_ARG, "%s: pt_offset, pts or radius missing", fn);
  if (pt_offset[0] != 0) return fail(MPLX_ERR_ARG, "%s: pt_offset[0] must be 0", fn);
  for (int q = 0; q < n_q; q++)
    if (pt_offset[q + 1] <= pt_offset[q])
      return fail(MPLX_ERR_ARG, "%s: query %d has no points (pt_offset must increase)", fn, q);
  const int dim = c->dim;

  // the path cells of every query, as mplx_set_search_region_path traces them
  std::vector<int> cells, owner;
  for (int q = 0; q < n_q; q++) {
    const size_t before = cells.size() / 3;
    region_path_cells(c, pts + (size_t)pt_offset[q] * dim, (int)(pt_offset[q + 1] - pt_offset[q]), dense, cells);
    owner.insert(owner.end(), cells.size() / 3 - before, q);
  }
  StampArgs A{};
  A.dim = dim;
  for (int k = 0; k < 3; k++) A.mdim[k] = c->P.mdim[k];
  region_radius_cells(c, radius, A.r);
  A.per_cell = tunnel_box_bricks(dim, A.r);
  const size_t n_slots = owner.size() * (size_t)A.per_cell;
  if (n_slots > (size_t)INT32_MAX)  // the unique count and the brick offsets are int
    return fail(MPLX_ERR_ARG, "%s: %zu (path cell, brick) pairs exceed 2^31 - 1", fn, n_slots);
  A.n_cells = (int)owner.size();
  const uint64_t sentinel = tunnel_key(n_q, 0);
  const int end_bit = 32 + bits_for((uint64_t)n_q);
  cudaStream_t st = c->stream;

  // the build's scratch: cells, owners, keys twice, the unique count and cub's temporary storage
  ScopedDevBuf<int> d_cells, d_owner, d_nu;
  ScopedDevBuf<uint64_t> k0, k1;
  ScopedDevBuf<unsigned char> tmp;
  size_t sort_tmp = 0, uniq_tmp = 0;
  CU(cub::DeviceRadixSort::SortKeys(nullptr, sort_tmp, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                    (int64_t)n_slots, 0, end_bit, st));
  CU(cub::DeviceSelect::Unique(nullptr, uniq_tmp, (const uint64_t *)nullptr, (uint64_t *)nullptr, (int *)nullptr,
                               (int64_t)n_slots, st));
  CU(d_cells.reserve(std::max<size_t>(cells.size(), 1)));
  CU(d_owner.reserve(std::max<size_t>(owner.size(), 1)));
  CU(d_nu.reserve(1));
  CU(k0.reserve(std::max<size_t>(n_slots, 1)));
  CU(k1.reserve(std::max<size_t>(n_slots, 1)));
  CU(tmp.reserve(std::max<size_t>(std::max(sort_tmp, uniq_tmp), 1)));
  CU(cudaMemsetAsync(d_nu.p, 0, sizeof(int), st));
  if (A.n_cells > 0) {
    CU(cudaMemcpyAsync(d_cells.p, cells.data(), cells.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(d_owner.p, owner.data(), owner.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  }
  A.cells = d_cells.p;
  A.owner = d_owner.p;

  TunnelStore T;  // built aside: the ctx keeps its tunnels until the new ones are complete
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
