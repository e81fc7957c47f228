// mplx_update.cu — sparse edits of the device grid (mplx_update_cells) and the read-back of the
// grid and its packed views (mplx_read_map).
//
// An edit of n voxels costs O(n) device work and 5n bytes over PCIe, instead of the full upload and
// the two full-grid packs of mplx_set_map:
//   1. the (index, value) pairs are sorted by index with a stable radix sort (skipped when the host
//      finds them already in order), so the last write of a voxel ends its run of equal indices;
//   2. scatter: the last entry of each run writes its byte into the grid;
//   3. every occupancy word holding an edited voxel is re-packed from its 32 bytes (pack_word);
//   4. every occ2 brick pair holding a voxel whose summary an edited voxel reaches is recomputed
//      (occ2_guard_brick_pair, from the occupancy words of step 3 and occ2_summary_word); the guard band
//      around the map never changes.
// Step 3 runs one thread per distinct word (the first entry of each word in sorted order), step 4 one
// thread per edited voxel that reaches a pair its predecessor does not.  Both use the rules of the full
// packs on the final grid and occupancy, so the result is bit-identical to mplx_set_map of the edited
// grid.  Two threads may recompute the same pair; they write the same value.
#include <cub/device/device_radix_sort.cuh>
#include <cuda_runtime.h>
#include <string.h>

#include "mplx_internal.h"
#include "mplx_pack.cuh"

namespace mplx {

// step 2: the last write of each voxel (equal indices are adjacent and in array order)
__global__ void scatter_last_kernel(const uint32_t *__restrict__ idx, const int8_t *__restrict__ val, int n,
                                    int8_t *__restrict__ map) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    if (k == n - 1 || idx[k + 1] != idx[k]) map[idx[k]] = val[k];
}

__device__ __forceinline__ bool first_of_word(const uint32_t *idx, int k) {
  return k == 0 || (idx[k - 1] >> 5) != (idx[k] >> 5);
}

// step 3
__global__ void repack_occ_kernel(const uint32_t *__restrict__ idx, int n, const int8_t *__restrict__ map, size_t nvox,
                                  uint32_t *__restrict__ occ) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    if (first_of_word(idx, k)) occ[idx[k] >> 5] = pack_word<true>(map, idx[k] >> 5, nvox);
}

// step 4: the summary of voxel (x,y,z) reads the occupancy of {x-1,x} x {y-1,y} (x {z-1,z}), so an edit of
// voxel v reaches the summaries of v + {0,1}^dim: the pairs of those cells are recomputed.  A voxel whose
// predecessor in the sorted list is the voxel before it in x within the same brick row (not at either end
// of the row) reaches no pair the predecessor does not, and is skipped; duplicates are skipped too.
__global__ void repack_occ2_kernel(const uint32_t *__restrict__ idx, int n, const uint32_t *__restrict__ occ, size_t nvox,
                                   int dim, int nx, int ny, int nz, uint32_t *__restrict__ occ2) {
  const size_t npairs = occ2_guard_pair_count(dim, nx, ny, nz);
  const size_t sxy = (size_t)nx * ny;
  const int pbx = occ2_guard_bricks_x(dim, nx), pby = occ2_guard_bricks_y(dim, ny);
  const int xmask = dim == 3 ? 7 : 31;  // x extent of a brick row - 1
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const uint32_t v = idx[k];
    const int x = (int)(v % nx), y = (int)(v / nx % ny), z = (int)(v / sxy);
    if (k > 0 && (idx[k - 1] == v || (idx[k - 1] == v - 1 && (x & xmask) != 0 && (x & xmask) != xmask))) continue;
    unsigned done[8];
    int nd = 0;
    for (int dz = 0; dz <= (dim == 3 ? 1 : 0); dz++)
      for (int dy = 0; dy <= 1; dy++)
        for (int dx = 0; dx <= 1; dx++) {
          if (x + dx >= nx || y + dy >= ny || z + dz >= nz) continue;
          const unsigned p = dim == 3 ? occ2_guard_pair<3>(x + dx, y + dy, z + dz, pbx, pby)
                                      : occ2_guard_pair<2>(x + dx, y + dy, 0, pbx, pby);
          bool seen = false;
          for (int i = 0; i < nd; i++) seen = seen || done[i] == p;
          if (seen) continue;
          done[nd++] = p;
          uint32_t o, s;
          occ2_guard_brick_pair(occ, p, nvox, dim, nx, ny, nz, o, s);
          occ2[p] = o;
          occ2[npairs + p] = s;
        }
  }
}

// The pairs in voxel order, as mplx_read_map returns them: pair w holds the occupancy word w and the summary
// bits of voxels 32w..32w+31, gathered from the bricks of the padded map; bits at i >= nvox read as they did
// in voxel order (occupancy 0, summary 1).
__global__ void unbrick_occ2_kernel(const uint32_t *__restrict__ occ2, size_t npairs, size_t nvox, int dim, int nx,
                                    int ny, uint2 *__restrict__ out) {
  const size_t nwords = (nvox + 31) >> 5, sxy = (size_t)nx * ny;
  const int pbx = occ2_guard_bricks_x(dim, nx), pby = occ2_guard_bricks_y(dim, ny);
  for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += (size_t)gridDim.x * blockDim.x) {
    uint32_t o = 0, s = 0;
    for (int b = 0; b < 32; b++) {
      const size_t i = (w << 5) + b;
      if (i >= nvox) {
        s |= 1u << b;
        continue;
      }
      const int x = (int)(i % nx), y = (int)(i / nx % ny), z = (int)(i / sxy);
      const unsigned p = dim == 3 ? occ2_guard_pair<3>(x, y, z, pbx, pby) : occ2_guard_pair<2>(x, y, 0, pbx, pby);
      const unsigned bit = dim == 3 ? occ2_bit<3>(x, y) : occ2_bit<2>(x, y);
      o |= ((occ2[p] >> bit) & 1u) << b;
      s |= ((occ2[npairs + p] >> bit) & 1u) << b;
    }
    out[w] = make_uint2(o, s);
  }
}

static int grid_for_entries(int n) {
  const int cap = sm_count() * 16;
  const int g = (n + 255) / 256;
  return g < 1 ? 1 : (g > cap ? cap : g);
}

}  // namespace mplx

using namespace mplx;

extern "C" int mplx_update_cells(mplx_ctx *c, const int32_t *idx, const int8_t *values, int n) {
  if (int r = mplx_bind(c)) return r;
  if (!c->has_map) return fail(MPLX_ERR_ARG, "mplx_set_map must be called first");
  if (n < 0) return fail(MPLX_ERR_ARG, "n = %d < 0", n);
  if (n == 0) return MPLX_OK;
  if (!idx || !values) return fail(MPLX_ERR_ARG, "idx/values is null");
  bool sorted = true;
  for (int k = 0; k < n; k++) {
    if (idx[k] < 0 || (size_t)idx[k] >= c->nvox)
      return fail(MPLX_ERR_ARG, "idx[%d] = %d is outside the grid [0, %zu)", k, idx[k], c->nvox);
    sorted = sorted && (k == 0 || idx[k] >= idx[k - 1]);
  }
  UpdateBufs &B = c->ub;
  cudaStream_t st = c->stream;
  CU(B.h_idx.reserve(n));
  CU(B.h_val.reserve(n));
  CU(B.idx.reserve(n));
  CU(B.val.reserve(n));
  memcpy(B.h_idx.p, idx, sizeof(int32_t) * n);
  memcpy(B.h_val.p, values, n);
  CU(cudaMemcpyAsync(B.idx.p, B.h_idx.p, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(B.val.p, B.h_val.p, n, cudaMemcpyHostToDevice, st));
  const uint32_t *d_idx = B.idx.p;
  const int8_t *d_val = B.val.p;
  if (!sorted) {
    int end_bit = 1;
    while (end_bit < 32 && ((c->nvox - 1) >> end_bit) != 0) end_bit++;
    CU(B.idx_sorted.reserve(n));
    CU(B.val_sorted.reserve(n));
    size_t tmp_bytes = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, B.idx.p, B.idx_sorted.p, B.val.p, B.val_sorted.p, n, 0, end_bit,
                                       st));
    CU(B.sort_tmp.reserve(tmp_bytes));
    CU(cub::DeviceRadixSort::SortPairs(B.sort_tmp.p, tmp_bytes, B.idx.p, B.idx_sorted.p, B.val.p, B.val_sorted.p, n, 0,
                                       end_bit, st));
    d_idx = B.idx_sorted.p;
    d_val = B.val_sorted.p;
  }
  const int grid = grid_for_entries(n);
  const int nx = c->P.mdim[0], ny = c->P.mdim[1], nz = c->dim == 3 ? c->P.mdim[2] : 1;
  scatter_last_kernel<<<grid, 256, 0, st>>>(d_idx, d_val, n, c->map.p);
  repack_occ_kernel<<<grid, 256, 0, st>>>(d_idx, n, c->map.p, c->nvox, c->occ.p);
  repack_occ2_kernel<<<grid, 256, 0, st>>>(d_idx, n, c->occ.p, c->nvox, c->dim, nx, ny, nz, c->occ2.p);
  CU(cudaGetLastError());
  c->launches += 3;
  CU(cudaStreamSynchronize(st));
  return MPLX_OK;
}

extern "C" int mplx_read_map(mplx_ctx *c, int8_t *grid, uint32_t *occ, uint32_t *occ2) {
  if (int r = mplx_bind(c)) return r;
  if (!c->has_map) return fail(MPLX_ERR_ARG, "mplx_set_map must be called first");
  const size_t nwords = (c->nvox + 31) / 32;
  cudaStream_t st = c->stream;
  if (grid) CU(cudaMemcpyAsync(grid, c->map.p, c->nvox, cudaMemcpyDeviceToHost, st));
  if (occ) CU(cudaMemcpyAsync(occ, c->occ.p, nwords * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  if (occ2) {
    ScopedDevBuf<uint2> tmp;
    CU(tmp.reserve(nwords));
    const int grid = grid_for_entries(nwords < (1u << 30) ? (int)nwords : 1 << 30);
    const size_t npairs = occ2_guard_pair_count(c->dim, c->P.mdim[0], c->P.mdim[1], c->dim == 3 ? c->P.mdim[2] : 1);
    unbrick_occ2_kernel<<<grid, 256, 0, st>>>(c->occ2.p, npairs, c->nvox, c->dim, c->P.mdim[0], c->P.mdim[1], tmp.p);
    CU(cudaGetLastError());
    c->launches += 1;
    CU(cudaMemcpyAsync(occ2, tmp.p, nwords * sizeof(uint2), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));  // before tmp is freed
  }
  CU(cudaStreamSynchronize(st));
  return MPLX_OK;
}
