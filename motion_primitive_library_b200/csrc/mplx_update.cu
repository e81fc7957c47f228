// mplx_update.cu — sparse edits of the device grid (mplx_update_cells) and the read-back of the
// grid and its packed views (mplx_read_map).
//
// An edit of n voxels costs O(n) device work and 5n bytes over PCIe, instead of the full upload and
// the two full-grid packs of mplx_set_map:
//   1. the (index, value) pairs are sorted by index with a stable radix sort (skipped when the host
//      finds them already in order), so the last write of a voxel ends its run of equal indices;
//   2. scatter: the last entry of each run writes its byte into the grid;
//   3. every occupancy word holding an edited voxel is re-packed from its 32 bytes (pack_word);
//   4. every occ2 pair whose summary can read such a word is recomputed (occ2_summary_word).
// Steps 3 and 4 run one thread per distinct word (the first entry of each word in sorted order) and
// use the rules of the full packs on the final grid and occupancy, so the result is bit-identical to
// mplx_set_map of the edited grid.  Step 4 may recompute a pair none of whose summary bits changed
// (a neighbour across a row or plane end); recomputing it rewrites the value it already has.
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

// step 4: the summary of voxel j reads the occupancy of j - {0,1} - {0,nx} (- {0,nx*ny}), so a change in
// word w reaches the voxels 32w + [0, 32] + dy*nx (+ dz*nx*ny): two words per (dy, dz).
__global__ void repack_occ2_kernel(const uint32_t *__restrict__ idx, int n, const uint32_t *__restrict__ occ, size_t nvox,
                                   int dim, int nx, int ny, uint2 *__restrict__ occ2) {
  const size_t nwords = (nvox + 31) >> 5, sxy = (size_t)nx * ny;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    if (!first_of_word(idx, k)) continue;
    const size_t w = idx[k] >> 5;
    for (int dz = 0; dz <= (dim == 3 ? 1 : 0); dz++)
      for (int dy = 0; dy <= 1; dy++) {
        const size_t w0 = w + ((dy * (size_t)nx + dz * sxy) >> 5);
        for (size_t t = w0; t <= w0 + 1 && t < nwords; t++)
          occ2[t] = make_uint2(occ[t], occ2_summary_word(occ, t, nvox, dim, nx, ny));
      }
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
  const int nx = c->P.mdim[0], ny = c->P.mdim[1];
  scatter_last_kernel<<<grid, 256, 0, st>>>(d_idx, d_val, n, c->map.p);
  repack_occ_kernel<<<grid, 256, 0, st>>>(d_idx, n, c->map.p, c->nvox, c->occ.p);
  repack_occ2_kernel<<<grid, 256, 0, st>>>(d_idx, n, c->occ.p, c->nvox, c->dim, nx, ny, c->occ2.p);
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
  if (occ2) CU(cudaMemcpyAsync(occ2, c->occ2.p, nwords * sizeof(uint2), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return MPLX_OK;
}
