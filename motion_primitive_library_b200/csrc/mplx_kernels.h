// mplx_kernels.h — host-callable launchers of the sm_90a kernels (internal).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/mplx.h"

namespace mplx {
struct EnvParams;
constexpr int kMaxU = 1024;  // |U| upper bound (125 is the largest set the reference's users build)

// force_seq != 0 selects the literal per-thread sample loop (expand_seq_kernel) instead of
// the flat kernel; results are identical.
struct FxScratch;
cudaError_t launch_expand(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes,
                          const mplx_succ_out &o, cudaStream_t st, int force_seq, const FxScratch *fs = nullptr);
// The dealing kernel (mplx_deal.cu): phases A/B for `rounds` batches of 256 items per CTA, then
// phase C pulled from a CTA-wide ticket queue.  rounds <= 0 picks it from the batch size.  |U| <= 256.
constexpr int kDealMaxRounds = 8;
cudaError_t launch_expand_deal(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes,
                               const mplx_succ_out &o, cudaStream_t st, int rounds);
// The fixed-point kernel (mplx_fx.cu): occupancy planning only (fx_supported), |U| <= 256.
bool fx_supported(const EnvParams &P);
cudaError_t launch_expand_fx(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes, const mplx_succ_out &o,
                             cudaStream_t st);
// The node-cooperative, flat-item variant for large batches (mplx_fxn.cu).  amb_q / amb_n: the global
// queue of ambiguous primitives (amb_cap records of fx_amb_record_bytes() in kFxSegments segments,
// kFxSegments counters), re-evaluated by a second launch on the same stream.
struct FxScratch {
  void *q = nullptr;
  unsigned *n = nullptr;
  unsigned cap = 0;
};
bool fxn_supported(const EnvParams &P, int n_nodes);
cudaError_t launch_expand_fxn(const EnvParams &P, const mplx_waypoint *d_nodes, int n_nodes, const mplx_succ_out &o,
                              cudaStream_t st, void *amb_q, unsigned *amb_n, unsigned amb_cap);
size_t fx_amb_record_bytes();
// SMs of the current device: the grid-size rules of the launchers scale with it
int sm_count();
// occupancy bits -> {occupancy word, candidate-summary word} per 32 voxels (mplx_fx.cu)
cudaError_t launch_pack_occ2(const uint32_t *d_occ, size_t nvox, int dim, int nx, int ny, uint2 *d_out, cudaStream_t st);
// bytes -> 1 bit/voxel: occ ? (byte == 100) : (byte != 0)
cudaError_t launch_pack_bits(const int8_t *d_bytes, size_t nvox, uint32_t *d_bits, bool occ, cudaStream_t st);
// sample-time table of `for (t = 0; t < T; t += T/n)` for n = 0..kNMax
cudaError_t launch_build_ttab(double T, double *d_ttab, int *d_tcount, double *d_tdt, cudaStream_t st);
}  // namespace mplx
