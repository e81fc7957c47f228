// mplx_packed.cu — mplx_expand_packed: the expansion with a dense, field-selected result stream
// for hosts on the far side of PCIe.
//
// The full get_succ contract returns, per successor, a 112-byte Waypoint + cost + action
// (env_map.h:147-149): 3.3 KB per 27-primitive expansion, which caps a PCIe Gen5 x16 link at
// ~15 M expansions/s.  What an A*/LPA* host actually consumes per successor is the lattice key
// (hm_[succ] lookup, graph_search.h:84), the edge cost, the action id, and — for a state it has
// not seen before — the state itself.  The fields of a Waypoint that ARE state are exactly the
// ones its control flag marks use_pos/use_vel/use_acc/use_jrk/use_yaw (waypoint.h:47-56); the
// others are copies of the control input or literal zeros (e.g. ACC: acc = 0+u, jrk = 0, yaw = 0,
// t = curr.t + dt) and are rebuilt by the host wrapper without arithmetic on the path.
// So: after the expansion kernel has written its per-node segments in HBM, pack_kernel gathers
// the kept successors (optionally dropping +inf ones, which A* skips: graph_search.h:81) into
// dense arrays {state, cost, action(u16), key}; chunks are double-buffered over two streams so
// that chunk k's results cross PCIe while chunk k+1 is expanded.
#include <cuda_runtime.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "mplx_internal.h"

namespace mplx {

// One warp per node.  Node i's successors sit at [i*nU, i*nU + count[i]) of the strided arrays
// (control order).  Kept successors of a node are written contiguously, in control order, at a
// position reserved with one atomicAdd per node; offset[i] records it.
__global__ void __launch_bounds__(256)
pack_kernel(int n_nodes, int nU, int dim, int control, int drop_inf, const int32_t *__restrict__ count,
            const mplx_waypoint *__restrict__ succ, const double *__restrict__ cost,
            const int32_t *__restrict__ action, const uint64_t *__restrict__ key, long long *__restrict__ total,
            int32_t *__restrict__ kcount, long long *__restrict__ offset, double *__restrict__ pstate,
            double *__restrict__ pcost, uint16_t *__restrict__ paction, uint64_t *__restrict__ pkey) {
  const int lane = threadIdx.x & 31;
  const int node = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (node >= n_nodes) return;
  const int cnt = count[node];
  const size_t s0 = (size_t)node * nU;
  int kept = 0;
  for (int j0 = 0; j0 < cnt; j0 += 32) {
    const int j = j0 + lane;
    const bool k = j < cnt && !(drop_inf && isinf(cost[s0 + j]));
    kept += __popc(__ballot_sync(0xffffffffu, k));
  }
  long long base = 0;
  if (lane == 0) {
    base = kept ? atomicAdd((unsigned long long *)total, (unsigned long long)kept) : 0;
    kcount[node] = kept;
    offset[node] = base;
  }
  base = __shfl_sync(0xffffffffu, base, 0);
  const int nfields = __popc(control & 15);
  const int nstate = dim * nfields + ((control & 16) ? 1 : 0);
  int written = 0;
  for (int j0 = 0; j0 < cnt; j0 += 32) {
    const int j = j0 + lane;
    const bool k = j < cnt && !(drop_inf && isinf(cost[s0 + j]));
    const unsigned bal = __ballot_sync(0xffffffffu, k);
    if (k) {
      const long long r = base + written + __popc(bal & ((1u << lane) - 1u));
      const mplx_waypoint *w = succ + s0 + j;
      if (pstate) {
        double *ps = pstate + r * nstate;
        int c = 0;
        for (int d = 0; d < dim; d++) ps[c++] = w->pos[d];
        if (nfields >= 2) for (int d = 0; d < dim; d++) ps[c++] = w->vel[d];
        if (nfields >= 3) for (int d = 0; d < dim; d++) ps[c++] = w->acc[d];
        if (nfields >= 4) for (int d = 0; d < dim; d++) ps[c++] = w->jrk[d];
        if (control & 16) ps[c++] = w->yaw;
      }
      if (pcost) pcost[r] = cost[s0 + j];
      if (paction) paction[r] = (uint16_t)action[s0 + j];
      if (pkey) pkey[r] = key[s0 + j];
    }
    written += __popc(bal);
  }
}

}  // namespace mplx

extern "C" int mplx_expand_packed(mplx_ctx *c, const mplx_waypoint *nodes, int n_nodes, int flags,
                                  mplx_packed_out *out) {
  if (int r = mplx_bind(c)) return r;
  if (int r = mplx_check_ready(c, n_nodes)) return r;
  if (!out || !out->count || !out->offset) return fail(MPLX_ERR_ARG, "out->count and out->offset are required");
  const int nU = c->P.nU, dim = c->P.dim, control = c->P.control;
  const int nstate = dim * __builtin_popcount(control & 15) + ((control & 16) ? 1 : 0);
  out->nstate = nstate;
  out->total = 0;
  if (n_nodes == 0) return MPLX_OK;
  if (!nodes) return fail(MPLX_ERR_ARG, "nodes is null");
  if (nU > 65535) return fail(MPLX_ERR_ARG, "action ids are uint16 in the packed stream");
  const int drop_inf = (flags & MPLX_PACK_DROP_INF) ? 1 : 0;

  // Pipeline: chunks of ~2^21 successor slots cycle through kPackBufs buffer sets.  Two compute streams
  // alternate (copy-in of chunk k+1 overlaps the kernels of chunk k), and a third stream carries every
  // device-to-host copy, so a chunk's results cross PCIe while the next chunks are already being expanded:
  // the copy engine — the longest stage — stays busy.  The host has to learn a chunk's record count before it
  // can size that chunk's copies; it waits for chunk k-2's count after queueing chunk k.
  // Chunks of 2^21 slots: 2^20 pays ~7 % more in per-copy overhead (four copies per chunk), 2^22 leaves too
  // few chunks to overlap at the bench's batch size.  MPLX_PACK_CHUNK_LOG2 overrides for tuning.
  int chunk_log2 = 21;
  if (const char *e = getenv("MPLX_PACK_CHUNK_LOG2")) chunk_log2 = atoi(e) < 10 ? 10 : (atoi(e) > 26 ? 26 : atoi(e));
  int chunk = (1 << chunk_log2) / nU;
  if (chunk < 1) chunk = 1;
  if (chunk > n_nodes) chunk = n_nodes;
  const size_t slots = (size_t)chunk * nU;
  if (!c->d2h_stream) CU(cudaStreamCreateWithFlags(&c->d2h_stream, cudaStreamNonBlocking));
  for (int b = 0; b < 2; b++)
    if (!c->cb[b].st) CU(cudaStreamCreateWithFlags(&c->cb[b].st, cudaStreamNonBlocking));
  for (int b = 0; b < kPackBufs; b++) {
    ChunkBufs &B = c->cb[b];
    if (!B.ready) CU(cudaEventCreateWithFlags(&B.ready, cudaEventDisableTiming));
    if (!B.drained) CU(cudaEventCreateWithFlags(&B.drained, cudaEventDisableTiming));
    // successor waypoints are produced only when the caller wants state fields: a keys-only stream
    // (state == NULL: the host rebuilds coordinates of NEW states itself, graph_search.h:84-88) never
    // writes the 112-byte records to HBM
    CU(B.nodes.reserve(chunk)); CU(B.count.reserve(chunk)); if (out->state) CU(B.succ.reserve(slots)); CU(B.cost.reserve(slots));
    CU(B.action.reserve(slots)); CU(B.key.reserve(slots)); CU(B.kcount.reserve(chunk)); CU(B.offset.reserve(chunk));
    CU(B.total.reserve(1)); CU(B.h_total.reserve(1));
    if (out->state) CU(B.pstate.reserve(slots * nstate));
    if (out->cost) CU(B.pcost.reserve(slots));
    if (out->action) CU(B.paction.reserve(slots));
    if (out->key) CU(B.pkey.reserve(slots));
  }
  CU(cudaStreamSynchronize(c->stream));  // set-up kernels of mplx_set_* run on the ctx stream

  const int nchunks = (n_nodes + chunk - 1) / chunk;

  // (Writing the records straight into the pinned host buffers from pack_kernel — no staging, one wait per
  // call — was measured: 2.28 vs 1.92 ms per 262 144-node step for the {key, action} stream and 5x slower
  // with state records; SM stores over PCIe do not reach the copy engines' rate.  Staged copies it is.)
  std::vector<long long> bases(nchunks, 0);
  long long written = 0;
  cudaStream_t ds = c->d2h_stream;
  auto drain = [&](int k) -> int {  // results of chunk k: wait for its count, then queue its copies on ds
    ChunkBufs &B = c->cb[k % kPackBufs];
    const int off = k * chunk;
    const int m = n_nodes - off < chunk ? n_nodes - off : chunk;
    CU(cudaEventSynchronize(B.ready));
    const long long tot = *B.h_total.p;
    bases[k] = written;
    if (written + tot > out->capacity)
      return fail(MPLX_ERR_ARG, "packed output capacity %lld too small (need > %lld)", (long long)out->capacity,
                  written + tot);
    CU(cudaMemcpyAsync(out->count + off, B.kcount.p, sizeof(int32_t) * m, cudaMemcpyDeviceToHost, ds));
    CU(cudaMemcpyAsync(out->offset + off, B.offset.p, sizeof(long long) * m, cudaMemcpyDeviceToHost, ds));
    if (tot > 0) {
      if (out->state)
        CU(cudaMemcpyAsync(out->state + written * nstate, B.pstate.p, sizeof(double) * tot * nstate, cudaMemcpyDeviceToHost, ds));
      if (out->cost) CU(cudaMemcpyAsync(out->cost + written, B.pcost.p, sizeof(double) * tot, cudaMemcpyDeviceToHost, ds));
      if (out->action) CU(cudaMemcpyAsync(out->action + written, B.paction.p, sizeof(uint16_t) * tot, cudaMemcpyDeviceToHost, ds));
      if (out->key) CU(cudaMemcpyAsync(out->key + written, B.pkey.p, sizeof(uint64_t) * tot, cudaMemcpyDeviceToHost, ds));
    }
    CU(cudaEventRecord(B.drained, ds));
    written += tot;
    return MPLX_OK;
  };

  const int ahead = 2;  // chunks queued before the host waits for a record count
  for (int k = 0; k < nchunks; k++) {
    ChunkBufs &B = c->cb[k % kPackBufs];
    cudaStream_t st = c->cb[k & 1].st;
    const int off = k * chunk;
    const int m = n_nodes - off < chunk ? n_nodes - off : chunk;
    if (k >= kPackBufs) CU(cudaStreamWaitEvent(st, B.drained, 0));  // chunk k-kPackBufs has left these buffers
    CU(cudaMemcpyAsync(B.nodes.p, nodes + off, sizeof(mplx_waypoint) * m, cudaMemcpyHostToDevice, st));
    mplx_succ_out d{B.count.p, out->state ? B.succ.p : nullptr, B.cost.p, B.action.p, B.key.p, nullptr};
    CU(B.fxq.reserve((size_t)m * nU));
    int launches = 0;
    CU(mplx::launch_expand(c->P, B.nodes.p, m, d, st, c->kernel, &B.fxq.view, &launches));
    CU(cudaMemsetAsync(B.total.p, 0, sizeof(long long), st));
    mplx::pack_kernel<<<(m + 7) / 8, 256, 0, st>>>(m, nU, dim, control, drop_inf, B.count.p,
                                                   out->state ? B.succ.p : nullptr, B.cost.p, B.action.p, B.key.p, B.total.p, B.kcount.p, B.offset.p,
                                                   out->state ? B.pstate.p : nullptr, out->cost ? B.pcost.p : nullptr,
                                                   out->action ? B.paction.p : nullptr, out->key ? B.pkey.p : nullptr);
    CU(cudaGetLastError());
    c->launches += launches + 1;
    CU(cudaMemcpyAsync(B.h_total.p, B.total.p, sizeof(long long), cudaMemcpyDeviceToHost, st));
    CU(cudaEventRecord(B.ready, st));
    if (k >= ahead)
      if (int r = drain(k - ahead)) return r;
  }
  for (int k = nchunks - ahead < 0 ? 0 : nchunks - ahead; k < nchunks; k++)
    if (int r = drain(k)) return r;
  CU(cudaStreamSynchronize(ds));
  CU(cudaStreamSynchronize(c->cb[0].st));
  CU(cudaStreamSynchronize(c->cb[1].st));
  // offsets were reserved per chunk: make them global
  for (int k = 1; k < nchunks; k++) {
    const int off = k * chunk;
    const int m = n_nodes - off < chunk ? n_nodes - off : chunk;
    for (int i = 0; i < m; i++) out->offset[off + i] += bases[k];
  }
  out->total = written;
  return MPLX_OK;
}
