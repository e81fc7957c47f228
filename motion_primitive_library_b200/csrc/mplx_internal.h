// mplx_internal.h — ctx layout and small helpers shared by the libmplx translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <vector>
#include "../../include/mplx.h"
#include "mplx_device.cuh"
#include "mplx_kernels.h"

namespace mplx {
int fail(int code, const char *fmt, ...);
}
using mplx::fail;

#define CU(call)                                                                              \
  do {                                                                                        \
    cudaError_t e_ = (call);                                                                  \
    if (e_ != cudaSuccess) {                                                                  \
      cudaGetLastError();                                                                     \
      return fail(e_ == cudaErrorMemoryAllocation ? MPLX_ERR_ALLOC : MPLX_ERR_CUDA,           \
                  "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    }                                                                                         \
  } while (0)

template <typename T>
struct DevBuf {
  T *p = nullptr;
  size_t cap = 0;  // elements
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaMalloc((void **)&p, n * sizeof(T));
    if (e == cudaSuccess) cap = n;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

// a function-local DevBuf that frees itself on every exit path
template <typename T>
struct ScopedDevBuf : DevBuf<T> {
  ScopedDevBuf() = default;
  ScopedDevBuf(const ScopedDevBuf &) = delete;
  ScopedDevBuf &operator=(const ScopedDevBuf &) = delete;
  ~ScopedDevBuf() { this->release(); }
};

// The device time of one batch of launches on a stream: an event pair that destroys itself on every exit path
struct TimedRun {
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  TimedRun() = default;
  TimedRun(const TimedRun &) = delete;
  TimedRun &operator=(const TimedRun &) = delete;
  ~TimedRun() {
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
  }
  // Records e0, calls launch(int *n) -> cudaError_t, which launches on st and counts its launches in *n, then
  // records e1; adds *n to launches whether or not a step failed.  Returns the first error.
  template <class F>
  cudaError_t run(cudaStream_t st, int64_t &launches, F &&launch) {
    cudaError_t e = cudaEventCreate(&e0);
    if (e == cudaSuccess) e = cudaEventCreate(&e1);
    if (e != cudaSuccess) return e;
    int n = 0;
    e = cudaEventRecord(e0, st);
    if (e == cudaSuccess) e = launch(&n);
    if (e == cudaSuccess) e = cudaEventRecord(e1, st);
    launches += n;
    return e;
  }
  // the time between the records, once the caller has synchronised the stream
  cudaError_t seconds(double *s) const {
    float ms = 0.f;
    const cudaError_t e = cudaEventElapsedTime(&ms, e0, e1);
    *s = ms * 1e-3;
    return e;
  }
};

template <typename T>
struct PinBuf {
  T *p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
    cudaError_t e = cudaHostAlloc((void **)&p, n * sizeof(T), cudaHostAllocDefault);
    if (e == cudaSuccess) cap = n;
    return e;
  }
  void release() {
    if (p) cudaFreeHost(p);
    p = nullptr;
    cap = 0;
  }
};

inline bool is_pinned(const void *p) {
  if (!p) return false;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeHost;
}

// Global queue of ambiguous primitives of the fixed-point kernels (mplx_fxn.cu), one per stream in use.
struct FxQueue {
  DevBuf<unsigned char> q;
  DevBuf<unsigned> n;
  mplx::FxScratch view;
  // room for a quarter of the batch's primitives (~5 % are ambiguous on the bench maps) + slack per segment
  cudaError_t reserve(size_t n_prims) {
    const size_t cap = ((n_prims / 4 + 64 * 4096 + 63) / 64) * 64;
    cudaError_t e = q.reserve(cap * mplx::fx_amb_record_bytes());
    if (e == cudaSuccess) e = n.reserve(64);
    if (e != cudaSuccess) return e;
    view.q = q.p;
    view.n = n.p;
    view.cap = (unsigned)(q.cap / mplx::fx_amb_record_bytes() / 64 * 64);
    return cudaSuccess;
  }
  void release() { q.release(); n.release(); view = mplx::FxScratch(); }
};

// One set of per-chunk device buffers + its stream: two sets let chunk k+1 compute while
// chunk k's results cross PCIe (mplx_expand_packed).
constexpr int kPackBufs = 4;  // chunk buffer sets of the packed pipeline
struct ChunkBufs {
  cudaStream_t st = nullptr;
  cudaEvent_t ready = nullptr;    // the chunk's records are packed and its record count is on the host
  cudaEvent_t drained = nullptr;  // the chunk's device-to-host copies have left the buffers
  DevBuf<mplx_waypoint> nodes, succ;
  DevBuf<int32_t> count, action;
  DevBuf<double> cost;
  DevBuf<uint64_t> key;
  // packed stream
  DevBuf<int32_t> kcount;
  DevBuf<long long> offset, total;
  DevBuf<double> pstate, pcost;
  DevBuf<uint16_t> paction;
  DevBuf<uint64_t> pkey;
  PinBuf<long long> h_total;
  FxQueue fxq;
  void release() {
    fxq.release();
    nodes.release(); succ.release(); count.release(); action.release(); cost.release(); key.release();
    kcount.release(); offset.release(); total.release(); pstate.release(); pcost.release(); paction.release();
    pkey.release(); h_total.release();
    if (ready) cudaEventDestroy(ready);
    if (drained) cudaEventDestroy(drained);
    if (st) cudaStreamDestroy(st);
    ready = drained = nullptr;
    st = nullptr;
  }
};

// staging of the edge re-validation queries (mplx_edges.cu)
struct EdgeBufs {
  DevBuf<mplx_waypoint> parents;
  DevBuf<int32_t> actions, cells, ids, owner, ids_sorted, owner_sorted;
  DevBuf<uint8_t> free_, scan_tmp;
  DevBuf<double> cost;
  DevBuf<long long> count, offset;
  void release() {
    parents.release(); actions.release(); cells.release(); free_.release(); scan_tmp.release(); cost.release();
    count.release(); offset.release(); ids.release(); owner.release(); ids_sorted.release(); owner_sorted.release();
  }
};

// staging of the sparse grid edits (mplx_update.cu)
struct UpdateBufs {
  PinBuf<uint32_t> h_idx;
  PinBuf<int8_t> h_val;
  DevBuf<uint32_t> idx, idx_sorted;
  DevBuf<int8_t> val, val_sorted;
  DevBuf<uint8_t> sort_tmp;
  void release() {
    h_idx.release(); h_val.release(); idx.release(); idx_sorted.release(); val.release(); val_sorted.release();
    sort_tmp.release();
  }
};

// inputs, outputs and per-waypoint scratch of mplx_traj_solve, mplx_traj_scale, mplx_traj_check and
// mplx_plan_batch_trajectories (mplx_traj.cu), sized by the largest batch so far; the second line of members is
// mplx_traj_scale's and mplx_traj_check's, the third mplx_traj_check's alone, the last
// mplx_plan_batch_trajectories'
struct TrajBufs {
  DevBuf<long long> offset;
  DevBuf<mplx_waypoint> wps;
  DevBuf<uint8_t> ctl, mono;
  DevBuf<int32_t> status;
  DevBuf<double> dts, seg_t, taus, coeff, samples, fac, dpos, dyaw;
  DevBuf<int32_t> n_cand, n_knot;
  DevBuf<double> par, total, seg_T, cand, cand_p, knot_t, knot_p, lam, lam_T;
  DevBuf<int32_t> n_pts;
  DevBuf<uint8_t> form, seg_free, seg_valid;
  DevBuf<double> cost;
  DevBuf<long long> slot_src;  // mplx_plan_batch_trajectories' per-slot inputs
  DevBuf<int32_t> slot_action;
  void release() {
    slot_src.release(); slot_action.release();
    offset.release(); wps.release(); ctl.release(); mono.release(); status.release(); dts.release(); seg_t.release();
    taus.release(); coeff.release(); samples.release(); fac.release(); dpos.release(); dyaw.release();
    n_cand.release(); n_knot.release(); par.release(); total.release(); seg_T.release(); cand.release();
    cand_p.release(); knot_t.release(); knot_p.release(); lam.release(); lam_T.release();
    n_pts.release(); form.release(); seg_free.release(); seg_valid.release(); cost.release();
  }
};

// Device memory one search call may take (arenas, per-query arrays and the result pool): a quarter of the
// free device memory, at most this much.  The slot count follows from it (mplx_search.cu, search_budget).
constexpr size_t kSearchArenaBudget = (size_t)8 << 30;

// the device search (mplx_search.cu): per-slot arenas kept across calls; per-slot successor scratch
// (succ, cost, key, action, count), the per-query arrays (queries, free_, ires, dres, offs) and the
// result pool (closed), reused by every call and round
enum TrajState : int { kTrajNone = 0, kTrajOff = 1, kTrajOn = 2 };
struct SearchBufs {
  DevBuf<unsigned char> arena;
  int64_t layout_bytes = 0;  // bytes per slot of the layout the arena was cleared for
  size_t cleared = 0;        // leading arena bytes cleared for that layout
  uint32_t next_epoch = 1;   // key-table entries of earlier queries carry smaller epochs
  DevBuf<mplx_waypoint> succ, queries;
  DevBuf<double> cost, dres;
  DevBuf<uint64_t> key, closed;
  DevBuf<int32_t> action, count, ires;
  DevBuf<uint8_t> free_;
  DevBuf<unsigned long long> offs;  // each query's place in the result pool, then the pool's fill counter
  // what mplx_plan_batch_grow_results copies: the last mplx_plan_batch_grow call's trajectories and
  // sorted closed keys, query q's at [offset[q], offset[q+1]); the other entry points leave them alone
  std::vector<int64_t> grow_aoff, grow_coff;
  std::vector<int32_t> grow_actions;
  std::vector<uint64_t> grow_closed;
  // trajectory recording (mplx_set_batch_trajectories): on, and the room asked for in bytes (0 = automatic)
  bool traj_on = false;
  int64_t traj_room_bytes = 0;
  // the recorded coordinates of the last search call: the rooms of its rounds one after the other, the first
  // traj_kept slots in use; toffs holds each query's place in the round's room, then the room's fill counter
  DevBuf<mplx_waypoint> traj;
  int64_t traj_kept = 0;
  DevBuf<unsigned long long> toffs;
  // what mplx_plan_batch_trajectories reads: kTrajNone before any search call (or after one that failed),
  // kTrajOff after one without recording, kTrajOn after one with.  Query q owns the waypoint slots
  // [traj_off[q], traj_off[q+1]); slot s holds the state traj[slot_src[s]] and the action id slot_action[s] of
  // the segment that starts there (-1 on a path's last slot)
  int traj_state = 0;
  std::vector<int64_t> traj_off, slot_src;
  std::vector<int32_t> slot_action;
  void release() {
    arena.release(); succ.release(); queries.release(); cost.release(); dres.release(); key.release();
    closed.release(); action.release(); count.release(); ires.release(); free_.release(); offs.release();
    traj.release(); toffs.release();
    traj_kept = 0;
    traj_state = 0;
    layout_bytes = 0;
    cleared = 0;
    next_epoch = 1;
  }
};

// The per-query tunnels of the batched searches (mplx_set_batch_regions, mplx_tunnel.cuh): query q owns the bricks
// [off[q], off[q+1]) of key and their tunnel_words(dim) mask words each in bits; n_q = 0 when none are set
struct TunnelStore {
  int n_q = 0;
  int64_t n_bricks = 0;
  DevBuf<uint64_t> key;
  DevBuf<uint32_t> bits;
  DevBuf<int64_t> off;
  size_t bytes() const { return key.cap * sizeof(uint64_t) + bits.cap * sizeof(uint32_t) + off.cap * sizeof(int64_t); }
  void release() {
    key.release(); bits.release(); off.release();
    n_q = 0;
    n_bricks = 0;
  }
};

struct mplx_ctx {
  int dim = 0, device = 0;
  cudaStream_t stream = nullptr;
  // static data in HBM
  DevBuf<int8_t> map, pot;
  DevBuf<uint32_t> region, occ;
  DevBuf<uint32_t> occ2;
  DevBuf<unsigned char> prow, row_axis;  // per-axis value tables of U (EnvParams::prow ...)
  DevBuf<double> row_u;
  int n_rows = 0;
  size_t occ2_window = 0;  // bytes of occ2 (from its start) covered by the L2 access-policy window (0 = none)
  size_t l2_persist = 0;   // persisting L2 set-aside this ctx last asked for (size_l2_window)
  DevBuf<double> U, ttab, tdt;
  DevBuf<int> tcount;
  int kernel = 0;  // mplx_set_kernel
  DevBuf<unsigned long long> stats;
  bool has_map = false, has_pot = false, has_region = false, has_params = false, stats_on = false;
  size_t nvox = 0;
  mplx::EnvParams P;
  // per-call staging (host-buffer entry point)
  DevBuf<mplx_waypoint> d_nodes, d_succ;
  DevBuf<int32_t> d_count, d_action, d_lattice;
  DevBuf<double> d_cost;
  DevBuf<uint64_t> d_key;
  PinBuf<mplx_waypoint> h_nodes, h_succ;
  PinBuf<int32_t> h_count, h_action, h_lattice;
  PinBuf<double> h_cost;
  PinBuf<uint64_t> h_key;
  ChunkBufs cb[kPackBufs];
  cudaStream_t d2h_stream = nullptr;  // result copies of the packed pipeline
  FxQueue fxq;
  EdgeBufs eb;
  UpdateBufs ub;
  SearchBufs sb;
  TunnelStore tun;
  TrajBufs tb;
  int64_t launches = 0;
  unsigned long long last_stats[2] = {0, 0};
};

namespace mplx {
// mplx_maps.cu: the grid the ray trace of MapPlanner::setSearchRegion walks (search::segment_cells) and the tunnel's
// half-widths, shared by mplx_set_search_region_path and the batch tunnel build (mplx_tunnel.cu)
namespace search {
struct Grid;
}
search::Grid region_grid(const mplx_ctx *c);
// mplx_api.cu: the L2 persisting set-aside and window for occ2, sized for the ctx's current plan
void size_l2_window(mplx_ctx *c);
void region_radius_cells(const mplx_ctx *c, const double *radius, int *rn);
// mplx_search.cu: the device memory one search call may take
int search_budget(const mplx_ctx *c, size_t &budget);
}  // namespace mplx

extern "C" {
int mplx_bind(mplx_ctx *ctx);
int mplx_check_ready(mplx_ctx *c, int n_nodes);
}
