// mplx_edges.cu — re-validation of STORED graph edges for the incremental (LPA*) callers of the
// expansion path.  An edge of the search graph is fully described by (parent state, action id):
// pr = Primitive(parent, U[action], dt) (env_base.h:228-231 forward_action).  Two batched queries:
//
//   mplx_edges_is_free  env_map<Dim>::is_free(pr) (env_map.h:60-76) — what StateSpace::decreaseCost
//                       asks for every +inf edge through a cleared voxel (state_space.h:236-243) —
//                       plus the cost it then installs, calculate_intrinsic_cost(pr)
//                       (env_base.h:343-345);
//   mplx_edges_cells    the voxels an edge passes through, as MapPlanner::getLinkedNodes walks them
//                       (src/mpl_planner/map_planner.cpp:135-151): the host builds the
//                       voxel -> edges table (lhm_) from it.
//
// Both sample the primitive as Primitive::sample(n) does (primitive.h:415-420): n = ceil(max_v*T/res)
// WITHOUT the max(5, .) of traverse_primitive, n+1 samples at t = i*(T/n) (a product, not the
// running sum of env_map.h:99).  One thread per edge: these are maintenance queries (thousands to a
// few million edges per map update), bandwidth is the occupancy bit grid in L2.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cuda_runtime.h>
#include <limits.h>
#include <math.h>

#include "mplx_dispatch.h"
#include "mplx_internal.h"
#include "mplx_prim.cuh"

namespace mplx {

// floatToInt (map_util.h:103-108): (int)std::round((p - origin)/res - 0.5), true division.
// NaN / out-of-int-range inputs convert to INT_MIN, the x86-64 cvttsd2si result the reference
// build produces for them (a sample there is outside every map).
__device__ __forceinline__ int float_to_int(double p, double origin, double res) {
  const double x = (p - origin) / res - 0.5;
  if (!(fabs(x) < 2147483648.0)) return INT_MIN;
  int k;
  round_haz(x, k);
  return k;
}

// Largest n = ceil(max_v*T/res) served.  Beyond it (unbounded speed, NaN state) the reference
// would try to allocate the n+1 sample Waypoints; such an edge is reported not free / no cells.
constexpr int kEdgeNMax = 1 << 20;

template <int DIM, int ORD>
struct EdgePrim {
  double cf[DIM * (ORD + 1)];
  double dt;
  int n;
};

// Primitive(parent, U[action], T), max_v over the axes, n and dt of sample(n).
template <int DIM, int ORD>
__device__ __forceinline__ void edge_build(const EnvParams &P, const mplx_waypoint &w, int action,
                                           EdgePrim<DIM, ORD> &e, double &J) {
  PrimState<DIM, ORD, false> pr;
  const double *u = P.U + (size_t)action * P.udim;
  double max_v = 0;
  bool nan_v = false;  // a NaN speed compares false above and would otherwise read as max_v = 0, n = 0
  J = 0;
#pragma unroll
  for (int k = 0; k < DIM; k++) {
    pr.ax[k].build(__ldg(u + k), w.pos[k], w.vel[k], w.acc[k], w.jrk[k]);
    const double mv = pr.ax[k].max_vel(P.T);
    if (mv > max_v) max_v = mv;
    nan_v = nan_v || mv != mv;
    J += pr.ax[k].J(P.T);  // Primitive::J sums the axes left to right (primitive.h:403-407)
  }
  fill_coef<DIM, ORD, false>(pr, false, e.cf);
  const double nd = ceil(max_v * P.T / P.res);
  e.n = (nan_v || !(nd <= (double)kEdgeNMax)) ? -1 : (int)nd;  // -1: more samples than any real edge has
  e.dt = P.T / e.n;
}

template <int DIM, int ORD>
__global__ void __launch_bounds__(128)
edges_free_kernel(const __grid_constant__ EnvParams P, const mplx_waypoint *__restrict__ parents,
                  const int32_t *__restrict__ actions, int n_edges, uint8_t *__restrict__ out_free,
                  double *__restrict__ out_cost) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  EdgePrim<DIM, ORD> ep;
  double J;
  edge_build<DIM, ORD>(P, parents[e], actions[e], ep, J);
  if (out_cost) out_cost[e] = J + P.w * P.T;
  bool free = ep.n >= 0;
  for (int i = 0; i <= ep.n && free; i++) {
    double pk[DIM];
    eval_pos<DIM, ORD>(ep.cf, i * ep.dt, pk);
    int pn[DIM];
    bool inside = true;
#pragma unroll
    for (int k = 0; k < DIM; k++) {
      pn[k] = float_to_int(pk[k], P.origin[k], P.res);
      inside = inside && (unsigned)pn[k] < (unsigned)P.mdim[k];
    }
    if (!inside) {  // isOutside (env_map.h:68)
      free = false;
      break;
    }
    int idx = pn[0] + P.mdim[0] * pn[1];
    if (DIM == 3) idx += P.mdim[0] * P.mdim[1] * pn[DIM - 1];
    if ((__ldg(P.occ_bits + (idx >> 5)) >> (idx & 31)) & 1u) free = false;  // isOccupied
    if (free && P.region_bits != nullptr && !((__ldg(P.region_bits + (idx >> 5)) >> (idx & 31)) & 1u))
      free = false;  // outside the tunnel (env_map.h:69-71)
  }
  out_free[e] = free ? 1 : 0;
}

// WRITE=false: count[e] = number of cells the walk emits; WRITE=true: emit them at offset[e].
template <int DIM, int ORD, bool WRITE>
__global__ void __launch_bounds__(128)
edges_cells_kernel(const __grid_constant__ EnvParams P, const mplx_waypoint *__restrict__ parents,
                   const int32_t *__restrict__ actions, int n_edges, long long *__restrict__ count,
                   const long long *__restrict__ offset, int32_t *__restrict__ cells, int32_t *__restrict__ ids,
                   int32_t *__restrict__ owner) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_edges) return;
  EdgePrim<DIM, ORD> ep;
  double J;
  edge_build<DIM, ORD>(P, parents[e], actions[e], ep, J);
  long long k_out = 0;
  int prev_id = -1;  // map_planner.cpp:143
  int32_t *dst = WRITE ? cells + offset[e] * DIM : nullptr;
  for (int i = 0; i <= ep.n; i++) {
    double pk[DIM];
    eval_pos<DIM, ORD>(ep.cf, i * ep.dt, pk);
    int pn[DIM];
#pragma unroll
    for (int k = 0; k < DIM; k++) pn[k] = float_to_int(pk[k], P.origin[k], P.res);
    // getIndex without a bounds test, int arithmetic wraps as on the reference's targets (:146)
    unsigned id = (unsigned)pn[0] + (unsigned)P.mdim[0] * (unsigned)pn[1];
    if (DIM == 3) id += (unsigned)P.mdim[0] * (unsigned)P.mdim[1] * (unsigned)pn[DIM - 1];
    if ((int)id != prev_id) {
      if (WRITE) {
#pragma unroll
        for (int k = 0; k < DIM; k++) dst[k_out * DIM + k] = pn[k];
        if (ids) {  // (voxel index, edge) pairs in emission order, for the inverted table
          ids[offset[e] + k_out] = (int)id;
          owner[offset[e] + k_out] = e;
        }
      }
      k_out++;
      prev_id = (int)id;
    }
  }
  if (!WRITE) count[e] = k_out;
}

static cudaError_t launch_free(const EnvParams &P, const mplx_waypoint *parents, const int32_t *actions, int n,
                               uint8_t *out_free, double *out_cost, cudaStream_t st) {
  return with_dim(P.dim, [&](auto DIM) {
    return with_order(P.control, [&](auto ORD) {
      edges_free_kernel<DIM, ORD><<<(n + 127) / 128, 128, 0, st>>>(P, parents, actions, n, out_free, out_cost);
      return cudaGetLastError();
    });
  });
}

template <bool WRITE>
static cudaError_t launch_cells(const EnvParams &P, const mplx_waypoint *parents, const int32_t *actions, int n,
                                long long *count, const long long *offset, int32_t *cells, int32_t *ids, int32_t *owner,
                                cudaStream_t st) {
  return with_dim(P.dim, [&](auto DIM) {
    return with_order(P.control, [&](auto ORD) {
      edges_cells_kernel<DIM, ORD, WRITE>
          <<<(n + 127) / 128, 128, 0, st>>>(P, parents, actions, n, count, offset, cells, ids, owner);
      return cudaGetLastError();
    });
  });
}

}  // namespace mplx

static int check_edges(mplx_ctx *c, const mplx_waypoint *parents, const int32_t *actions, int n_edges) {
  if (int r = mplx_bind(c)) return r;
  if (int r = mplx_check_ready(c, n_edges)) return r;
  if (n_edges > 0 && (!parents || !actions)) return fail(MPLX_ERR_ARG, "parents/actions is null");
  for (int i = 0; i < n_edges; i++)
    if (actions[i] < 0 || actions[i] >= c->P.nU)
      return fail(MPLX_ERR_ARG, "edge %d: action id %d outside [0, %d)", i, actions[i], c->P.nU);
  return MPLX_OK;
}

extern "C" int mplx_edges_is_free(mplx_ctx *c, const mplx_waypoint *parents, const int32_t *actions, int n_edges,
                                  uint8_t *out_free, double *out_cost) {
  if (int r = check_edges(c, parents, actions, n_edges)) return r;
  if (n_edges == 0) return MPLX_OK;
  if (!out_free) return fail(MPLX_ERR_ARG, "out_free is null");
  EdgeBufs &B = c->eb;
  CU(B.parents.reserve(n_edges)); CU(B.actions.reserve(n_edges)); CU(B.free_.reserve(n_edges));
  if (out_cost) CU(B.cost.reserve(n_edges));
  cudaStream_t st = c->stream;
  CU(cudaMemcpyAsync(B.parents.p, parents, sizeof(mplx_waypoint) * n_edges, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(B.actions.p, actions, sizeof(int32_t) * n_edges, cudaMemcpyHostToDevice, st));
  CU(mplx::launch_free(c->P, B.parents.p, B.actions.p, n_edges, B.free_.p, out_cost ? B.cost.p : nullptr, st));
  c->launches += 1;
  CU(cudaMemcpyAsync(out_free, B.free_.p, n_edges, cudaMemcpyDeviceToHost, st));
  if (out_cost) CU(cudaMemcpyAsync(out_cost, B.cost.p, sizeof(double) * n_edges, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return MPLX_OK;
}

extern "C" int mplx_edges_cells(mplx_ctx *c, const mplx_waypoint *parents, const int32_t *actions, int n_edges,
                                int64_t *out_offset, int32_t *out_cells, int64_t capacity, int64_t *out_total,
                                int32_t *out_table_voxel, int32_t *out_table_edge) {
  if (int r = check_edges(c, parents, actions, n_edges)) return r;
  if (!out_offset || !out_total) return fail(MPLX_ERR_ARG, "out_offset and out_total are required");
  if ((out_table_voxel == nullptr) != (out_table_edge == nullptr))
    return fail(MPLX_ERR_ARG, "out_table_voxel and out_table_edge go together");
  const bool table = out_table_voxel != nullptr;
  *out_total = 0;
  out_offset[0] = 0;
  if (n_edges == 0) return MPLX_OK;
  EdgeBufs &B = c->eb;
  const int dim = c->dim;
  CU(B.parents.reserve(n_edges)); CU(B.actions.reserve(n_edges));
  CU(B.count.reserve((size_t)n_edges + 1)); CU(B.offset.reserve((size_t)n_edges + 1));
  cudaStream_t st = c->stream;
  CU(cudaMemcpyAsync(B.parents.p, parents, sizeof(mplx_waypoint) * n_edges, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(B.actions.p, actions, sizeof(int32_t) * n_edges, cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(B.count.p + n_edges, 0, sizeof(long long), st));
  CU(mplx::launch_cells<false>(c->P, B.parents.p, B.actions.p, n_edges, B.count.p, nullptr, nullptr, nullptr, nullptr, st));
  // exclusive scan over n_edges+1 counts: offset[n_edges] = total
  size_t tmp_bytes = 0;
  CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, B.count.p, B.offset.p, n_edges + 1, st));
  CU(B.scan_tmp.reserve(tmp_bytes));
  CU(cub::DeviceScan::ExclusiveSum(B.scan_tmp.p, tmp_bytes, B.count.p, B.offset.p, n_edges + 1, st));
  static_assert(sizeof(long long) == sizeof(int64_t), "offset width");
  CU(cudaMemcpyAsync(out_offset, B.offset.p, sizeof(int64_t) * ((size_t)n_edges + 1), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  c->launches += 2;
  const int64_t total = out_offset[n_edges];
  *out_total = total;
  if (total > capacity || (total > 0 && !out_cells))
    return fail(MPLX_ERR_ARG, "out_cells capacity %lld too small (need %lld entries)", (long long)capacity,
                (long long)total);
  if (total == 0) return MPLX_OK;
  if (total >= ((int64_t)1 << 31)) return fail(MPLX_ERR_ARG, "more than 2^31 linked voxels in one query");
  CU(B.cells.reserve((size_t)total * dim));
  if (table) {
    CU(B.ids.reserve(total)); CU(B.owner.reserve(total)); CU(B.ids_sorted.reserve(total)); CU(B.owner_sorted.reserve(total));
  }
  int32_t *ids = table ? B.ids.p : nullptr, *own = table ? B.owner.p : nullptr;
  CU(mplx::launch_cells<true>(c->P, B.parents.p, B.actions.p, n_edges, nullptr, B.offset.p, B.cells.p, ids, own, st));
  c->launches += 1;
  CU(cudaMemcpyAsync(out_cells, B.cells.p, sizeof(int32_t) * (size_t)total * dim, cudaMemcpyDeviceToHost, st));
  if (table) {
    // voxel -> edges table: the pairs sorted by voxel index; the radix sort is stable, so the
    // edges of one voxel stay in emission order (the push_back order of lhm_[id], map_planner.cpp:149)
    size_t sort_bytes = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, B.ids.p, B.ids_sorted.p, B.owner.p, B.owner_sorted.p, (int)total,
                                       0, 32, st));
    CU(B.scan_tmp.reserve(sort_bytes));
    CU(cub::DeviceRadixSort::SortPairs(B.scan_tmp.p, sort_bytes, B.ids.p, B.ids_sorted.p, B.owner.p, B.owner_sorted.p,
                                       (int)total, 0, 32, st));
    CU(cudaMemcpyAsync(out_table_voxel, B.ids_sorted.p, sizeof(int32_t) * (size_t)total, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out_table_edge, B.owner_sorted.p, sizeof(int32_t) * (size_t)total, cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  return MPLX_OK;
}
