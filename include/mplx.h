/*
 * mplx.h — C ABI of libmplx.so, the H100 (sm_90a) node-expansion engine.
 *
 * This is the drop-in boundary for ONE path of sikang/motion_primitive_library: the body of
 *   env_map<Dim>::get_succ               include/mpl_planner/env/env_map.h:147-172
 * (called from GraphSearch::Astar  include/mpl_planner/common/graph_search.h:75 and
 *  GraphSearch::LPAstar :266) — batched over many frontier nodes.  The reference has no
 * FFI layer; its operator API for this path is the virtual
 *   env_base<Dim>::get_succ(curr, succ, succ_cost, action_idx)
 *                                        include/mpl_planner/common/env_base.h:358-362
 * and the setters that feed it.  Each entry point below names the reference interface it
 * replaces.  INTEGRATION.md shows the env_map subclass a maintainer adds on the reference
 * side to bind these.
 *
 * Conventions: extern "C", opaque handle, plain pointers and sizes, int status
 * (0 = MPLX_OK, non-zero = error, text from mplx_last_error()), no exceptions cross the
 * boundary.  There is NO CPU fallback: every compute entry point fails with
 * MPLX_ERR_CUDA when no CUDA device is usable.
 *
 * One ctx = one device + one stream; a ctx is not thread-safe (the reference's get_succ is
 * not re-entrant either: env_base.h:402-404).  Any number of ctxs may coexist.
 */
#ifndef MPLX_H
#define MPLX_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPLX_OK 0
#define MPLX_ERR_ARG 1    /* bad argument / state not configured */
#define MPLX_ERR_CUDA 2   /* CUDA runtime error or no device */
#define MPLX_ERR_ALLOC 3  /* out of memory (host or device) */

/* Control::Control, include/mpl_basis/control.h:10-20 */
#define MPLX_VEL 0x01
#define MPLX_ACC 0x03
#define MPLX_JRK 0x07
#define MPLX_SNP 0x0f
#define MPLX_VELxYAW 0x11
#define MPLX_ACCxYAW 0x13
#define MPLX_JRKxYAW 0x17
#define MPLX_SNPxYAW 0x1f

#define MPLX_LATTICE_MAX 13 /* 3 axes x {pos,vel,acc,jrk} + yaw */

/* Waypoint<Dim> payload, include/mpl_basis/waypoint.h:33-38.  2D uses [0],[1] of each
 * vector ([2] ignored on input, 0 on output).  `control` is per-ctx (mplx_set_params), as it
 * is per-plan in the reference (goal.control = start.control, test/test_planner_2d.cpp:46);
 * enable_t is never set by the reference's planners and is treated as false. 112 bytes. */
typedef struct {
  double pos[3], vel[3], acc[3], jrk[3];
  double yaw;
  double t;
} mplx_waypoint;

typedef struct mplx_ctx mplx_ctx;

/* Output of one batched expansion.  Successors of node i occupy slots
 * [i*nU, i*nU + count[i]) of every array, in increasing control index (the order
 * env_map::get_succ push_back()s them, env_map.h:155-170).  An entry exists iff
 * !(tn == curr) && validate_primitive(...) (env_map.h:158-160); cost may be +inf
 * (colliding but dynamically valid — LPA* keeps those, graph_search.h:284-311).
 * Any pointer except `count` may be NULL to skip that field.  All pointers are HOST
 * pointers for mplx_expand and DEVICE pointers for mplx_expand_device. */
typedef struct {
  int32_t *count;      /* [n_nodes]                                                       */
  mplx_waypoint *succ; /* [n_nodes*nU]   succ      (vec_E<Waypoint<Dim>>&, env_map.h:147)   */
  double *cost;        /* [n_nodes*nU]   succ_cost (std::vector<decimal_t>&, env_map.h:148) */
  int32_t *action;     /* [n_nodes*nU]   action_idx (std::vector<int>&, env_map.h:149)      */
  uint64_t *key;       /* [n_nodes*nU]   hash_value(succ), include/mpl_basis/waypoint.h:93  */
  int32_t *lattice;    /* [n_nodes*nU*13] the rounded ints fed to hash_combine, in hash
                          order (waypoint.h:96-122); unused tail slots are 0               */
} mplx_succ_out;

/* ---- lifecycle -------------------------------------------------------------------- */

/* Replaces `new env_map<Dim>(map_util)` in MapPlanner::setMapUtil
 * (src/mpl_planner/map_planner.cpp:14-18).  dim is 2 or 3; device is a CUDA ordinal. */
int mplx_create(int dim, int device, mplx_ctx **out);
int mplx_destroy(mplx_ctx *ctx);
/* Thread-local text of the last error returned on this thread. */
const char *mplx_last_error(void);

/* ---- static per-plan data (SURVEY.md §8 a9) ----------------------------------------- */

/* MapUtil<Dim>::setMap (include/mpl_collision/map_util.h:85-91).  `data` is the x-fastest
 * int8 grid (occupied 100 / free 0 / unknown -1, map_util.h:309-313); it is copied to HBM.
 * dim/origin have ctx-dim entries.  Clears any potential map and search region
 * (their sizes are tied to the grid). */
int mplx_set_map(mplx_ctx *ctx, const int8_t *data, const int32_t *dim, const double *origin,
                 double res);

/* env_map::set_potential_map / set_potential_weight / set_gradient_weight
 * (include/mpl_planner/env/env_map.h:181-186, 175-178).  data == NULL restores
 * potential_map_.empty().  Same size as the grid. */
int mplx_set_potential(mplx_ctx *ctx, const int8_t *data, double potential_weight,
                       double gradient_weight);

/* env_map::set_potential_weight / set_gradient_weight alone (env_map.h:175-178): the potential map
 * already on the device (mplx_set_potential or mplx_update_potential_map) is kept. */
int mplx_set_potential_weights(mplx_ctx *ctx, double potential_weight, double gradient_weight);

/* env_base::set_search_region (include/mpl_planner/common/env_base.h:301-303).
 * One byte per voxel, non-zero = inside the tunnel; NULL restores search_region_.empty(). */
int mplx_set_search_region(mplx_ctx *ctx, const uint8_t *in_region);

/* MapPlanner<Dim>::updatePotentialMap(pos) with createMask (src/mpl_planner/map_planner.cpp:286-391),
 * on the device grid: builds the potential field around every cell with map > 0 (inside the optional
 * source range: `range` = potential_map_range_, `pos` its centre; NULL or all-zero range = whole
 * map), radius = potential_radius_ (metres; radius[0] is used for x and y as in the reference,
 * radius[2] for z), pow = pow_ (map_planner.h:113).  Like the reference it then OVERWRITES the grid
 * with the result (map_util_->setMap(dmap), :387) and installs it as the potential map (:388) with
 * the given weights.  out_map (host, one int8 per voxel) receives the new grid, or NULL. */
int mplx_update_potential_map(mplx_ctx *ctx, const double *radius, double pow, const double *range,
                              const double *pos, double potential_weight, double gradient_weight,
                              int8_t *out_map);

/* MapPlanner<Dim>::setSearchRegion(path, dense) (src/mpl_planner/map_planner.cpp:46-95): the tunnel
 * of half-width ceil(radius/res) cells around the ray-traced path (n_pts points of ctx-dim doubles)
 * becomes the search region.  out_region (host, one byte per voxel) receives it, or NULL. */
int mplx_set_search_region_path(mplx_ctx *ctx, const double *path, int n_pts, const double *radius,
                                int dense, uint8_t *out_region);

/* env_base::set_u / set_dt / set_w / set_wyaw / set_v_max / set_a_max / set_j_max /
 * set_yaw_max (env_base.h:234-287) and the Waypoint control flag.  U is nU x udim row-major,
 * udim = dim (+1 when the control carries a yaw rate, primitive.h:235-248). */
int mplx_set_params(mplx_ctx *ctx, int control, double T, double w, double wyaw, double v_max,
                    double a_max, double j_max, double yaw_max, const double *U, int nU, int udim);

/* ---- the hot path ------------------------------------------------------------------- */

/* Batched env_map::get_succ with HOST buffers: copies `nodes` to the device, runs the
 * expansion kernel, copies every non-NULL output back (pinned staging inside the ctx),
 * and returns when the results are in the caller's buffers.  Batches of up to 4096 successor
 * slots (n_nodes * nU) skip the copies: the kernel reads the nodes from and writes the outputs to
 * pinned host memory directly — the caller's arrays when they come from mplx_host_alloc, else the
 * ctx's staging buffers — so a single-node get_succ is one launch and one wait. */
int mplx_expand(mplx_ctx *ctx, const mplx_waypoint *nodes, int n_nodes, const mplx_succ_out *out);

/* Same, but `d_nodes` and the arrays in `out` are DEVICE pointers on the ctx's device.
 * `stream` is a cudaStream_t (NULL = the ctx's own stream).  Asynchronous: returns after
 * the launch. */
int mplx_expand_device(mplx_ctx *ctx, const void *d_nodes, int n_nodes, const mplx_succ_out *out,
                       void *stream);

/* ---- packed result stream (hosts across PCIe) ------------------------------------------ */

/* Drop successors whose edge cost is +inf (A* skips them: graph_search.h:81; LPA* keeps them). */
#define MPLX_PACK_DROP_INF 1

/* Dense result of mplx_expand_packed.  Record r of node i, r in [offset[i], offset[i]+count[i]),
 * in increasing control index.  `state` holds only the Waypoint fields the control flag marks as
 * state (use_pos, use_vel, use_acc, use_jrk, use_yaw: include/mpl_basis/waypoint.h:47-56), as
 * nstate = Dim*popcount(control&15) + (yaw?1:0) doubles per record laid out
 * [pos[Dim], vel[Dim], (acc[Dim]), (jrk[Dim]), (yaw)].  The remaining Waypoint fields of a
 * successor are copies, not results: evaluated derivative above the state order = 0 + U[action]
 * (next one) or 0, yaw = 0 without a yaw control, t = curr.t + dt (env_map.h:161).
 * state/cost/action/key may be NULL to skip; capacity is in records. */
typedef struct {
  int32_t *count;   /* [n_nodes]                                              */
  int64_t *offset;  /* [n_nodes] first record of node i                        */
  double *state;    /* [capacity*nstate]                                       */
  double *cost;     /* [capacity]   succ_cost                                  */
  uint16_t *action; /* [capacity]   action_idx                                 */
  uint64_t *key;    /* [capacity]   hash_value(succ), waypoint.h:93            */
  int64_t capacity; /* in: records the arrays can hold (n_nodes*nU always suffices) */
  int64_t total;    /* out: records written                                    */
  int32_t nstate;   /* out: doubles per state record                           */
} mplx_packed_out;

/* Batched env_map::get_succ with HOST buffers and the packed result stream: chunks of the
 * batch are expanded, packed on the device and copied back double-buffered over two streams,
 * so the PCIe transfer of one chunk overlaps the expansion of the next.  Pinned host buffers
 * (mplx_host_alloc) are needed for that overlap; pageable ones work but serialise. */
int mplx_expand_packed(mplx_ctx *ctx, const mplx_waypoint *nodes, int n_nodes, int flags,
                       mplx_packed_out *out);

/* ---- stored-edge re-validation (the incremental / LPA* callers of the path) ------------ */
/* An edge of the search graph is (parent state, action id): pr = Primitive(parent, U[action], dt)
 * (env_base::forward_action, include/mpl_planner/common/env_base.h:228-231).  Host buffers. */

/* env_map<Dim>::is_free(const Primitive&) (include/mpl_planner/env/env_map.h:60-76) for n_edges
 * edges: out_free[e] = 1 iff none of the n+1 samples of pr.sample(n), n = ceil(max_v*T/res)
 * (primitive.h:415-420), is occupied, outside the map or outside the search region.  out_cost
 * (NULL or n_edges doubles) receives calculate_intrinsic_cost(pr) (env_base.h:343-345), the cost
 * StateSpace::decreaseCost installs for a re-opened edge (state_space.h:236-243). */
int mplx_edges_is_free(mplx_ctx *ctx, const mplx_waypoint *parents, const int32_t *actions, int n_edges,
                       uint8_t *out_free, double *out_cost);

/* The voxel walk of MapPlanner<Dim>::getLinkedNodes (src/mpl_planner/map_planner.cpp:135-151): for
 * edge e the cells floatToInt(w.pos) of the samples w of pr.sample(n), an entry being emitted
 * whenever getIndex differs from the previous sample's.  Edge e owns entries
 * [out_offset[e], out_offset[e+1]) of out_cells, ctx-dim int32 each; out_offset has n_edges+1
 * entries and *out_total = out_offset[n_edges].  If capacity (entries) is too small the call fails
 * with MPLX_ERR_ARG after filling out_offset and *out_total, so the caller can size and retry.
 * out_table_voxel / out_table_edge (both NULL, or capacity int32 each) receive the inverted table
 * the reference keeps in lhm_ (map_planner.h:15-16,101): entry k says edge out_table_edge[k] passes
 * through voxel getIndex = out_table_voxel[k]; sorted by voxel index, the edges of one voxel in
 * emission order (edge index, then position along the edge) as lhm_[id] lists them. */
int mplx_edges_cells(mplx_ctx *ctx, const mplx_waypoint *parents, const int32_t *actions, int n_edges,
                     int64_t *out_offset, int32_t *out_cells, int64_t capacity, int64_t *out_total,
                     int32_t *out_table_voxel, int32_t *out_table_edge);

/* Kernel selection (diagnostics): 0 = auto (occupancy planning without a yaw control: the fixed-point
 * kernels, 5; otherwise the dealing kernel for JRK/SNP controls, yaw controls and potential-field
 * planning once a batch fills the GPU, else the register kernel),
 * 1 = the sequential kernel that keeps traverse_primitive's literal per-primitive loop
 * (env_map.h:99-130), 2 = the register kernel, 3 = the flat (sample-parallel, shared-memory
 * staged) kernel, 4 = the dealing kernel (sampling pulled from a CTA-wide ticket queue), 5 = the
 * fixed-point kernel (cells of the sample loop from one fused Horner chain per axis, exact FP64 only
 * for samples within 2^-25 cell of a boundary next to an obstacle; occupancy planning only, else auto).
 * All produce identical results.  The environment variable MPLX_KERNEL sets the initial value of a new ctx. */
int mplx_set_kernel(mplx_ctx *ctx, int which);

/* Synchronise the ctx stream. */
int mplx_sync(mplx_ctx *ctx);

/* ---- introspection ------------------------------------------------------------------ */

/* Number of kernel launches issued by this ctx since creation (expand + setup kernels). */
int64_t mplx_launch_count(const mplx_ctx *ctx);
/* Total voxel samples visited by the last mplx_expand* call when stats were enabled
 * (mplx_enable_stats(ctx,1)); used to compute the algorithmic bytes of SURVEY.md §8d. */
int mplx_enable_stats(mplx_ctx *ctx, int on);
int mplx_last_stats(mplx_ctx *ctx, int64_t *samples, int64_t *successors);
/* The ctx's cudaStream_t, for callers that time with CUDA events. */
void *mplx_stream(mplx_ctx *ctx);
/* Pinned (page-locked) host memory.  Buffers obtained here (or any cudaHostRegister'ed
 * memory) are DMA'd directly by mplx_expand; ordinary pageable buffers go through the ctx's
 * internal pinned staging plus one host memcpy. */
void *mplx_host_alloc(size_t bytes);
void mplx_host_free(void *p);
/* "libmplx sm_90a; <build flags>" */
const char *mplx_build_info(void);

#ifdef __cplusplus
}
#endif
#endif
