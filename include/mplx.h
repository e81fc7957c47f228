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
 * pointers for mplx_expand and DEVICE pointers for mplx_expand_device.
 * mplx_expand and mplx_expand_device may also write the slots [i*nU + count[i], (i+1)*nU)
 * of every non-NULL array; what they hold there is unspecified.  Nothing outside
 * [0, n_nodes*nU) is written. */
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
 * (their sizes are tied to the grid).  Edits of a few voxels of the same grid: mplx_update_cells.
 * Ordered only against the ctx's own stream: it does not wait for an expansion that
 * mplx_expand_device still runs on a caller's stream; synchronise that stream first. */
int mplx_set_map(mplx_ctx *ctx, const int8_t *data, const int32_t *dim, const double *origin,
                 double res);

/* Sparse MapUtil edit: grid[idx[k]] = values[k] for k < n, applied in array order (a later entry for
 * the same voxel wins).  idx are getIndex() values (map_util.h:34-41), 0 <= idx < nvox.  Updates the
 * int8 grid and both packed views derived from it (occupancy bits, occ2 pairs) with O(n) device work
 * and 5n bytes over PCIe: no pass over the full grid.  The result is bit-identical to mplx_set_map of
 * the edited grid.  Unlike mplx_set_map, the potential map and the search region are kept (the
 * reference env holds its own copies of both: env_map.h:181-183,290; env_base.h:301-303).
 * Synchronous, like mplx_set_map.  n == 0 is a no-op.  Any invalid argument (n < 0, a NULL array
 * with n > 0, an index outside the grid) -> MPLX_ERR_ARG with nothing applied.  Like mplx_set_map,
 * ordered only against the ctx's own stream: an expansion still running on a caller's stream from
 * mplx_expand_device may read the grid while it changes; synchronise that stream first. */
int mplx_update_cells(mplx_ctx *ctx, const int32_t *idx, const int8_t *values, int n);

/* Diagnostics: copy the device grid (nvox bytes), the occupancy words and the occ2 pairs
 * ((nvox+31)/32 each; a pair is {occupancy word, candidate-summary word}, 2 uint32 per pair) to
 * host buffers; any pointer may be NULL. */
int mplx_read_map(mplx_ctx *ctx, int8_t *grid, uint32_t *occ, uint32_t *occ2);

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

/* ---- batched A* on the device ---------------------------------------------------------------- */

/* Results of mplx_plan_batch (HOST arrays).  Query q's trajectory is actions[action_offset[q],
 * action_offset[q+1]) (action ids from start to goal; recoverTraj, graph_search.h:369-455); its closed
 * set is closed_keys[closed_offset[q], closed_offset[q+1]) sorted ascending (NULL closed_keys skips it).
 * Both capacities must be at least n_q*max_expand, which always suffices. */
typedef struct {
  int32_t *valid;          /* [n_q] a trajectory was found (or the start is already a goal)      */
  double *cost;            /* [n_q] its cost; +inf when none                                     */
  int32_t *expanded;       /* [n_q] expansion iterations (pops)                                  */
  int32_t *n_closed;       /* [n_q] closed states                                                */
  int64_t *action_offset;  /* [n_q+1]                                                            */
  int32_t *actions;
  int64_t action_capacity;
  int64_t *closed_offset;  /* [n_q+1], needed with closed_keys                                   */
  uint64_t *closed_keys;
  int64_t closed_capacity;
  int32_t slots;           /* out: queries searched at once (arena slots)                        */
  int64_t arena_bytes;     /* out: device bytes of one slot's arena                              */
  double seconds;          /* out: device time of the search (CUDA events)                       */
} mplx_batch_out;

/* Graph search A* (graph_search.h:39-182, setEpsilon(eps), setMaxNum(max_expand)) for n_q independent
 * (starts[q], goals[q]) queries on the ctx's map and parameters, entirely on the device: each query gives
 * what the host planner (MPL::AstarStepper with env_map's goal test and heuristic) gives, bit for bit.
 * The goal test is env_map::is_goal with tolerances tol_pos / tol_vel / tol_acc / tol_yaw (< 0 = off).
 * start_free[q] != 0 says the start is free (planner_base.h:283-287); NULL = is_free(start.pos) on the
 * device grid.  Occupancy planning only (mplx_plan_batch_cost_terms serves the rest): the call fails
 * with MPLX_ERR_ARG, and does nothing, when a potential map is installed, the control carries yaw,
 * max_expand <= 0, nU > 256, or the map or the parameters are missing, and with MPLX_ERR_ALLOC, also
 * doing nothing, when one worst-case arena does not fit the budget (mplx_plan_batch_fits).  Every query
 * slot owns an arena for the worst case (1 + max_expand*nU states), so no query can overflow; the arenas
 * stay in the ctx for the next call.  Synchronous. */
int mplx_plan_batch(mplx_ctx *ctx, const mplx_waypoint *starts, const mplx_waypoint *goals, const uint8_t *start_free,
                    int n_q, double eps, int max_expand, double tol_pos, double tol_vel, double tol_acc,
                    double tol_yaw, mplx_batch_out *out);

/* Whether mplx_plan_batch can run n_q queries with this max_expand (with_closed: the closed keys are
 * asked for) on the ctx as it stands: MPLX_OK with the slots and bytes per slot it would use, MPLX_ERR_ALLOC
 * when one worst-case arena next to the results exceeds the device-memory budget (a quarter of the free
 * device memory, counting the search buffers the ctx holds, at most 8 GiB), MPLX_ERR_ARG for the plans
 * mplx_plan_batch refuses.  Allocates and changes nothing.  slots / arena_bytes may be NULL. */
int mplx_plan_batch_fits(mplx_ctx *ctx, int n_q, int max_expand, int with_closed, int32_t *slots,
                         int64_t *arena_bytes);

/* mplx_plan_batch for every plan the ctx can hold: besides occupancy planning, potential-field planning
 * (mplx_set_potential or mplx_update_potential_map, with or without a gradient weight), yaw controls
 * (with wyaw and yaw_max) and search regions.  The sample loop sums the potential, gradient and
 * yaw-alignment terms per sample in the reference's loop order, so each query again gives what the host
 * planner gives, cost bit for bit.  The goal test and the start-is-free test read the ctx's grid, as the
 * host planner reads its map: after mplx_update_potential_map that grid is the field, after
 * mplx_set_potential it stays the occupancy map.  Same arguments, outputs, memory budget and refusals as
 * mplx_plan_batch, except that a potential map or a yaw control is not refused: MPLX_ERR_ARG when
 * max_expand <= 0, nU > 256, or the map or the parameters are missing, MPLX_ERR_ALLOC when one worst-case
 * arena does not fit; either leaves outputs and ctx untouched.  Occupancy plans give the same results as
 * through mplx_plan_batch, whose kernel skips the cost-term code.  Synchronous. */
int mplx_plan_batch_cost_terms(mplx_ctx *ctx, const mplx_waypoint *starts, const mplx_waypoint *goals,
                               const uint8_t *start_free, int n_q, double eps, int max_expand, double tol_pos,
                               double tol_vel, double tol_acc, double tol_yaw, mplx_batch_out *out);

/* mplx_plan_batch_fits for mplx_plan_batch_cost_terms: the slots and bytes per slot that call would use,
 * MPLX_ERR_ALLOC / MPLX_ERR_ARG as it would refuse.  Allocates and changes nothing. */
int mplx_plan_batch_cost_terms_fits(mplx_ctx *ctx, int n_q, int max_expand, int with_closed, int32_t *slots,
                                    int64_t *arena_bytes);

/* Results of mplx_plan_batch_grow (HOST arrays of n_q entries, all required).  The trajectories and closed
 * keys follow with mplx_plan_batch_grow_results. */
typedef struct {
  int32_t *valid;     /* [n_q] as mplx_batch_out                                                    */
  double *cost;       /* [n_q]                                                                      */
  int32_t *expanded;  /* [n_q]                                                                      */
  int32_t *n_closed;  /* [n_q]                                                                      */
  int32_t *n_actions; /* [n_q] trajectory length                                                    */
  int32_t *searched;  /* [n_q] 1: the fields above are the query's result; 0: its search needed more than
                         the largest capacity (its fields are 0 / +inf)                              */
  int32_t rounds;     /* out: kernel launches this call made                                        */
  int32_t slots;      /* out: slots (arenas) of the first round                                     */
  int64_t first_cap, last_cap; /* out: records per arena in the first and the last round            */
  int64_t arena_bytes; /* out: bytes of one first-round arena                                       */
  int64_t reruns;     /* out: query searches abandoned and searched again (arena or result pool full) */
  double seconds;     /* out: device time of all rounds (CUDA events)                               */
} mplx_grow_out;

/* Graph search A* for n_q queries as mplx_plan_batch (cost_terms = 0: the occupancy search, with its
 * refusals) or mplx_plan_batch_cost_terms (cost_terms = 1, with its refusals) runs it, with arenas sized
 * for the batch rather than for the worst case, so that unbounded searches (max_expand <= 0, the
 * reference's default setMaxNum(-1)) and caps whose worst case does not fit run on the device too.  Each
 * searched query gives exactly what the host planner gives: a query that outgrows its arena is abandoned
 * and searched again from scratch, and a search's result does not depend on its arena's size.
 *
 * Capacity: an arena of cap records holds cap states and cap predecessor records.  A query's need is the
 * larger of its final state and predecessor-record counts (the records, one per finite successor,
 * normally bind); it finishes in an arena with cap >= need and is abandoned in one with cap < need.
 *
 * Budget: as mplx_plan_batch_fits (a quarter of the free device memory counting the search buffers the
 * ctx holds, at most 8 GiB).  The per-query arrays (a few hundred bytes per query) and the automatic
 * result pool (an eighth of the budget) come off it first; the arenas share the rest.
 *
 * Round schedule (each round is one kernel launch over the round's pending queries, each query with a
 * fresh key-table epoch):
 *   cap_max = the largest capacity at which one arena fits the rest of the budget, at most max_cap when
 *             max_cap > 0, and at most 1 + max_expand*nU (the worst case) when max_expand > 0;
 *   cap_0   = first_cap when first_cap > 0, else the largest capacity at which min(n_q, resident CTAs)
 *             arenas fit the rest of the budget; then clipped to [1, cap_max].  A bounded plan whose worst
 *             case fits therefore runs in one round.
 *   Round r runs its pending queries in max(1, min(pending, resident CTAs, arenas that fit)) slots.  A query that
 *   finishes takes its room in the result pool; one that finds the pool full stays pending at the same
 *   capacity; one that overflows moves on.  The pool-full queries run again first, at the same capacity;
 *   then the overflowed ones at min(4*cap, cap_max).  A query that overflows at cap_max gets searched = 0.
 *   reruns counts every query that was queued again (pool full or overflowed below cap_max).
 *
 * Result pool: completed queries reserve room for their closed keys (with_closed) and action ids in one
 * device pool, one atomicAdd per query; the pool is drained to the host after each round.  pool_bytes > 0
 * sets its size (a diagnostic), 0 takes an eighth of the budget.  The rerun of queries that found the pool
 * full gets a pool that holds the largest of them, so every round completes at least one query.  No result
 * is truncated or written out of bounds.
 *
 * Refusals, each with the outputs and the ctx untouched and no launch: MPLX_ERR_ARG for cost_terms not 0
 * or 1, a potential map or a yaw control with cost_terms = 0, nU > 256, a missing map or parameters, a NULL
 * out or output array, missing query arrays, n_q < 0, or a negative first_cap, max_cap or pool_bytes;
 * MPLX_ERR_ALLOC when not even an arena of one record fits next to the per-query arrays and the pool.
 * The arenas stay in the ctx and are shared with mplx_plan_batch and mplx_plan_batch_cost_terms.
 * Synchronous. */
int mplx_plan_batch_grow(mplx_ctx *ctx, int cost_terms, const mplx_waypoint *starts, const mplx_waypoint *goals,
                         const uint8_t *start_free, int n_q, double eps, int max_expand, double tol_pos,
                         double tol_vel, double tol_acc, double tol_yaw, int with_closed, int64_t first_cap,
                         int64_t max_cap, int64_t pool_bytes, mplx_grow_out *out);

/* The trajectories (action ids from start to goal) and the closed keys (sorted ascending; with_closed) of
 * the last mplx_plan_batch_grow call on this ctx: query q's at actions[action_offset[q], action_offset[q+1])
 * and closed_keys[closed_offset[q], closed_offset[q+1]) (offsets have n_q+1 entries; closed_keys NULL skips
 * them, and a call without with_closed has none).  MPLX_ERR_ARG, writing nothing, when no call was made,
 * an array is missing, or a capacity is below the sum of n_actions / n_closed. */
int mplx_plan_batch_grow_results(mplx_ctx *ctx, int64_t *action_offset, int32_t *actions, int64_t action_capacity,
                                 int64_t *closed_offset, uint64_t *closed_keys, int64_t closed_capacity);

/* ---- the planned trajectories of the batched searches ------------------------------------------ */

/* Record the trajectories of the following mplx_plan_batch / _cost_terms / _grow calls on this ctx (on = 1;
 * 0 = off, the default).  pool_bytes > 0 sizes the trajectory room (a diagnostic); 0 = automatic, an eighth of
 * the call's search budget.  With recording on, a finished query with a trajectory of n actions also copies the
 * stored coordinates of its path's n + 1 states (recoverTraj's best_child_) into the room, which stays on the
 * device; a query that finds the room full is searched again in a later round whose room holds all such queries
 * (the kept buffer grows past the share only by what the trajectories themselves take), so
 * mplx_plan_batch and mplx_plan_batch_cost_terms may then take more than one kernel launch.  The room comes off
 * the budget, so fewer arenas may fit; no query's results depend on the room's size.  With recording off, every
 * search call makes the launches it made without this call.  MPLX_ERR_ARG for on not 0 or 1 or pool_bytes < 0. */
int mplx_set_batch_trajectories(mplx_ctx *ctx, int on, int64_t pool_bytes);

/* Results of mplx_plan_batch_trajectories (HOST arrays), slots as mplx_traj_out's. */
typedef struct {
  int64_t *offset;       /* [n_q+1] query q owns waypoint slots [offset[q], offset[q+1]): n_actions+1 when its
                            trajectory has at least one segment, else 0 (no trajectory, start already a goal,
                            not searched)                                                                      */
  mplx_waypoint *nodes;  /* [capacity] the stored coordinates of the path's states, start to goal (best_child_) */
  double *seg_t;         /* [capacity] dt per segment (the ctx's T); the path's last slot 0                    */
  double *coeff;         /* [capacity*(dim+1)*6] forward_action(nodes[j], U[action j], T) Primitive
                            coefficients, mplx_traj_out's layout (highest order first, axes, then yaw; the
                            yaw axis is 0 without a yaw control); the path's last slot 0                       */
  double *samples;       /* NULL or [n_q*(n_samples+1)*(4*dim+3)] Trajectory::sample(n_samples) rows as
                            mplx_traj_out's; zeros for a query without trajectory                              */
  int64_t capacity;      /* in: waypoint slots the arrays hold                                                  */
  int64_t total;         /* out: slots needed                                                                   */
  double seconds;        /* out: device time of the kernels (CUDA events)                                       */
} mplx_batch_traj_out;

/* The trajectories of the last search call (mplx_plan_batch, mplx_plan_batch_cost_terms or mplx_plan_batch_grow)
 * on this ctx, which must have run with recording on (mplx_set_batch_trajectories), for its n_q queries in query
 * order.  Segment j of query q is Primitive(nodes[offset[q] + j], U[actions[j]], T) (env_base::forward_action)
 * built from the coordinates the search stored for the path's states, as recoverTraj builds it; a replay of the
 * action ids from the start can differ where a state's best predecessor is not the one that first created it.
 * The coefficients are bit for bit the host's Primitive and the samples the host's Trajectory::sample.  The
 * output feeds mplx_traj_check and mplx_traj_scale as it stands.  Capacity: when capacity < total the call fills
 * offset and total and fails with MPLX_ERR_ARG.  Refusals, each with MPLX_ERR_ARG, the outputs untouched and no
 * launch: no completed search call yet, the last one ran without recording, n_samples < 0, samples given with
 * n_samples == 0, and a NULL out, offset, nodes, seg_t or coeff.  The kept coordinates stay until the next search
 * call replaces them.  A constant number of launches per call.  Synchronous. */
int mplx_plan_batch_trajectories(mplx_ctx *ctx, int n_samples, mplx_batch_traj_out *out);

/* ---- one tunnel per query of the batched searches ---------------------------------------------- */

/* MapPlanner<Dim>::setSearchRegion(path, dense) once per query for the following mplx_plan_batch / _cost_terms /
 * _grow calls: query q's tunnel is built from the points pts[pt_offset[q] .. pt_offset[q+1]) (ctx-dim doubles
 * each) with the one radius (ctx-dim doubles) and dense flag of the batch, and is exactly the region
 * mplx_set_search_region_path builds from those points.  Those calls must then have exactly n_q queries (else
 * MPLX_ERR_ARG, doing nothing); query q searches in tunnel q, which replaces the ctx-wide region for it, as
 * setSearchRegion replaces search_region_.  The expansion, edge and trajectory-check calls keep the ctx-wide region.
 * n_q = 0 clears the tunnels.  mplx_set_map drops them; mplx_update_cells keeps them.
 *
 * A tunnel is stored as the 8x8x8 bricks (8x8 tiles in 2-D) it touches, with one bit per cell, so its memory grows
 * with the tunnel, not the map (mplx_batch_regions_info reports it).  The store comes off the search calls' budget
 * (mplx_plan_batch_fits); MPLX_ERR_ALLOC, with the tunnels unchanged, when it alone exceeds that budget.  A constant
 * number of launches whatever n_q.  Refusals, each with MPLX_ERR_ARG, nothing changed and no launch: no map,
 * n_q < 0, a NULL array (n_q > 0), pt_offset[0] != 0, and a query with no points (pt_offset must increase).
 * Synchronous. */
int mplx_set_batch_regions(mplx_ctx *ctx, int n_q, const int64_t *pt_offset, const double *pts, const double *radius,
                           int dense);

/* mplx_set_batch_regions with paths the last search call recorded, so that a replanning loop (MapPlanner::
 * iterativePlan) builds each round's tunnels without bringing the paths to the host: query j's tunnel is
 * MapPlanner<Dim>::setSearchRegion(path, dense) where path is, for from[j] >= 0, the recorded path of query from[j]
 * of the last mplx_plan_batch / _cost_terms / _grow call (the positions of its stored path states from start to
 * goal, the nodes mplx_plan_batch_trajectories returns and MapPlanner::getWaypointPositions gives on the host), and
 * for from[j] < 0 the points pts[pt_offset[j] .. pt_offset[j+1]), as in mplx_set_batch_regions.  pt_offset and pts
 * may be NULL when every from[j] >= 0; otherwise pt_offset has n_q + 1 entries, starts at 0 and never decreases, and
 * increases at every j with from[j] < 0.  The paths are traced on the device, by the same walk as
 * mplx_set_search_region_path's, so each tunnel is exactly that call's region of the same points.  The recorded
 * paths are read at this call; the next search call replaces them.  Everything else as mplx_set_batch_regions:
 * the next search calls must have exactly n_q queries, n_q = 0 clears the tunnels, the store, its budget
 * (MPLX_ERR_ALLOC, tunnels unchanged), mplx_set_map / mplx_update_cells, mplx_read_batch_region, and a constant
 * number of launches whatever n_q.  Refusals, each with MPLX_ERR_ARG, the tunnels unchanged and no launch: no map,
 * n_q < 0, a NULL from or radius (n_q > 0), no completed search call (none yet, or the last one failed), a last
 * call without recording (mplx_set_batch_trajectories), from[j] at or past the last call's query count, a selected
 * query with no recorded path (no trajectory, start already a goal, or not searched), and from[j] < 0 without
 * points (NULL pt_offset or pts, or a pt_offset as above it is not).  Synchronous. */
int mplx_set_batch_regions_recorded(mplx_ctx *ctx, int n_q, const int32_t *from, const int64_t *pt_offset,
                                    const double *pts, const double *radius, int dense);

/* The tunnels set on the ctx: their query count (0 = none), bricks and device bytes.  Any pointer may be NULL. */
int mplx_batch_regions_info(mplx_ctx *ctx, int32_t *n_q, int64_t *n_bricks, int64_t *bytes);

/* Diagnostics: query q's tunnel as one byte per voxel (1 = inside), the layout mplx_set_search_region_path's
 * out_region has.  MPLX_ERR_ARG when no tunnels are set, q is out of range or out is NULL.  Synchronous. */
int mplx_read_batch_region(mplx_ctx *ctx, int q, uint8_t *out);

/* ---- trajectories through waypoints (TrajSolver) ----------------------------------------------- */

/* Results of mplx_traj_solve (HOST arrays).  Path p owns the waypoint slots [offset[p], offset[p+1]); segment j
 * of path p (j < n_wp(p) - 1) is at slot offset[p] + j, and the path's last slot holds zeros. */
typedef struct {
  int32_t *status;  /* [n_paths] 1: at least 2 waypoints and every coefficient finite; else 0                 */
  double *seg_t;    /* [n_wp] segment duration (the given dts, or |p_j+1 - p_j|_inf / v)                     */
  double *coeff;    /* [n_wp*(dim+1)*6] Primitive1D coefficients, highest order first, axes x, y, (z), yaw:
                       what the segment's Primitive holds after TrajSolver::solve                           */
  double *samples;  /* NULL, or [n_paths*(n_samples+1)*(4*dim+3)] Trajectory::sample(n_samples) rows
                       {pos, vel, acc, jrk, yaw, yaw_dot, t}; zeros for status-0 paths                       */
  double seconds;   /* out: device time of the kernels (CUDA events)                                        */
} mplx_traj_out;

/* TrajSolver<Dim>(control, yaw_control) (include/mpl_traj_solver/traj_solver.h) for n_paths independent paths
 * on the device: the piecewise polynomial through each path's waypoints that minimises the integral of the
 * squared velocity (VEL), acceleration (ACC) or jerk (JRK) — with or without YAW, the yaw axis from its own
 * pass — for Dim = the ctx's dimension.  No map or parameters are needed.
 *   wp_control NULL: setPath — only wps[].pos is read; the endpoints take `control`, the interior waypoints
 *     VEL (position fixed), every other derivative and the yaw are 0.
 *   wp_control given: setWaypoints — waypoint i fixes the derivatives its flags wp_control[i] name (use_pos,
 *     use_vel, use_acc below the solver's order) at wps[i].pos / vel / acc; the yaw pass reads wps[i].yaw.
 *   The yaw pass fixes the yaw at every waypoint, and at the endpoints also the derivatives yaw_control names
 *     (as 0).
 *   dts NULL: segment times |p_j+1 - p_j|_inf / v (TrajSolver::allocate_time); else dts[offset[p] + j] is
 *     segment j's duration ([n_wp] slots as the outputs).
 * Each path is what the host TrajSolver gives, within floating-point rounding: the reference's dense
 * (S*N) x (S*N) formulation becomes one O(S) block-tridiagonal Cholesky sweep per path.  Two waypoints with
 * free derivatives leave those at 0; a zero-length or non-finite segment time gives status 0.  The samples
 * are the host Trajectory's sample(n_samples) of seg_t and coeff bit for bit.  Each path's outputs do not
 * depend on the other paths of the batch.  Scratch is sized from the batch and kept in the ctx.
 * Refusals, each with MPLX_ERR_ARG, the outputs untouched and no launch: control not VEL / ACC / JRK (with
 * or without YAW; SNP has no solver in the reference), yaw_control not VEL / ACC / JRK, dts NULL with
 * v <= 0, n_paths < 0, offset NULL, offset[0] != 0 or decreasing, out / status / seg_t / coeff NULL, wps NULL
 * with waypoints, and samples given with n_samples <= 0.  Synchronous. */
int mplx_traj_solve(mplx_ctx *ctx, int n_paths, const int64_t *offset, const mplx_waypoint *wps,
                    const uint8_t *wp_control, const double *dts, double v, int control, int yaw_control,
                    int n_samples, mplx_traj_out *out);

/* ---- time scaling of trajectories (Trajectory::scale / scale_down) ------------------------------ */

#define MPLX_TRAJ_SCALE 1      /* Trajectory::scale(ri, rf)          */
#define MPLX_TRAJ_SCALE_DOWN 2 /* Trajectory::scale_down(mv, ri, rf) */

/* Results of mplx_traj_scale (HOST arrays), slots as mplx_traj_out's. */
typedef struct {
  int32_t *status;   /* [n_paths] 1: scaled; 2: SCALE_DOWN found no velocity above mv (max_l <= 1), unchanged;
                        0: not scaled (fewer than 2 waypoints, a segment time <= 0 or not finite, a coefficient
                        not finite, or ri, rf or (SCALE_DOWN) mv not finite and > 0)                         */
  double *total_t;   /* [n_paths] the trajectory's total time after the call (0 for status 0)                  */
  double *seg_T;     /* [n_wp] getSegmentTimes(): Ts[j+1] - Ts[j] of the scaled waypoint times; the path's last
                        slot and every slot of a status-0 path hold 0                                          */
  int32_t *n_lambda; /* NULL, or [n_paths] lambda segments of the path (0 unless status 1)                    */
  double *lambda;    /* NULL, or [n_wp*5*dim*7] lambda segments {a3, a2, a1, a0, ti, tf, dT}: path p's start at
                        slot offset[p]*5*dim, unused slots hold 0                                             */
  double *samples;   /* NULL, or [n_paths*(n_samples+1)*(4*dim+3)] Trajectory::sample(n_samples) rows after the
                        scaling, mplx_traj_out's row format; zeros for status-0 paths                          */
  double seconds;    /* out: device time of the kernels (CUDA events)                                        */
} mplx_traj_scale_out;

/* Trajectory<Dim>::scale(ri, rf) (mode MPLX_TRAJ_SCALE) or scale_down(mv, ri, rf) (MPLX_TRAJ_SCALE_DOWN) on
 * n_paths trajectories on the device, Dim = the ctx's dimension.  Path p's segment j has the duration
 * seg_t[offset[p] + j] and the coefficients coeff[(offset[p] + j)*(dim+1)*6 ...], exactly mplx_traj_out's
 * layout, so mplx_traj_solve's output feeds straight in.  mv, ri and rf are per-path arrays; mv may be NULL
 * for SCALE.
 *   scale: lambda(tau) is the cubic from 1/ri (slope 0) at tau = 0 to 1/rf (slope 0) at the end.
 *   scale_down: each segment and axis whose max_vel exceeds mv adds a knot at its velocity extrema, at its
 *     start (except segment 0) and at its end where |v| / mv > 1; between (0, ri) and (end, rf) the knots
 *     take the largest ratio max_l.  Note ri, rf here against 1/ri, 1/rf for scale, as in the reference.
 * Then t = integral of lambda maps real time to polynomial time; sampling inverts it per sample by the
 * closed-form quartic root (Lambda::getTau).  Each path is what the host Trajectory gives (mpl_host.hpp),
 * bit for bit where only arithmetic is involved (VEL and ACC paths, lambda constant), else within 1e-9
 * relative: cbrt, acos and cos are CUDA's (DESIGN.md §8).  As in the reference, the last sample can land an
 * ulp past the final lambda segment, and is then the trajectory's start state.  Each path's outputs do not
 * depend on the other paths.  Scratch is kept in the ctx.
 * Refusals, each with MPLX_ERR_ARG, the outputs untouched and no launch: an unknown mode, mv NULL for
 * SCALE_DOWN, ri or rf NULL, n_paths < 0, offset NULL, offset[0] != 0 or decreasing, out / status / total_t /
 * seg_T NULL, seg_t or coeff NULL with waypoints, and samples given with n_samples <= 0.  Synchronous. */
int mplx_traj_scale(mplx_ctx *ctx, int n_paths, const int64_t *offset, const double *seg_t, const double *coeff,
                    int mode, const double *mv, const double *ri, const double *rf, int n_samples,
                    mplx_traj_scale_out *out);

/* ---- checking trajectories against the map and the limits ------------------------------------ */

/* Largest sample count n that a trajectory or segment check evaluates (traverse_trajectory's N, is_free's n).
 * Beyond it the reference would allocate n + 1 samples; the checks report the path not evaluated or the
 * segment not free instead. */
#define MPLX_SAMPLE_N_MAX (1 << 20)

/* Results of mplx_traj_check (HOST arrays), slots as mplx_traj_out's. */
typedef struct {
  int32_t *status;    /* [n_paths] 1: cost evaluated; 0: not (fewer than 2 waypoints, a segment time <= 0 or not
                         finite, a coefficient not finite, or N = ceil(v_max * total / res) outside
                         [1, MPLX_SAMPLE_N_MAX])                                                             */
  double *cost;       /* [n_paths] env_map::traverse_trajectory: +inf when a counted sample leaves the map or
                         hits an obstacle, else the potential terms' sum (0 without a potential map); 0 for
                         status 0                                                                            */
  uint8_t *seg_free;  /* NULL, or [n_wp] env_map::is_free(segment j) at slot offset[p] + j; the path's last slot
                         and every slot of a path with a bad segment time or coefficient hold 0              */
  uint8_t *seg_valid; /* NULL, or [n_wp] validate_primitive(segment j, v_max, a_max, j_max, yaw_max), slots as
                         seg_free's                                                                          */
  double seconds;     /* out: device time of the kernels (CUDA events)                                       */
} mplx_traj_check_out;

/* Checks n_paths trajectories against the ctx's map and parameters on the device, as the reference's env_map
 * and validate_primitive do after the same mplx_set_map / mplx_set_potential (or mplx_update_potential_map) /
 * mplx_set_search_region / mplx_set_params calls.  The trajectories are mplx_traj_out's layout (offset, seg_t,
 * coeff), so mplx_traj_solve's output feeds straight in; total_t, n_lambda and lambda (mplx_traj_scale_out's,
 * all three or none) add mplx_traj_scale's time scaling, path p scaled when n_lambda[p] > 0.  control[p] is the
 * control flag of path p's segments (a TrajSolver segment carries its first waypoint's control); it may be
 * NULL when seg_valid is.
 *   cost: traverse_trajectory (env_map.h:228-255).  N = ceil(v_max * total / res) with the path's (scaled)
 *     total time; the N + 1 rows of Trajectory::sample(N).  A sample counts when its getIndex(floatToInt(pos)),
 *     wrapped to 32 bits, differs from the previous sample's (-1 before the first).  A counted sample outside
 *     the map, or with a potential map installed at a potential >= 100, or without one in an occupied cell,
 *     makes the cost +inf; otherwise, with a potential map, a counted sample with 0 < potential < 100 adds
 *     potential_weight * potential + gradient_weight * |vel|, summed in sample order.  No search-region test.
 *   seg_free: is_free(segment) (env_map.h:60-76): the n + 1 samples of Primitive::sample(n), n =
 *     ceil(max_v * T / res), max_v the largest Primitive::max_vel over the axes; a sample that is occupied,
 *     outside the map or outside the search region makes it not free.  A stationary segment (n = 0) samples at
 *     t = NaN, outside the map: not free.  n above MPLX_SAMPLE_N_MAX: not free.  No time scaling enters.
 *   seg_valid: validate_primitive (primitive.h:449-525) by control[p]: validate_xxx per axis (max_vel,
 *     max_acc, max_jrk; a limit <= 0 passes) and validate_yaw at the segment's two ends.
 * Each path is what the host env_map_host / validate_primitive give (mpl_host.hpp): cost and status bit for bit
 * without scaling; seg_free and seg_valid bit for bit for VEL and ACC segments, and for JRK ones except where
 * CUDA's cbrt / acos / cos put max_vel on the other side of an integer or a limit; with a yaw control
 * validate_yaw uses CUDA's sin / cos, so seg_valid may also differ where d is within 1e-12 of cos(yaw_max).  A
 * scaled path's samples pass through the closed-form quartic of Lambda::getTau, whose roots are not bitwise the
 * host's, so its cost may differ in three ways (DESIGN.md §8): a sample within 1e-9 (1 + |x|) of a cell boundary
 * can change cell; with a gradient weight, the |vel| = v / lambda of the terms carries the root's rounding, so the
 * sum may differ by about 1e-9 relative where every cell agrees; and the final sample, whose time can land an ulp
 * past the last lambda segment, can be the start state on one side and a root near the end on the other.  Each
 * path's outputs do not depend on the other paths.  Scratch is kept in the ctx.
 * Refusals, each with MPLX_ERR_ARG, the outputs untouched and no launch: no map or no parameters, n_paths < 0,
 * offset NULL, offset[0] != 0 or decreasing, out / status / cost NULL, seg_t or coeff NULL with waypoints,
 * control NULL with seg_valid, only some of total_t / n_lambda / lambda given, and n_lambda[p] outside
 * [0, n_wp(p) * 5 * dim].  Synchronous. */
int mplx_traj_check(mplx_ctx *ctx, int n_paths, const int64_t *offset, const double *seg_t, const double *coeff,
                    const uint8_t *control, const double *total_t, const int32_t *n_lambda, const double *lambda,
                    mplx_traj_check_out *out);

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
