"""Python mirror of the reference's operator interface for the node-expansion path.

`env_map` here has the method names, argument meaning and error behaviour of
MPL::env_map<Dim> / env_base<Dim> (reference include/mpl_planner/env/env_map.h,
include/mpl_planner/common/env_base.h:234-303) for the setters that feed get_succ, and
`get_succ` itself (env_map.h:147-172) plus the batched `expand` the B200 engine adds.
All computation happens in libmplx.so (CUDA, sm_90a); this file only marshals arguments.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import abi
from .abi import LATTICE_MAX, WAYPOINT_DTYPE, PackedOut, SuccOut
from .traj import pack_lambda, pack_paths, split_slots


class MapUtil:
    """MPL::MapUtil<Dim> storage + setMap (reference include/mpl_collision/map_util.h:85-91).

    Holds the x-fastest int8 grid (occupied 100 / free 0 / unknown -1, map_util.h:309-313).
    """

    def __init__(self):
        self.map = None
        self.dim = None
        self.origin = None
        self.res = None

    def setMap(self, ori, dim, map_, res):
        dim = np.asarray(dim, dtype=np.int32)
        map_ = np.ascontiguousarray(map_, dtype=np.int8).reshape(-1)
        if map_.size != int(np.prod(dim.astype(np.int64))):
            raise ValueError("map size does not match dim")
        self.origin = np.asarray(ori, dtype=np.float64)
        self.dim = dim
        self.map = map_
        self.res = float(res)

    def getRes(self):
        return self.res

    def getDim(self):
        return self.dim

    def getOrigin(self):
        return self.origin

    def getMap(self):
        return self.map


@dataclass
class Expansion:
    """Result of a batched expansion; segment i is [i*nU, i*nU+count[i]) of every array."""

    nU: int
    count: np.ndarray
    succ: np.ndarray | None
    cost: np.ndarray | None
    action: np.ndarray | None
    key: np.ndarray | None
    lattice: np.ndarray | None

    def node(self, i: int):
        """(succ, cost, action) of node i, exactly what env_map::get_succ returns."""
        s = slice(i * self.nU, i * self.nU + int(self.count[i]))
        return (
            None if self.succ is None else self.succ[s],
            None if self.cost is None else self.cost[s],
            None if self.action is None else self.action[s],
        )


class env_map:
    """GPU-backed MPL::env_map<Dim>.  One instance owns one libmplx ctx (one device, one stream)."""

    def __init__(self, map_util: MapUtil, device: int = 0):
        self._lib = abi.load()
        self.Dim = int(len(map_util.dim))
        h = C.c_void_p()
        abi.check(self._lib.mplx_create(self.Dim, device, C.byref(h)))
        self._h = h
        self.map_util_ = map_util
        # defaults: reference env_base.h:368-392, env_map.h:294-296
        self.w_, self.wyaw_, self.dt_ = 10.0, 1.0, 1.0
        self.v_max_ = self.a_max_ = self.j_max_ = self.yaw_max_ = -1.0
        self.U_ = None
        self.control = None
        self.potential_weight_, self.gradient_weight_ = 0.1, 0.0
        self._potential = None
        self._dirty = True
        self._last_nq = 0  # queries of the last plan_batch* call (batch_trajectories' offset length)
        self.upload_map()

    # -- lifecycle ------------------------------------------------------------------------
    def close(self):
        for p in getattr(self, "_pins", []):
            self._lib.mplx_host_free(p)  # numpy views handed out by _pinned_empty die with the env
        self._pins = []
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.mplx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def upload_map(self):
        """Stage the MapUtil grid into HBM (mplx_set_map).  The reference env shares the MapUtil by
        pointer (env_map.h:288); call this again after mutating it."""
        mu = self.map_util_
        dim = np.ascontiguousarray(mu.dim, dtype=np.int32)
        org = np.ascontiguousarray(mu.origin, dtype=np.float64)
        abi.check(self._lib.mplx_set_map(self._h, mu.map.ctypes.data, dim.ctypes.data, org.ctypes.data, mu.res))
        self._potential = None

    def update_cells(self, idx_or_cells, values):
        """Set a few voxels of the MapUtil grid, in place, and on the device (mplx_update_cells).
        `idx_or_cells` is either getIndex() values (1-D) or n x Dim cell coordinates; `values` has one
        int8 per entry, and a later entry for the same voxel wins.  Costs O(n), not a re-upload, and
        unlike upload_map() keeps the potential map and the search region."""
        mu = self.map_util_
        a = np.asarray(idx_or_cells)
        if a.ndim == 2:
            cells = a.astype(np.int64).reshape(-1, self.Dim)
            dims = np.asarray(mu.dim, dtype=np.int64)
            if ((cells < 0) | (cells >= dims)).any():
                raise ValueError("cell outside the map")
            idx = cells[:, 0] + dims[0] * cells[:, 1]
            if self.Dim == 3:
                idx = idx + dims[0] * dims[1] * cells[:, 2]
        else:
            idx = a.astype(np.int64).reshape(-1)
        vals = np.ascontiguousarray(values, dtype=np.int8).reshape(-1)
        if vals.size != idx.size:
            raise ValueError("one value per cell")
        if ((idx < 0) | (idx >= mu.map.size)).any():
            raise ValueError("index outside the map")
        idx32 = np.ascontiguousarray(idx, dtype=np.int32)
        abi.check(self._lib.mplx_update_cells(self._h, idx32.ctypes.data, vals.ctypes.data, idx32.size))
        # last write wins: the first occurrence of each index in the reversed arrays
        u, first = np.unique(idx32[::-1], return_index=True)
        mu.map[u] = vals[::-1][first]

    def read_map(self):
        """The device grid, occupancy words and occ2 pairs (mplx_read_map): (int8[nvox], uint32[nw], uint32[nw, 2])."""
        nvox = self.map_util_.map.size
        nw = (nvox + 31) // 32
        grid = np.empty(nvox, dtype=np.int8)
        occ = np.empty(nw, dtype=np.uint32)
        occ2 = np.empty((nw, 2), dtype=np.uint32)
        abi.check(self._lib.mplx_read_map(self._h, grid.ctypes.data, occ.ctypes.data, occ2.ctypes.data))
        return grid, occ, occ2

    # -- setters (env_base.h:234-303, env_map.h:175-186) -------------------------------------
    def set_u(self, U):
        self.U_ = np.ascontiguousarray(U, dtype=np.float64)
        if self.U_.ndim != 2:
            raise ValueError("U must be |U| x udim")
        self._dirty = True

    def set_control(self, control: int):
        """The Waypoint control flag of the plan (start.control; waypoint.h:47-56)."""
        self.control = int(control)
        self._dirty = True

    def set_dt(self, dt):
        self.dt_ = float(dt)
        self._dirty = True

    def set_w(self, w):
        self.w_ = float(w)
        self._dirty = True

    def set_wyaw(self, w):
        self.wyaw_ = float(w)
        self._dirty = True

    def set_v_max(self, v):
        self.v_max_ = float(v)
        self._dirty = True

    def set_a_max(self, a):
        self.a_max_ = float(a)
        self._dirty = True

    def set_j_max(self, j):
        self.j_max_ = float(j)
        self._dirty = True

    def set_yaw_max(self, y):
        self.yaw_max_ = float(y)
        self._dirty = True

    def set_potential_weight(self, w):
        self.potential_weight_ = float(w)
        self._push_potential()

    def set_gradient_weight(self, w):
        self.gradient_weight_ = float(w)
        self._push_potential()

    def set_potential_map(self, pmap):
        self._potential = None if pmap is None or len(pmap) == 0 else np.ascontiguousarray(pmap, dtype=np.int8).reshape(-1)
        if self._potential is not None and self._potential.size != self.map_util_.map.size:
            raise ValueError("potential map size does not match the grid")
        self._push_potential()

    def _push_potential(self):
        p = None if self._potential is None else self._potential.ctypes.data
        abi.check(self._lib.mplx_set_potential(self._h, p, self.potential_weight_, self.gradient_weight_))

    def set_search_region(self, region):
        if region is None or len(region) == 0:
            abi.check(self._lib.mplx_set_search_region(self._h, None))
            return
        r = np.ascontiguousarray(region).reshape(-1).astype(np.uint8)
        if r.size != self.map_util_.map.size:
            raise ValueError("search region size does not match the grid")
        abi.check(self._lib.mplx_set_search_region(self._h, r.ctypes.data))

    def update_potential_map(self, radius, pow_=1.0, range_=None, pos=None):
        """MapPlanner::updatePotentialMap on the device (mplx_update_potential_map).  As in the
        reference (map_planner.cpp:387-388) the MapUtil grid is replaced by the potential field,
        which also becomes the env's potential map.  Returns the new grid."""
        rad = np.ascontiguousarray(radius, dtype=np.float64)
        rng = None if range_ is None else np.ascontiguousarray(range_, dtype=np.float64)
        p = None if pos is None else np.ascontiguousarray(pos, dtype=np.float64)
        out = np.empty(self.map_util_.map.size, dtype=np.int8)
        abi.check(self._lib.mplx_update_potential_map(self._h, rad.ctypes.data, float(pow_), abi.ptr(rng), abi.ptr(p),
                                                      self.potential_weight_, self.gradient_weight_, out.ctypes.data))
        self.map_util_.map = out
        self._potential = out
        return out

    def set_search_region_path(self, path, radius, dense=False):
        """MapPlanner::setSearchRegion on the device (mplx_set_search_region_path); returns the region bytes."""
        path = np.ascontiguousarray(path, dtype=np.float64).reshape(-1, self.Dim)
        rad = np.ascontiguousarray(radius, dtype=np.float64)
        out = np.empty(self.map_util_.map.size, dtype=np.uint8)
        abi.check(self._lib.mplx_set_search_region_path(self._h, path.ctypes.data, len(path), rad.ctypes.data,
                                                        1 if dense else 0, out.ctypes.data))
        return out

    def set_batch_regions(self, paths, radius, dense=False):
        """One tunnel per query of the following plan_batch* calls (mplx_set_batch_regions): query q searches inside
        set_search_region_path(paths[q], radius, dense)'s region, in place of the env-wide one, and those calls must
        then have len(paths) queries.  Each path is points x Dim; an empty list clears the tunnels.  upload_map()
        drops them, update_cells() keeps them."""
        if len(paths) == 0:
            abi.check(self._lib.mplx_set_batch_regions(self._h, 0, None, None, None, 0))
            return
        pts = [np.ascontiguousarray(p, dtype=np.float64).reshape(-1, self.Dim) for p in paths]
        off = np.zeros(len(pts) + 1, np.int64)
        off[1:] = np.cumsum([len(p) for p in pts])
        flat = np.ascontiguousarray(np.concatenate(pts) if off[-1] else np.zeros((1, self.Dim)))
        rad = np.ascontiguousarray(radius, dtype=np.float64)
        abi.check(self._lib.mplx_set_batch_regions(self._h, len(pts), off.ctypes.data, flat.ctypes.data,
                                                   rad.ctypes.data, 1 if dense else 0))

    def set_batch_regions_recorded(self, from_, radius, dense=False, paths=None):
        """set_batch_regions from the paths the last plan_batch* call recorded (trajectories=True), traced on the
        device (mplx_set_batch_regions_recorded): query j's tunnel is built from the recorded path of query from_[j]
        of that call when from_[j] >= 0 (the positions of batch_trajectories()[from_[j]]["nodes"]), else from
        paths[j] (points x Dim; paths may be None when every from_[j] >= 0).  Read the recorded paths before the
        next plan_batch* call replaces them."""
        fr = np.ascontiguousarray(from_, dtype=np.int32).reshape(-1)
        rad = np.ascontiguousarray(radius, dtype=np.float64)
        off = flat = None
        if paths is not None:
            pts = [np.ascontiguousarray(p, dtype=np.float64).reshape(-1, self.Dim) for p in paths]
            if len(pts) != fr.size:
                raise ValueError("paths must hold one entry per query")
            off = np.zeros(len(pts) + 1, np.int64)
            off[1:] = np.cumsum([len(p) for p in pts])
            flat = np.ascontiguousarray(np.concatenate(pts) if off[-1] else np.zeros((1, self.Dim)))
        abi.check(self._lib.mplx_set_batch_regions_recorded(self._h, fr.size, fr.ctypes.data, abi.ptr(off),
                                                            abi.ptr(flat), rad.ctypes.data, 1 if dense else 0))

    def batch_regions_info(self):
        """The tunnels set_batch_regions installed: dict(n_q, n_bricks, bytes) (n_q = 0: none)."""
        n, b, by = C.c_int32(), C.c_int64(), C.c_int64()
        abi.check(self._lib.mplx_batch_regions_info(self._h, C.byref(n), C.byref(b), C.byref(by)))
        return dict(n_q=n.value, n_bricks=b.value, bytes=by.value)

    def read_batch_region(self, q):
        """Query q's tunnel as one byte per voxel, set_search_region_path's layout (mplx_read_batch_region)."""
        out = np.empty(self.map_util_.map.size, dtype=np.uint8)
        abi.check(self._lib.mplx_read_batch_region(self._h, int(q), out.ctypes.data))
        return out

    def _sync_params(self):
        if not self._dirty:
            return
        if self.U_ is None or self.control is None:
            raise RuntimeError("set_u() and set_control() must be called before get_succ()")
        abi.check(
            self._lib.mplx_set_params(
                self._h, self.control, self.dt_, self.w_, self.wyaw_, self.v_max_, self.a_max_, self.j_max_,
                self.yaw_max_, self.U_.ctypes.data, self.U_.shape[0], self.U_.shape[1],
            )
        )
        self._dirty = False

    def _sync_limits(self):
        """The device parameters for calls that read only the limits (mplx_traj_check): the env's own once set_u and
        set_control were called; before that, the limits with a stand-in control set of one zero VEL input.  The
        stand-in leaves the env marked unsynced, so the next expand sends the real U and control (or refuses without
        them, as before)."""
        if self.U_ is not None and self.control is not None:
            self._sync_params()
            return
        u = np.zeros((1, self.Dim))
        abi.check(self._lib.mplx_set_params(self._h, abi.VEL, self.dt_, self.w_, self.wyaw_, self.v_max_, self.a_max_,
                                            self.j_max_, self.yaw_max_, u.ctypes.data, 1, self.Dim))
        self._dirty = True

    # -- the hot path -----------------------------------------------------------------------
    def expand(self, nodes: np.ndarray, want=("succ", "cost", "action", "key"), pinned: bool = False) -> Expansion:
        """Batched env_map::get_succ through mplx_expand (HOST buffers)."""
        self._sync_params()
        nodes = np.ascontiguousarray(nodes, dtype=WAYPOINT_DTYPE).reshape(-1)
        n, nU = nodes.size, self.U_.shape[0]
        alloc = self._pinned_empty if pinned else (lambda shape, dt: np.empty(shape, dtype=dt))
        count = alloc(n, np.int32)
        succ = alloc(n * nU, WAYPOINT_DTYPE) if "succ" in want else None
        cost = alloc(n * nU, np.float64) if "cost" in want else None
        action = alloc(n * nU, np.int32) if "action" in want else None
        key = alloc(n * nU, np.uint64) if "key" in want else None
        lattice = alloc((n * nU, LATTICE_MAX), np.int32) if "lattice" in want else None
        out = SuccOut(abi.ptr(count), abi.ptr(succ), abi.ptr(cost), abi.ptr(action), abi.ptr(key), abi.ptr(lattice))
        abi.check(self._lib.mplx_expand(self._h, nodes.ctypes.data, n, C.byref(out)))
        return Expansion(nU, count, succ, cost, action, key, lattice)

    def expand_packed(self, nodes: np.ndarray, drop_inf: bool = False, pinned: bool = True, buffers=None):
        """mplx_expand_packed: dense {state, cost, action, key} records (see include/mplx.h).
        Returns a dict with count, offset, state[total, nstate], cost, action, key, total."""
        self._sync_params()
        nodes = np.ascontiguousarray(nodes, dtype=WAYPOINT_DTYPE).reshape(-1)
        n, nU = nodes.size, self.U_.shape[0]
        nstate = self.Dim * bin(self.control & 15).count("1") + (1 if self.control & 16 else 0)
        cap = n * nU
        if buffers is None:
            alloc = self._pinned_empty if pinned else (lambda shape, dt: np.empty(shape, dtype=dt))
            buffers = dict(count=alloc(n, np.int32), offset=alloc(n, np.int64), state=alloc(cap * nstate, np.float64),
                           cost=alloc(cap, np.float64), action=alloc(cap, np.uint16), key=alloc(cap, np.uint64))
        b = buffers
        out = PackedOut(abi.ptr(b["count"]), abi.ptr(b["offset"]), abi.ptr(b.get("state")), abi.ptr(b.get("cost")),
                        abi.ptr(b.get("action")), abi.ptr(b.get("key")), cap, 0, 0)
        abi.check(self._lib.mplx_expand_packed(self._h, nodes.ctypes.data, n, abi.PACK_DROP_INF if drop_inf else 0,
                                               C.byref(out)))
        tot = int(out.total)
        return dict(count=b["count"], offset=b["offset"], total=tot, nstate=int(out.nstate),
                    state=None if b.get("state") is None else b["state"][: tot * out.nstate].reshape(tot, out.nstate),
                    cost=None if b.get("cost") is None else b["cost"][:tot],
                    action=None if b.get("action") is None else b["action"][:tot],
                    key=None if b.get("key") is None else b["key"][:tot], buffers=b)

    def _pinned_empty(self, shape, dt):
        dt = np.dtype(dt)
        n = int(np.prod(shape)) if not isinstance(shape, int) else shape
        p = self._lib.mplx_host_alloc(max(1, n * dt.itemsize))
        if not p:
            raise MemoryError(self._lib.mplx_last_error().decode())
        buf = (C.c_char * (n * dt.itemsize)).from_address(p)
        arr = np.frombuffer(buf, dtype=dt, count=n).reshape(shape)
        self._pins = getattr(self, "_pins", [])
        self._pins.append(p)
        return arr

    def get_succ(self, curr):
        """env_map::get_succ(curr, succ, succ_cost, action_idx) for one node (env_map.h:147-172)."""
        node = np.zeros(1, dtype=WAYPOINT_DTYPE)
        node[0] = curr
        e = self.expand(node)
        return e.node(0)

    def is_free_edges(self, parents: np.ndarray, actions: np.ndarray):
        """env_map::is_free(pr) (env_map.h:60-76) for the stored edges pr = Primitive(parents[i],
        U[actions[i]], dt), batched on the device.  Returns (free uint8[n], intrinsic cost[n]);
        the cost is what StateSpace::decreaseCost installs for a re-opened edge (state_space.h:243)."""
        self._sync_params()
        parents = np.ascontiguousarray(parents, dtype=WAYPOINT_DTYPE).reshape(-1)
        actions = np.ascontiguousarray(actions, dtype=np.int32).reshape(-1)
        if actions.size != parents.size:
            raise ValueError("one action id per parent state")
        free = np.zeros(parents.size, dtype=np.uint8)
        cost = np.zeros(parents.size, dtype=np.float64)
        abi.check(self._lib.mplx_edges_is_free(self._h, parents.ctypes.data, actions.ctypes.data, parents.size,
                                               free.ctypes.data, cost.ctypes.data))
        return free, cost

    def traverse_trajectories(self, results, control, scaled=None, segments=True):
        """Checks trajectories against this env on the device (mplx_traj_check): per path the cost of
        env_map::traverse_trajectory (+inf when the trajectory leaves the map or hits an obstacle) and, with
        `segments`, env_map::is_free and validate_primitive(v_max, a_max, j_max, yaw_max) of every segment.
        results: dicts with `seg_t` and `coeff`, as TrajSolverBatch.solve returns them; control: the segments'
        control flag (a TrajSolver segment carries its first waypoint's), one for all paths or one per path;
        scaled: None, or TrajSolverBatch.scale's results for the same paths (with_lambda=True), whose time
        scaling then applies.  The checks read the map, the potential field, the search region and the limits;
        set_u and set_control are not needed (see _sync_limits).  Returns (results,
        seconds): one dict per path with `status` (1: cost evaluated; 0: not — fewer than 2 waypoints, a bad
        segment time or coefficient, or N = ceil(v_max * total / res) outside [1, 2^20]), `cost` and, with
        segments, `seg_free` and `seg_valid` (uint8 per segment); seconds is the device time of the kernels."""
        self._sync_limits()
        n_paths = len(results)
        if scaled is not None and len(scaled) != n_paths:
            raise ValueError("one scaled result per path")
        n, offset, seg_t, coeff = pack_paths(results, self.Dim)
        ctl = np.ascontiguousarray(np.broadcast_to(np.asarray(control, dtype=np.uint8), (n_paths,)))
        total_t = n_lambda = lam = None
        if scaled is not None:
            total_t, n_lambda, lam = pack_lambda(scaled, offset, self.Dim)
        status = np.zeros(max(n_paths, 1), dtype=np.int32)
        cost = np.zeros(max(n_paths, 1))
        free = np.zeros(seg_t.size, dtype=np.uint8) if segments else None
        valid = np.zeros(seg_t.size, dtype=np.uint8) if segments else None
        out = abi.TrajCheckOut(status.ctypes.data, cost.ctypes.data, abi.ptr(free), abi.ptr(valid), 0.0)
        abi.check(self._lib.mplx_traj_check(self._h, n_paths, offset.ctypes.data, seg_t.ctypes.data,
                                            coeff.ctypes.data, ctl.ctypes.data if n_paths else None, abi.ptr(total_t),
                                            abi.ptr(n_lambda), abi.ptr(lam), C.byref(out)))
        res = []
        for p in range(n_paths):
            r = dict(status=int(status[p]), cost=float(cost[p]))
            if segments:
                s = max(int(n[p]) - 1, 0)
                r["seg_free"] = free[offset[p]:offset[p] + s].copy()
                r["seg_valid"] = valid[offset[p]:offset[p] + s].copy()
            res.append(r)
        return res, out.seconds

    def edge_cells(self, parents: np.ndarray, actions: np.ndarray, table: bool = False):
        """The voxel walk of MapPlanner::getLinkedNodes (map_planner.cpp:135-151) for stored edges:
        returns (offset int64[n+1], cells int32[total, Dim]); edge i passes through
        cells[offset[i]:offset[i+1]] (consecutive repeats removed).  With table=True also the
        inverted voxel -> edges table (the reference's lhm_) as (voxel int32[total], edge int32[total]),
        sorted by voxel index, edges of one voxel in emission order."""
        self._sync_params()
        parents = np.ascontiguousarray(parents, dtype=WAYPOINT_DTYPE).reshape(-1)
        actions = np.ascontiguousarray(actions, dtype=np.int32).reshape(-1)
        if actions.size != parents.size:
            raise ValueError("one action id per parent state")
        n = parents.size
        off = np.zeros(n + 1, dtype=np.int64)
        total = C.c_int64(0)
        cap = max(1, 8 * n)
        for _ in range(2):
            cells = np.zeros((cap, self.Dim), dtype=np.int32)
            tv = np.zeros(cap, dtype=np.int32) if table else None
            te = np.zeros(cap, dtype=np.int32) if table else None
            rc = self._lib.mplx_edges_cells(self._h, parents.ctypes.data, actions.ctypes.data, n, off.ctypes.data,
                                            cells.ctypes.data, cap, C.byref(total), abi.ptr(tv), abi.ptr(te))
            if rc == 0:
                t = total.value
                return (off, cells[:t], tv[:t], te[:t]) if table else (off, cells[:t])
            if total.value <= cap:
                abi.check(rc)
            cap = int(total.value)
        abi.check(rc)

    def plan_batch(self, starts, goals, eps=1.0, max_expand=1000, tol_pos=0.5, tol_vel=-1.0, tol_acc=-1.0,
                   tol_yaw=-1.0, start_free=None, closed=True, trajectories=False, n_samples=0, traj_room_bytes=0):
        """mplx_plan_batch: the A* searches of n (start, goal) queries on the device (occupancy planning;
        plan_batch_cost_terms serves potential-field and yaw planning).  Returns a dict: valid, cost, expanded,
        n_closed (arrays), actions / closed (one array per query), slots, arena_bytes, seconds.  Raises
        MplxError (code MPLX_ERR_ARG) for the plans it refuses.

        trajectories=True records the searches' trajectories (mplx_set_batch_trajectories; traj_room_bytes > 0
        sizes the device room, a diagnostic) and adds `trajectories`, one dict per query (see _trajectories), and
        `traj_seconds`, the device time of mplx_plan_batch_trajectories."""
        return self._plan_batch(self._lib.mplx_plan_batch, starts, goals, eps, max_expand, tol_pos, tol_vel, tol_acc,
                                tol_yaw, start_free, closed, trajectories, n_samples, traj_room_bytes)

    def plan_batch_cost_terms(self, starts, goals, eps=1.0, max_expand=1000, tol_pos=0.5, tol_vel=-1.0, tol_acc=-1.0,
                              tol_yaw=-1.0, start_free=None, closed=True, trajectories=False, n_samples=0,
                              traj_room_bytes=0):
        """mplx_plan_batch_cost_terms: plan_batch for every plan, including a potential map (with or without a
        gradient weight), a yaw control and a search region; the sample loop sums the potential, gradient and
        yaw-alignment terms.  tol_yaw >= 0 adds |yaw - goal yaw| <= tol_yaw to the goal test.  Same results dict;
        raises MplxError for max_expand <= 0, more than 256 primitives, a missing map or parameters
        (MPLX_ERR_ARG) and search memory beyond the budget (MPLX_ERR_ALLOC).  trajectories, n_samples and
        traj_room_bytes as plan_batch."""
        return self._plan_batch(self._lib.mplx_plan_batch_cost_terms, starts, goals, eps, max_expand, tol_pos, tol_vel,
                                tol_acc, tol_yaw, start_free, closed, trajectories, n_samples, traj_room_bytes)

    def plan_batch_grow(self, starts, goals, eps=1.0, max_expand=-1, tol_pos=0.5, tol_vel=-1.0, tol_acc=-1.0,
                        tol_yaw=-1.0, start_free=None, closed=True, cost_terms=False, first_cap=0, max_cap=0,
                        pool_bytes=0, trajectories=False, n_samples=0, traj_room_bytes=0):
        """mplx_plan_batch_grow: plan_batch (cost_terms=False) or plan_batch_cost_terms (cost_terms=True) with
        arenas sized for the batch and grown for the queries that outgrow them, so max_expand <= 0 (unbounded)
        is served too.  first_cap / max_cap / pool_bytes: 0 = automatic (include/mplx.h has the round schedule).
        Returns plan_batch's dict plus searched (0: the query needed more than the largest arena; its fields are
        0 / +inf and its lists empty), rounds, reruns, first_cap and last_cap.  trajectories, n_samples and
        traj_room_bytes as plan_batch (a query with searched 0 has no trajectory)."""
        self._sync_params()
        self._record(trajectories, traj_room_bytes)
        starts = np.ascontiguousarray(starts, dtype=WAYPOINT_DTYPE).reshape(-1)
        goals = np.ascontiguousarray(goals, dtype=WAYPOINT_DTYPE).reshape(-1)
        n = starts.size
        valid, expanded, n_closed, n_actions, searched = (np.zeros(n, np.int32) for _ in range(5))
        cost = np.zeros(n)
        sf = None if start_free is None else np.ascontiguousarray(start_free, dtype=np.uint8)
        out = abi.GrowOut(valid.ctypes.data, cost.ctypes.data, expanded.ctypes.data, n_closed.ctypes.data,
                          n_actions.ctypes.data, searched.ctypes.data, 0, 0, 0, 0, 0, 0, 0.0)
        abi.check(self._lib.mplx_plan_batch_grow(
            self._h, 1 if cost_terms else 0, starts.ctypes.data, goals.ctypes.data, abi.ptr(sf), n, float(eps),
            int(max_expand), float(tol_pos), float(tol_vel), float(tol_acc), float(tol_yaw), 1 if closed else 0,
            int(first_cap), int(max_cap), int(pool_bytes), C.byref(out)))
        self._last_nq = n
        na, nc = int(n_actions.sum()), int(n_closed.sum()) if closed else 0
        aoff, coff = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
        acts, keys = np.zeros(max(na, 1), np.int32), np.zeros(max(nc, 1), np.uint64)
        abi.check(self._lib.mplx_plan_batch_grow_results(self._h, aoff.ctypes.data, acts.ctypes.data, acts.size,
                                                         coff.ctypes.data, keys.ctypes.data if closed else None,
                                                         keys.size))
        return self._batch_result(valid, cost, expanded, n_closed, aoff, acts, coff, keys if closed else None,
                                  trajectories, n_samples, searched=searched, slots=int(out.slots),
                                  arena_bytes=int(out.arena_bytes), seconds=float(out.seconds),
                                  rounds=int(out.rounds), reruns=int(out.reruns), first_cap=int(out.first_cap),
                                  last_cap=int(out.last_cap))

    def _record(self, trajectories, traj_room_bytes):
        abi.check(self._lib.mplx_set_batch_trajectories(self._h, 1 if trajectories else 0, int(traj_room_bytes)))

    def batch_trajectories(self, n_samples=0, capacity=1):
        """mplx_plan_batch_trajectories: the trajectories of the last plan_batch* call, which ran with
        trajectories=True.  Returns (one dict per query, device seconds).  A dict holds `nodes` (WAYPOINT_DTYPE,
        the stored coordinates of the path's states from start to goal; their positions are a path for
        TrajSolverBatch.solve), `seg_t` (one T per segment), `coeff` (segments x (Dim+1) x 6: Primitive
        coefficients, axes then yaw) and, with n_samples > 0, `samples` (Trajectory::sample(n_samples) rows
        {pos, vel, acc, jrk, yaw, yaw_dot, t}).  A query without a trajectory has no nodes and no segments.  The
        dicts go as they are into traverse_trajectories and TrajSolverBatch.scale.  capacity: the waypoint slots
        to try first (a query with n > 0 actions takes n + 1)."""
        dim = self.Dim
        n_q = self._last_nq
        offset = np.zeros(n_q + 1, np.int64)
        samples = np.zeros((n_q, n_samples + 1, 4 * dim + 3)) if n_samples > 0 else None
        cap = max(int(capacity), 1)
        for _ in range(2):  # the first call reports the slots needed when cap is too small
            nodes = np.zeros(cap, dtype=WAYPOINT_DTYPE)
            seg_t = np.zeros(cap)
            coeff = np.zeros((cap, dim + 1, 6))
            out = abi.BatchTrajOut(offset.ctypes.data, nodes.ctypes.data, seg_t.ctypes.data, coeff.ctypes.data,
                                   abi.ptr(samples), cap, 0, 0.0)
            rc = self._lib.mplx_plan_batch_trajectories(self._h, int(n_samples), C.byref(out))
            if rc == 0 or out.total <= cap:
                break
            cap = int(out.total)
        abi.check(rc)
        return split_slots(offset, nodes, seg_t, coeff, samples), float(out.seconds)

    def _plan_batch(self, fn, starts, goals, eps, max_expand, tol_pos, tol_vel, tol_acc, tol_yaw, start_free, closed,
                    trajectories=False, n_samples=0, traj_room_bytes=0):
        self._sync_params()
        self._record(trajectories, traj_room_bytes)
        starts = np.ascontiguousarray(starts, dtype=WAYPOINT_DTYPE).reshape(-1)
        goals = np.ascontiguousarray(goals, dtype=WAYPOINT_DTYPE).reshape(-1)
        n = starts.size
        cap = max(1, n * max(int(max_expand), 0))
        valid, expanded, n_closed = (np.zeros(n, np.int32) for _ in range(3))
        cost = np.zeros(n)
        aoff, coff = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
        acts = np.zeros(cap, np.int32)
        keys = np.zeros(cap, np.uint64) if closed else None
        sf = None if start_free is None else np.ascontiguousarray(start_free, dtype=np.uint8)
        out = abi.BatchOut(valid.ctypes.data, cost.ctypes.data, expanded.ctypes.data, n_closed.ctypes.data,
                           aoff.ctypes.data, acts.ctypes.data, cap, coff.ctypes.data, abi.ptr(keys), cap if closed else 0,
                           0, 0, 0.0)
        abi.check(fn(self._h, starts.ctypes.data, goals.ctypes.data, abi.ptr(sf), n, float(eps), int(max_expand),
                     float(tol_pos), float(tol_vel), float(tol_acc), float(tol_yaw), C.byref(out)))
        self._last_nq = n
        return self._batch_result(valid, cost, expanded, n_closed, aoff, acts, coff, keys, trajectories, n_samples,
                                  slots=int(out.slots), arena_bytes=int(out.arena_bytes), seconds=float(out.seconds))

    def _batch_result(self, valid, cost, expanded, n_closed, aoff, acts, coff, keys, trajectories, n_samples,
                      **extra):
        """The results dict of the plan_batch* calls: the per-query arrays, the actions and closed lists (keys None:
        closed None), the call's own fields (extra) and, with trajectories, `trajectories` and `traj_seconds`."""
        n = valid.size
        res = dict(valid=valid, cost=cost, expanded=expanded, n_closed=n_closed,
                   actions=[acts[aoff[q]:aoff[q + 1]].copy() for q in range(n)],
                   closed=None if keys is None else [keys[coff[q]:coff[q + 1]].copy() for q in range(n)], **extra)
        if trajectories:
            res["trajectories"], res["traj_seconds"] = self.batch_trajectories(
                n_samples, sum(len(a) + 1 for a in res["actions"] if len(a)))
        return res

    def set_kernel(self, which: int):
        """0 = auto, 1 = literal sequential loop, 2 = register kernel, 3 = flat kernel, 4 = dealing kernel."""
        abi.check(self._lib.mplx_set_kernel(self._h, int(which)))

    def enable_stats(self, on=True):
        abi.check(self._lib.mplx_enable_stats(self._h, 1 if on else 0))

    def last_stats(self):
        a, b = C.c_int64(), C.c_int64()
        abi.check(self._lib.mplx_last_stats(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def launch_count(self) -> int:
        return int(self._lib.mplx_launch_count(self._h))
