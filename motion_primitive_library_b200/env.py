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
