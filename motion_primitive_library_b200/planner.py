"""ctypes binding of libmpl_host.so: the C++ host planner (MPL::MapPlanner with the GPU env,
MPL::MultiQueryPlanner) behind flat C structs.  See host/plan_capi.hpp."""
import ctypes as C
import functools
from pathlib import Path

import numpy as np

from .traj import split_slots

PKG =Path(__file__).resolve().parent
LIB = PKG / "lib" / "libmpl_host.so"

class Waypoint(C.Structure):
    _fields_ = [("pos", C.c_double * 3), ("vel", C.c_double * 3), ("acc", C.c_double * 3), ("jrk", C.c_double * 3),
                ("yaw", C.c_double), ("t", C.c_double)]


class PlanArgs(C.Structure):
    _fields_ = [
        ("dim", C.c_int32), ("control", C.c_int32), ("map", C.c_void_p), ("mdim", C.c_int32 * 3),
        ("origin", C.c_double * 3), ("res", C.c_double), ("U", C.c_void_p), ("nU", C.c_int32), ("udim", C.c_int32),
        ("T", C.c_double), ("w", C.c_double), ("wyaw", C.c_double), ("eps", C.c_double),
        ("v_max", C.c_double), ("a_max", C.c_double), ("j_max", C.c_double), ("yaw_max", C.c_double),
        ("tol_pos", C.c_double), ("tol_vel", C.c_double), ("tol_acc", C.c_double),
        ("start", Waypoint), ("goal", Waypoint), ("max_num", C.c_int32), ("speculate", C.c_int32),
        ("device", C.c_int32), ("potential", C.c_void_p), ("potential_weight", C.c_double),
        ("gradient_weight", C.c_double), ("heur_ignore_dynamics", C.c_int32),
    ]


class PlanResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("cost", C.c_double), ("expanded", C.c_int32), ("n_closed", C.c_int32),
                ("n_open", C.c_int32), ("n_actions", C.c_int32), ("gpu_nodes", C.c_int64), ("gpu_calls", C.c_int64),
                ("gpu_launches", C.c_int64), ("seconds", C.c_double)]


class QueryResult(C.Structure):
    _fields_ = [("valid", C.c_int32), ("cost", C.c_double), ("expanded", C.c_int32), ("n_closed", C.c_int32),
                ("n_actions", C.c_int32)]


class LpaStep(C.Structure):
    _fields_ = [("op", C.c_int32), ("n", C.c_int32), ("cells", C.c_void_p)]


class LpaOut(C.Structure):
    _fields_ = [("valid", C.c_int32), ("cost", C.c_double), ("expanded", C.c_int32), ("n_actions", C.c_int32),
                ("n_states", C.c_int32), ("n_closed", C.c_int32), ("n_open", C.c_int32), ("state_hash", C.c_uint64),
                ("n_linked", C.c_int64), ("linked_hash", C.c_uint64), ("seconds", C.c_double)]


OP_PLAN, OP_LINK, OP_BLOCK, OP_CLEAR, OP_SUBTREE = range(5)

WAYPOINT_DTYPE = np.dtype(
    [("pos", "<f8", 3), ("vel", "<f8", 3), ("acc", "<f8", 3), ("jrk", "<f8", 3), ("yaw", "<f8"), ("t", "<f8")]
)


_vp, _i, _i64, _d = C.c_void_p, C.c_int, C.c_int64, C.c_double
_i32p, _i64p, _argp, _resp = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(PlanArgs), C.POINTER(PlanResult)
# (argtypes, restype) of every function libmpl_host.so exports (host/mpl_host_capi.cpp)
SIGNATURES = {
    "mplh_last_error": ([], C.c_char_p),
    "mplh_plan": ([_argp, _resp, _vp, _i, _vp, _i], _i),
    "mplh_plan_trace": ([_argp, _resp, _vp, _i, _i32p], _i),
    "mplh_plan_trajectory": ([_argp, _i, _resp, _vp, _vp, _vp, _i, _i32p, _vp], _i),
    "mplh_iterative_plan": ([_argp, _vp, _i, _resp, _resp, _vp, _vp, _i, _vp, _i], _i),
    "mplh_lpa_run": ([_argp, C.POINTER(LpaStep), _i, C.POINTER(LpaOut), _vp, _i], _i),
    "mplh_batch_open": ([_argp], _vp),
    "mplh_batch_plan": ([_vp, _vp, _vp, _i, _d, _i, _vp, _vp], _i),
    "mplh_batch_plan_keep": ([_vp, _vp, _vp, _i, _d, _i, _i, _vp, _vp], _i),
    "mplh_batch_kept": ([_vp, _vp, _vp, _i64, _vp, _vp, _i64], _i),
    "mplh_batch_update_cells": ([_vp, _vp, _vp, _i], _i),
    "mplh_batch_map_uploads": ([_vp, _i64p, _i64p], _i),
    "mplh_batch_set_path": ([_vp, _i], _i),
    "mplh_batch_set_grow_caps": ([_vp, _i64, _i64], _i),
    "mplh_batch_grow_stats": ([_vp, _i32p, _i64p, _i64p, _i64p, _i32p], _i),
    "mplh_batch_last_path": ([_vp, _i32p, _i32p, _i64p], _i),
    "mplh_batch_close": ([_vp, C.POINTER(_d)], _i),
    "mplh_batch_set_trajectories": ([_vp, _i], _i),
    "mplh_batch_set_regions": ([_vp, _i, _vp, _vp, _vp, _i], _i),
    "mplh_batch_iterative_plan": ([_vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _d, _i, _vp, _vp], _i),
    "mplh_batch_trajectories": ([_vp, _i, _vp, _vp, _vp, _vp, _vp, _i64, _i64p], _i),
    "mplh_traj_solve": ([_i, _i, _i, _vp, _vp, _i, _vp, _d, _i, _i32p, _vp, _vp, _vp, _vp], _i),
    "mplh_traj_sample": ([_i, _i, _vp, _vp, _i, _i, _vp, _vp], _i),
    "mplh_traj_scale": ([_i, _i, _vp, _vp, _i, _i, _d, _d, _d, _i, _i32p, C.POINTER(_d), _vp, _i32p, _vp, _vp], _i),
    "mplh_solve": ([_d] * 5 + [_i32p, _vp], _i),
    "mplh_traj_check": ([_i, _vp, _vp, _vp, _d, _vp, _d, _d, _vp, _d, _d, _d, _d, _i, _vp, _vp, _vp, _vp, _vp, _vp,
                         _vp, _i, _vp, _vp, _vp, _vp], _i),
}
# the reference's mplh_traj_scale, with a trailing per-row flags array
SIGNATURES["reft_traj_scale"] = (SIGNATURES["mplh_traj_scale"][0] + [_vp], _i)


@functools.cache
def _lib():
    """libmpl_host.so, opened once, with every function declared from SIGNATURES."""
    if not LIB.exists():
        raise ImportError(f"{LIB} not built (python -c 'import __graft_entry__ as g; g.build()')")
    lib = C.CDLL(str(LIB))
    for name, (argtypes, restype) in SIGNATURES.items():
        if name.startswith("mplh_"):
            f = getattr(lib, name)
            f.argtypes, f.restype = argtypes, restype
    return lib


def _host():
    """(libmpl_host.so, its mplh_plan), the pair callers of earlier versions unpack."""
    lib = _lib()
    return lib, lib.mplh_plan


def bind(path, name, like=None):
    """(lib, fn): the function `name` of the shared library at `path`, declared with the signature of `like`
    (default `name`) in SIGNATURES: a driver function that mirrors an mplh_* entry point."""
    lib = C.CDLL(str(path))
    fn = getattr(lib, name)
    fn.argtypes, fn.restype = SIGNATURES[like or name]
    return lib, fn


# the loaders of earlier versions, kept as public names: bind() with the mirrored entry point fixed
load_fn = functools.partial(bind, like="mplh_plan")
load_lpa_fn = functools.partial(bind, like="mplh_lpa_run")
load_traj_fn = functools.partial(bind, like="mplh_plan_trajectory")
load_iter_fn = functools.partial(bind, like="mplh_iterative_plan")
load_traj_solve_fn = functools.partial(bind, like="mplh_traj_solve")
load_solve_fn = functools.partial(bind, like="mplh_solve")
load_traj_check_fn = functools.partial(bind, like="mplh_traj_check")


def load_traj_scale_fn(path, fn, flags=False):
    """bind() with mplh_traj_scale's signature, plus the reference driver's trailing per-row flags when `flags`."""
    return bind(path, fn, "reft_traj_scale" if flags else "mplh_traj_scale")


def _check(lib, rc):
    """Raise RuntimeError with lib's mplh_last_error() when rc is nonzero."""
    if rc != 0:
        err = getattr(lib, "mplh_last_error", None)
        if err is None:
            raise RuntimeError(f"call failed rc={rc}")
        err.restype = C.c_char_p
        raise RuntimeError(err().decode())


def make_args(dim, control, grid, mdim, origin, res, U, start, goal, T=1.0, w=10.0, wyaw=1.0, eps=1.0, v_max=-1.0,
              a_max=-1.0, j_max=-1.0, yaw_max=-1.0, tol_pos=0.5, tol_vel=-1.0, tol_acc=-1.0, max_num=-1, speculate=0,
              potential=None, potential_weight=0.1, gradient_weight=0.0, heur_ignore_dynamics=True):
    keep = dict(grid=np.ascontiguousarray(grid, dtype=np.int8), U=np.ascontiguousarray(U, dtype=np.float64))
    a = PlanArgs()
    a.dim, a.control = dim, control
    a.map = keep["grid"].ctypes.data
    for k in range(3):
        a.mdim[k] = int(mdim[k]) if k < dim else 1
        a.origin[k] = float(origin[k]) if k < dim else 0.0
    a.res = res
    a.U = keep["U"].ctypes.data
    a.nU, a.udim = keep["U"].shape
    a.T, a.w, a.wyaw, a.eps = T, w, wyaw, eps
    a.v_max, a.a_max, a.j_max, a.yaw_max = v_max, a_max, j_max, yaw_max
    a.tol_pos, a.tol_vel, a.tol_acc = tol_pos, tol_vel, tol_acc
    for name, src in (("start", start), ("goal", goal)):
        w_ = getattr(a, name)
        for f in ("pos", "vel", "acc", "jrk"):
            v = src.get(f, ())
            for k in range(len(v)):
                getattr(w_, f)[k] = float(v[k])
        w_.yaw = float(src.get("yaw", 0.0))
    a.max_num, a.speculate, a.device = max_num, speculate, 0
    if potential is not None:
        keep["pot"] = np.ascontiguousarray(potential, dtype=np.int8)
        a.potential = keep["pot"].ctypes.data
    a.potential_weight, a.gradient_weight = potential_weight, gradient_weight
    a.heur_ignore_dynamics = 1 if heur_ignore_dynamics else 0
    a._keep = keep
    return a


def run_plan(fn, lib, args, cap=1 << 21):
    r = PlanResult()
    closed = np.zeros(cap, dtype=np.uint64)
    actions = np.zeros(65536, dtype=np.int32)
    _check(lib, fn(C.byref(args), C.byref(r), closed.ctypes.data, cap, actions.ctypes.data, actions.size))
    out = {k: getattr(r, k) for k, _ in PlanResult._fields_}
    out["closed"] = closed[: min(r.n_closed, cap)].copy()
    out["actions"] = actions[: r.n_actions].copy()
    return out


def run_lpa(fn, lib, args, script, cap_actions=4096):
    """Run a scripted LPA* session.  script: list of ("plan",), ("link",), ("block", cells[n, dim]),
    ("clear", cells[n, dim]), ("subtree", k).  Returns one dict per step (fields of mplh_lpa_out, plus
    the action ids of the trajectory for plan steps)."""
    ops = dict(plan=OP_PLAN, link=OP_LINK, block=OP_BLOCK, clear=OP_CLEAR, subtree=OP_SUBTREE)
    steps = (LpaStep * len(script))()
    keep = []
    for k, st in enumerate(script):
        steps[k].op = ops[st[0]]
        if st[0] in ("block", "clear"):
            cells = np.ascontiguousarray(st[1], dtype=np.int32).reshape(-1, args.dim)
            keep.append(cells)
            steps[k].n = len(cells)
            steps[k].cells = cells.ctypes.data
        elif st[0] == "subtree":
            steps[k].n = int(st[1])
    outs = (LpaOut * len(script))()
    actions = np.full((len(script), cap_actions), -1, dtype=np.int32)
    _check(lib, fn(C.byref(args), steps, len(script), outs, actions.ctypes.data, cap_actions))
    res = []
    for k in range(len(script)):
        d = {name: getattr(outs[k], name) for name, _ in LpaOut._fields_}
        d["op"] = script[k][0]
        d["actions"] = actions[k, : min(d["n_actions"], cap_actions)].copy()
        res.append(d)
    return res


def lpa_session(args, script):
    """MPL::MapPlanner with setLPAstar(true) and the GPU env: plan / getLinkedNodes / updateBlockedNodes /
    updateClearedNodes / getSubStateSpace as scripted; expansion, the linked-voxel walk and the
    is_free(pr) re-validation run on the device."""
    lib = _lib()
    return run_lpa(lib.mplh_lpa_run, lib, args, script)


def run_trajectory(fn, lib, args, n_samples=50, cap_wp=4096):
    """plan(), then the recovered Trajectory (trajectory.h): dict with `commands` = sample(N) rows
    {pos, vel, acc, jrk, yaw, yaw_dot, t}, `total_time`, `J`, `Jyaw`, `segments`, `waypoints` =
    getWaypoints() rows {pos, vel, acc, jrk, yaw, t} and `evaluated` = evaluate(t) at the sample times."""
    dim = args.dim
    r = PlanResult()
    samples = np.zeros((n_samples + 1, 4 * dim + 3))
    totals = np.zeros(4)
    wps = np.zeros((cap_wp, 4 * dim + 2))
    mids = np.zeros((n_samples + 1, 4 * dim + 2))
    n_wp = C.c_int32(0)
    _check(lib, fn(C.byref(args), n_samples, C.byref(r), samples.ctypes.data, totals.ctypes.data, wps.ctypes.data,
                   cap_wp, C.byref(n_wp), mids.ctypes.data))
    out = {k: getattr(r, k) for k, _ in PlanResult._fields_}
    out.update(commands=samples, total_time=totals[0], J=totals[1], Jyaw=totals[2], segments=int(totals[3]),
               waypoints=wps[: min(n_wp.value, cap_wp)].copy(), evaluated=mids)
    return out


def plan_trajectory(args, n_samples=50):
    """MPL::MapPlanner::plan() with the GPU env + the recovered Trajectory (sample / waypoints / efforts)."""
    lib = _lib()
    return run_trajectory(lib.mplh_plan_trajectory, lib, args, n_samples)


def run_iterative(fn, lib, args, search_radius, max_iter=3, cap=1 << 21):
    """plan() followed by MapPlanner::iterativePlan() from that trajectory.  Returns (first, last):
    dicts of the plan-result fields; `last` also has closed keys, action ids, `iterations` (plan() calls
    iterativePlan made; 0 when the driver cannot know) and `ok` (its return value)."""
    first, last = PlanResult(), PlanResult()
    info = np.zeros(2, dtype=np.int32)
    rad = np.zeros(3)
    rad[: len(search_radius)] = search_radius
    closed = np.zeros(cap, dtype=np.uint64)
    actions = np.zeros(65536, dtype=np.int32)
    _check(lib, fn(C.byref(args), rad.ctypes.data, int(max_iter), C.byref(first), C.byref(last), info.ctypes.data,
                   closed.ctypes.data, cap, actions.ctypes.data, actions.size))
    f = {k: getattr(first, k) for k, _ in PlanResult._fields_}
    l = {k: getattr(last, k) for k, _ in PlanResult._fields_}
    l["closed"] = closed[: min(last.n_closed, cap)].copy()
    l["actions"] = actions[: last.n_actions].copy()
    l["iterations"], l["ok"] = int(info[0]), int(info[1])
    return f, l


def iterative_plan(args, search_radius, max_iter=3):
    """MPL::MapPlanner::plan() + iterativePlan() with the GPU env (tunnels built on the device)."""
    lib = _lib()
    return run_iterative(lib.mplh_iterative_plan, lib, args, search_radius, max_iter)


def plan(args):
    """MPL::MapPlanner<Dim>::plan() with the GPU env (one query)."""
    lib = _lib()
    return run_plan(lib.mplh_plan, lib, args)


def plan_trace(args, cap=1 << 20):
    """plan() with the GPU env, returning also the expanded nodes in A* pop order (WAYPOINT_DTYPE array)."""
    lib = _lib()
    r = PlanResult()
    trace = np.zeros(cap, dtype=WAYPOINT_DTYPE)
    n = C.c_int32(0)
    _check(lib, lib.mplh_plan_trace(C.byref(args), C.byref(r), trace.ctypes.data, cap, C.byref(n)))
    out = {k: getattr(r, k) for k, _ in PlanResult._fields_}
    out["trace"] = trace[: n.value].copy()
    return out


def plan_batch(args, starts, goals, path="auto"):
    """MPL::MultiQueryPlanner over many (start, goal) pairs, one session opened and closed around the call.
    path: "auto" (a device search for a bounded search once the batch is large enough, else the lock-step
    loop: one device launch per iteration expands the current node of every live query), "lockstep",
    "device" or "device_cost_terms" (see BatchPlanner).  starts/goals: WAYPOINT_DTYPE arrays."""
    s = BatchPlanner(args, path=path)
    try:
        res, tot = s.plan(starts, goals)
    finally:
        tot_release = s.close()
    tot["t_release"] = tot_release
    return res, tot


_QRES = [("valid", "i4"), ("cost", "f8"), ("expanded", "i4"), ("n_closed", "i4"), ("n_actions", "i4")]


class BatchPlanner:
    """A MPL::MultiQueryPlanner session: the map is uploaded once, and the search states of one query set
    are recycled for the next (a planner that answers batch after batch allocates its state memory once).
    `args` supplies the map, the controls and the limits (its start/goal are ignored).

    path: "auto" runs each query's whole A* on the device for at most 256 primitives once the batch is large
    enough: for max_num > 0 occupancy planning (no potential map, no yaw control) with mplx_plan_batch, potential-
    field and yaw planning with mplx_plan_batch_cost_terms; for max_num <= 0 (unbounded, the reference's default)
    every plan with mplx_plan_batch_grow; otherwise the lock-step loop.  "lockstep" always runs the lock-step
    loop, "device" mplx_plan_batch whenever the plan allows it, "device_cost_terms" mplx_plan_batch_cost_terms
    for every plan the cap and the control set allow, "device_grow" mplx_plan_batch_grow for every plan the
    control set allows (the queries that outgrow its largest arena go through the lock-step loop).  Every path
    gives each query the same result; the choice is a diagnostic.  The totals of plan() say which ran ("path":
    "device", "device_cost_terms", "device_grow" or "lockstep"; for "device_grow" also grow_rounds,
    grow_reruns, grow_first_cap, grow_last_cap and grow_lockstep, the queries handed to the lock-step loop)."""

    PATHS = {"auto": 0, "lockstep": 1, "device": 2, "device_cost_terms": 3, "device_grow": 4}
    _RAN = {0: "lockstep", 1: "device", 2: "device_cost_terms", 3: "device_grow"}

    def __init__(self, args, path="auto"):
        self._lib = _lib()
        self._args = args  # keeps the arrays the struct points at alive
        self._h = self._lib.mplh_batch_open(C.byref(args))
        _check(self._lib, 0 if self._h else 1)
        self.set_path(path)

    def _call(self, name, *a):
        _check(self._lib, getattr(self._lib, name)(self._h, *a))

    def set_path(self, path):
        if path not in self.PATHS:
            raise ValueError(f"path must be one of {sorted(self.PATHS)}")
        self._call("mplh_batch_set_path", self.PATHS[path])

    def set_grow_caps(self, first_cap=0, max_cap=0):
        """Diagnostics: the growing device search's first and largest arena capacity in records (0 = automatic;
        see mplx_plan_batch_grow).  Queries that outgrow max_cap run through the lock-step loop."""
        self._call("mplh_batch_set_grow_caps", int(first_cap), int(max_cap))

    def set_search_regions(self, paths, radius, dense=False):
        """One tunnel per query of the following plans (MultiQueryPlanner::setSearchRegions): query q searches inside
        MapPlanner::setSearchRegion(paths[q], dense) with the search radius `radius` (Dim metres), in place of any
        env-wide region, and those plans must have len(paths) queries.  Each path is points x Dim; an empty list
        clears them.  The device searches build every tunnel at once; the lock-step loop plans tunnelled queries one
        at a time (correct, and slow)."""
        dim = self._args.dim
        if len(paths) == 0:
            self._call("mplh_batch_set_regions", 0, None, None, None, 0)
            return
        pts = [np.ascontiguousarray(p, dtype=np.float64).reshape(-1, dim) for p in paths]
        off = np.zeros(len(pts) + 1, np.int64)
        off[1:] = np.cumsum([len(p) for p in pts])
        flat = np.ascontiguousarray(np.concatenate(pts) if off[-1] else np.zeros((1, dim)))
        rad = np.ascontiguousarray(radius, dtype=np.float64)
        self._call("mplh_batch_set_regions", len(pts), off.ctypes.data, flat.ctypes.data, rad.ctypes.data,
                   1 if dense else 0)

    def _last_path(self):
        dev, slots, nbytes = C.c_int32(0), C.c_int32(0), C.c_int64(0)
        self._call("mplh_batch_last_path", C.byref(dev), C.byref(slots), C.byref(nbytes))
        d = dict(path=self._RAN[dev.value], slots=int(slots.value), arena_bytes=int(nbytes.value))
        rounds, lockstep = C.c_int32(0), C.c_int32(0)
        reruns, first_cap, last_cap = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        self._call("mplh_batch_grow_stats", C.byref(rounds), C.byref(reruns), C.byref(first_cap), C.byref(last_cap),
                   C.byref(lockstep))
        d.update(grow_rounds=int(rounds.value), grow_reruns=int(reruns.value), grow_first_cap=int(first_cap.value),
                 grow_last_cap=int(last_cap.value), grow_lockstep=int(lockstep.value))
        return d

    def _plan(self, name, starts, goals, eps, max_num, *keep):
        """mplh_batch_plan or, with keep = (collect_closed,), mplh_batch_plan_keep: (per-query results, totals)."""
        starts = np.ascontiguousarray(starts, dtype=WAYPOINT_DTYPE)
        goals = np.ascontiguousarray(goals, dtype=WAYPOINT_DTYPE)
        nq = len(starts)
        out = (QueryResult * max(nq, 1))()
        totals = np.zeros(7)
        self._call(name, starts.ctypes.data, goals.ctypes.data, nq, self._args.eps if eps is None else eps,
                   self._args.max_num if max_num is None else max_num, *keep, out, totals.ctypes.data)
        res = np.zeros(nq, dtype=_QRES)
        for q in range(nq):
            res[q] = (out[q].valid, out[q].cost, out[q].expanded, out[q].n_closed, out[q].n_actions)
        return res, totals

    def plan_detail(self, starts, goals, eps=None, max_num=None, closed=True, trajectories=False, n_samples=0):
        """plan() that also returns every query's trajectory (action ids) and closed set (sorted lattice keys):
        (res, totals, actions, closed) with one array per query in actions / closed.  Any max_num, including
        max_num <= 0 (unbounded): the outputs are sized from the results.

        trajectories=True collects every query's planned trajectory on whichever path runs
        (MultiQueryPlanner::setCollectTrajectories) and returns (res, totals, actions, closed, trajectories):
        one dict per query as env_map.batch_trajectories gives them (nodes, seg_t, coeff and, with n_samples > 0,
        samples)."""
        self._call("mplh_batch_set_trajectories", 1 if trajectories else 0)
        try:
            res, totals = self._plan("mplh_batch_plan_keep", starts, goals, eps, max_num, 1 if closed else 0)
        finally:
            if trajectories:
                self._call("mplh_batch_set_trajectories", 0)
        nq = len(res)
        out = (res, self._totals(totals)) + self.kept(res, closed)
        if not trajectories:
            return out
        return out + (self._trajectories(nq, int(sum(n + 1 for n in res["n_actions"] if n)), n_samples),)

    def kept(self, res, closed=True):
        """(actions, closed): every query's trajectory (action ids) and, with closed, closed set (sorted lattice
        keys) of the last plan_detail or iterative_plan, one array per query; res is that call's results."""
        nq = len(res)
        na, nc = int(res["n_actions"].sum()), int(res["n_closed"].sum()) if closed else 0
        aoff, coff = np.zeros(nq + 1, np.int64), np.zeros(nq + 1, np.int64)
        acts = np.zeros(max(na, 1), np.int32)
        keys = np.zeros(max(nc, 1), np.uint64) if closed else None
        self._call("mplh_batch_kept", aoff.ctypes.data, acts.ctypes.data, acts.size, coff.ctypes.data,
                   None if keys is None else keys.ctypes.data, 0 if keys is None else keys.size)
        return ([acts[aoff[q]:aoff[q + 1]].copy() for q in range(nq)],
                [keys[coff[q]:coff[q + 1]].copy() for q in range(nq)] if closed else None)

    def iterative_plan(self, starts, goals, radius, max_iter=3, raw_paths=None, eps=None, max_num=None,
                       trajectories=False, n_samples=0):
        """MapPlanner::iterativePlan for every query as one batch (mplh_batch_iterative_plan): query q replans inside
        tunnels of `radius` (Dim metres) around its last trajectory until the cost stops changing, its plan fails or
        max_iter plans were made.  raw_paths (one points x Dim array per query) are the first round's tunnels; None
        plans the batch first and iterates from those trajectories, as iterative_plan() does for one query (a query
        whose first plan fails reports 0 iterations and that plan).  Returns (res, iterations, ok): res as plan()'s,
        for each query's last plan (kept() gives its actions and closed set), iterations the plan() calls
        iterativePlan made and ok its return value; with trajectories=True also the last plans' trajectories in
        plan_detail's layout.  The session's tunnels and settings are unchanged afterwards."""
        dim = self._args.dim
        starts = np.ascontiguousarray(starts, dtype=WAYPOINT_DTYPE)
        goals = np.ascontiguousarray(goals, dtype=WAYPOINT_DTYPE)
        nq = len(starts)
        off = flat = None
        if raw_paths is not None:
            pts = [np.ascontiguousarray(p, dtype=np.float64).reshape(-1, dim) for p in raw_paths]
            if len(pts) != nq:
                raise ValueError("one raw path per query")
            off = np.zeros(nq + 1, np.int64)
            off[1:] = np.cumsum([len(p) for p in pts])
            flat = np.ascontiguousarray(np.concatenate(pts) if off[-1] else np.zeros((1, dim)))
        rad = np.ascontiguousarray(radius, dtype=np.float64)
        out = (QueryResult * max(nq, 1))()
        info = np.zeros(2 * max(nq, 1), np.int32)
        self._call("mplh_batch_set_trajectories", 1 if trajectories else 0)
        try:
            self._call("mplh_batch_iterative_plan", starts.ctypes.data, goals.ctypes.data, nq,
                       None if off is None else off.ctypes.data, None if flat is None else flat.ctypes.data,
                       rad.ctypes.data, int(max_iter), self._args.eps if eps is None else eps,
                       self._args.max_num if max_num is None else max_num, out, info.ctypes.data)
        finally:
            if trajectories:
                self._call("mplh_batch_set_trajectories", 0)
        res = np.zeros(nq, dtype=_QRES)
        for q in range(nq):
            res[q] = (out[q].valid, out[q].cost, out[q].expanded, out[q].n_closed, out[q].n_actions)
        its, ok = info[0:2 * nq:2].copy(), info[1:2 * nq:2].astype(bool)
        if not trajectories:
            return res, its, ok
        return res, its, ok, self._trajectories(nq, int(sum(n + 1 for n in res["n_actions"] if n)), n_samples)

    def _trajectories(self, nq, cap, n_samples):
        """mplh_batch_trajectories: the last plan's trajectories, one dict per query."""
        dim = self._args.dim
        cap = max(cap, 1)
        offset, total = np.zeros(nq + 1, np.int64), C.c_int64(0)
        nodes = np.zeros(cap, dtype=WAYPOINT_DTYPE)
        seg_t, coeff = np.zeros(cap), np.zeros((cap, dim + 1, 6))
        samples = np.zeros((nq, n_samples + 1, 4 * dim + 3)) if n_samples > 0 else None
        self._call("mplh_batch_trajectories", int(n_samples), offset.ctypes.data, nodes.ctypes.data, seg_t.ctypes.data,
                   coeff.ctypes.data, None if samples is None else samples.ctypes.data, cap, C.byref(total))
        return split_slots(offset, nodes, seg_t, coeff, samples)

    def _totals(self, totals):
        t = dict(iterations=int(totals[0]), nodes=int(totals[1]), seconds=float(totals[2]), t_pop=float(totals[3]),
                 t_device=float(totals[4]), t_relax=float(totals[5]), t_release=0.0)
        t.update(self._last_path())
        return t

    def plan(self, starts, goals, eps=None, max_num=None):
        res, totals = self._plan("mplh_batch_plan", starts, goals, eps, max_num)
        return res, self._totals(totals)

    def update_cells(self, cells, values):
        """MapUtil::setCells on the session's map: cells[k] (n x Dim cell coordinates) := values[k], a later
        entry for the same cell winning.  The next plan() sends only these voxels to the device."""
        cells = np.ascontiguousarray(cells, dtype=np.int32).reshape(-1, self._args.dim)
        values = np.ascontiguousarray(values, dtype=np.int8).reshape(-1)
        if values.size != len(cells):
            raise ValueError("one value per cell")
        self._call("mplh_batch_update_cells", cells.ctypes.data, values.ctypes.data, len(cells))

    def map_uploads(self):
        """(full, delta): whole-grid uploads and sparse updates the session's env has made."""
        full, delta = C.c_int64(0), C.c_int64(0)
        self._call("mplh_batch_map_uploads", C.byref(full), C.byref(delta))
        return full.value, delta.value

    def close(self) -> float:
        """Free the session (incl. the kept search states); returns the seconds that took."""
        if not self._h:
            return 0.0
        rel = C.c_double(0.0)
        self._lib.mplh_batch_close(self._h, C.byref(rel))
        self._h = None
        return rel.value

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def run_traj_solve(fn, lib, dim, control, pos=None, waypoints=None, wp_control=None, dts=None, v=1.0, yaw_control=0x01,
                   n_samples=50):
    """TrajSolver<dim>(control, yaw_control) on one path: setPath(pos) (n x dim), or setWaypoints(waypoints
    (WAYPOINT_DTYPE) with controls wp_control); setDts(dts) when given; setV(v); solve().  Returns a dict:
    `segments`, `seg_t` (getDts), `coeff` (segments x (dim+1) x 6: Primitive1D coefficients, axes then yaw),
    `samples` = sample(n_samples) rows {pos, vel, acc, jrk, yaw, yaw_dot, t} and `waypoints` = getWaypoints()
    rows {pos, vel, acc, jrk, yaw, t}."""
    if waypoints is None:
        pos = np.asarray(pos, dtype=np.float64).reshape(-1, dim)
        wps = np.zeros(len(pos), dtype=WAYPOINT_DTYPE)
        wps["pos"][:, :dim] = pos
        ctl = None
    else:
        wps = np.ascontiguousarray(waypoints, dtype=WAYPOINT_DTYPE)
        ctl = np.ascontiguousarray(wp_control, dtype=np.uint8)
        assert len(ctl) == len(wps)
    n = len(wps)
    d = None if dts is None else np.ascontiguousarray(dts, dtype=np.float64)
    assert d is None or len(d) == max(n - 1, 0)
    seg_t = np.zeros(max(n - 1, 1))
    coeff = np.zeros((max(n - 1, 1), dim + 1, 6))
    samples = np.zeros((n_samples + 1, 4 * dim + 3))
    wout = np.zeros((max(n, 1), 4 * dim + 2))
    n_seg = C.c_int32(0)
    _check(lib, fn(dim, control, yaw_control, wps.ctypes.data if n else None, None if ctl is None else ctl.ctypes.data,
                   n, None if d is None else d.ctypes.data, float(v), n_samples, C.byref(n_seg), seg_t.ctypes.data,
                   coeff.ctypes.data, samples.ctypes.data, wout.ctypes.data))
    s = n_seg.value
    return dict(segments=s, seg_t=seg_t[: max(n - 1, 0)].copy(), coeff=coeff[:s].copy(), samples=samples,
                waypoints=wout[: s + 1 if s else 0].copy())


def traj_solve(dim, control, **kw):
    """MPL::TrajSolver on the host (mpl_host.hpp: the reference's dense formulation, one path).  Arguments as
    run_traj_solve."""
    lib = _lib()
    return run_traj_solve(lib.mplh_traj_solve, lib, dim, control, **kw)


def traj_sample(dim, seg_t, coeff, control, n_samples):
    """Trajectory<dim> built on the host from segment times and Primitive1D coefficients (segments x (dim+1) x 6,
    axes then yaw), each segment with the control flag `control`: (sample(n_samples), getWaypoints()) as arrays
    of rows {pos, vel, acc, jrk, yaw, yaw_dot, t} and {pos, vel, acc, jrk, yaw, t}."""
    lib = _lib()
    seg_t = np.ascontiguousarray(seg_t, dtype=np.float64)
    coeff = np.ascontiguousarray(coeff, dtype=np.float64).reshape(len(seg_t), dim + 1, 6)
    samples = np.zeros((n_samples + 1, 4 * dim + 3))
    wout = np.zeros((len(seg_t) + 1, 4 * dim + 2))
    _check(lib, lib.mplh_traj_sample(dim, len(seg_t), seg_t.ctypes.data, coeff.ctypes.data, control, n_samples,
                                     samples.ctypes.data, wout.ctypes.data))
    return samples, wout[: len(seg_t) + 1 if len(seg_t) else 0]


def run_traj_scale(fn, lib, dim, seg_t, coeff, mode, mv=1.0, ri=1.0, rf=1.0, control=0x07, n_samples=50, flags=False):
    """Trajectory<dim> from segment times and Primitive1D coefficients (segments x (dim+1) x 6, axes then yaw),
    then scale(ri, rf) (mode 1) or scale_down(mv, ri, rf) (mode 2).  Returns a dict: `status` (1 scaled,
    2 unchanged, 0 not scaled), `total_t`, `seg_T` (getSegmentTimes, segments entries), `lambda` (n x 7 rows
    {a3, a2, a1, a0, ti, tf, dT}), `samples` = sample(n_samples) rows {pos, vel, acc, jrk, yaw, yaw_dot, t} and,
    with flags, `flags` (1 on the rows whose lambda the reference leaves indeterminate)."""
    seg_t = np.ascontiguousarray(seg_t, dtype=np.float64)
    n = len(seg_t)
    coeff = np.ascontiguousarray(coeff, dtype=np.float64).reshape(n, dim + 1, 6)
    st, nl, tot = C.c_int32(0), C.c_int32(0), C.c_double(0)
    seg_T = np.zeros(n + 1)
    lam = np.zeros(((n + 1) * 5 * dim, 7))
    samples = np.zeros((n_samples + 1, 4 * dim + 3))
    fl = np.zeros(n_samples + 1, dtype=np.uint8)
    args = [dim, n, seg_t.ctypes.data, coeff.ctypes.data, control, mode, float(mv), float(ri), float(rf), n_samples,
            C.byref(st), C.byref(tot), seg_T.ctypes.data, C.byref(nl), lam.ctypes.data, samples.ctypes.data]
    _check(lib, fn(*(args + ([fl.ctypes.data] if flags else []))))
    r = dict(status=st.value, total_t=tot.value, seg_T=seg_T[:n].copy(), **{"lambda": lam[: nl.value].copy()},
             samples=samples)
    if flags:
        r["flags"] = fl
    return r


def traj_scale(dim, seg_t, coeff, mode, **kw):
    """Trajectory::scale / scale_down on the host (mpl_host.hpp, one path).  Arguments as run_traj_scale.

    As in the reference, sample(N)'s last time N * (total / N) can land an ulp past the last lambda segment;
    getTau then finds no root and that row is the trajectory's start state."""
    lib = _lib()
    return run_traj_scale(lib.mplh_traj_scale, lib, dim, seg_t, coeff, mode, **kw)


def run_solve(fn, a, b, c, d, e):
    """solve(a, b, c, d, e) of math.h: the real roots of a t^4 + b t^3 + c t^2 + d t + e, in solver order."""
    n = C.c_int32(0)
    r = np.zeros(4)
    fn(float(a), float(b), float(c), float(d), float(e), C.byref(n), r.ctypes.data)
    return r[: n.value].copy()


def solve_roots(a, b, c, d, e):
    """The host's closed-form root solver (mpl_host.hpp), as run_solve."""
    return run_solve(_lib().mplh_solve, a, b, c, d, e)


def run_traj_check(fn, lib, dim, grid, mdim, origin, res, paths, control, potential=None, potential_weight=0.1,
                   gradient_weight=0.0, region=None, v_max=-1.0, a_max=-1.0, j_max=-1.0, yaw_max=-1.0, scaled=None,
                   nthreads=1):
    """The map and parameters given directly, the trajectories as TrajSolverBatch results (dicts with `seg_t` and
    `coeff`; `scaled` as TrajSolverBatch.scale's, with `total_t` and `lambda`), control one flag or one per path.
    Returns a dict of arrays: `status`, `cost` (one per path), `seg_free` and `seg_valid` (one per waypoint slot,
    mplx_traj_out's layout) and `offset`."""
    from .traj import pack_lambda, pack_paths

    _, offset, seg_t, coeff = pack_paths(paths, dim)
    n_paths = len(paths)
    ctl = np.ascontiguousarray(np.broadcast_to(np.asarray(control, dtype=np.uint8), (max(n_paths, 1),)))
    total_t = n_lambda = lam = None
    if scaled is not None:
        total_t, n_lambda, lam = pack_lambda(scaled, offset, dim)
    grid = np.ascontiguousarray(grid, dtype=np.int8).reshape(-1)
    mdim = np.ascontiguousarray(mdim, dtype=np.int32)
    origin = np.ascontiguousarray(origin, dtype=np.float64)
    pot = None if potential is None else np.ascontiguousarray(potential, dtype=np.int8).reshape(-1)
    reg = None if region is None else np.ascontiguousarray(region, dtype=np.uint8).reshape(-1)
    status = np.zeros(max(n_paths, 1), dtype=np.int32)
    cost = np.zeros(max(n_paths, 1))
    free = np.zeros(seg_t.size, dtype=np.uint8)
    valid = np.zeros(seg_t.size, dtype=np.uint8)

    def p(a):
        return None if a is None else a.ctypes.data

    _check(lib, fn(dim, grid.ctypes.data, mdim.ctypes.data, origin.ctypes.data, float(res), p(pot),
                   float(potential_weight), float(gradient_weight), p(reg), float(v_max), float(a_max), float(j_max),
                   float(yaw_max), n_paths, offset.ctypes.data, seg_t.ctypes.data, coeff.ctypes.data, ctl.ctypes.data,
                   p(total_t), p(n_lambda), p(lam), int(nthreads), status.ctypes.data, cost.ctypes.data,
                   free.ctypes.data, valid.ctypes.data))
    return dict(status=status[:n_paths], cost=cost[:n_paths], seg_free=free[:int(offset[-1])],
                seg_valid=valid[:int(offset[-1])], offset=offset)


def traj_check(dim, grid, mdim, origin, res, paths, control, **kw):
    """env_map_host::traverse_trajectory, is_free and validate_primitive on the host (mpl_host.hpp) for a batch of
    trajectories, as mplx_traj_check computes them on the device.  Arguments as run_traj_check."""
    lib = _lib()
    return run_traj_check(lib.mplh_traj_check, lib, dim, grid, mdim, origin, res, paths, control, **kw)
