"""ctypes binding of oracle/liboracle.so — TEST INFRASTRUCTURE (the checker, never the product)."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

from reference_record import reference

ROOT = Path(__file__).resolve().parent.parent
ORACLE_DIR = ROOT / "oracle"
LIB = ORACLE_DIR / "liboracle.so"

WAYPOINT_DTYPE = np.dtype(
    [("pos", "<f8", 3), ("vel", "<f8", 3), ("acc", "<f8", 3), ("jrk", "<f8", 3), ("yaw", "<f8"), ("t", "<f8")]
)
LATTICE_MAX = 13


class OrcEnv(C.Structure):
    _fields_ = [
        ("dim", C.c_int32), ("control", C.c_int32),
        ("T", C.c_double), ("w", C.c_double), ("wyaw", C.c_double),
        ("v_max", C.c_double), ("a_max", C.c_double), ("j_max", C.c_double), ("yaw_max", C.c_double),
        ("nU", C.c_int32), ("udim", C.c_int32), ("U", C.c_void_p),
        ("mdim", C.c_int32 * 3), ("origin", C.c_double * 3), ("res", C.c_double),
        ("map", C.c_void_p), ("potential", C.c_void_p),
        ("potential_weight", C.c_double), ("gradient_weight", C.c_double),
        ("region", C.c_void_p),
    ]


_lib = None


def build():
    src_new = max((ORACLE_DIR / f).stat().st_mtime for f in ("mpl_oracle.cpp", "mpl_oracle.h"))
    if not LIB.exists() or LIB.stat().st_mtime < src_new:
        subprocess.check_call(["make", "-C", str(ORACLE_DIR), "liboracle.so"], stdout=subprocess.DEVNULL)


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(str(LIB))
        vp = C.c_void_p
        L.orc_get_succ.argtypes = [C.POINTER(OrcEnv), vp, vp, vp, vp, vp, vp]
        L.orc_get_succ.restype = C.c_int
        L.orc_expand_batch.argtypes = [C.POINTER(OrcEnv), vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_int]
        L.orc_expand_batch.restype = C.c_int
        L.orc_expand_batch_timed.argtypes = [C.POINTER(OrcEnv), vp, C.c_int, C.c_int, C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int64), C.POINTER(C.c_double)]
        L.orc_expand_batch_timed.restype = C.c_int
        L.orc_hash.argtypes = [C.POINTER(OrcEnv), vp, vp, vp]
        L.orc_hash.restype = C.c_uint64
        L.orc_sample_count.argtypes = [C.c_double, C.c_int]
        L.orc_sample_count.restype = C.c_int
        L.orc_max_vel.argtypes = [C.POINTER(OrcEnv), vp, C.c_int, C.c_int]
        L.orc_max_vel.restype = C.c_double
        L.orc_last_samples.argtypes = []
        L.orc_last_samples.restype = C.c_int64
        L.orc_edges_is_free.argtypes = [C.POINTER(OrcEnv), vp, vp, C.c_int, vp, vp]
        L.orc_edges_is_free.restype = C.c_int
        L.orc_edges_cells.argtypes = [C.POINTER(OrcEnv), vp, vp, C.c_int, vp, vp, C.c_int64]
        L.orc_edges_cells.restype = C.c_int64
        _lib = L
    return _lib


class OracleEnv:
    """Holds the numpy arrays an orc_env points at."""

    def __init__(self, dim, control, U, grid, mdim, origin, res, T=1.0, w=10.0, wyaw=1.0, v_max=-1.0, a_max=-1.0,
                 j_max=-1.0, yaw_max=-1.0, potential=None, potential_weight=0.1, gradient_weight=0.0, region=None):
        self.U = np.ascontiguousarray(U, dtype=np.float64)
        self.grid = np.ascontiguousarray(grid, dtype=np.int8).reshape(-1)
        self.potential = None if potential is None else np.ascontiguousarray(potential, dtype=np.int8).reshape(-1)
        self.region = None if region is None else np.ascontiguousarray(region).reshape(-1).astype(np.uint8)
        e = OrcEnv()
        e.dim, e.control = dim, control
        e.T, e.w, e.wyaw = T, w, wyaw
        e.v_max, e.a_max, e.j_max, e.yaw_max = v_max, a_max, j_max, yaw_max
        e.nU, e.udim = self.U.shape
        e.U = self.U.ctypes.data
        for k in range(3):
            e.mdim[k] = int(mdim[k]) if k < dim else 1
            e.origin[k] = float(origin[k]) if k < dim else 0.0
        e.res = res
        e.map = self.grid.ctypes.data
        e.potential = None if self.potential is None else self.potential.ctypes.data
        e.potential_weight, e.gradient_weight = potential_weight, gradient_weight
        e.region = None if self.region is None else self.region.ctypes.data
        self.e = e
        self.nU = int(e.nU)

    @classmethod
    def from_scenario(cls, sc, region=None):
        return cls(sc.Dim, sc.control, sc.U, sc.grid(), sc.dim_cells, sc.origin, sc.res, T=sc.T, w=sc.w, wyaw=sc.wyaw,
                   v_max=sc.v_max, a_max=sc.a_max, j_max=sc.j_max, yaw_max=sc.yaw_max, potential=sc.potential(),
                   potential_weight=sc.potential_weight, gradient_weight=sc.gradient_weight, region=region)

    def expand(self, nodes, nthreads=1, lattice=True):
        nodes = np.ascontiguousarray(nodes, dtype=WAYPOINT_DTYPE).reshape(-1)
        n, nU = nodes.size, self.nU
        succ = np.zeros(n * nU, dtype=WAYPOINT_DTYPE)
        cost = np.zeros(n * nU)
        action = np.zeros(n * nU, dtype=np.int32)
        key = np.zeros(n * nU, dtype=np.uint64)
        lat = np.zeros((n * nU, LATTICE_MAX), dtype=np.int32) if lattice else None
        count = np.zeros(n, dtype=np.int32)
        lib().orc_expand_batch(C.byref(self.e), nodes.ctypes.data, n, succ.ctypes.data, cost.ctypes.data,
                               action.ctypes.data, key.ctypes.data, None if lat is None else lat.ctypes.data,
                               count.ctypes.data, nthreads)
        return dict(count=count, succ=succ, cost=cost, action=action, key=key, lattice=lat, nU=nU)

    def get_succ(self, node):
        r = self.expand(np.array([node], dtype=WAYPOINT_DTYPE))
        c = int(r["count"][0])
        return {k: (v[:c] if isinstance(v, np.ndarray) and k != "count" else v) for k, v in r.items()}

    def edges_is_free(self, parents, actions):
        """env_map::is_free(pr) + calculate_intrinsic_cost(pr) for stored edges (parent, action)."""
        parents = np.ascontiguousarray(parents, dtype=WAYPOINT_DTYPE).reshape(-1)
        actions = np.ascontiguousarray(actions, dtype=np.int32).reshape(-1)
        free = np.zeros(parents.size, dtype=np.uint8)
        cost = np.zeros(parents.size)
        lib().orc_edges_is_free(C.byref(self.e), parents.ctypes.data, actions.ctypes.data, parents.size,
                                free.ctypes.data, cost.ctypes.data)
        return free, cost

    def edges_cells(self, parents, actions):
        """The getLinkedNodes voxel walk per edge: (offset[n+1], cells[total, dim])."""
        parents = np.ascontiguousarray(parents, dtype=WAYPOINT_DTYPE).reshape(-1)
        actions = np.ascontiguousarray(actions, dtype=np.int32).reshape(-1)
        dim = int(self.e.dim)
        off = np.zeros(parents.size + 1, dtype=np.int64)
        total = lib().orc_edges_cells(C.byref(self.e), parents.ctypes.data, actions.ctypes.data, parents.size,
                                      off.ctypes.data, None, 0)
        cells = np.zeros((total, dim), dtype=np.int32)
        lib().orc_edges_cells(C.byref(self.e), parents.ctypes.data, actions.ctypes.data, parents.size,
                              off.ctypes.data, cells.ctypes.data, total)
        return off, cells

    def timed(self, nodes, nthreads=1):
        nodes = np.ascontiguousarray(nodes, dtype=WAYPOINT_DTYPE).reshape(-1)
        a, b, s = C.c_int64(), C.c_int64(), C.c_double()
        lib().orc_expand_batch_timed(C.byref(self.e), nodes.ctypes.data, nodes.size, nthreads, C.byref(a), C.byref(b),
                                     C.byref(s))
        return dict(seconds=s.value, successors=a.value, samples=b.value)


def wp(pos, vel=None, acc=None, jrk=None, yaw=0.0, t=0.0):
    w = np.zeros((), dtype=WAYPOINT_DTYPE)
    for name, v in (("pos", pos), ("vel", vel), ("acc", acc), ("jrk", jrk)):
        if v is not None:
            w[name][: len(v)] = v
    w["yaw"], w["t"] = yaw, t
    return w


# ---- oracle/_ref: the unmodified reference headers behind the same C ABI -------------------------
REF_LIB = ORACLE_DIR / "_ref" / "libmplref.so"
_ref = None


def ref_available() -> bool:
    return REF_LIB.exists()


def ref_info() -> str:
    return reference(REF_LIB, lambda: ref_lib().ref_info().decode())


def ref_lib():
    """oracle/_ref/libmplref.so (built by `make -C oracle ref` where the reference sources are present)."""
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_LIB))
        vp = C.c_void_p
        L.ref_expand_batch.argtypes = [C.POINTER(OrcEnv), vp, C.c_int, vp, vp, vp, vp, vp, C.c_int]
        L.ref_expand_batch.restype = C.c_int
        L.ref_expand_batch_timed.argtypes = [C.POINTER(OrcEnv), vp, C.c_int, C.c_int, C.POINTER(C.c_int64),
                                             C.POINTER(C.c_double)]
        L.ref_expand_batch_timed.restype = C.c_int
        L.ref_info.argtypes = []
        L.ref_info.restype = C.c_char_p
        L.ref_edges_is_free.argtypes = [C.POINTER(OrcEnv), vp, vp, C.c_int, vp, vp]
        L.ref_edges_is_free.restype = C.c_int
        _ref = L
    return _ref


def ref_expand(env: "OracleEnv", nodes, nthreads=1):
    """Run the REFERENCE's env_map<Dim>::get_succ on `nodes` with the parameters held by `env`.  Inside a test
    without oracle/_ref: its recorded result, with only the emitted slots of each field (valid_only)."""
    full = {}

    def live():
        full.update(_ref_expand(env, nodes, nthreads))
        return emitted(full)

    recorded = reference(REF_LIB, live)
    return full or recorded


def emitted(r):
    """The fields a comparison reads: count, and action/succ/cost/key of the emitted slots only."""
    if r.get("valid_only"):
        return r
    valid = (np.arange(r["nU"])[None, :] < r["count"][:, None]).reshape(-1)
    return dict(valid_only=True, nU=r["nU"], count=r["count"], action=r["action"][valid], succ=r["succ"][valid],
                cost=r["cost"][valid], key=r["key"][valid])


def _ref_expand(env: "OracleEnv", nodes, nthreads=1):
    nodes = np.ascontiguousarray(nodes, dtype=WAYPOINT_DTYPE).reshape(-1)
    n, nU = nodes.size, env.nU
    succ = np.zeros(n * nU, dtype=WAYPOINT_DTYPE)
    cost = np.zeros(n * nU)
    action = np.zeros(n * nU, dtype=np.int32)
    key = np.zeros(n * nU, dtype=np.uint64)
    count = np.zeros(n, dtype=np.int32)
    ref_lib().ref_expand_batch(C.byref(env.e), nodes.ctypes.data, n, succ.ctypes.data, cost.ctypes.data,
                               action.ctypes.data, key.ctypes.data, count.ctypes.data, nthreads)
    return dict(count=count, succ=succ, cost=cost, action=action, key=key, lattice=None, nU=nU)


def ref_edges_is_free(env: "OracleEnv", parents, actions):
    """The REFERENCE's env_map::is_free(pr) / calculate_intrinsic_cost(pr) for stored edges."""
    return reference(REF_LIB, lambda: _ref_edges_is_free(env, parents, actions))


def _ref_edges_is_free(env, parents, actions):
    parents = np.ascontiguousarray(parents, dtype=WAYPOINT_DTYPE).reshape(-1)
    actions = np.ascontiguousarray(actions, dtype=np.int32).reshape(-1)
    free = np.zeros(parents.size, dtype=np.uint8)
    cost = np.zeros(parents.size)
    ref_lib().ref_edges_is_free(C.byref(env.e), parents.ctypes.data, actions.ctypes.data, parents.size,
                                free.ctypes.data, cost.ctypes.data)
    return free, cost


def ref_timed(env: "OracleEnv", nodes, nthreads=1):
    nodes = np.ascontiguousarray(nodes, dtype=WAYPOINT_DTYPE).reshape(-1)
    a, s = C.c_int64(), C.c_double()
    ref_lib().ref_expand_batch_timed(C.byref(env.e), nodes.ctypes.data, nodes.size, nthreads, C.byref(a), C.byref(s))
    return dict(seconds=s.value, successors=a.value)
