"""Planner bindings for the tests: the product's (motion_primitive_library_b200.planner) plus the
TEST-ONLY harness oracle/liboracle_planner.so (same host A*, CPU-oracle env)."""
import subprocess
from pathlib import Path

from motion_primitive_library_b200.planner import (PlanArgs, PlanResult, QueryResult, Waypoint, bind,  # noqa: F401
                                                   iterative_plan, lpa_session, make_args, plan, plan_batch,
                                                   plan_trajectory, run_iterative, run_lpa, run_plan, run_trajectory)
from reference_record import reference

ROOT = Path(__file__).resolve().parent.parent
ORACLE_PLANNER = ROOT / "oracle" / "liboracle_planner.so"


def plan_gpu(args):
    return plan(args)


def plan_oracle(args):
    if not ORACLE_PLANNER.exists():
        subprocess.check_call(["make", "-C", str(ROOT / "oracle"), "liboracle_planner.so"], stdout=subprocess.DEVNULL)
    lib, fn = bind(ORACLE_PLANNER, "orcp_plan", "mplh_plan")
    return run_plan(fn, lib, args)


REF_PLANNER = ROOT / "oracle" / "_ref" / "libmplref_planner.so"


def lpa_oracle(args, script):
    """The product's host LPA* driven by the CPU-oracle env (TEST-ONLY harness)."""
    lib, fn = bind(ORACLE_PLANNER, "orcp_lpa_run", "mplh_lpa_run")
    return run_lpa(fn, lib, args, script)


def lpa_reference(args, script):
    """The REFERENCE's LPA* (setLPAstar / plan / getLinkedNodes / updateBlockedNodes / updateClearedNodes /
    getSubStateSpace, unmodified sources + Eigen/Boost stand-ins) on the same script."""
    def live():
        lib, fn = bind(REF_PLANNER, "refp_lpa_run", "mplh_lpa_run")
        return run_lpa(fn, lib, args, script)

    return reference(REF_PLANNER, live)


def iterative_oracle(args, search_radius, max_iter=3):
    """The product's host plan() + iterativePlan() driven by the CPU-oracle env (TEST-ONLY harness)."""
    lib, fn = bind(ORACLE_PLANNER, "orcp_iterative_plan", "mplh_iterative_plan")
    return run_iterative(fn, lib, args, search_radius, max_iter)


def iterative_reference(args, search_radius, max_iter=3):
    """The REFERENCE's plan() + MapPlanner::iterativePlan(start, goal, getTraj(), max_iter)."""
    def live():
        lib, fn = bind(REF_PLANNER, "refp_iterative_plan", "mplh_iterative_plan")
        return run_iterative(fn, lib, args, search_radius, max_iter)

    return reference(REF_PLANNER, live)


def trajectory_oracle(args, n_samples=50):
    lib, fn = bind(ORACLE_PLANNER, "orcp_plan_trajectory", "mplh_plan_trajectory")
    return run_trajectory(fn, lib, args, n_samples)


def trajectory_reference(args, n_samples=50):
    """The REFERENCE's plan() + its own Trajectory::sample / getWaypoints / evaluate / J."""
    def live():
        lib, fn = bind(REF_PLANNER, "refp_plan_trajectory", "mplh_plan_trajectory")
        return run_trajectory(fn, lib, args, n_samples)

    return reference(REF_PLANNER, live)


def ref_planner_available():
    return REF_PLANNER.exists()


def plan_reference(args):
    """The REFERENCE's MapPlanner<Dim>::plan() (unmodified sources + Eigen/Boost stand-ins)."""
    def live():
        lib, fn = bind(REF_PLANNER, "refp_plan", "mplh_plan")
        return run_plan(fn, lib, args)

    return reference(REF_PLANNER, live)


def reference_potential_map(args, radius, n_cells, range_=None, pos=None, record_all=False):
    """MapPlanner::updatePotentialMap (src/mpl_planner/map_planner.cpp:323-391) on args' map.  record_all: the
    recording keeps the whole map (a test that uses it as input data), not only its digest."""
    import ctypes as C

    import numpy as np

    def live():
        lib = C.CDLL(str(REF_PLANNER))
        out = np.zeros(n_cells, dtype=np.int8)
        rad = np.asarray(radius, dtype=np.float64)
        rng = None if range_ is None else np.asarray(range_, dtype=np.float64)
        p = None if pos is None else np.asarray(pos, dtype=np.float64)
        lib.refp_update_potential_map.argtypes = [C.POINTER(PlanArgs), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.refp_update_potential_map(C.byref(args), rad.ctypes.data, None if rng is None else rng.ctypes.data,
                                      None if p is None else p.ctypes.data, out.ctypes.data)
        return out

    return reference(REF_PLANNER, live, max_bytes=None) if record_all else reference(REF_PLANNER, live)


def reference_search_region(args, path, radius, n_cells, dense=False):
    """MapPlanner::setSearchRegion (src/mpl_planner/map_planner.cpp:46-95)."""
    import ctypes as C

    import numpy as np

    def live():
        lib = C.CDLL(str(REF_PLANNER))
        out = np.zeros(n_cells, dtype=np.uint8)
        p = np.ascontiguousarray(path, dtype=np.float64)
        rad = np.asarray(radius, dtype=np.float64)
        lib.refp_set_search_region.argtypes = [C.POINTER(PlanArgs), C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        lib.refp_set_search_region(C.byref(args), p.ctypes.data, len(p), rad.ctypes.data, 1 if dense else 0,
                                   out.ctypes.data)
        return out

    return reference(REF_PLANNER, live)


REF_B200 = ROOT / "oracle" / "_ref" / "libmplref_b200.so"


def ref_b200_available():
    return REF_B200.exists()


def plan_reference_b200(args):
    """The REFERENCE's MapPlanner<Dim>::plan() with integration/env_map_b200.h (libmplx behind the
    reference's virtual get_succ) installed through the virtual setMapUtil — the drop-in of INTEGRATION.md."""
    lib, fn = bind(REF_B200, "refb_plan", "mplh_plan")
    lib.mplh_last_error = lib.refb_last_error
    return run_plan(fn, lib, args)
