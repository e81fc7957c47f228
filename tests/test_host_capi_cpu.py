"""The C entry points of libmpl_host.so without a GPU: the exported functions are exactly those planner.py declares,
and every entry point that dispatches on the dimension refuses one outside {2, 3} before it touches the device, as
the test harness's planner entry points do."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import fixtures
import planner_bindings as pb
from motion_primitive_library_b200 import planner as P

DIM_ERROR = "dim must be 2 or 3"


def args4():
    c = fixtures.corridor()
    return P.make_args(4, 0x03, c["grid"], (*c["dim"], 1), (*c["origin"], 0.0), c["res"], fixtures.U_2d(),
                       start=dict(pos=c["start"]), goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0)


def test_exports_match_the_signature_table():
    out = subprocess.run(["nm", "-D", "--defined-only", str(P.LIB)], capture_output=True, text=True, check=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if line.split() and line.split()[-1].startswith("mplh_")}
    assert exported == {k for k in P.SIGNATURES if k.startswith("mplh_")}


def _dim4_calls():
    a = args4()
    r, r2 = P.PlanResult(), P.PlanResult()
    buf = np.zeros(4096)
    i32 = C.c_int32(0)
    i32b = C.c_int32(0)
    d = C.c_double(0)
    wps = np.zeros(2, dtype=P.WAYPOINT_DTYPE)
    step = (P.LpaStep * 1)()
    outs = (P.LpaOut * 1)()
    mdim = np.array([4, 4, 4, 4], dtype=np.int32)
    grid = np.zeros(256, dtype=np.int8)
    offset = np.zeros(1, dtype=np.int64)
    status = np.zeros(1, dtype=np.int32)
    return {
        "mplh_plan": lambda L: L.mplh_plan(C.byref(a), C.byref(r), buf.ctypes.data, 1, buf.ctypes.data, 1),
        "mplh_plan_trace": lambda L: L.mplh_plan_trace(C.byref(a), C.byref(r), buf.ctypes.data, 1, C.byref(i32)),
        "mplh_plan_trajectory": lambda L: L.mplh_plan_trajectory(C.byref(a), 5, C.byref(r), buf.ctypes.data,
                                                                 buf.ctypes.data, buf.ctypes.data, 1, C.byref(i32),
                                                                 buf.ctypes.data),
        "mplh_iterative_plan": lambda L: L.mplh_iterative_plan(C.byref(a), buf.ctypes.data, 2, C.byref(r), C.byref(r2),
                                                               buf.ctypes.data, buf.ctypes.data, 1, buf.ctypes.data, 1),
        "mplh_lpa_run": lambda L: L.mplh_lpa_run(C.byref(a), step, 1, outs, buf.ctypes.data, 1),
        "mplh_traj_solve": lambda L: L.mplh_traj_solve(4, 0x03, 0x01, wps.ctypes.data, None, 2, None, 1.0, 0,
                                                       C.byref(i32), None, None, None, None),
        "mplh_traj_sample": lambda L: L.mplh_traj_sample(4, 0, None, None, 0x03, 0, None, None),
        "mplh_traj_scale": lambda L: L.mplh_traj_scale(4, 0, None, None, 0x07, 1, 1.0, 1.0, 1.0, 0, C.byref(i32),
                                                       C.byref(d), buf.ctypes.data, C.byref(i32b), None, None),
        "mplh_traj_check": lambda L: L.mplh_traj_check(4, grid.ctypes.data, mdim.ctypes.data, buf.ctypes.data, 1.0,
                                                       None, 0.0, 0.0, None, -1.0, -1.0, -1.0, -1.0, 0,
                                                       offset.ctypes.data, None, None, None, None, None, None, 1,
                                                       status.ctypes.data, buf.ctypes.data, None, None),
    }


@pytest.mark.parametrize("name", sorted(_dim4_calls()))
def test_entry_point_refuses_dim_4(name):
    lib = P._lib()
    assert lib.mplh_batch_set_path(None, 0) == 1  # leaves another message behind
    assert lib.mplh_last_error().decode() != DIM_ERROR
    assert _dim4_calls()[name](lib) == 1
    assert lib.mplh_last_error().decode() == DIM_ERROR


def test_batch_open_refuses_dim_4():
    lib = P._lib()
    assert lib.mplh_batch_set_path(None, 0) == 1
    assert not lib.mplh_batch_open(C.byref(args4()))
    assert lib.mplh_last_error().decode() == DIM_ERROR
    with pytest.raises(RuntimeError, match=DIM_ERROR):
        P.BatchPlanner(args4())


@pytest.mark.parametrize("call", [lambda a: pb.plan_oracle(a), lambda a: pb.lpa_oracle(a, [("plan",)]),
                                  lambda a: pb.iterative_oracle(a, (0.5,) * 3), lambda a: pb.trajectory_oracle(a, 5)],
                         ids=["orcp_plan", "orcp_lpa_run", "orcp_iterative_plan", "orcp_plan_trajectory"])
def test_harness_refuses_dim_4(call):
    with pytest.raises(RuntimeError, match=DIM_ERROR):
        call(args4())
