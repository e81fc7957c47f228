"""The host TrajSolver restatement (MPL::TrajSolver / PolySolver, mpl_host.hpp) against the reference's own
TrajSolver (src/mpl_traj_solver, live where oracle/_ref is built, else its recording): bit for bit in the
segment times, the Primitive1D coefficients, sample(N) and getWaypoints()."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
import traj_bindings as TB
from motion_primitive_library_b200 import planner as P
from reference_record import same_array

VEL, ACC, JRK, ACCxYAW = 0x01, 0x03, 0x07, 0x13
NS = 50


def same(got, ref, finite=True):
    assert got["segments"] == ref["segments"]
    for k in ("seg_t", "coeff", "samples", "waypoints"):
        if finite:
            assert np.isfinite(got[k]).all(), k
            same_array(got[k], ref[k], k, bits=True)
        else:
            np.testing.assert_array_equal(np.isfinite(got[k]), np.isfinite(ref[k]), err_msg=k)


def both(dim, control, max_bytes=256, **kw):
    return (TB.traj_solve(dim, control, n_samples=NS, **kw),
            TB.traj_reference(dim, control, max_bytes=max_bytes, n_samples=NS, **kw))


@pytest.mark.parametrize("control", [VEL, ACC, JRK])
def test_reference_test_program(control):
    """test/test_traj_solver.cpp: path (0,0), (1,0), (2,1), (5,1), setV(1)."""
    got, ref = both(2, control, pos=[(0, 0), (1, 0), (2, 1), (5, 1)], v=1.0)
    assert got["segments"] == 3
    same(got, ref)


def planned_waypoints(args, dim):
    t = pb.trajectory_oracle(args, 8)
    assert t["valid"] == 1
    rows = t["waypoints"]
    w = np.zeros(len(rows), dtype=P.WAYPOINT_DTYPE)
    for k, f in enumerate(("pos", "vel", "acc", "jrk")):
        w[f][:, :dim] = rows[:, k * dim:(k + 1) * dim]
    w["yaw"] = rows[:, 4 * dim]
    return w, np.diff(rows[:, 4 * dim + 1])


@pytest.mark.parametrize("control,yaw_control", [(ACC, VEL), (ACCxYAW, VEL), (ACCxYAW, ACC), (ACCxYAW, JRK)])
def test_planned_corridor_waypoints(control, yaw_control):
    """setWaypoints + setDts from the host planner's trajectory on the corridor map."""
    c = fixtures.corridor()
    U = fixtures.U_2d_yaw() if control & 0x10 else fixtures.U_2d()
    kw = dict(yaw_max=0.7, max_num=3000) if control & 0x10 else {}
    a = pb.make_args(2, control, c["grid"], c["dim"], c["origin"], c["res"], U, start=dict(pos=c["start"]),
                     goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, **kw)
    w, dts = planned_waypoints(a, 2)
    ctl = np.full(len(w), control, dtype=np.uint8)
    got, ref = both(2, control, waypoints=w, wp_control=ctl, dts=dts, yaw_control=yaw_control)
    assert got["segments"] == len(w) - 1
    same(got, ref)


def test_planned_voxel_jrk_waypoints():
    import scenarios as S

    sc = S.scaled(S.cfg3(), 48)
    nodes = sc.frontier(16, seed=4, max_steps=0)
    done = 0
    for q in range(0, 16, 2):
        a = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=nodes["pos"][q]),
                         goal=dict(pos=nodes["pos"][q + 1]), v_max=sc.v_max, a_max=sc.a_max, max_num=600)
        if not pb.trajectory_oracle(a, 8)["valid"]:
            continue
        w, dts = planned_waypoints(a, 3)
        got, ref = both(3, JRK, waypoints=w, wp_control=np.full(len(w), sc.control, dtype=np.uint8), dts=dts)
        same(got, ref)
        done += 1
        if done == 3:
            break
    assert done >= 2


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("control", [VEL, ACC, JRK, 0x11, ACCxYAW, 0x17])
def test_random_paths(dim, control):
    rng = np.random.default_rng(dim * 100 + control)
    for trial in range(3):
        n = int(rng.integers(2, 61))
        if trial == 0:
            kw = dict(pos=np.cumsum(rng.uniform(-2, 2, (n, dim)), axis=0), v=float(rng.uniform(0.5, 2)))
        else:
            w = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
            w["pos"][:, :dim] = np.cumsum(rng.uniform(-2, 2, (n, dim)), axis=0)
            w["vel"][:, :dim] = rng.uniform(-1, 1, (n, dim))
            w["acc"][:, :dim] = rng.uniform(-1, 1, (n, dim))
            w["yaw"] = rng.uniform(-1, 1, n)
            ctl = rng.choice([VEL, ACC, JRK, ACCxYAW], n).astype(np.uint8)
            kw = dict(waypoints=w, wp_control=ctl, dts=rng.uniform(0.05, 5, n - 1),
                      yaw_control=int(rng.choice([VEL, ACC, JRK])))
        got, ref = both(dim, control, **kw)
        same(got, ref)


def test_two_waypoints_with_free_derivatives():
    """ACC waypoints under a JRK solver: the accelerations are free and the reference skips the free solve."""
    w = np.zeros(2, dtype=P.WAYPOINT_DTYPE)
    w["pos"][:, :2] = [(0, 0), (2, 1)]
    w["vel"][:, :2] = [(0.5, 0), (0, -0.5)]
    got, ref = both(2, JRK, waypoints=w, wp_control=np.array([ACC, ACC], dtype=np.uint8), dts=[1.5])
    same(got, ref)
    assert got["waypoints"][0, 4:6].tolist() == [0.0, 0.0]  # the free accelerations are 0
    assert np.abs(got["waypoints"][1, 4:6]).max() < 1e-9


def test_zero_length_segment():
    got, ref = both(2, ACC, max_bytes=None, pos=[(0, 0), (1, 0), (1, 0), (2, 1)], v=1.0)
    assert got["seg_t"][1] == 0.0 and not np.isfinite(got["coeff"]).all()
    same(got, ref, finite=False)
