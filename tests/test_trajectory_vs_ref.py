"""The recovered Trajectory (include/mpl_basis/trajectory.h, primitive.h): sample(N) commands,
getWaypoints, evaluate(t), total time and effort integrals of the host planner's Trajectory/Primitive
restatement against the reference's own classes — bit for bit (same flags, same operand order)."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
from reference_record import same_array
VEL, ACC, JRK, ACCxYAW = 0x01, 0x03, 0x07, 0x13


def same(a, b):
    assert a["valid"] == b["valid"] == 1 and a["segments"] == b["segments"] > 0
    for k in ("total_time", "J", "Jyaw"):
        assert a[k] == b[k], (k, a[k], b[k])
    for k in ("commands", "waypoints", "evaluated"):
        same_array(a[k], b[k], k, bits=True)


@pytest.mark.parametrize("control,U,kw", [(ACC, "U_2d", {}), (VEL, "U_2d_vel", {}), (ACCxYAW, "U_2d_yaw", dict(yaw_max=0.7, max_num=3000))])
@pytest.mark.parametrize("n_samples", [7, 50])
def test_corridor_trajectory(control, U, kw, n_samples):
    c = fixtures.corridor()
    Us = dict(U_2d=fixtures.U_2d(), U_2d_vel=fixtures.U_2d(1.0, 1.0), U_2d_yaw=fixtures.U_2d_yaw())[U]
    a = pb.make_args(2, control, c["grid"], c["dim"], c["origin"], c["res"], Us, start=dict(pos=c["start"]),
                     goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, **kw)
    ref = pb.trajectory_reference(a, n_samples)
    got = pb.trajectory_oracle(a, n_samples)
    same(got, ref)  # bit for bit, so the checks below hold for both
    assert got["total_time"] == got["segments"] * 1.0 and got["waypoints"].shape[0] == got["segments"] + 1
    np.testing.assert_array_equal(got["commands"][:, -1], np.arange(n_samples + 1) * (got["total_time"] / n_samples))


def test_voxel_jrk_trajectory():
    import scenarios as S

    sc = S.scaled(S.cfg3(), 48)
    nodes = sc.frontier(16, seed=4, max_steps=0)
    done = 0
    for q in range(0, 16, 2):
        a = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=nodes["pos"][q]),
                         goal=dict(pos=nodes["pos"][q + 1]), v_max=sc.v_max, a_max=sc.a_max, max_num=600)
        ref = pb.trajectory_reference(a, 33)
        if not ref["valid"]:
            continue
        same(pb.trajectory_oracle(a, 33), ref)
        done += 1
    assert done >= 2
