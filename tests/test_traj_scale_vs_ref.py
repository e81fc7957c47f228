"""The host's trajectory time scaling (Trajectory::scale / scale_down, Lambda and the root solvers, mpl_host.hpp)
against the reference's own classes (live where oracle/_ref is built, else their recordings): bit for bit in the
status, the total time, getSegmentTimes, the lambda segments and every sample field, except vel / acc / jrk on
the rows whose lambda the reference leaves indeterminate, where the host's defined value is checked instead."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
import traj_scale_bindings as SB
from motion_primitive_library_b200 import planner as P
from reference_record import same_array

VEL, ACC, JRK = 0x01, 0x03, 0x07
SCALE, SCALE_DOWN = 1, 2
NS = 50


def roots_same(args):
    got, ref = SB.solve_roots(*args), SB.solve_reference(*args)
    same_array(got, ref, args, bits=True)
    return got


def test_root_solver_branches():
    cases = [
        (0, 1, 0, 1, 1),           # cubic, D > 0
        (0, 1, 0, -3, 2),          # cubic, D = 0: (t - 1)^2 (t + 2)
        (0, 1, -6, 11, -6),        # cubic, D < 0: (t - 1)(t - 2)(t - 3)
        (1, 0, 0, 0, -1),          # quartic, R = 0 (the resolvent's root is exactly 0), E NaN
        (1, 0, 0, 0, 1),           # quartic, D and E NaN
        (1, -10, 35, -50, 24),     # quartic, four real roots
        (1, 0, 1, 0, 1),           # quartic without real roots
        (0, 0, 1, -3, 2),          # a = b = 0: quadratic
        (0, 0, 1, 0, 1),           # quadratic without real roots
        (0, 0, 0, 2, 1),           # linear
        (0, 0, 0, 0, 1),           # constant: no root
        (0, 0, 0, 0, 0),
    ]
    n = [len(roots_same(c)) for c in cases]
    assert n[0] == 1 and n[1] == 2 and n[2] == 3 and n[7] == 2 and n[8] == 0 and n[9] == 1 and n[10] == 0
    assert len(SB.solve_roots(1, 0, 0, 0, -1)) == 2 and n[4] == 0


def test_root_solver_random():
    rng = np.random.default_rng(7)
    for _ in range(200):
        c = rng.normal(size=5) * rng.choice([1e-3, 1, 1e3], 5)
        c[: int(rng.integers(0, 3))] = 0
        roots_same(tuple(float(x) for x in c))


def traj_input(dim, control, yaw, seed, n=None):
    """A TrajSolver output: setPath (no yaw) or setWaypoints with yaws and ACCxYAW-style flags (yaw)."""
    rng = np.random.default_rng(seed)
    n = n or int(rng.integers(2, 25))
    if not yaw:
        r = P.traj_solve(dim, control, pos=np.cumsum(rng.uniform(-2, 2, (n, dim)), axis=0), v=float(rng.uniform(0.5, 2)),
                         n_samples=1)
    else:
        w = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
        w["pos"][:, :dim] = np.cumsum(rng.uniform(-2, 2, (n, dim)), axis=0)
        w["yaw"] = rng.uniform(-3, 3, n)
        r = P.traj_solve(dim, control | 0x10, waypoints=w, wp_control=np.full(n, control | 0x10, dtype=np.uint8),
                         dts=rng.uniform(0.3, 3, n - 1), yaw_control=int(rng.choice([VEL, ACC, JRK])), n_samples=1)
    assert r["segments"] == n - 1
    return r["seg_t"], r["coeff"]


def check(dim, seg_t, coeff, mode, ref=None, **kw):
    got = SB.traj_scale(dim, seg_t, coeff, mode, n_samples=NS, **kw)
    if ref is None:
        ref = SB.scale_reference(dim, seg_t, coeff, mode, n_samples=NS, **kw)
    assert got["status"] == ref["status"]
    assert float(got["total_t"]).hex() == float(ref["total_t"]).hex()
    same_array(got["seg_T"], ref["seg_T"], "seg_T", bits=True)
    same_array(got["lambda"], ref["lambda"], "lambda", bits=True)
    flags = ref["flags"]
    s = got["samples"].copy()
    if flags.any():
        assert got["status"] == 1
        want = SB.end_row_derivatives(dim, seg_t, coeff, got["lambda"])
        for i in np.nonzero(flags)[0]:
            assert s[i, dim:4 * dim].tobytes() == want.tobytes(), i
        s[flags == 1, dim:4 * dim] = 0.0
    same_array(s, ref["samples"], "samples", bits=True)
    return got, ref


CASES = [(dim, control, yaw) for dim in (2, 3) for control in (VEL, ACC, JRK) for yaw in (False, True)]


@pytest.mark.parametrize("dim,control,yaw", CASES)
def test_scale(dim, control, yaw):
    for k, (ri, rf) in enumerate([(1.0, 1.0), (2.0, 0.5), (0.7, 1.3)]):
        seg_t, coeff = traj_input(dim, control, yaw, 100 * dim + 10 * control + k + yaw)
        got, _ = check(dim, seg_t, coeff, SCALE, ri=ri, rf=rf)
        assert got["status"] == 1 and len(got["lambda"]) == 1
        if ri == rf == 1.0:
            assert got["lambda"][0, :4].tolist() == [0.0, 0.0, 0.0, 1.0]


def test_scale_zeroes_small_lambda_coefficients():
    seg_t, coeff = traj_input(3, JRK, False, 5)
    got, _ = check(3, seg_t, coeff, SCALE, ri=1.0, rf=1.0 / (1 + 1e-9))
    a = got["lambda"][0, :4]
    assert a[0] == 0 and a[1] == 0 and a[3] == 1.0


def scale_down_2d(seg_t, coeff, **kw):
    """The 2-D host against the reference's 3-D path with the z coefficients 0."""
    c3 = np.zeros((len(seg_t), 4, 6))
    c3[:, :2] = coeff[:, :2]
    c3[:, 3] = coeff[:, 2]
    ref = SB.scale_reference(3, seg_t, c3, SCALE_DOWN, n_samples=NS, max_bytes=None, **kw)
    cols = [0, 1, 3, 4, 6, 7, 9, 10, 12, 13, 14]
    assert not ref["samples"][:, [2, 5, 8, 11]].any()
    ref2 = dict(ref, samples=ref["samples"][:, cols].copy())
    return check(2, seg_t, coeff, SCALE_DOWN, ref=ref2, **kw)


@pytest.mark.parametrize("dim,control,yaw", CASES)
def test_scale_down(dim, control, yaw):
    statuses = []
    for k, (mv, ri, rf) in enumerate([(0.5, 1.0, 1.0), (0.8, 1.5, 0.5), (1e6, 1.0, 1.0), (0.3, 0.9, 1.1)]):
        seg_t, coeff = traj_input(dim, control, yaw, 1000 * dim + 10 * control + k + yaw)
        if dim == 2:
            got, _ = scale_down_2d(seg_t, coeff, mv=mv, ri=ri, rf=rf)
        else:
            got, _ = check(dim, seg_t, coeff, SCALE_DOWN, mv=mv, ri=ri, rf=rf)
        statuses.append(got["status"])
    assert statuses[2] == 2 and statuses[0] == 1


def planned(dim, control, args):
    """A planned trajectory as segment times and coefficients: each segment's Primitive from its start state
    and the control that state's next derivative holds (Primitive(p, u, t))."""
    t = pb.trajectory_oracle(args, 8)
    assert t["valid"] == 1
    rows = t["waypoints"]
    order = {VEL: 1, ACC: 2, JRK: 3}[control & 0x0F]
    coeff = np.zeros((len(rows) - 1, dim + 1, 6))
    for j in range(len(rows) - 1):
        for k in range(order + 1):  # pos, vel, acc, jrk at c[5], c[4], c[3], c[2]
            coeff[j, :dim, 5 - k] = rows[j, k * dim:(k + 1) * dim]
    return np.diff(rows[:, 4 * dim + 1]), coeff


@pytest.mark.parametrize("control", [ACC, JRK])
def test_planned_corridor(control):
    c = fixtures.corridor()
    a = pb.make_args(2, control, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                     goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0)
    seg_t, coeff = planned(2, control, a)
    check(2, seg_t, coeff, SCALE, ri=1.0, rf=2.0)
    scale_down_2d(seg_t, coeff, mv=0.6, ri=1.0, rf=1.0)


def test_planned_voxel():
    import scenarios as S

    sc = S.scaled(S.cfg3(), 48)
    nodes = sc.frontier(16, seed=4, max_steps=0)
    done = 0
    for q in range(0, 16, 2):
        a = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=nodes["pos"][q]),
                         goal=dict(pos=nodes["pos"][q + 1]), v_max=sc.v_max, a_max=sc.a_max, max_num=600)
        if not pb.trajectory_oracle(a, 8)["valid"]:
            continue
        seg_t, coeff = planned(3, sc.control, a)
        check(3, seg_t, coeff, SCALE_DOWN, mv=0.5 * sc.v_max, ri=1.0, rf=1.0)
        check(3, seg_t, coeff, SCALE, ri=1.2, rf=0.8)
        done += 1
        if done == 2:
            break
    assert done == 2


def test_final_sample_at_the_start_state():
    """sample(N)'s last time can land an ulp past the last lambda segment; getTau then returns -1 and the last
    row is the trajectory's start, on the host as in the reference.  Under scale(1, 1) the last row's tau is
    often exactly the last tf, where the reference's lambda is indeterminate."""
    start_rows = flagged = 0
    for seed in range(30):
        seg_t, coeff = traj_input(3, JRK, False, 50_000 + seed)
        got, _ = check(3, seg_t, coeff, SCALE_DOWN, mv=1.0, ri=1.0, rf=1.0)
        if got["status"] == 1:
            s = got["samples"]
            start_rows += int(s[-1, :3].tobytes() == s[0, :3].tobytes() and s[-1, 14] != 0)
        _, ref = check(3, seg_t, coeff, SCALE, ri=1.0, rf=1.0)
        flagged += int(ref["flags"][-1]) + 100 * int(ref["flags"][:-1].any())
    assert start_rows >= 1 and 1 <= flagged < 100


def test_not_scaled():
    seg_t, coeff = traj_input(2, ACC, False, 3)
    for kw in (dict(ri=0.0), dict(rf=np.inf), dict(mv=-1.0), dict(mv=np.nan)):
        got = SB.traj_scale(2, seg_t, coeff, SCALE_DOWN, n_samples=NS, **kw)
        assert got["status"] == 0 and got["total_t"] == 0 and not got["samples"].any() and len(got["lambda"]) == 0
    bad = seg_t.copy()
    bad[0] = 0.0
    assert SB.traj_scale(2, bad, coeff, SCALE, n_samples=NS)["status"] == 0
    c = coeff.copy()
    c[-1, 2, 0] = np.nan
    assert SB.traj_scale(2, seg_t, c, SCALE, n_samples=NS)["status"] == 0
