"""The host's trajectory checks (env_map_host::traverse_trajectory, is_free(Primitive), validate_primitive,
mpl_host.hpp) against the reference's own env_map and validate_primitive (live where oracle/_ref is built, else
their recordings): bit for bit in the status, the cost and every segment's flags, on TrajSolver outputs, planned
trajectories and their time-scaled versions, on occupancy and potential maps, with and without a search region.
The defined behaviours where the reference is undefined are checked on the host against their statement."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
import traj_check_bindings as CB
from motion_primitive_library_b200 import planner as P
from test_traj_scale_vs_ref import planned

VEL, ACC, JRK, YAW = CB.VEL, CB.ACC, CB.JRK, CB.YAW
SCALE, SCALE_DOWN = 1, 2
MDIM3, RES3, ORIGIN3 = (40, 36, 12), 0.25, (-5.0, -4.5, -1.5)
MDIM2, RES2, ORIGIN2 = (48, 40), 0.2, (-4.8, -4.0)


def compare(dim, grid, mdim, origin, res, paths, control, **kw):
    got = CB.traj_check(dim, grid, mdim, origin, res, paths, control, nthreads=4, **kw)
    ref = CB.check_reference(dim, grid, mdim, origin, res, paths, control, **kw)
    assert got["status"].tobytes() == ref["status"].tobytes()
    assert got["cost"].tobytes() == ref["cost"].tobytes(), (got["cost"], ref["cost"])
    assert got["seg_free"].tobytes() == ref["seg_free"].tobytes()
    assert got["seg_valid"].tobytes() == ref["seg_valid"].tobytes()
    return got


def world(dim, seed):
    if dim == 3:
        return CB.random_grid(MDIM3, seed), MDIM3, ORIGIN3, RES3
    return CB.random_grid(MDIM2, seed, p_occ=0.02), MDIM2, ORIGIN2, RES2


def box(dim, mdim, origin, res, margin=0.1):
    """the box the waypoints are drawn from: the map, `margin` of it kept clear on each side (negative: beyond)"""
    lo = np.asarray(origin, dtype=np.float64)
    ext = np.asarray(mdim) * res
    return lo + margin * ext, lo + (1 - margin) * ext


CASES = [(dim, control, yaw) for dim in (2, 3) for control in (VEL, ACC, JRK) for yaw in (False, True)]


@pytest.mark.parametrize("dim,control,yaw", CASES)
def test_solved_occupancy(dim, control, yaw):
    grid, mdim, origin, res = world(dim, 10 * dim + control + yaw)
    lo, hi = box(dim, mdim, origin, res)
    paths, ctl = CB.solved_paths(dim, control, yaw, 24, 100 * dim + control + yaw, lo, hi)
    got = compare(dim, grid, mdim, origin, res, paths, ctl, v_max=2.0, a_max=1.5, j_max=2.0, yaw_max=0.8)
    assert got["status"].all()
    # some paths collide and some do not; some segments fail each check
    assert np.isinf(got["cost"]).any() and (got["cost"] == 0).any()
    real = np.ones(got["seg_free"].size, dtype=bool)
    real[got["offset"][1:] - 1] = False  # every path's last slot holds 0
    assert got["seg_free"][real].any() and not got["seg_free"][real].all()
    if control != VEL or yaw:
        assert not got["seg_valid"][real].all()


@pytest.mark.parametrize("dim,control,yaw", CASES)
def test_solved_leaving_the_map(dim, control, yaw):
    """waypoints beyond the map: samples outside it, segments that leave and come back, ends outside"""
    grid, mdim, origin, res = world(dim, 7 + dim)
    lo, hi = box(dim, mdim, origin, res, margin=-0.15)
    paths, ctl = CB.solved_paths(dim, control, yaw, 24, 300 * dim + control + yaw, lo, hi)
    got = compare(dim, grid, mdim, origin, res, paths, ctl, v_max=1.0)
    assert np.isinf(got["cost"]).any()


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("gradient", [0.0, 0.7])
@pytest.mark.parametrize("with_region", [False, True])
def test_solved_potential(dim, gradient, with_region):
    """a potential field from the reference's updatePotentialMap, with and without a gradient weight and a search
    region"""
    grid, mdim, origin, res = world(dim, 40 + dim)
    grid[grid < 0] = 0
    args = pb.make_args(dim, ACC, grid, mdim, origin, res, np.zeros((1, dim)), start=dict(pos=np.zeros(dim)),
                        goal=dict(pos=np.zeros(dim)))
    pot = pb.reference_potential_map(args, [0.75] * dim, grid.size, record_all=True)
    assert (pot > 0).any() and (pot < 100).any() and (pot >= 100).any()
    region = None
    if with_region:
        rng = np.random.default_rng(dim)
        region = (rng.random(grid.size) < 0.9).astype(np.uint8)
    lo, hi = box(dim, mdim, origin, res)
    paths, ctl = CB.solved_paths(dim, JRK, dim == 2, 24, 500 * dim, lo, hi)
    got = compare(dim, pot, mdim, origin, res, paths, ctl, potential=pot, potential_weight=0.3,
                  gradient_weight=gradient, region=region, v_max=1.5, a_max=2.0, yaw_max=1.0)
    fin = got["cost"][np.isfinite(got["cost"])]
    assert (fin > 0).any()


@pytest.mark.parametrize("dim,control", [(2, ACC), (3, JRK), (3, ACC)])
def test_scaled(dim, control):
    """scale and scale_down results of the host (Trajectory::scale / scale_down) checked with their lambda"""
    grid, mdim, origin, res = world(dim, 60 + dim)
    lo, hi = box(dim, mdim, origin, res)
    paths, ctl = CB.solved_paths(dim, control, False, 16, 700 * dim + control, lo, hi)
    for mode, kw in ((SCALE, dict(ri=0.8, rf=1.5)), (SCALE_DOWN, dict(mv=0.6, ri=1.0, rf=1.0))):
        sc = [P.traj_scale(dim, p["seg_t"], p["coeff"], mode, control=control, n_samples=1, **kw) for p in paths]
        assert any(s["status"] == 1 for s in sc)
        scaled = [dict(total_t=s["total_t"], **{"lambda": s["lambda"]}) for s in sc]
        got = compare(dim, grid, mdim, origin, res, paths, ctl, scaled=scaled, v_max=1.2, a_max=1.0)
        assert got["status"].all()


@pytest.mark.parametrize("control", [ACC, JRK])
def test_planned_corridor(control):
    c = fixtures.corridor()
    a = pb.make_args(2, control, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                     goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0)
    seg_t, coeff = planned(2, control, a)
    paths = [dict(seg_t=seg_t, coeff=coeff)]
    got = compare(2, c["grid"], c["dim"], c["origin"], c["res"], paths, [control], v_max=1.0, a_max=1.0)
    assert got["status"][0] == 1 and got["cost"][0] == 0 and got["seg_free"][:-1].all() and got["seg_valid"][:-1].all()
    sc = P.traj_scale(2, seg_t, coeff, SCALE, control=control, ri=1.0, rf=2.0, n_samples=1)
    compare(2, c["grid"], c["dim"], c["origin"], c["res"], paths, [control], v_max=1.0, a_max=1.0,
            scaled=[dict(total_t=sc["total_t"], **{"lambda": sc["lambda"]})])


def test_planned_voxel():
    import scenarios as S

    sc = S.scaled(S.cfg3(), 48)
    nodes = sc.frontier(16, seed=4, max_steps=0)
    paths = []
    for q in range(0, 16, 2):
        a = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=nodes["pos"][q]),
                         goal=dict(pos=nodes["pos"][q + 1]), v_max=sc.v_max, a_max=sc.a_max, max_num=600)
        if pb.trajectory_oracle(a, 8)["valid"]:
            seg_t, coeff = planned(3, sc.control, a)
            paths.append(dict(seg_t=seg_t, coeff=coeff))
        if len(paths) == 2:
            break
    assert len(paths) == 2
    got = compare(3, sc.grid(), sc.dim_cells, sc.origin, sc.res, paths, sc.control, v_max=sc.v_max, a_max=sc.a_max)
    assert (got["cost"] == 0).all()


def test_ends_in_obstacles_and_grazing():
    """paths that start or end in an occupied cell, and straight paths along a cell boundary"""
    mdim, res, origin = (20, 20), 0.5, (0.0, 0.0)
    grid = np.zeros(400, dtype=np.int8)
    grid[5 + 20 * 5] = 100
    grid[15 + 20 * 12] = 100
    ends = [((2.75, 2.75), (8.0, 8.0)), ((1.0, 1.0), (7.75, 6.25)), ((0.0, 3.0), (9.0, 3.0)), ((3.0, 0.25), (3.0, 9.99)),
            ((-0.01, 4.0), (5.0, 4.0)), ((2.5, 2.5), (2.5, 2.5 + 1e-9))]
    paths = [P.traj_solve(2, ACC, pos=np.array(e), v=1.0, n_samples=1) for e in ends]
    paths = [dict(seg_t=p["seg_t"], coeff=p["coeff"]) for p in paths]
    got = compare(2, grid, mdim, origin, res, paths, ACC, v_max=1.0)
    # x = 0 is floatToInt's cell round(-0.5) = -1: the path along the map's edge starts outside it
    assert np.isinf(got["cost"][:3]).all() and got["cost"][3] == 0 and np.isinf(got["cost"][4])


def test_stationary_segments():
    """a segment that does not move: is_free samples at t = NaN (outside the map), so it is not free"""
    grid, mdim, origin, res = world(2, 3)
    grid[:] = 0
    w = np.zeros(3, dtype=P.WAYPOINT_DTYPE)
    w["pos"][:, :2] = [[0.0, 0.0], [0.0, 0.0], [1.0, 0.5]]
    r = P.traj_solve(2, ACC, waypoints=w, wp_control=np.full(3, ACC, dtype=np.uint8), dts=[1.0, 1.0], n_samples=1)
    paths = [dict(seg_t=r["seg_t"], coeff=r["coeff"]), dict(seg_t=[1.0], coeff=np.zeros((1, 3, 6)))]
    got = compare(2, grid, mdim, origin, res, paths, ACC, v_max=1.0)
    assert got["seg_free"][0] == 0 and got["seg_free"][1] == 1 and got["seg_free"][3] == 0
    # the stationary path samples one cell: cost 0, evaluated only when N >= 1
    assert got["status"][1] == 1 and got["cost"][1] == 0


@pytest.mark.parametrize("dim,control", [(2, ACC), (3, JRK), (3, ACC | YAW)])
def test_limits_at_the_maxima(dim, control):
    """v_max / a_max (and the yaw limit) just above and just below the trajectory's largest value"""
    grid, mdim, origin, res = world(dim, 80 + dim)
    lo, hi = box(dim, mdim, origin, res)
    yaw = bool(control & YAW)
    paths, ctl = CB.solved_paths(dim, control & 15, yaw, 6, 900 * dim + control, lo, hi)
    vmax = max(CB.max_abs(c[a], t, 1) for p in paths for t, c in zip(p["seg_t"], p["coeff"]) for a in range(dim))
    amax = max(CB.max_abs(c[a], t, 2) for p in paths for t, c in zip(p["seg_t"], p["coeff"]) for a in range(dim))
    for f, want in ((1 + 1e-12, 1), (1 - 1e-12, 0)):
        got = compare(dim, grid, mdim, origin, res, paths, ctl, v_max=vmax * f, a_max=amax * f)
        last = np.cumsum([len(p["seg_t"]) + 1 for p in paths]) - 1
        flags = np.delete(got["seg_valid"], last)
        assert flags.all() if want else not flags.all()


def test_defined_behaviours():
    grid, mdim, origin, res = world(3, 5)
    lo, hi = box(3, mdim, origin, res)
    paths, ctl = CB.solved_paths(3, ACC, False, 4, 11, lo, hi)
    # N < 1: v_max < 0 (the default) or 0 -> status 0, cost 0; the segments are still checked
    for vm in (-1.0, 0.0):
        got = CB.traj_check(3, grid, mdim, origin, res, paths, ctl, v_max=vm)
        assert not got["status"].any() and not got["cost"].any()
        ref = CB.traj_check(3, grid, mdim, origin, res, paths, ctl, v_max=1.0)
        assert got["seg_free"].tobytes() == ref["seg_free"].tobytes()
    # N above MPLX_SAMPLE_N_MAX: status 0
    got = CB.traj_check(3, grid, mdim, origin, res, paths, ctl, v_max=1e9)
    assert not got["status"].any()
    # bad segment time / coefficient, fewer than 2 waypoints: status 0 and no segment results
    bad = [dict(p) for p in paths]
    bad[0]["seg_t"] = np.array(bad[0]["seg_t"]); bad[0]["seg_t"][0] = 0.0
    bad[1]["seg_t"] = np.array(bad[1]["seg_t"]); bad[1]["seg_t"][-1] = np.inf
    bad[2]["coeff"] = np.array(bad[2]["coeff"]); bad[2]["coeff"][0, 1, 3] = np.nan
    bad.append(dict(seg_t=np.zeros(0), coeff=np.zeros((0, 4, 6))))
    got = CB.traj_check(3, grid, mdim, origin, res, bad, np.append(ctl, ACC), v_max=1.0)
    assert got["status"].tolist() == [0, 0, 0, 1, 0] and got["cost"][:3].tolist() == [0, 0, 0]
    o = got["offset"]
    assert not got["seg_free"][:o[3]].any() and not got["seg_valid"][:o[3]].any()


def test_wrapped_index_rule():
    """getIndex of a cell outside the map wraps in 32 bits (defined behaviour 4): with N = 1 the end sample's index
    2^32 wraps to the start's index 0, so the end is not counted and the cost is 0 although the end is outside the
    map; a 64-bit or signed index would count it and give +inf.  With N = 2 the middle sample (index 2^31) differs
    from both, is counted, lies outside and gives +inf."""
    grid, mdim, origin, res, paths = CB.wrapped_index_case()
    one = compare(3, grid, mdim, origin, res, paths, VEL, v_max=1.0 / 65536)
    assert one["status"][0] == 1 and one["cost"][0] == 0
    two = compare(3, grid, mdim, origin, res, paths, VEL, v_max=2.0 / 65536)
    assert two["status"][0] == 1 and np.isinf(two["cost"][0])
