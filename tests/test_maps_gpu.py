"""SURVEY.md §8f row 2 on the device: mplx_update_potential_map = MapPlanner::updatePotentialMap,
mplx_set_search_region_path = MapPlanner::setSearchRegion.  Bit-exact against the REFERENCE's own
functions (oracle/_ref planner library, built from the unmodified sources, or its recorded results where
it is not built) and against the literal numpy restatement of the stamping rule
(tests/test_maps_inputs_restatement_vs_ref.py), unknown cells included."""
import numpy as np
import pytest

import oracle_bindings as ob
import planner_bindings as pb
from reference_record import same_array
from parity import assert_expansion_equal

pytestmark = pytest.mark.gpu
ACC = 0x03


def gpu_env(grid, dims, origin, res):
    from motion_primitive_library_b200 import MapUtil, env_map

    mu = MapUtil()
    mu.setMap(origin, dims, grid, res)
    return env_map(mu)


def ref_args(grid, dims, origin, res):
    D = len(dims)
    return pb.make_args(D, ACC, grid, dims, origin, res, np.zeros((1, D)), start=dict(pos=(0,) * D), goal=dict(pos=(0,) * D))


def test_potential_map_3d_matches_reference():
    from test_maps_inputs_restatement_vs_ref import restate_potential

    rng = np.random.default_rng(3)
    for dims, res, rad, powv in (((40, 36, 30), 0.1, (0.5, 0.5, 0.3), 1.0), ((33, 31, 29), 0.25, (1.0, 1.0, 0.5), 1.0),
                                 ((32, 32, 32), 0.1, (0.45, 0.45, 0.45), 1.0)):
        g = (rng.random(int(np.prod(dims))) < 0.015).astype(np.int8) * 100
        g[rng.integers(0, g.size, 50)] = -1  # unknown cells stay untouched unless stamped
        origin = (-1.0, 0.5, 0.0)
        got = gpu_env(g, dims, origin, res).update_potential_map(rad, powv)
        np.testing.assert_array_equal(got, restate_potential(g, dims, origin, res, rad, powv))
        same_array(got, pb.reference_potential_map(ref_args(g, dims, origin, res), rad, g.size))


def test_potential_map_2d_and_source_range():
    import fixtures

    c = fixtures.corridor()
    dims, origin, res = tuple(int(x) for x in c["dim"]), tuple(c["origin"]), c["res"]
    for rad, rng_, pos in (((0.5, 0.5), None, None), ((1.0, 1.0), (4.0, 2.0), (12.0, -1.0))):
        got = gpu_env(c["grid"], dims, origin, res).update_potential_map(rad + (0.0,), 1.0, None if rng_ is None else rng_ + (0.0,),
                                                                          None if pos is None else pos + (0.0,))
        ref = pb.reference_potential_map(ref_args(c["grid"], dims, origin, res), rad, c["grid"].size, rng_, pos)
        same_array(got, ref)
        assert (got > 0).sum() > (c["grid"] > 0).sum()


def test_search_region_matches_reference():
    import fixtures

    c = fixtures.corridor()
    dims, origin, res = tuple(int(x) for x in c["dim"]), tuple(c["origin"]), c["res"]
    path = np.array([[2.5, -3.5], [6.0, -3.0], [6.2, 1.0], [20.0, 2.0], [45.0, 2.5]])  # last point leaves the map
    for dense in (False, True):
        got = gpu_env(c["grid"], dims, origin, res).set_search_region_path(path, (0.5, 0.35), dense)
        ref = pb.reference_search_region(ref_args(c["grid"], dims, origin, res), path, (0.5, 0.35), c["grid"].size, dense)
        same_array(got, ref)
        assert 0 < got.sum() < got.size
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 48)
    path3 = np.array([[-2.0, -2.0, -2.0], [0.0, 1.0, 0.5], [2.0, 2.0, 2.0]])
    got = gpu_env(sc.grid(), sc.dim_cells, sc.origin, sc.res).set_search_region_path(path3, (0.3, 0.3, 0.2))
    ref = pb.reference_search_region(ref_args(sc.grid(), sc.dim_cells, sc.origin, sc.res), path3, (0.3, 0.3, 0.2), sc.grid().size)
    same_array(got, ref)


def test_expansion_after_device_side_potential_and_tunnel():
    """The distance-map planner flow (test/test_distance_map_planner_2d.cpp:77-94): tunnel around a path,
    potential field from the grid, then get_succ — all device-side, against the oracle fed the same arrays."""
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 64)
    env = gpu_env(sc.grid(), sc.dim_cells, sc.origin, sc.res)
    env.set_control(sc.control)
    env.set_u(sc.U)
    env.set_v_max(sc.v_max)
    env.set_potential_weight(0.5)
    path = np.array([[-2.5, -2.5, -2.5], [0.0, 0.0, 0.0], [2.5, 2.5, 2.5]])
    region = env.set_search_region_path(path, (1.5, 1.5, 1.5))
    pot = env.update_potential_map((0.5, 0.5, 0.5))
    nodes = sc.frontier(2000, seed=8)
    o = ob.OracleEnv(3, sc.control, sc.U, pot, sc.dim_cells, sc.origin, sc.res, v_max=sc.v_max, potential=pot,
                     potential_weight=0.5, region=region).expand(nodes, nthreads=8)
    g = env.expand(nodes, want=("succ", "cost", "action", "key", "lattice"))
    st = assert_expansion_equal(g, o)
    assert 0 < st["finite"] < st["successors"]
