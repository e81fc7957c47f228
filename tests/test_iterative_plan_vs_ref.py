"""MapPlanner::iterativePlan (src/mpl_planner/map_planner.cpp:393-433): replanning inside a tunnel
(setSearchRegion, :46-95) around the previous trajectory until the cost stops changing.  The host
planner's restatement, driven by the CPU oracle env, against the reference's own code: the final
plan's validity, cost, closed set, open-set size and action sequence must be identical — which also
pins the checker env's CPU tunnel builder against the reference's setSearchRegion."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
from reference_record import same_array
ACC, JRK = 0x03, 0x07


def same(a, b):
    fa, la = a
    fb, lb = b
    for k in ("valid", "cost", "n_closed", "n_open", "n_actions"):
        assert fa[k] == fb[k], ("first", k, fa[k], fb[k])
    assert la["ok"] == lb["ok"] and la["valid"] == lb["valid"]
    assert la["n_closed"] == lb["n_closed"] and la["n_open"] == lb["n_open"]
    same_array(la["closed"], lb["closed"], "closed")
    same_array(la["actions"], lb["actions"], "actions")
    if lb["valid"]:
        assert la["cost"] == lb["cost"]


@pytest.mark.parametrize("radius,max_iter", [((0.5, 0.5), 3), ((0.15, 0.15), 3), ((1.0, 0.3), 1)])
def test_corridor_tunnel_replanning(radius, max_iter):
    c = fixtures.corridor()
    a = pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                     goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0)
    ref = pb.iterative_reference(a, radius, max_iter)
    assert ref[0]["valid"] == 1 and ref[1]["ok"] == 1
    assert ref[1]["n_closed"] <= ref[0]["n_closed"]          # the tunnel prunes the search
    got = pb.iterative_oracle(a, radius, max_iter)
    same(got, ref)
    assert 1 <= got[1]["iterations"] <= max_iter


def test_corridor_with_potential_field():
    """test/test_distance_map_planner_2d.cpp's setting: a potential field makes the tunnel-constrained
    replans cost something different from the first plan, so more than one iteration runs."""
    c = fixtures.corridor()
    a0 = pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                      goal=dict(pos=c["goal"]))
    # the field of the reference's own MapPlanner::updatePotentialMap (radius 0.5 m), used as plain input data
    pot = pb.reference_potential_map(a0, (0.5, 0.5), int(np.prod(c["dim"])), record_all=True)
    assert 0 < (pot > 0).sum() and pot.max() == 100
    a = pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                     goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, potential=pot, potential_weight=0.5)
    ref = pb.iterative_reference(a, (0.5, 0.5), 3)
    got = pb.iterative_oracle(a, (0.5, 0.5), 3)
    assert ref[0]["valid"] == 1
    same(got, ref)


def test_voxel_map_tunnel():
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 64)
    nodes = sc.frontier(16, seed=4, max_steps=0)
    a = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=nodes["pos"][0]),
                     goal=dict(pos=nodes["pos"][1]), v_max=sc.v_max, a_max=sc.a_max, max_num=4000)
    ref = pb.iterative_reference(a, (0.6, 0.6, 0.4), 3)
    assert ref[0]["valid"] == 1
    same(pb.iterative_oracle(a, (0.6, 0.6, 0.4), 3), ref)
