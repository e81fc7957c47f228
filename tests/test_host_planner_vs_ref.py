"""Pins the host side (row a10): this repository's planner (mpl_host.hpp: heap, state space, A*,
recoverTraj) against the REFERENCE's own MapPlanner::plan(), compiled unmodified from
/root/reference (graph_search.h, state_space.h, planner_base.h, map_planner.cpp) with the
Eigen/Boost stand-ins of oracle/shim.  Both use a CPU env here; everything must agree exactly:
validity, cost, expansion count, closed set (lattice keys), open-set size, action sequence.
Also pins the potential-field generator against MapPlanner::updatePotentialMap.  Where oracle/_ref is
not built, the reference's side is its recorded results (tests/reference_record.py)."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
from reference_record import same_array
ACC, JRK, ACCxYAW, VEL = 0x03, 0x07, 0x13, 0x01


def same(a, b):
    assert a["valid"] == b["valid"]
    # the reference stores expand_iteration_ only when the goal was reached (graph_search.h:173), so
    # getExpandedNum() is 0 after a max-expand / empty-queue abort; A* closes one state per iteration
    assert a["expanded"] == (b["expanded"] if b["valid"] else b["n_closed"])
    assert a["n_closed"] == b["n_closed"] and a["n_open"] == b["n_open"]
    same_array(a["closed"], b["closed"], "closed")
    same_array(a["actions"], b["actions"], "actions")
    if b["valid"]:
        assert a["cost"] == b["cost"]


def test_config1_test_planner_2d():
    """test/test_planner_2d.cpp on data/corridor.yaml (BASELINE.json configs[0])."""
    c = fixtures.corridor()
    a = pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                     goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0)
    ref = pb.plan_reference(a)
    assert ref["valid"] == 1 and ref["expanded"] > 100
    same(pb.plan_oracle(a), ref)


def test_corridor_yaw_and_eps_and_max_expand():
    c = fixtures.corridor()
    for kw in (dict(control=ACCxYAW, U=fixtures.U_2d_yaw(), yaw_max=0.7, max_num=3000), dict(control=ACC, U=fixtures.U_2d(), eps=2.0),
               dict(control=ACC, U=fixtures.U_2d(), max_num=77), dict(control=VEL, U=fixtures.U_2d(1.0, 1.0), eps=1.0)):
        control, U = kw.pop("control"), kw.pop("U")
        a = pb.make_args(2, control, c["grid"], c["dim"], c["origin"], c["res"], U, start=dict(pos=c["start"]),
                         goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, **kw)
        same(pb.plan_oracle(a), pb.plan_reference(a))


def test_3d_voxel_maps_acc_and_jrk():
    import scenarios as S

    for sc, maxn in ((S.scaled(S.cfg_headline(), 64), 1500), (S.scaled(S.cfg3(), 48), 300)):
        nodes = sc.frontier(16, seed=4, max_steps=0)
        for q in range(0, 16, 2):
            a = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U,
                             start=dict(pos=nodes["pos"][q]), goal=dict(pos=nodes["pos"][q + 1]), v_max=sc.v_max,
                             a_max=sc.a_max, max_num=maxn)
            same(pb.plan_oracle(a), pb.plan_reference(a))


def test_potential_field_generator_vs_updatePotentialMap():
    import scenarios as S

    rng = np.random.default_rng(2)
    for dims, res, rad in (((30, 28, 26), 0.1, (0.5, 0.5, 0.3)), ((24, 24, 24), 0.25, (1.0, 1.0, 0.5))):
        g = (rng.random(int(np.prod(dims))) < 0.02).astype(np.int8) * 100
        a = pb.make_args(3, ACC, g, dims, (0.0, 0.0, 0.0), res, np.zeros((1, 3)), start=dict(pos=(0, 0, 0)),
                         goal=dict(pos=(0, 0, 0)))
        ref = pb.reference_potential_map(a, rad, g.size)
        same_array(S.potential_from_map(g, dims, res, rad), ref)


def test_heuristic_with_dynamics_is_not_provided():
    """setHeurIgnoreDynamics(false) selects env_base::cal_heur's minimum-time branches (env_base.h:66-211),
    which SURVEY.md §2 puts outside the expansion path: the host planner reports it and keeps the default
    (admissible) Linf heuristic, so the plan is the default plan."""
    c = fixtures.corridor()
    kw = dict(start=dict(pos=c["start"]), goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0)
    a = pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), heur_ignore_dynamics=False, **kw)
    b = pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), **kw)
    same(pb.plan_oracle(a), pb.plan_oracle(b))

