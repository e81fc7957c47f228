"""Pins the host side of the incremental planner (row a10 LPA* + §8f-3): this repository's LPAstar,
StateSpace::updateNode / increaseCost / decreaseCost / getSubStateSpace and MapPlanner::getLinkedNodes /
updateBlockedNodes / updateClearedNodes (mpl_host.hpp), driven by the CPU oracle env, against the
REFERENCE's own code (graph_search.h:194-365, state_space.h:116-285, map_planner.cpp:124-185)
compiled unmodified with the Eigen/Boost stand-ins of oracle/shim, on scripted replanning sessions.
After EVERY step the whole search state must agree: validity, cost, expansion count, trajectory
actions, and a hash over (key, g, rhs, flags) of all states; after LINK the voxel->edges table."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
from reference_record import same_array
ACC, JRK, VEL = 0x03, 0x07, 0x01
FIELDS = ("valid", "n_states", "n_closed", "n_open", "state_hash", "n_linked", "linked_hash", "n_actions")


def same_session(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        for f in FIELDS:
            assert x[f] == y[f], (x["op"], f, x[f], y[f])
        if x["op"] == "plan":
            same_array(x["actions"], y["actions"], "actions")
            if y["valid"]:
                assert x["cost"] == y["cost"] and x["expanded"] == y["expanded"]


def corridor_args(**kw):
    c = fixtures.corridor()
    a = pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                     goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, **kw)
    return a, c


def trajectory_cells(c, ref_first, every=3):
    """cells under the first plan's trajectory (positions integrated from the action ids)"""
    U = fixtures.U_2d()
    p = np.array(c["start"], dtype=float)
    v = np.zeros(2)
    cells = []
    for k, act in enumerate(ref_first["actions"]):
        u = U[act]
        p = p + v + 0.5 * u
        v = v + u
        if k % every == 0:
            cells.append(np.floor((p - np.asarray(c["origin"])) / c["res"]).astype(int))
    return np.asarray(cells, dtype=np.int32)


def test_lpastar_first_plan_matches_reference_and_astar_cost():
    a, c = corridor_args()
    ref = pb.lpa_reference(a, [("plan",)])
    assert ref[0]["valid"] == 1 and ref[0]["n_closed"] > 100
    same_session(pb.lpa_oracle(a, [("plan",)]), ref)
    # LPA* on an unchanged map finds the A* optimum (eps = 1)
    assert ref[0]["cost"] == pb.plan_reference(a)["cost"]


def wall_at(cells, idx, half):
    x, y = cells[idx]
    return np.array([[x, yy] for yy in range(y - half, y + half + 1)], dtype=np.int32)


@pytest.mark.parametrize("idx,half", [(5, 0), (10, 2), (20, 0), (30, 2)])
def test_block_replan_clear_replan_session(idx, half):
    """A new obstacle on the first trajectory, replan, remove it, replan (and a no-op block+clear)."""
    a, c = corridor_args()
    first = pb.lpa_reference(a, [("plan",)])[0]
    cells = trajectory_cells(c, first, every=1)
    wall = wall_at(cells, idx, half)
    script = [("plan",), ("link",), ("block", wall), ("plan",), ("link",), ("clear", wall), ("plan",),
              ("link",), ("block", cells[:3]), ("clear", cells[:3]), ("plan",)]
    ref = pb.lpa_reference(a, script)
    assert ref[1]["n_linked"] > 1000
    assert ref[2]["state_hash"] != ref[0]["state_hash"]            # the block changed the search state
    if idx <= 10:
        assert ref[3]["valid"] == 1 and ref[3]["cost"] >= ref[0]["cost"]
    assert ref[6]["valid"] == 1 and ref[6]["cost"] == ref[0]["cost"]   # obstacle removed: optimum restored
    same_session(pb.lpa_oracle(a, script), ref)


def test_subtree_replanning_session():
    a, c = corridor_args()
    script = [("plan",), ("subtree", 3), ("plan",), ("link",), ("subtree", 2), ("plan",)]
    ref = pb.lpa_reference(a, script)
    assert ref[0]["valid"] == 1 and ref[2]["valid"] == 1 and ref[1]["n_states"] < ref[0]["n_states"]
    same_session(pb.lpa_oracle(a, script), ref)


def integrate_cells(control, U, start_pos, actions, origin, res, T=1.0):
    """cells at the nodes of a trajectory given by action ids (states start at rest)"""
    dim = len(start_pos)
    p, v, acc = np.array(start_pos, dtype=float), np.zeros(dim), np.zeros(dim)
    cells = []
    for act in actions:
        u = np.asarray(U[act][:dim], dtype=float)
        if control == VEL:
            p = p + u * T
        elif control == ACC:
            p, v = p + v * T + 0.5 * u * T * T, v + u * T
        else:
            p, v, acc = p + v * T + 0.5 * acc * T * T + u * T ** 3 / 6, v + acc * T + 0.5 * u * T * T, acc + u * T
        cells.append(np.floor((p - np.asarray(origin)) / res).astype(int))
    return np.asarray(cells, dtype=np.int32)


def voxel_session_args(sc, q, max_num):
    nodes = sc.frontier(16, seed=4, max_steps=0)
    return pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=nodes["pos"][q]),
                        goal=dict(pos=nodes["pos"][q + 1]), v_max=sc.v_max, a_max=sc.a_max, max_num=max_num)


def voxel_script(sc, a, first):
    cells = integrate_cells(sc.control, sc.U, [a.start.pos[k] for k in range(3)], first["actions"], sc.origin, sc.res)
    mid = cells[len(cells) // 2: len(cells) // 2 + 1]
    blob = np.array([mid[0] + (dx, dy, dz) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1)], dtype=np.int32)
    return [("plan",), ("link",), ("block", blob), ("plan",), ("link",), ("clear", blob), ("plan",), ("subtree", 1),
            ("plan",), ("link",), ("block", cells[-2:-1]), ("plan",)]


@pytest.mark.parametrize("which,q", [("acc", 0), ("acc", 4), ("jrk", 2)])
def test_voxel_map_sessions(which, q):
    import scenarios as S

    sc, maxn = (S.scaled(S.cfg_headline(), 64), 4000) if which == "acc" else (S.scaled(S.cfg3(), 48), 600)
    a = voxel_session_args(sc, q, maxn)
    first = pb.lpa_reference(a, [("plan",)])[0]
    if not first["valid"]:
        pytest.skip("no first trajectory within the expansion budget")
    script = voxel_script(sc, a, first)
    ref = pb.lpa_reference(a, script)
    assert ref[1]["n_linked"] > 100
    same_session(pb.lpa_oracle(a, script), ref)


def test_degenerate_updates_match_reference():
    """Cells outside the map (getIndex aliases them onto other voxels, as in the reference), repeated
    cells, an empty list, LINK before any plan-changing step, and clearing cells that were never blocked."""
    a, c = corridor_args()
    first = pb.lpa_reference(a, [("plan",)])[0]
    cells = trajectory_cells(c, first, every=1)
    outside = np.array([[-3, 5], [int(c["dim"][0]) + 2, 7], [4, -1]], dtype=np.int32)
    twice = np.concatenate([cells[8:10], cells[8:10]])
    script = [("plan",), ("link",), ("block", outside), ("plan",), ("block", twice), ("plan",), ("link",),
              ("clear", np.zeros((0, 2), dtype=np.int32)), ("clear", cells[20:22]), ("clear", twice), ("plan",)]
    ref = pb.lpa_reference(a, script)
    assert ref[10]["valid"] == 1
    same_session(pb.lpa_oracle(a, script), ref)
