"""Pins the oracle planner (planner_bindings.plan_oracle: the host A* on the CPU oracle env) against the reference
planner on the inputs of tests/test_device_search_cost_terms_gpu.py, before the cost-term device-search tests rely
on the oracle env: the instantiation matrix (2-D/3-D x VEL/ACC/JRK/SNP x yaw/no yaw) crossed with a potential
field, a field with a gradient weight, wyaw > 0, wyaw 0 with yaw_max, and yaw with a field, and the reference's
distance-map and yaw configurations on the corridor.  The bar: validity, cost bits, expansions, the closed set
and the action sequence.  The reference's results are recorded under tests/golden/reference
(tests/reference_record.py), so these run without oracle/_ref too.

The search-region case of the matrix is not here: the reference planner takes a search region only from a path
(MapPlanner::setSearchRegion), not the arbitrary tunnel of that case; the device search is compared there with the
same bookkeeping driven by the oracle env with that tunnel."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
import test_device_search_cost_terms_gpu as cs
from reference_record import reference, same_array


def plan_reference(args):
    """The reference's MapPlanner::plan() on args, potential map included.  The reference driver installs
    args.potential in its iterativePlan entry only; with max_iter 0 that entry reports the plan() it ran first.
    A plan without a trajectory is recorded with cost +inf and no closed keys or actions: the reference leaves
    getTrajCost() unset then, and the driver exports the closed set only for a trajectory."""
    def live():
        lib, fn = pb.bind(pb.REF_PLANNER, "refp_iterative_plan", "mplh_iterative_plan")
        _, r = pb.run_iterative(fn, lib, args, (0.5,) * args.dim, max_iter=0)
        out = {k: r[k] for k in ("valid", "cost", "expanded", "n_closed", "closed", "actions")}
        if not out["valid"]:
            out.update(cost=float("inf"), closed=np.zeros(0, np.uint64), actions=np.zeros(0, np.int32))
        return out

    return reference(pb.REF_PLANNER, live)


def same_as_reference(mine, ref, what, yaw_cost_tol=None):
    """mine: dict of one query (valid, cost, expanded, n_closed, closed sorted, actions)."""
    assert int(mine["valid"]) == ref["valid"], what
    # the reference keeps its expansion count only when the goal was reached (graph_search.h:173)
    assert int(mine["expanded"]) == ref["expanded"] or (not ref["valid"] and ref["expanded"] == 0), what
    assert int(mine["n_closed"]) == ref["n_closed"], what
    if ref["valid"]:
        same_array(np.sort(np.asarray(mine["closed"], np.uint64)), ref["closed"], ("closed", what))
        same_array(np.asarray(mine["actions"], np.int32), ref["actions"], ("actions", what))
        if yaw_cost_tol is None:
            assert np.float64(mine["cost"]).tobytes() == np.float64(ref["cost"]).tobytes(), what
        else:
            assert abs(mine["cost"] - ref["cost"]) <= yaw_cost_tol * abs(ref["cost"]), what


def query_args(base, S, G, q, dim):
    a = base
    for k in range(3):
        a.start.pos[k] = float(S["pos"][q][k]) if k < dim else 0.0
        a.goal.pos[k] = float(G["pos"][q][k]) if k < dim else 0.0
    a.start.yaw, a.goal.yaw = float(S["yaw"][q]), float(G["yaw"][q])
    return a


NO_REGION = tuple(c for c in cs.CASES if c != "pot_region")


@pytest.mark.parametrize("case", NO_REGION)
@pytest.mark.parametrize("dim,order,yaw", cs.MATRIX, ids=[f"{d}d-{o}-{'yaw' if y else 'noyaw'}" for d, o, y in cs.MATRIX])
def test_matrix_inputs(dim, order, yaw, case):
    control = cs.ORDERS[order] | (cs.YAW_BIT if yaw else 0)
    U = cs.control_set(dim, cs.ORDER_OF[order], yaw)
    p = cs.case_params(case, yaw)
    w = cs.small_world(dim)
    nq, mx, eps = 8, 40 if dim == 3 else 60, 2.0
    S, G = cs.queries(w, dim, nq, seed=11 + dim, yaw=yaw)
    base = cs.args_for(w, dim, control, U, p, mx, eps)
    for q in range(nq):
        a = query_args(base, S, G, q, dim)
        same_as_reference(pb.plan_oracle(a), plan_reference(a), (case, q))


@pytest.mark.parametrize("name", cs.CORRIDOR_CONFIGS)
def test_corridor_configuration_inputs(name):
    args, S, G, _ = cs.corridor_config(name)
    for q in range(len(S)):
        a = query_args(args, S, G, q, 2)
        same_as_reference(pb.plan_oracle(a), plan_reference(a), (name, q))
