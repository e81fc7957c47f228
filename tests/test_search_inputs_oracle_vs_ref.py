"""Pins the oracle planner (planner_bindings.plan_oracle: the host A* on the CPU oracle env) against the reference
planner on the input classes of tests/test_device_search_paths_gpu.py, before the device-search tests rely on it:
2-D JRK/SNP and 3-D VEL plans, control sets of 1 to 256 primitives (products and random rows, with dynamic
limits that reject some of them), eps 0/1/2/5 with re-opened states, equal-f ties, max_expand 1 and a goal popped
at the cap, the tolerances, and goals and starts of every class.  The bar: validity, cost bits, expansions, the
closed set and the action sequence.  The reference's results are recorded under tests/golden/reference
(tests/reference_record.py), so these run without oracle/_ref too."""
import numpy as np
import pytest

import planner_bindings as pb
import test_device_search_paths_gpu as ds
from reference_record import reference, same_array


def plan_reference(args):
    """pb.plan_reference, with the cost of a plan that found no trajectory recorded as +inf: the reference
    leaves getTrajCost() unset when the start is not free, so that value differs from run to run."""
    def live():
        lib, fn = pb.bind(pb.REF_PLANNER, "refp_plan", "mplh_plan")
        r = pb.run_plan(fn, lib, args)
        if not r["valid"]:
            r["cost"] = float("inf")
        return r

    return reference(pb.REF_PLANNER, live)


def same_as_reference(sc, S, G):
    for q in range(len(S)):
        a = sc.args(S[q], G[q])
        o, r = pb.plan_oracle(a), plan_reference(a)
        assert o["valid"] == r["valid"], q
        # the reference keeps its expansion count only when the goal was reached (graph_search.h:173)
        assert o["expanded"] == r["expanded"] or (not r["valid"] and r["expanded"] == 0), q
        assert o["n_closed"] == r["n_closed"], q
        same_array(o["closed"], r["closed"], ("closed", q))
        same_array(o["actions"], r["actions"], ("actions", q))
        if r["valid"]:
            assert np.float64(o["cost"]).tobytes() == np.float64(r["cost"]).tobytes(), q


@pytest.mark.parametrize("dim,control", [(2, ds.JRK), (2, ds.SNP), (3, ds.VEL)])
def test_instantiation_inputs(dim, control):
    same_as_reference(*ds.matrix_case(dim, control))


@pytest.mark.parametrize("nU,kind,dim", ds.WIDTH_CASES, ids=[f"{n}-{k}-{d}d" for n, k, d in ds.WIDTH_CASES])
def test_control_set_width_inputs(nU, kind, dim):
    sc = ds.width_scene(nU, kind, dim)
    same_as_reference(sc, *ds.random_queries(sc, 8, seed=nU + 7 * dim, near=(1.5, 3.0)))


@pytest.mark.parametrize("eps", [0.0, 1.0, 2.0, 5.0])
def test_eps_inputs(eps):
    same_as_reference(*ds.eps_case(eps))


def test_equal_f_tie_inputs():
    sc, S, G = ds.tie_case()
    for mx in (2, 3, 150):
        same_as_reference(sc.with_(max_expand=mx), S, G)


def test_max_expand_inputs():
    sc, S, G, q, cap = ds.cap_case()
    same_as_reference(sc.with_(max_expand=1), S, G)
    for mx in (cap, cap - 1):
        same_as_reference(sc.with_(max_expand=mx), S[q:q + 1], G[q:q + 1])


@pytest.mark.parametrize("tol", ds.TOLERANCES)
def test_tolerance_inputs(tol):
    sc, S, G = ds.tolerance_case()
    same_as_reference(sc.with_(**tol), S, G)


def test_goal_class_inputs():
    sc, S, G, _ = ds.goal_class_case()
    same_as_reference(sc, S, G)
    same_as_reference(*ds.tol_pos_zero_case())


def test_start_class_inputs():
    sc, S, G, _ = ds.start_class_case()
    same_as_reference(sc, S, G)
