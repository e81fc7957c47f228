"""MultiQueryPlanner::iterativePlan (BatchPlanner.iterative_plan, mplh_batch_iterative_plan) against the
single-query MapPlanner::iterativePlan on the GPU env (mplh_iterative_plan), query by query: return value,
iterations, validity, cost bits, expansions, closed keys and actions of the last plan.  tests/test_iterative_plan_gpu.py
and tests/test_iterative_plan_vs_ref.py chain that single-query call to the reference's own iterativePlan.

Covers the corridor at the radii of test_iterative_plan_vs_ref.py, the reference's iterative test's settings (potential
radius 1.0, potential weight 0.5, search radius 0.5, max_iter 10), the 3-D voxel map, and every planner path forced in
turn (AUTO, DEVICE, DEVICE_COST_TERMS, DEVICE_GROW with caps that make it rerun and hand queries to the lock-step
loop, LOCKSTEP).  The queries converge in different rounds, include a blocked start and a start already in the goal,
and the session's own tunnels come back unchanged."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
from motion_primitive_library_b200 import MapUtil, env_map
from motion_primitive_library_b200 import planner as P

pytestmark = pytest.mark.gpu
ACC = 0x03
PATHS = ["auto", "lockstep", "device", "device_cost_terms", "device_grow", "grow_fallback"]


def corridor_queries(c, n, seed):
    """The corridor's own query, then random free start/goal pairs, a blocked start and a start already in the goal."""
    grid = np.asarray(c["grid"]).reshape(tuple(reversed(c["dim"])))
    free = np.argwhere(grid == 0)
    rng = np.random.default_rng(seed)
    res, org = c["res"], np.asarray(c["origin"], float)
    centre = lambda cell: (np.asarray(cell[::-1], float) + 0.5) * res + org  # noqa: E731
    S = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
    G = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
    S["pos"][0, :2], G["pos"][0, :2] = c["start"], c["goal"]
    for q in range(1, n):
        S["pos"][q, :2] = centre(free[rng.integers(len(free))])
        G["pos"][q, :2] = centre(free[rng.integers(len(free))])
    blocked = np.argwhere(grid != 0)
    S["pos"][n - 2, :2] = centre(blocked[len(blocked) // 2])  # a start that is not free
    S["pos"][n - 1] = G["pos"][n - 1]                            # a start already in the goal
    return S, G


def single(args_kw, S, G, radius, max_iter):
    out = []
    for q in range(len(S)):
        a = pb.make_args(start=dict(pos=S["pos"][q, :args_kw["dim"]]), goal=dict(pos=G["pos"][q, :args_kw["dim"]]),
                         **{k: v for k, v in args_kw.items() if k != "dim"}, dim=args_kw["dim"])
        out.append(pb.iterative_plan(a, radius, max_iter))
    return out


def batched(args_kw, S, G, radius, max_iter, path, tunnels=None):
    a = pb.make_args(start=dict(pos=S["pos"][0, :args_kw["dim"]]), goal=dict(pos=G["pos"][0, :args_kw["dim"]]),
                     **{k: v for k, v in args_kw.items() if k != "dim"}, dim=args_kw["dim"])
    s = P.BatchPlanner(a, path="device_grow" if path == "grow_fallback" else path)
    try:
        if path == "grow_fallback":
            s.set_grow_caps(2, 40)  # small arenas: reruns, and queries handed to the lock-step loop
        if tunnels is not None:
            s.set_search_regions(*tunnels)
            before = s.plan_detail(S, G)
        res, its, ok = s.iterative_plan(S, G, radius, max_iter)
        acts, closed = s.kept(res)
        ran = s._last_path()
        if tunnels is not None:  # the caller's tunnels are back
            after = s.plan_detail(S, G)
            for x, y in zip(before[2] + before[3], after[2] + after[3]):
                assert np.array_equal(x, y)
            assert np.array_equal(before[0], after[0])
    finally:
        s.close()
    return res, its, ok, acts, closed, ran


def check(single_out, got):
    res, its, ok, acts, closed, _ = got
    for q, (first, last) in enumerate(single_out):
        assert int(its[q]) == last["iterations"], q
        assert int(ok[q]) == last["ok"], q
        assert int(res["valid"][q]) == last["valid"], q
        if first["valid"]:  # a failed first plan: the single-query call exports its fields only partly
            assert int(res["expanded"][q]) == last["expanded"] and int(res["n_closed"][q]) == last["n_closed"], q
            assert np.float64(res["cost"][q]).tobytes() == np.float64(last["cost"]).tobytes(), q
            assert np.array_equal(acts[q], last["actions"]), q
            assert np.array_equal(closed[q], np.sort(last["closed"])), q


CASES = {}


def case(name):
    if name in CASES:
        return CASES[name]
    c = fixtures.corridor()
    kw = dict(dim=2, control=ACC, grid=c["grid"], mdim=c["dim"], origin=c["origin"], res=c["res"], U=fixtures.U_2d(),
              v_max=1.0, a_max=1.0, max_num=2000)
    if name.startswith("corridor"):
        radius, max_iter = {"corridor-0.5": ((0.5, 0.5), 3), "corridor-0.15": ((0.15, 0.15), 3),
                            "corridor-aniso": ((1.0, 0.3), 1)}[name]
        S, G = corridor_queries(c, 12, seed=len(name))
    elif name == "potential":
        mu = MapUtil()
        mu.setMap(c["origin"], c["dim"], np.asarray(c["grid"], np.int8), c["res"])
        e = env_map(mu, device=0)
        pot = e.update_potential_map((1.0, 1.0))
        e.close()
        kw.update(potential=pot, potential_weight=0.5)
        radius, max_iter = (0.5, 0.5), 10
        S, G = corridor_queries(c, 12, seed=5)
    else:
        import scenarios as SC

        sc = SC.scaled(SC.cfg_headline(), 64)
        nodes = sc.frontier(16, seed=4, max_steps=0)
        kw = dict(dim=3, control=sc.control, grid=sc.grid(), mdim=sc.dim_cells, origin=sc.origin, res=sc.res, U=sc.U,
                  v_max=sc.v_max, a_max=sc.a_max, max_num=4000)
        S = np.zeros(6, dtype=P.WAYPOINT_DTYPE)
        G = np.zeros(6, dtype=P.WAYPOINT_DTYPE)
        for q in range(6):
            S["pos"][q], G["pos"][q] = nodes["pos"][2 * q], nodes["pos"][2 * q + 1]
        S["pos"][5] = G["pos"][5]
        radius, max_iter = (0.6, 0.6, 0.4), 3
    ref = single(kw, S, G, radius, max_iter)
    CASES[name] = (kw, S, G, radius, max_iter, ref)
    return CASES[name]


def make_kw(kw):
    return kw


@pytest.mark.parametrize("name", ["corridor-0.5", "corridor-0.15", "corridor-aniso", "potential", "voxel"])
@pytest.mark.parametrize("path", PATHS)
def test_batch_equals_single_query(name, path):
    kw, S, G, radius, max_iter, ref = case(name)
    got = batched(kw, S, G, radius, max_iter, path)
    check(ref, got)
    ran = got[5]
    if path == "lockstep":
        assert ran["path"] == "lockstep"
    if name == "potential":
        assert len(set(int(i) for i in got[1])) >= 2  # queries converge in different rounds
    # the blocked start fails in round 1 of the first plan: 0 iterations; the start in the goal converges in one
    if kw["dim"] == 2:
        assert int(got[1][-2]) == 0 and not got[2][-2]
    assert int(got[1][-1]) == 1 and got[2][-1] and int(got[0]["valid"][-1]) == 1 and got[0]["cost"][-1] == 0.0


@pytest.mark.parametrize("path", ["device", "lockstep"])
def test_raw_paths_and_restored_tunnels(path):
    kw, S, G, radius, max_iter, ref = case("corridor-0.5")
    # the first plans' trajectories as raw paths give what the batch's own first plan gives
    a = pb.make_args(start=dict(pos=S["pos"][0, :2]), goal=dict(pos=G["pos"][0, :2]),
                     **{k: v for k, v in kw.items() if k != "dim"}, dim=2)
    s = P.BatchPlanner(a, path=path)
    try:
        res0, _, _, _, trajs = s.plan_detail(S, G, trajectories=True)
    finally:
        s.close()
    keep = [q for q in range(len(S)) if res0["valid"][q]]
    raw = [trajs[q]["nodes"]["pos"][:, :2] if len(trajs[q]["nodes"]) else S["pos"][q:q + 1, :2] for q in keep]
    s = P.BatchPlanner(a, path=path)
    try:
        res, its, ok = s.iterative_plan(S[keep], G[keep], radius, max_iter, raw_paths=raw)
    finally:
        s.close()
    for i, q in enumerate(keep):
        first, last = ref[q]
        assert (int(its[i]), int(ok[i])) == (last["iterations"], last["ok"]), q
        assert np.float64(res["cost"][i]).tobytes() == np.float64(last["cost"]).tobytes(), q
    # the session's own tunnels and plans are unchanged by an iterative plan
    tunnels = ([np.stack([S["pos"][q, :2], G["pos"][q, :2]]) for q in range(len(S))], (0.8, 0.8))
    got = batched(kw, S, G, radius, max_iter, path, tunnels=tunnels)
    assert len(got[1]) == len(S)


@pytest.mark.parametrize("path", ["device", "lockstep"])
def test_max_iter_one(path):
    kw, S, G, radius, _, _ = case("corridor-0.5")
    ref = single(kw, S, G, radius, 1)
    check(ref, batched(kw, S, G, radius, 1, path))
