"""The device search's bookkeeping on the CPU: mplx_search.cuh (heap, key table, predecessor lists, relax
step, goal test, trace-back), compiled by g++ and fed successors from the oracle's get_succ, must give every
query what the host planner gives with the oracle env (planner_bindings.plan_oracle): validity, cost (bit
for bit), expansions, the closed set and the action sequence."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import fixtures
import oracle_bindings as ob
import planner_bindings as pb

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
VEL, ACC, JRK = 0x01, 0x03, 0x07


def build_sbk(directory):
    """Compile tests/search_bookkeeping_host.cpp with the oracle into directory/libsbk.so and load it."""
    so = Path(directory) / "libsbk.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(so),
                           str(HERE / "search_bookkeeping_host.cpp"), str(ROOT / "oracle" / "mpl_oracle.cpp")])
    L = C.CDLL(str(so))
    vp = C.c_void_p
    L.sbk_plan.argtypes = [C.POINTER(ob.OrcEnv), vp, vp, C.c_double, C.c_int, C.c_double, C.c_double, C.c_double,
                           vp, vp, vp, vp, vp, vp, vp]
    L.sbk_plan.restype = C.c_int
    return L


@pytest.fixture(scope="module")
def sbk(tmp_path_factory):
    return build_sbk(tmp_path_factory.mktemp("sbk"))


def run_sbk(L, env, start, goal, eps, max_expand, tol_pos=0.5, tol_vel=-1.0, tol_acc=-1.0):
    s = np.zeros(1, dtype=ob.WAYPOINT_DTYPE)
    g = np.zeros(1, dtype=ob.WAYPOINT_DTYPE)
    s[0], g[0] = start, goal
    valid, expanded, n_closed, n_actions = (np.zeros(1, np.int32) for _ in range(4))
    cost = np.zeros(1)
    closed = np.zeros(max_expand, np.uint64)
    actions = np.zeros(max_expand, np.int32)
    assert L.sbk_plan(C.byref(env.e), s.ctypes.data, g.ctypes.data, eps, max_expand, tol_pos, tol_vel, tol_acc,
                      valid.ctypes.data, cost.ctypes.data, expanded.ctypes.data, n_closed.ctypes.data,
                      closed.ctypes.data, actions.ctypes.data, n_actions.ctypes.data) == 0
    return dict(valid=int(valid[0]), cost=float(cost[0]), expanded=int(expanded[0]), n_closed=int(n_closed[0]),
                closed=closed[: n_closed[0]].copy(), actions=actions[: n_actions[0]].copy())


def check_same(mine, ref):
    assert mine["valid"] == ref["valid"]
    assert mine["expanded"] == ref["expanded"]
    assert mine["n_closed"] == ref["n_closed"]
    assert np.array_equal(mine["closed"], np.sort(ref["closed"]))
    assert np.array_equal(mine["actions"], ref["actions"])
    if ref["valid"]:
        assert np.float64(mine["cost"]).tobytes() == np.float64(ref["cost"]).tobytes()
    else:
        assert np.isinf(mine["cost"])


def corridor_points(n, seed):
    c = fixtures.corridor()
    rng = np.random.default_rng(seed)
    free = np.nonzero(c["grid"].reshape(199, 799) == 0)
    pick = rng.choice(len(free[0]), size=2 * n, replace=False)
    pts = np.stack([(free[1][pick] + 0.5) * c["res"] + c["origin"][0], (free[0][pick] + 0.5) * c["res"] + c["origin"][1]], 1)
    return c, pts[:n], pts[n:]


@pytest.mark.parametrize("control,eps,tol", [(ACC, 1.0, {}), (ACC, 2.0, {}), (ACC, 0.0, {}), (VEL, 1.0, {}),
                                             (ACC, 1.0, dict(tol_vel=0.5)), (ACC, 1.0, dict(tol_vel=1.0, tol_acc=0.5))])
def test_corridor_matches_host_planner(sbk, control, eps, tol):
    c, S, G = corridor_points(6, seed=3)
    U = fixtures.U_2d()
    if control == VEL:
        U = U * 2.0
    # the corridor's own start/goal, a start that is already a goal, a start on an occupied cell
    occ = np.argwhere(c["grid"].reshape(199, 799) == 100)[0]
    occ_pos = np.array([(occ[1] + 0.5) * c["res"] + c["origin"][0], (occ[0] + 0.5) * c["res"] + c["origin"][1]])
    starts = [np.asarray(c["start"]), S[0]] + list(S[1:])
    goals = [np.asarray(c["goal"]), S[0] + 0.1] + list(G[1:])
    starts.append(occ_pos)
    goals.append(G[0])
    max_num = 400
    for s, g in zip(starts, goals):
        args = pb.make_args(2, control, c["grid"], c["dim"], c["origin"], c["res"], U, start=dict(pos=s),
                            goal=dict(pos=g), v_max=1.0, a_max=1.0, eps=eps, max_num=max_num, **tol)
        ref = pb.plan_oracle(args)
        env = ob.OracleEnv(2, control, U, c["grid"], c["dim"], c["origin"], c["res"], v_max=1.0, a_max=1.0)
        mine = run_sbk(sbk, env, ob.wp(s), ob.wp(g), eps, max_num, tol_vel=tol.get("tol_vel", -1.0),
                       tol_acc=tol.get("tol_acc", -1.0))
        check_same(mine, ref)


def test_voxel_map_matches_host_planner(sbk):
    import scenarios as S

    sc = S.scaled(S.cfg3(), 32)
    nodes = sc.frontier(12, seed=7, max_steps=0)
    env = ob.OracleEnv.from_scenario(sc)
    for q in range(6):
        s, g = nodes["pos"][q], nodes["pos"][6 + q]
        args = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=s),
                            goal=dict(pos=g), T=sc.T, w=sc.w, v_max=sc.v_max, a_max=sc.a_max, eps=2.0, max_num=60)
        ref = pb.plan_oracle(args)
        mine = run_sbk(sbk, env, ob.wp(s), ob.wp(g), 2.0, 60)
        check_same(mine, ref)
