"""The capacity check of the device search's bookkeeping on the CPU: mplx_search.cuh's consume<true>, compiled
by g++ and fed successors from the oracle's get_succ.  Each query is first run unbounded in a large arena for
its result and its need (the larger of its final state and predecessor-record counts).  In an arena of exactly
`need` records it must give that result bit for bit; in any smaller arena it must end in kOverflow and write
nothing.  The round schedule of mplx_plan_batch_grow (include/mplx.h) is restated here from the needs, for the
GPU test to compare the device's counters with."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import fixtures
import oracle_bindings as ob

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
VEL, ACC, JRK = 0x01, 0x03, 0x07
K_OVERFLOW = 5
GROW_FACTOR = 4
GUARD_I, GUARD_F, GUARD_K = -7, -7.5, np.uint64(0xDEADBEEFDEADBEEF)


def build_sgr(directory):
    """Compile tests/search_grow_host.cpp with the oracle into directory/libsgr.so and load it."""
    so = Path(directory) / "libsgr.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(so),
                           str(HERE / "search_grow_host.cpp"), str(ROOT / "oracle" / "mpl_oracle.cpp")])
    L = C.CDLL(str(so))
    vp, i64 = C.c_void_p, C.c_int64
    L.sgr_plan.argtypes = [C.POINTER(ob.OrcEnv), vp, vp, C.c_double, C.c_int, i64, C.c_double, C.c_double,
                           C.c_double, vp, vp, vp, vp, vp, vp, vp, i64, vp, i64, vp]
    L.sgr_plan.restype = C.c_int
    L.sgr_layout_for.argtypes = [C.c_int, C.c_int, vp]
    L.sgr_layout_cap.argtypes = [i64, vp]
    return L


@pytest.fixture(scope="module")
def sgr(tmp_path_factory):
    return build_sgr(tmp_path_factory.mktemp("sgr"))


def run_sgr(L, env, start, goal, eps, cap, max_expand=-1, tol_pos=0.5, tol_vel=-1.0, tol_acc=-1.0, room=1 << 16):
    """One query in an arena of `cap` records.  Returns (status, result dict or None); the result arrays are
    checked to hold their guard values when the query overflowed."""
    s = np.zeros(1, dtype=ob.WAYPOINT_DTYPE)
    g = np.zeros(1, dtype=ob.WAYPOINT_DTYPE)
    s[0], g[0] = start, goal
    status = np.zeros(1, np.int32)
    need = np.full(1, GUARD_I, np.int64)
    valid, expanded, n_closed, n_actions = (np.full(1, GUARD_I, np.int32) for _ in range(4))
    cost = np.full(1, GUARD_F)
    closed = np.full(room, GUARD_K, np.uint64)
    actions = np.full(room, GUARD_I, np.int32)
    assert L.sgr_plan(C.byref(env.e), s.ctypes.data, g.ctypes.data, eps, max_expand, int(cap), tol_pos, tol_vel,
                      tol_acc, status.ctypes.data, need.ctypes.data, valid.ctypes.data, cost.ctypes.data,
                      expanded.ctypes.data, n_closed.ctypes.data, closed.ctypes.data, room, actions.ctypes.data, room,
                      n_actions.ctypes.data) == 0
    if status[0] == K_OVERFLOW:
        for a, v in ((need, GUARD_I), (valid, GUARD_I), (expanded, GUARD_I), (n_closed, GUARD_I),
                     (n_actions, GUARD_I), (actions, GUARD_I)):
            assert (a == v).all()
        assert (cost == GUARD_F).all() and (closed == GUARD_K).all()
        return int(status[0]), None
    assert n_closed[0] <= room and n_actions[0] <= room
    return int(status[0]), dict(need=int(need[0]), valid=int(valid[0]), cost=float(cost[0]),
                                expanded=int(expanded[0]), n_closed=int(n_closed[0]),
                                closed=closed[: n_closed[0]].copy(), actions=actions[: n_actions[0]].copy())


def unbounded(L, env, start, goal, eps, max_expand=-1, **tol):
    """The query's result and need: run in arenas growing by GROW_FACTOR until it does not overflow."""
    cap = 1024
    while True:
        st, r = run_sgr(L, env, start, goal, eps, cap, max_expand, **tol)
        if r is not None:
            return r
        cap *= GROW_FACTOR


def same(a, b):
    assert a["valid"] == b["valid"] and a["expanded"] == b["expanded"] and a["n_closed"] == b["n_closed"]
    assert np.float64(a["cost"]).tobytes() == np.float64(b["cost"]).tobytes()
    assert np.array_equal(a["closed"], b["closed"]) and np.array_equal(a["actions"], b["actions"])


def check_caps(L, env, start, goal, eps, max_expand=-1, **tol):
    ref = unbounded(L, env, start, goal, eps, max_expand, **tol)
    need = ref["need"]
    st, r = run_sgr(L, env, start, goal, eps, max(need, 1), max_expand, **tol)
    assert st != K_OVERFLOW
    same(r, ref)
    assert r["need"] == need
    if need > 1:
        for cap in sorted({need - 1, max(1, need // 2), max(1, need // 4), 1}):
            st, r = run_sgr(L, env, start, goal, eps, cap, max_expand, **tol)
            assert st == K_OVERFLOW and r is None, cap
    return ref


def schedule(needs, cap0, cap_max, factor=GROW_FACTOR):
    """mplx_plan_batch_grow's round schedule (include/mplx.h) from the queries' needs, with a result pool that
    never fills: dict(rounds, reruns, first_cap, last_cap, searched[n])."""
    cap_max = max(1, int(cap_max))
    cap = max(1, min(int(cap0), cap_max))
    out = dict(rounds=0, reruns=0, first_cap=cap, last_cap=0, searched=np.ones(len(needs), np.int32))
    pending = list(range(len(needs)))
    while pending:
        out["rounds"] += 1
        out["last_cap"] = cap
        over = [q for q in pending if needs[q] > cap]
        if cap >= cap_max:
            out["searched"][over] = 0
            break
        out["reruns"] += len(over)
        pending = over
        cap = min(cap * factor, cap_max)
    return out


def corridor_crop():
    """A 6 m x 4 m window of the corridor map (config 1) with a sealed pocket: a goal inside it cannot be
    reached, and a search for it exhausts the window's reachable lattice."""
    c = fixtures.corridor()
    g = c["grid"].reshape(199, 799)[40:120, 20:140].copy()
    g[30:50, 90:110] = 100
    g[36:44, 96:104] = 0  # the pocket, walled in on every side
    origin = np.array([c["origin"][0] + 20 * c["res"], c["origin"][1] + 40 * c["res"]])
    return dict(grid=g.reshape(-1), dim=np.array([120, 80], np.int32), origin=origin, res=c["res"])


def cell_pos(m, ij):
    return np.array([(ij[1] + 0.5) * m["res"] + m["origin"][0], (ij[0] + 0.5) * m["res"] + m["origin"][1]])


def corridor_queries(m, n, seed):
    g = m["grid"].reshape(80, 120)
    rng = np.random.default_rng(seed)
    free = np.argwhere(g == 0)
    free = free[~((free[:, 0] >= 30) & (free[:, 0] < 50) & (free[:, 1] >= 90) & (free[:, 1] < 110))]
    pick = free[rng.choice(len(free), size=2 * n, replace=False)]
    starts = [cell_pos(m, ij) for ij in pick[:n]]
    goals = [cell_pos(m, ij) for ij in pick[n:]]
    goals[-1] = cell_pos(m, (40, 100))  # in the pocket: unreachable
    return starts, goals


@pytest.mark.parametrize("control,eps", [(ACC, 1.0), (ACC, 0.0), (ACC, 2.0), (VEL, 1.0)])
def test_corridor_capacity_boundary(sgr, control, eps):
    m = corridor_crop()
    U = fixtures.U_2d() * (2.0 if control == VEL else 1.0)
    env = ob.OracleEnv(2, control, U, m["grid"], m["dim"], m["origin"], m["res"], v_max=1.0, a_max=1.0)
    starts, goals = corridor_queries(m, 3, seed=11)
    refs = [check_caps(sgr, env, ob.wp(s), ob.wp(g), eps) for s, g in zip(starts, goals)]
    assert refs[-1]["valid"] == 0 and any(r["valid"] for r in refs[:-1])


def test_corridor_bounded_capacity_boundary(sgr):
    """A capped search (max_num 200): the need is below the worst case, and the boundary holds the same way."""
    m = corridor_crop()
    env = ob.OracleEnv(2, ACC, fixtures.U_2d(), m["grid"], m["dim"], m["origin"], m["res"], v_max=1.0, a_max=1.0)
    starts, goals = corridor_queries(m, 2, seed=5)
    for s, g in zip(starts, goals):
        ref = check_caps(sgr, env, ob.wp(s), ob.wp(g), 1.0, max_expand=200)
        assert ref["need"] <= 1 + 200 * 9


@pytest.mark.parametrize("control", [ACC, JRK])
def test_voxel_map_capacity_boundary(sgr, control):
    import scenarios as S

    sc = S.scaled(S.cfg3(), 12)
    env = ob.OracleEnv.from_scenario(sc)
    if control != sc.control:
        env = ob.OracleEnv(3, control, sc.U, sc.grid(), sc.dim_cells, sc.origin, sc.res, T=sc.T, w=sc.w,
                           v_max=sc.v_max, a_max=sc.a_max, j_max=max(sc.a_max, 1.0))
    nodes = sc.frontier(6, seed=7, max_steps=0)
    for q in range(3):
        s, g = nodes["pos"][q], nodes["pos"][3 + q]
        check_caps(sgr, env, ob.wp(s), ob.wp(g), 1.0, max_expand=60)
    # a goal outside the map is never reached: the search ends when its cap or the lattice runs out
    check_caps(sgr, env, ob.wp(nodes["pos"][0]), ob.wp(np.asarray(sc.origin) - 5.0), 1.0, max_expand=60)


def old_layout_for(max_expand, nU):
    """layout_for as it stood before the capacity was split out (SState 152 B, SPred 24 B, SHeapItem 16 B,
    SSlot 16 B, regions rounded up to 256 B)."""
    cap = 1 + max_expand * nU
    tab = 1
    while tab < 2 * cap:
        tab <<= 1
    r = lambda b: (b + 255) & ~255
    st, pr, hp = r(cap * 152), r(cap * 24), r(cap * 16)
    return [cap, tab, st, st + pr, st + pr + hp, st + pr + hp + tab * 16]


def test_layout_for_unchanged(sgr):
    out = np.zeros(6, np.int64)
    out2 = np.zeros(6, np.int64)
    for mx in (1, 2, 7, 60, 400, 1000, 20000, 10 ** 6):
        for nU in (1, 9, 27, 28, 125, 256):
            sgr.sgr_layout_for(mx, nU, out.ctypes.data)
            assert out.tolist() == old_layout_for(mx, nU), (mx, nU)
            sgr.sgr_layout_cap(1 + mx * nU, out2.ctypes.data)
            assert out2.tolist() == out.tolist()


def test_schedule_restatement():
    needs = [5, 40, 700, 3000, 1]
    s = schedule(needs, 10, 10 ** 6)
    # 10: {40, 700, 3000} overflow; 40: {700, 3000}; 160: same; 640: {700, 3000}; 2560: {3000}; 10240: none
    assert (s["rounds"], s["first_cap"], s["last_cap"]) == (6, 10, 10240)
    assert s["reruns"] == 3 + 2 + 2 + 2 + 1 and s["searched"].all()
    s = schedule(needs, 10, 700)
    assert s["last_cap"] == 700 and s["searched"].tolist() == [1, 1, 1, 0, 1]
    assert schedule(needs, 5000, 10 ** 6)["rounds"] == 1
