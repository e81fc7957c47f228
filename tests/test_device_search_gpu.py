"""The device search (mplx_plan_batch, MultiQueryPlanner's device path) must give every query exactly what the
lock-step loop and the single-query planner give: validity, cost (bit for bit), expansions, the closed set
(sorted lattice keys) and the action sequence."""
import numpy as np
import pytest

import fixtures
import planner_bindings as pb
from motion_primitive_library_b200 import abi
from motion_primitive_library_b200 import planner as P

pytestmark = pytest.mark.gpu
VEL, ACC, JRK, SNP, ACCxYAW = 0x01, 0x03, 0x07, 0x0F, 0x13


def both_paths(args, starts, goals, **kw):
    out = {}
    for path in ("device", "lockstep"):
        s = P.BatchPlanner(args, path=path)
        try:
            out[path] = s.plan_detail(starts, goals, **kw)
        finally:
            s.close()
    assert out["device"][1]["path"] == "device" and out["lockstep"][1]["path"] == "lockstep"
    return out["device"], out["lockstep"]


def assert_same(d, l):
    rd, td, ad, cd = d
    rl, tl, al, cl = l
    for f in ("valid", "expanded", "n_closed", "n_actions"):
        assert np.array_equal(rd[f], rl[f]), f
    assert rd["cost"].tobytes() == rl["cost"].tobytes()
    for q in range(len(rd)):
        assert np.array_equal(ad[q], al[q]), q
        assert np.array_equal(cd[q], cl[q]), q
    assert td["nodes"] == int(rd["expanded"].sum()) and td["iterations"] == int(rd["expanded"].max(initial=0))
    assert td["t_pop"] == 0 and td["t_relax"] == 0


def wps(pts, dim):
    w = np.zeros(len(pts), dtype=P.WAYPOINT_DTYPE)
    w["pos"][:, :dim] = pts
    return w


def corridor_set(nq=24, seed=1):
    c = fixtures.corridor()
    rng = np.random.default_rng(seed)
    free = np.nonzero(c["grid"].reshape(199, 799) == 0)
    pick = rng.choice(len(free[0]), size=2 * nq, replace=False)
    pts = np.stack([(free[1][pick] + 0.5) * c["res"] + c["origin"][0], (free[0][pick] + 0.5) * c["res"] + c["origin"][1]], 1)
    return c, pts[:nq], pts[nq:]


def corridor_args(c, control=ACC, U=None, **kw):
    base = dict(v_max=1.0, a_max=1.0, max_num=800)
    base.update(kw)
    return pb.make_args(2, control, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d() if U is None else U,
                        start=dict(pos=c["start"]), goal=dict(pos=c["goal"]), **base)


@pytest.mark.parametrize("control,eps", [(ACC, 1.0), (ACC, 2.0), (ACC, 0.0), (VEL, 1.0), (VEL, 2.0)])
def test_corridor_device_equals_lockstep_and_single(control, eps):
    c, S, G = corridor_set()
    # special queries: the corridor's own pair, start == goal, an occupied start, a start outside the map
    occ = np.argwhere(c["grid"].reshape(199, 799) == 100)[0]
    occ_pos = [(occ[1] + 0.5) * c["res"] + c["origin"][0], (occ[0] + 0.5) * c["res"] + c["origin"][1]]
    S = np.vstack([S, [c["start"][:2], S[0], occ_pos, [-5.0, -5.0]]])
    G = np.vstack([G, [c["goal"][:2], S[0], G[0], G[1]]])
    args = corridor_args(c, control, eps=eps)
    d, l = both_paths(args, wps(S, 2), wps(G, 2))
    assert_same(d, l)
    assert d[0]["valid"].sum() > 0 and (d[0]["valid"] == 0).sum() > 0
    for q in range(0, len(S), 4):
        a = corridor_args(c, control, eps=eps)
        a.start.pos[0], a.start.pos[1] = S[q]
        a.goal.pos[0], a.goal.pos[1] = G[q]
        one = pb.plan_gpu(a)
        assert (one["valid"], one["expanded"], one["n_closed"]) == (d[0]["valid"][q], d[0]["expanded"][q], d[0]["n_closed"][q])
        assert np.array_equal(np.sort(one["closed"]), d[3][q]) and np.array_equal(one["actions"], d[2][q])
        if one["valid"]:
            assert np.float64(one["cost"]).tobytes() == np.float64(d[0]["cost"][q]).tobytes()


@pytest.mark.parametrize("tol", [dict(tol_vel=0.5), dict(tol_vel=1.0, tol_acc=0.5), dict(tol_pos=2.0)])
def test_corridor_goal_tolerances(tol):
    c, S, G = corridor_set(16, seed=4)
    d, l = both_paths(corridor_args(c, ACC, **tol), wps(S, 2), wps(G, 2))
    assert_same(d, l)


def test_blocked_straight_line_goals_and_max_expand():
    # generous position tolerance: many popped states are within tol of the goal, and the walkRay test decides
    c, S, G = corridor_set(24, seed=9)
    d, l = both_paths(corridor_args(c, ACC, tol_pos=8.0, max_num=50), wps(S, 2), wps(G, 2))
    assert_same(d, l)
    assert (d[0]["expanded"] == 50).any()


def test_unreachable_goal_empties_the_heap():
    c = fixtures.corridor()
    g = c["grid"].reshape(199, 799).copy()
    g[:, 400] = 100  # a wall across the corridor
    args = pb.make_args(2, ACC, g, c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                        goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, max_num=20000)
    free = np.nonzero(g == 0)
    left = np.nonzero(free[1] < 30)[0][:2]
    right = np.nonzero(free[1] > 700)[0][:2]
    pos = lambda i: [(free[1][i] + 0.5) * c["res"] + c["origin"][0], (free[0][i] + 0.5) * c["res"] + c["origin"][1]]
    S = wps(np.array([pos(i) for i in left]), 2)
    G = wps(np.array([pos(i) for i in right]), 2)
    d, l = both_paths(args, S, G)
    assert_same(d, l)
    assert (d[0]["valid"] == 0).all() and (d[0]["expanded"] < 20000).all()


@pytest.mark.parametrize("control,n", [(ACC, 64), (JRK, 64), (SNP, 48)])
def test_voxel_map_controls(control, n):
    import scenarios as S

    sc = S.scaled(S.cfg3(), 64)
    U = sc.U
    if control == ACC:
        U = S.cfg_headline().U
    elif control == SNP:
        U = np.array([[x, y, z] for x in (-1.0, 0.0, 1.0) for y in (-1.0, 1.0) for z in (-1.0, 1.0)])
    nodes = sc.frontier(2 * n, seed=5, max_steps=0)
    args = pb.make_args(3, control, sc.grid(), sc.dim_cells, sc.origin, sc.res, U, start=dict(pos=nodes["pos"][0]),
                        goal=dict(pos=nodes["pos"][1]), T=sc.T, w=sc.w, v_max=sc.v_max, a_max=sc.a_max,
                        j_max=sc.j_max, max_num=150, eps=2.0)
    d, l = both_paths(args, nodes[:n].copy(), nodes[n:].copy())
    assert_same(d, l)


def test_two_passes_with_update_cells():
    c, S, G = corridor_set(20, seed=6)
    args = corridor_args(c, ACC)
    dev = P.BatchPlanner(args, path="device")
    lck = P.BatchPlanner(args, path="lockstep")
    try:
        first = dev.plan_detail(wps(S, 2), wps(G, 2))
        assert_same(first, lck.plan_detail(wps(S, 2), wps(G, 2)))
        cells = np.array([[x, y] for x in range(380, 384) for y in range(0, 199)], dtype=np.int32)
        for s in (dev, lck):
            s.update_cells(cells, np.full(len(cells), 100, np.int8))
        second = dev.plan_detail(wps(S, 2), wps(G, 2))
        assert_same(second, lck.plan_detail(wps(S, 2), wps(G, 2)))
        assert dev.map_uploads() == (1, 1)
    finally:
        dev.close()
        lck.close()


def test_refusals_and_automatic_fallback():
    from motion_primitive_library_b200 import MapUtil, env_map

    c, S, G = corridor_set(4, seed=2)
    mu = MapUtil()
    mu.setMap(c["origin"], c["dim"], c["grid"], c["res"])
    e = env_map(mu, device=0)
    e.set_control(ACC)
    e.set_u(fixtures.U_2d())
    e.set_dt(1.0)
    e.set_w(10.0)
    e.set_v_max(1.0)
    e.set_a_max(1.0)
    r = e.plan_batch(wps(S, 2), wps(G, 2), eps=1.0, max_expand=200)
    assert r["slots"] >= 1 and r["arena_bytes"] > 0
    with pytest.raises(abi.MplxError) as ex:
        e.plan_batch(wps(S, 2), wps(G, 2), max_expand=0)
    assert ex.value.code == abi.MPLX_ERR_ARG
    e.set_potential_map(np.zeros(c["grid"].size, np.int8))
    with pytest.raises(abi.MplxError) as ex:
        e.plan_batch(wps(S, 2), wps(G, 2), max_expand=200)
    assert ex.value.code == abi.MPLX_ERR_ARG
    e.close()
    # BatchPlanner keeps the lock-step loop for every plan the device search refuses
    pot = np.zeros(c["grid"].size, np.int8)
    for args, mx in ((corridor_args(c, ACC, potential=pot), 200), (corridor_args(c, ACC), -1),
                     (corridor_args(c, ACCxYAW, U=fixtures.U_2d_yaw()), 200)):
        s = P.BatchPlanner(args, path="device")
        try:
            _, tot = s.plan(wps(S, 2), wps(G, 2), max_num=mx)
            assert tot["path"] == "lockstep"
        finally:
            s.close()


def test_cfg5_full_set_identical():
    import cfg5_bench
    import scenarios as S

    sc = S.cfg3()
    q = cfg5_bench.make_queries(sc, 4096, 20.0)
    args = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=q["start"]["pos"][0]),
                        goal=dict(pos=q["goal"]["pos"][0]), v_max=sc.v_max, a_max=sc.a_max, T=sc.T, w=sc.w, max_num=1000,
                        eps=2.0)
    d, l = both_paths(args, q["start"], q["goal"])
    assert_same(d, l)
    assert d[1]["slots"] < 4096  # arenas are reused
    if pb.ref_planner_available():
        for k in range(32):
            a = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U,
                             start=dict(pos=q["start"]["pos"][k]), goal=dict(pos=q["goal"]["pos"][k]), v_max=sc.v_max,
                             a_max=sc.a_max, T=sc.T, w=sc.w, max_num=1000, eps=2.0)
            o = pb.plan_reference(a)
            assert o["n_closed"] == d[0]["n_closed"][k] and o["valid"] == d[0]["valid"][k]
            assert np.array_equal(np.sort(o["closed"]), d[3][k]) and np.array_equal(o["actions"], d[2][k])
            if o["valid"]:
                assert o["cost"] == d[0]["cost"][k]


def test_auto_falls_back_to_lockstep_when_search_memory_does_not_fit():
    # a cap whose worst-case arena (1 + max_num*|U| states, about 20 GB here) exceeds any device-memory budget:
    # AUTO keeps the lock-step loop, which served these plans before, and forcing the device search fails
    c = fixtures.corridor()
    S = wps(np.tile(np.asarray(c["start"])[:2], (16, 1)), 2)
    G = wps(np.tile(np.asarray(c["goal"])[:2], (16, 1)), 2)
    big = 10 ** 7
    args = corridor_args(c, ACC, max_num=big)
    auto = P.BatchPlanner(args)
    lck = P.BatchPlanner(args, path="lockstep")
    dev = P.BatchPlanner(args, path="device")
    try:
        res, tot = auto.plan(S, G)
        assert tot["path"] == "lockstep"
        ref, tref = lck.plan(S, G)
        assert np.array_equal(res, ref) and res["cost"].tobytes() == ref["cost"].tobytes()
        assert res["valid"].all()
        with pytest.raises(RuntimeError, match="budget"):
            dev.plan_detail(S[:2], G[:2])
        # the refused detail call left no closed-set collection behind, and the session still plans on the device
        res2, tot2 = dev.plan(S, G, max_num=800)
        assert tot2["path"] == "device" and res2["valid"].all()
        d = dev.plan_detail(S, G, max_num=800)
        assert np.array_equal(d[0], res2)
    finally:
        auto.close()
        lck.close()
        dev.close()


def test_unknown_start():
    c, S, G = corridor_set(16, seed=8)
    grid = c["grid"].reshape(199, 799).copy()
    for k in (0, 3):  # two starts on unknown (-1) cells: never started, as on an occupied cell
        ix = int((S[k][0] - c["origin"][0]) / c["res"])
        iy = int((S[k][1] - c["origin"][1]) / c["res"])
        grid[iy, ix] = -1
    args = pb.make_args(2, ACC, grid, c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                        goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, max_num=800)
    d, l = both_paths(args, wps(S, 2), wps(G, 2))
    assert_same(d, l)
    assert d[0]["expanded"][0] == 0 and d[0]["valid"][0] == 0 and d[0]["expanded"][3] == 0


@pytest.mark.parametrize("dim", [2, 3])
def test_search_region_matches_bookkeeping_on_oracle(tmp_path, dim):
    # inside a tunnel the sample loop reads the region bits (sample_group's non-plain branch); the reference
    # for each query is the same bookkeeping driven on the CPU by the oracle env with the same region
    import oracle_bindings as ob
    import scenarios as Sc
    from test_search_bookkeeping_cpu import build_sbk, run_sbk

    from motion_primitive_library_b200 import MapUtil, env_map

    L = build_sbk(tmp_path)
    if dim == 2:
        c, S, G = corridor_set(12, seed=12)
        grid, mdim, origin, res, U = c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d()
        region = np.ones((199, 799), np.uint8)
        region[60:140, 200:600] = 0  # a hole in the tunnel
        kw = dict(T=1.0, w=10.0, v_max=1.0, a_max=1.0, j_max=-1.0)
        control, mx = ACC, 400
    else:
        sc = Sc.scaled(Sc.cfg3(), 48)
        nodes = sc.frontier(24, seed=4, max_steps=0)
        S, G = nodes["pos"][:12], nodes["pos"][12:]
        grid, mdim, origin, res, U = sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U
        region = np.ones(tuple(int(x) for x in mdim[::-1]), np.uint8)
        region[:, :, : int(mdim[0]) // 3] = 0
        kw = dict(T=sc.T, w=sc.w, v_max=sc.v_max, a_max=sc.a_max, j_max=sc.j_max)
        control, mx = sc.control, 80
    mu = MapUtil()
    mu.setMap(origin, mdim, grid, res)
    e = env_map(mu, device=0)
    e.set_control(control)
    e.set_u(U)
    e.set_dt(kw["T"])
    e.set_w(kw["w"])
    e.set_v_max(kw["v_max"])
    e.set_a_max(kw["a_max"])
    e.set_j_max(kw["j_max"])
    r0 = e.plan_batch(wps(S[:, :dim], dim), wps(G[:, :dim], dim), eps=1.0, max_expand=mx)
    e.set_search_region(region.reshape(-1))
    r = e.plan_batch(wps(S[:, :dim], dim), wps(G[:, :dim], dim), eps=1.0, max_expand=mx)
    e.close()
    env = ob.OracleEnv(dim, control, U, grid, mdim, origin, res, region=region.reshape(-1), **kw)
    for q in range(len(S)):
        ref = run_sbk(L, env, ob.wp(S[q][:dim]), ob.wp(G[q][:dim]), 1.0, mx)
        assert (r["valid"][q], r["expanded"][q], r["n_closed"][q]) == (ref["valid"], ref["expanded"], ref["n_closed"])
        assert np.array_equal(r["closed"][q], ref["closed"]) and np.array_equal(r["actions"][q], ref["actions"])
        assert np.float64(r["cost"][q]).tobytes() == np.float64(ref["cost"]).tobytes()
    # the tunnel changed what the searches did
    assert any(not np.array_equal(a, b) for a, b in zip(r0["closed"], r["closed"]))
    if dim == 2:
        assert r["valid"].sum() > 0


def _raw_plan_batch(lib, h, nq, max_expand):
    """mplx_plan_batch with sentinel-filled outputs: returns (rc, outputs)."""
    S = wps(np.zeros((nq, 2)), 2)
    o = dict(valid=np.full(nq, 7, np.int32), cost=np.full(nq, 7.0), expanded=np.full(nq, 7, np.int32),
             n_closed=np.full(nq, 7, np.int32), aoff=np.full(nq + 1, 7, np.int64),
             acts=np.full(max(1, nq * max(max_expand, 1)), 7, np.int32), coff=np.full(nq + 1, 7, np.int64),
             keys=np.full(max(1, nq * max(max_expand, 1)), 7, np.uint64))
    out = abi.BatchOut(o["valid"].ctypes.data, o["cost"].ctypes.data, o["expanded"].ctypes.data, o["n_closed"].ctypes.data,
                       o["aoff"].ctypes.data, o["acts"].ctypes.data, o["acts"].size, o["coff"].ctypes.data,
                       o["keys"].ctypes.data, o["keys"].size, 7, 7, 7.0)
    rc = lib.mplx_plan_batch(h, S.ctypes.data, S.ctypes.data, None, nq, 1.0, max_expand, 0.5, -1.0, -1.0, -1.0,
                             __import__("ctypes").byref(out))
    o["meta"] = (out.slots, out.arena_bytes, out.seconds)
    return rc, o


def _untouched(o):
    return all((v == 7).all() for k, v in o.items() if k != "meta") and o["meta"] == (7, 7, 7.0)


def test_refusals_leave_outputs_and_ctx_untouched():
    import ctypes as C

    from motion_primitive_library_b200 import MapUtil, env_map

    lib = abi.load()
    # no map, no parameters
    h = C.c_void_p()
    assert lib.mplx_create(2, 0, C.byref(h)) == abi.MPLX_OK
    rc, o = _raw_plan_batch(lib, h, 3, 50)
    assert rc == abi.MPLX_ERR_ARG and _untouched(o)
    assert lib.mplx_plan_batch_fits(h, 3, 50, 1, None, None) == abi.MPLX_ERR_ARG
    lib.mplx_destroy(h)

    c = fixtures.corridor()
    mu = MapUtil()
    mu.setMap(c["origin"], c["dim"], c["grid"], c["res"])

    def make(control, U):
        e = env_map(mu, device=0)
        e.set_control(control)
        e.set_u(U)
        e.set_dt(1.0)
        e.set_w(10.0)
        e.set_v_max(1.0)
        e.set_a_max(1.0)
        e._sync_params()
        return e

    many = np.array([[0.01 * i, 0.0] for i in range(300)])  # nU = 300 > 256
    for control, U, mx in ((ACCxYAW, fixtures.U_2d_yaw(), 50), (ACC, many, 50), (ACC, fixtures.U_2d(), 0),
                           (ACC, fixtures.U_2d(), -3)):
        e = make(control, U)
        n0 = e.launch_count()
        rc, o = _raw_plan_batch(lib, e.handle, 3, mx)
        assert rc == abi.MPLX_ERR_ARG and _untouched(o), (control, len(U), mx)
        assert e.launch_count() == n0
        e.close()
    # memory that does not fit: refused with MPLX_ERR_ALLOC before anything is touched, and the ctx still plans
    e = make(ACC, fixtures.U_2d())
    c2, S, G = corridor_set(4, seed=2)
    before = e.plan_batch(wps(S, 2), wps(G, 2), max_expand=200)
    n0 = e.launch_count()
    slots, nbytes = C.c_int32(-1), C.c_int64(-1)
    assert lib.mplx_plan_batch_fits(e.handle, 3, 10 ** 9, 0, C.byref(slots), C.byref(nbytes)) == abi.MPLX_ERR_ALLOC
    assert (slots.value, nbytes.value) == (-1, -1) and e.launch_count() == n0
    assert lib.mplx_plan_batch_fits(e.handle, 4, 200, 1, C.byref(slots), C.byref(nbytes)) == abi.MPLX_OK
    assert slots.value == before["slots"] and nbytes.value == before["arena_bytes"]
    after = e.plan_batch(wps(S, 2), wps(G, 2), max_expand=200)
    for f in ("valid", "cost", "expanded", "n_closed"):
        assert np.array_equal(before[f], after[f])
    e.close()


def test_voxel_map_single_query_plans():
    import scenarios as S

    sc = S.scaled(S.cfg3(), 64)
    nodes = sc.frontier(32, seed=5, max_steps=0)
    args = pb.make_args(3, JRK, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=nodes["pos"][0]),
                        goal=dict(pos=nodes["pos"][1]), T=sc.T, w=sc.w, v_max=sc.v_max, a_max=sc.a_max, max_num=150,
                        eps=2.0)
    s = P.BatchPlanner(args, path="device")
    try:
        res, tot, acts, closed = s.plan_detail(nodes[:16].copy(), nodes[16:].copy())
    finally:
        s.close()
    for q in range(16):
        a = pb.make_args(3, JRK, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=nodes["pos"][q]),
                         goal=dict(pos=nodes["pos"][16 + q]), T=sc.T, w=sc.w, v_max=sc.v_max, a_max=sc.a_max,
                         max_num=150, eps=2.0)
        one = pb.plan_gpu(a)
        assert (one["valid"], one["expanded"], one["n_closed"]) == (res["valid"][q], res["expanded"][q], res["n_closed"][q])
        assert np.array_equal(np.sort(one["closed"]), closed[q]) and np.array_equal(one["actions"], acts[q])
        if one["valid"]:
            assert np.float64(one["cost"]).tobytes() == np.float64(res["cost"][q]).tobytes()
