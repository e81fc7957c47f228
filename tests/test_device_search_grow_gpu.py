"""The growing device search (mplx_plan_batch_grow, MultiQueryPlanner's DEVICE_GROW path and AUTO for unbounded
plans) must give every query exactly what the lock-step loop and the bounded device searches give: validity, cost
(bit for bit), expansions, the closed set and the action sequence, whatever its arenas' sizes, rounds and reruns.
The rounds, reruns and capacities must follow the schedule include/mplx.h states (restated in
test_search_grow_cpu.schedule from each query's need, measured on the CPU)."""
import ctypes as C

import numpy as np
import pytest

import fixtures
import oracle_bindings as ob
import planner_bindings as pb
import test_device_search_cost_terms_gpu as CT
import test_device_search_paths_gpu as PT
import test_search_grow_cpu as GC
from motion_primitive_library_b200 import abi
from motion_primitive_library_b200 import planner as P
from reference_record import same_array

pytestmark = pytest.mark.gpu
ACC, ACCxYAW = 0x03, 0x13


@pytest.fixture(scope="module")
def sgr(tmp_path_factory):
    return GC.build_sgr(tmp_path_factory.mktemp("sgr"))


def wps(pts, dim=2):
    w = np.zeros(len(pts), dtype=P.WAYPOINT_DTYPE)
    w["pos"][:, :dim] = np.asarray(pts, dtype=np.float64).reshape(len(pts), dim)
    return w


def walled_corridor():
    """The corridor (config 1) with a wall across it at x cell 400: goals beyond it cannot be reached, and their
    unbounded searches exhaust the part of the lattice their start reaches."""
    c = fixtures.corridor()
    g = c["grid"].reshape(199, 799).copy()
    g[:, 400] = 100
    return dict(c, grid=g.reshape(-1))


def corridor_pairs(c, n, seed, n_unreachable=0):
    g = c["grid"].reshape(199, 799)
    rng = np.random.default_rng(seed)
    free = np.argwhere(g == 0)
    left, right = free[free[:, 1] < 390], free[free[:, 1] > 410]
    pos = lambda ij: [(ij[1] + 0.5) * c["res"] + c["origin"][0], (ij[0] + 0.5) * c["res"] + c["origin"][1]]
    S = [pos(left[rng.integers(len(left))]) for _ in range(n)]
    G = [pos(left[rng.integers(len(left))]) for _ in range(n - n_unreachable)]
    G += [pos(right[rng.integers(len(right))]) for _ in range(n_unreachable)]
    return wps(S), wps(G)


def config1_args(c, **kw):
    """test/test_planner_2d.cpp's parameters: ACC, 9 primitives, v_max = a_max = 1, eps 1, max_num -1."""
    return pb.make_args(2, ACC, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                        goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, **kw)


def detail(args, S, G, path, **kw):
    s = P.BatchPlanner(args, path=path)
    try:
        return s.plan_detail(S, G, **kw)
    finally:
        s.close()


def as_dict(d):
    res, tot, acts, closed = d
    return dict(valid=res["valid"], cost=res["cost"], expanded=res["expanded"], n_closed=res["n_closed"],
                actions=acts, closed=closed)


def same(a, b, what=""):
    PT.same_results(a, b, what)


def corridor_env(c, control=ACC, U=None):
    from motion_primitive_library_b200 import MapUtil, env_map

    mu = MapUtil()
    mu.setMap(c["origin"], c["dim"], c["grid"], c["res"])
    e = env_map(mu, device=0)
    e.set_control(control)
    e.set_u(fixtures.U_2d() if U is None else U)
    e.set_dt(1.0)
    e.set_w(10.0)
    e.set_v_max(1.0)
    e.set_a_max(1.0)
    e._sync_params()
    return e


def needs_of(sgr, c, S, G, eps=1.0, max_expand=-1):
    env = ob.OracleEnv(2, ACC, fixtures.U_2d(), c["grid"], c["dim"], c["origin"], c["res"], v_max=1.0, a_max=1.0)
    return [GC.unbounded(sgr, env, ob.wp(S["pos"][q][:2]), ob.wp(G["pos"][q][:2]), eps, max_expand)["need"]
            for q in range(len(S))]


# ---- unbounded batches through every path -----------------------------------------------------------------
def test_config1_unbounded_equals_reference_and_lockstep():
    c = fixtures.corridor()
    args = config1_args(c)
    ref = pb.plan_reference(args)  # MapPlanner::plan with the reference's defaults
    S, G = corridor_pairs(c, 15, seed=3)
    S, G = np.concatenate([wps([c["start"][:2]]), S]), np.concatenate([wps([c["goal"][:2]]), G])
    a = detail(args, S, G, "auto")
    assert a[1]["path"] == "device_grow" and a[1]["grow_lockstep"] == 0
    same(as_dict(a), as_dict(detail(args, S, G, "lockstep")), "lockstep")
    same(as_dict(a), as_dict(detail(args, S, G, "device_grow")), "device_grow")
    # the closed set is recorded in the reference's own order (as a digest): its size is compared here, and its
    # keys through the lock-step loop, which the other GPU tests pin to the reference
    assert a[0]["valid"][0] == ref["valid"] == 1 and a[0]["n_closed"][0] == ref["n_closed"]
    assert a[0]["expanded"][0] == ref["expanded"]
    same_array(a[2][0], ref["actions"], "actions")
    assert a[0]["cost"][0] == ref["cost"]


def test_unbounded_walled_corridor_paths_agree():
    c = walled_corridor()
    args = config1_args(c)
    S, G = corridor_pairs(c, 20, seed=7, n_unreachable=3)
    a = detail(args, S, G, "auto")
    assert a[1]["path"] == "device_grow"
    l = detail(args, S, G, "lockstep")
    same(as_dict(a), as_dict(l), "lockstep")
    same(as_dict(a), as_dict(detail(args, S, G, "device_grow")), "device_grow")
    assert (a[0]["valid"][-3:] == 0).all() and a[0]["valid"][:-3].any()


# ---- the round schedule ------------------------------------------------------------------------------------
def test_forced_rounds_follow_the_schedule(sgr):
    c = walled_corridor()
    S, G = corridor_pairs(c, 12, seed=9, n_unreachable=2)
    needs = needs_of(sgr, c, S, G)
    e = corridor_env(c)
    try:
        one = e.plan_batch_grow(S, G, first_cap=max(needs))
        assert one["rounds"] == 1 and one["reruns"] == 0 and one["searched"].all()
        top = max(needs)
        for rounds in (1, 2, 3):
            cap0 = max(1, -(-top // GC.GROW_FACTOR ** (rounds - 1)))
            want = GC.schedule(needs, cap0, 10 ** 8)
            assert want["rounds"] == rounds
            n0 = e.launch_count()
            r = e.plan_batch_grow(S, G, first_cap=cap0)
            assert e.launch_count() == n0 + want["rounds"]
            for k in ("rounds", "reruns", "first_cap", "last_cap"):
                assert r[k] == want[k], (rounds, k, r[k], want[k])
            assert r["searched"].all()
            same(r, one, f"{rounds} rounds")
        # max_cap below some needs: those queries are not searched, the others are as before
        cut = sorted(needs)[len(needs) // 2]
        want = GC.schedule(needs, 64, cut)
        r = e.plan_batch_grow(S, G, first_cap=64, max_cap=cut)
        assert r["searched"].tolist() == want["searched"].tolist() and not want["searched"].all()
        for k in ("rounds", "reruns", "first_cap", "last_cap"):
            assert r[k] == want[k], k
        for q in np.nonzero(want["searched"] == 0)[0]:
            assert r["valid"][q] == 0 and np.isinf(r["cost"][q]) and r["expanded"][q] == 0
            assert len(r["actions"][q]) == 0 and len(r["closed"][q]) == 0
        for q in np.nonzero(want["searched"])[0]:
            assert r["expanded"][q] == one["expanded"][q] and np.array_equal(r["closed"][q], one["closed"][q])
    finally:
        e.close()


def test_small_result_pool_reruns_and_stays_complete():
    c = walled_corridor()
    S, G = corridor_pairs(c, 16, seed=12, n_unreachable=1)
    e = corridor_env(c)
    try:
        one = e.plan_batch_grow(S, G)
        assert one["reruns"] == 0 and one["rounds"] == 1
        cap = one["first_cap"]
        # a pool of one uint64: every round completes at least the first query that reserves, at one capacity
        r = e.plan_batch_grow(S, G, first_cap=cap, pool_bytes=8)
        assert r["reruns"] > 0 and 1 < r["rounds"] <= len(S) + 1 and r["last_cap"] == cap
        same(r, one, "small pool")
        # the results come back whole, and nothing is written past the caller's arrays
        n = len(S)
        na, nc = sum(len(a) for a in r["actions"]), sum(len(k) for k in r["closed"])
        lib, h = e._lib, e._h
        guard = 64
        aoff = np.full(n + 1 + guard, -3, np.int64)
        coff = np.full(n + 1 + guard, -3, np.int64)
        acts = np.full(na + guard, -3, np.int32)
        keys = np.full(nc + guard, 7, np.uint64)
        abi.check(lib.mplx_plan_batch_grow_results(h, aoff.ctypes.data, acts.ctypes.data, na, coff.ctypes.data,
                                                   keys.ctypes.data, nc))
        assert (aoff[n + 1:] == -3).all() and (coff[n + 1:] == -3).all()
        assert (acts[na:] == -3).all() and (keys[nc:] == 7).all()
        assert aoff[n] == na and coff[n] == nc
        for q in range(n):
            assert np.array_equal(acts[aoff[q]:aoff[q + 1]], r["actions"][q])
            assert np.array_equal(keys[coff[q]:coff[q + 1]], r["closed"][q])
        # a capacity one short is refused with nothing written
        acts2 = np.full(na, -5, np.int32)
        aoff2 = np.full(n + 1, -5, np.int64)
        assert lib.mplx_plan_batch_grow_results(h, aoff2.ctypes.data, acts2.ctypes.data, na - 1, None, None, 0) \
            == abi.MPLX_ERR_ARG
        assert (acts2 == -5).all() and (aoff2 == -5).all()
    finally:
        e.close()


def test_max_cap_queries_go_to_lockstep_through_the_planner(sgr):
    c = walled_corridor()
    args = config1_args(c)
    S, G = corridor_pairs(c, 16, seed=21, n_unreachable=2)
    l = detail(args, S, G, "lockstep")
    needs = needs_of(sgr, c, S, G)
    cut = sorted(needs)[-3]
    want = GC.schedule(needs, 256, cut)
    s = P.BatchPlanner(args, path="device_grow")
    try:
        s.set_grow_caps(256, cut)
        g = s.plan_detail(S, G)
    finally:
        s.close()
    assert g[1]["path"] == "device_grow"
    assert g[1]["grow_lockstep"] == int((want["searched"] == 0).sum()) >= 2
    assert (g[1]["grow_rounds"], g[1]["grow_reruns"], g[1]["grow_last_cap"]) == \
        (want["rounds"], want["reruns"], want["last_cap"])
    same(as_dict(g), as_dict(l), "device_grow with lock-step for the queries past max_cap")


# ---- every instantiation, each with a forced overflow round ---------------------------------------------------
@pytest.mark.parametrize("dim,control", PT.MATRIX, ids=[f"{d}d-{PT.NAME[c]}" for d, c in PT.MATRIX])
def test_occupancy_instantiations_with_overflow(dim, control):
    sc, S, G = PT.matrix_case(dim, control)
    mx = sc.search["max_expand"]
    l = PT.batch_run(sc, S, G, "lockstep")
    env = sc.env()
    try:
        s = sc.search
        r = env.plan_batch_grow(S, G, eps=s["eps"], max_expand=mx, tol_pos=s["tol_pos"], tol_vel=s["tol_vel"],
                                tol_acc=s["tol_acc"], first_cap=8)
        assert r["rounds"] > 1 and r["reruns"] > 0 and r["searched"].all()
        same(r, l, "grow vs lockstep")
    finally:
        env.close()


@pytest.mark.parametrize("dim,order,yaw", CT.MATRIX, ids=[f"{d}d-{o}-{'yaw' if y else 'noyaw'}" for d, o, y in CT.MATRIX])
def test_cost_term_instantiations_with_overflow(dim, order, yaw):
    control = CT.ORDERS[order] | (CT.YAW_BIT if yaw else 0)
    U = CT.control_set(dim, CT.ORDER_OF[order], yaw)
    p = CT.case_params("yaw_pot" if yaw else "pot", yaw)
    w = CT.small_world(dim)
    nq, mx, eps = 8, 40 if dim == 3 else 60, 2.0
    S, G = CT.queries(w, dim, nq, seed=11 + dim, yaw=yaw)
    l = as_dict(detail(CT.args_for(w, dim, control, U, p, mx, eps), S, G, "lockstep"))
    e = CT.env_for(w, dim, control, U, p)
    try:
        r = e.plan_batch_grow(S, G, eps=eps, max_expand=mx, cost_terms=True, first_cap=8)
    finally:
        e.close()
    # a plan whose every successor collides never needs more than its start state
    assert (r["rounds"] > 1 and r["reruns"] > 0) or (r["expanded"] <= 1).all()
    assert r["searched"].all()
    for f in ("valid", "expanded", "n_closed"):
        assert np.array_equal(r[f], l[f]), f
    for q in range(nq):
        assert np.array_equal(r["actions"][q], l["actions"][q]) and np.array_equal(r["closed"][q], l["closed"][q])
    if yaw:
        np.testing.assert_allclose(r["cost"], l["cost"], rtol=1e-12)
    else:
        assert r["cost"].tobytes() == l["cost"].tobytes()


# ---- bounded plans ---------------------------------------------------------------------------------------------
def test_cfg5_bounded_grow_equals_device():
    import cfg5_bench
    import scenarios as S

    sc = S.cfg3()
    q = cfg5_bench.make_queries(sc, 4096, 20.0)
    args = pb.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=q["start"]["pos"][0]),
                        goal=dict(pos=q["goal"]["pos"][0]), v_max=sc.v_max, a_max=sc.a_max, T=sc.T, w=sc.w, max_num=1000,
                        eps=2.0)
    d = detail(args, q["start"], q["goal"], "device")
    g = detail(args, q["start"], q["goal"], "device_grow")
    assert g[1]["path"] == "device_grow" and g[1]["grow_lockstep"] == 0
    assert g[1]["grow_first_cap"] <= g[1]["grow_last_cap"] <= 1 + 1000 * len(sc.U)
    same(as_dict(g), as_dict(d), "cfg5")
    # first_cap at the worst case: one round, as the bounded device search
    s = P.BatchPlanner(args, path="device_grow")
    try:
        s.set_grow_caps(1 + 1000 * len(sc.U), 0)
        one = s.plan_detail(q["start"][:256], q["goal"][:256])
    finally:
        s.close()
    assert one[1]["grow_rounds"] == 1 and one[1]["grow_reruns"] == 0
    d256 = detail(args, q["start"][:256], q["goal"][:256], "device")
    same(as_dict(one), as_dict(d256), "cfg5 worst-case arenas")


def test_huge_cap_refused_by_device_runs_on_grow():
    c = fixtures.corridor()
    S, G = corridor_pairs(c, 16, seed=31)
    args = config1_args(c, max_num=10 ** 7)
    dev = P.BatchPlanner(args, path="device")
    try:
        with pytest.raises(RuntimeError, match="budget"):
            dev.plan(S[:2], G[:2])
    finally:
        dev.close()
    g = detail(args, S, G, "device_grow")
    assert g[1]["path"] == "device_grow"
    same(as_dict(g), as_dict(detail(args, S, G, "lockstep")), "cap 1e7")


# ---- one ctx, every entry point -------------------------------------------------------------------------------
def test_one_ctx_alternating_entry_points_equals_fresh_ctx():
    c = walled_corridor()
    S, G = corridor_pairs(c, 10, seed=41, n_unreachable=1)
    e = corridor_env(c)

    def fresh(fn):
        f = corridor_env(c)
        try:
            return fn(f)
        finally:
            f.close()

    try:
        seq = [
            ("grow", lambda x: x.plan_batch_grow(S, G, first_cap=256)),
            ("batch", lambda x: x.plan_batch(S, G, max_expand=300)),
            ("grow", lambda x: x.plan_batch_grow(S, G)),
            ("cost_terms", lambda x: x.plan_batch_cost_terms(S, G, max_expand=300)),
            ("grow_ct", lambda x: x.plan_batch_grow(S, G, cost_terms=True, first_cap=1000)),
            ("batch", lambda x: x.plan_batch(S[:3], G[:3], max_expand=50)),
            ("grow", lambda x: x.plan_batch_grow(S[:3], G[:3], max_expand=50, first_cap=16)),
        ]
        for name, fn in seq:
            same(fn(e), fresh(fn), name)
        # a map edit, a search region and a new control set between calls
        cells = np.array([[x, y] for x in range(100, 103) for y in range(0, 199)], np.int32)
        idx = cells[:, 0] + 799 * cells[:, 1]
        e.update_cells(idx, np.full(len(idx), 100, np.int8))
        g2 = c["grid"].copy()
        g2[idx] = 100
        c2 = dict(c, grid=g2)
        f = corridor_env(c2)
        try:
            same(e.plan_batch_grow(S, G, first_cap=512), f.plan_batch_grow(S, G, first_cap=512), "update_cells")
            region = np.ones(g2.size, np.uint8)
            region[: g2.size // 4] = 0
            e.set_search_region(region)
            f.set_search_region(region)
            same(e.plan_batch_grow(S, G, cost_terms=True), f.plan_batch_grow(S, G, cost_terms=True), "region")
            e.set_search_region(None)
            f.set_search_region(None)
            U2 = fixtures.U_2d() * 0.5
            e.set_u(U2)
            f.set_u(U2)
            same(e.plan_batch_grow(S, G, first_cap=300), f.plan_batch_grow(S, G, first_cap=300), "set_u")
            same(e.plan_batch(S, G, max_expand=200), f.plan_batch(S, G, max_expand=200), "plan_batch after grow")
        finally:
            f.close()
    finally:
        e.close()


def _grow_results(e, n, n_actions, n_closed):
    aoff, coff = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
    acts, keys = np.zeros(max(n_actions, 1), np.int32), np.zeros(max(n_closed, 1), np.uint64)
    abi.check(e._lib.mplx_plan_batch_grow_results(e._h, aoff.ctypes.data, acts.ctypes.data, acts.size,
                                                  coff.ctypes.data, keys.ctypes.data, keys.size))
    return aoff, acts, coff, keys


def test_bounded_calls_leave_the_grow_results_alone():
    """mplx_plan_batch and mplx_plan_batch_cost_terms search through the same device result pool as
    mplx_plan_batch_grow, but mplx_plan_batch_grow_results keeps returning the last grow call's results."""
    c = walled_corridor()
    S, G = corridor_pairs(c, 10, seed=43, n_unreachable=1)
    e = corridor_env(c)
    try:
        g = e.plan_batch_grow(S, G, first_cap=256)
        na, nc = sum(map(len, g["actions"])), sum(map(len, g["closed"]))
        before = _grow_results(e, len(S), na, nc)
        assert np.array_equal(before[1][:na], np.concatenate(g["actions"]))
        assert np.array_equal(before[3][:nc], np.concatenate(g["closed"]))
        # other queries, so that the bounded calls fill the pool with other keys and actions
        S2, G2 = corridor_pairs(c, 24, seed=44)
        b = e.plan_batch(S2, G2, max_expand=400)
        ct = e.plan_batch_cost_terms(S2[::-1], G2[::-1], max_expand=150)
        assert b["n_closed"].sum() > 0 and ct["n_closed"].sum() > 0
        after = _grow_results(e, len(S), na, nc)
        for x, y in zip(before, after):
            assert np.array_equal(x, y)
    finally:
        e.close()


# ---- refusals ----------------------------------------------------------------------------------------------
def _raw_out(n):
    arrs = dict(valid=np.full(n, -9, np.int32), cost=np.full(n, -9.0), expanded=np.full(n, -9, np.int32),
                n_closed=np.full(n, -9, np.int32), n_actions=np.full(n, -9, np.int32),
                searched=np.full(n, -9, np.int32))
    out = abi.GrowOut(*[arrs[k].ctypes.data for k in ("valid", "cost", "expanded", "n_closed", "n_actions", "searched")],
                      -9, -9, -9, -9, -9, -9, -9.0)
    return arrs, out


def _untouched(arrs, out):
    assert all((a == -9).all() for a in arrs.values())
    assert (out.rounds, out.slots, out.first_cap, out.last_cap, out.arena_bytes, out.reruns, out.seconds) == \
        (-9, -9, -9, -9, -9, -9, -9.0)


def test_refusals_leave_outputs_and_ctx_untouched():
    from motion_primitive_library_b200 import MapUtil, env_map

    c = fixtures.corridor()
    S, G = corridor_pairs(c, 4, seed=51)
    e = corridor_env(c)
    lib = e._lib
    before = e.plan_batch_grow(S, G, first_cap=128)
    kept = [np.zeros(5, np.int64), np.zeros(10 ** 5, np.int32)]
    abi.check(lib.mplx_plan_batch_grow_results(e._h, kept[0].ctypes.data, kept[1].ctypes.data, kept[1].size, None,
                                               None, 0))

    def call(env, cost_terms=0, first_cap=0, max_cap=0, pool=0, n=len(S)):
        arrs, out = _raw_out(len(S))
        n0 = env.launch_count()
        rc = lib.mplx_plan_batch_grow(env._h, cost_terms, S.ctypes.data, G.ctypes.data, None, n, 1.0, -1, 0.5, -1.0,
                                      -1.0, -1.0, 1, first_cap, max_cap, pool, C.byref(out))
        assert rc == abi.MPLX_ERR_ARG, rc
        assert env.launch_count() == n0
        _untouched(arrs, out)

    for kw in (dict(first_cap=-1), dict(max_cap=-1), dict(pool=-8), dict(cost_terms=2), dict(n=-1)):
        call(e, **kw)
    # cost_terms = 0 with a potential map or a yaw control
    e.set_potential_map(np.zeros(c["grid"].size, np.int8))
    e._sync_params()
    call(e, cost_terms=0)
    e.set_potential_map(None)
    y = corridor_env(c, ACCxYAW, fixtures.U_2d_yaw())
    call(y, cost_terms=0)
    y.close()
    # 257 primitives
    wide = corridor_env(c, ACC, np.tile(fixtures.U_2d(), (29, 1))[:257])
    call(wide, cost_terms=1)
    wide.close()
    # missing map or parameters
    h = C.c_void_p()
    abi.check(lib.mplx_create(2, 0, C.byref(h)))
    try:
        arrs, out = _raw_out(len(S))
        assert lib.mplx_plan_batch_grow(h, 1, S.ctypes.data, G.ctypes.data, None, len(S), 1.0, -1, 0.5, -1.0, -1.0,
                                        -1.0, 1, 0, 0, 0, C.byref(out)) == abi.MPLX_ERR_ARG
        _untouched(arrs, out)
    finally:
        lib.mplx_destroy(h)
    # the refused calls left the last call's results in place, and the ctx plans as before
    again = [np.zeros(5, np.int64), np.zeros(10 ** 5, np.int32)]
    abi.check(lib.mplx_plan_batch_grow_results(e._h, again[0].ctypes.data, again[1].ctypes.data, again[1].size, None,
                                               None, 0))
    assert np.array_equal(kept[0], again[0]) and np.array_equal(kept[1], again[1])
    same(e.plan_batch_grow(S, G, first_cap=128), before, "after refusals")
    e.close()


# ---- plan_detail with max_num <= 0 --------------------------------------------------------------------------
def test_plan_detail_unbounded_on_every_path():
    c = walled_corridor()
    args = config1_args(c, max_num=200)
    S, G = corridor_pairs(c, 16, seed=61, n_unreachable=1)
    outs = {p: detail(args, S, G, p, max_num=-1) for p in ("auto", "device_grow", "lockstep")}
    assert outs["auto"][1]["path"] == "device_grow" and outs["lockstep"][1]["path"] == "lockstep"
    same(as_dict(outs["auto"]), as_dict(outs["lockstep"]), "auto")
    same(as_dict(outs["device_grow"]), as_dict(outs["lockstep"]), "device_grow")
    assert outs["lockstep"][0]["expanded"].max() > 200
