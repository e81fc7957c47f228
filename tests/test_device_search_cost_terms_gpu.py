"""The cost-term device search (mplx_plan_batch_cost_terms, MultiQueryPlanner's path "device_cost_terms") serves
potential-field, gradient and yaw planning.  Every query is compared with two independent results:
  - the lock-step loop of MultiQueryPlanner: validity, cost bits, expansions, closed set and actions equal;
  - the search bookkeeping (mplx_search.cuh) compiled by g++ and driven by the oracle env on the CPU: without
    yaw the cost bits are equal, with yaw the cost is within 1e-12 relative (the device turns the yaw angle
    with a rotation recurrence, the oracle calls sincos per sample: DESIGN §2) and everything else equal."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import fixtures
import oracle_bindings as ob
import planner_bindings as pb
from motion_primitive_library_b200 import abi
from motion_primitive_library_b200 import planner as P
from reference_record import same_array

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
ORDERS = {"VEL": 0x01, "ACC": 0x03, "JRK": 0x07, "SNP": 0x0F}
ORDER_OF = {"VEL": 1, "ACC": 2, "JRK": 3, "SNP": 4}
YAW_BIT = 0x10
COST_TERMS_MIN_QUERIES = 16  # MultiQueryPlanner::kDeviceCostTermsMinQueries


# ---- which search_kernel<DIM, ORD, YAW, COST> a plan runs (csrc/mplx_search.cu: with_search_kernel) ----
def search_kernel_for(dim, control, cost_terms):
    ord_ = {0x01: 1, 0x03: 2, 0x07: 3, 0x0F: 4}[control & 15]
    if not cost_terms:
        return (dim, ord_, False, False)
    return (dim, ord_, bool(control & YAW_BIT), True)


MATRIX = [(dim, o, yaw) for dim in (2, 3) for o in ORDERS for yaw in (False, True)]
CASES = ("pot", "pot_grad", "pot_region", "wyaw", "wyaw0_yawmax", "yaw_pot")


def test_matrix_reaches_every_cost_term_instantiation():
    got = {search_kernel_for(dim, ORDERS[o] | (YAW_BIT if yaw else 0), True) for dim, o, yaw in MATRIX}
    assert len(got) == 16 and all(k[3] for k in got)
    # the occupancy entry point keeps its own 8 instantiations
    occ = {search_kernel_for(dim, ORDERS[o], False) for dim, o, _ in MATRIX}
    assert len(occ) == 8 and not (occ & got)


# ---- CPU bookkeeping -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sbkc(tmp_path_factory):
    so = tmp_path_factory.mktemp("sbkc") / "libsbkc.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(so),
                           str(HERE / "search_bookkeeping_cost_host.cpp"), str(ROOT / "oracle" / "mpl_oracle.cpp")])
    L = C.CDLL(str(so))
    vp = C.c_void_p
    L.sbkc_plan.argtypes = [C.POINTER(ob.OrcEnv), vp, vp, C.c_double, C.c_int, C.c_double, C.c_double, C.c_double,
                            C.c_double, vp, vp, vp, vp, vp, vp, vp]
    L.sbkc_plan.restype = C.c_int
    return L


def run_sbkc(L, env, start, goal, eps, max_expand, tol_pos=0.5, tol_vel=-1.0, tol_acc=-1.0, tol_yaw=-1.0):
    s = np.zeros(1, dtype=ob.WAYPOINT_DTYPE)
    g = np.zeros(1, dtype=ob.WAYPOINT_DTYPE)
    s[0], g[0] = start, goal
    valid, expanded, n_closed, n_actions = (np.zeros(1, np.int32) for _ in range(4))
    cost = np.zeros(1)
    closed = np.zeros(max_expand, np.uint64)
    actions = np.zeros(max_expand, np.int32)
    assert L.sbkc_plan(C.byref(env.e), s.ctypes.data, g.ctypes.data, eps, max_expand, tol_pos, tol_vel, tol_acc, tol_yaw,
                       valid.ctypes.data, cost.ctypes.data, expanded.ctypes.data, n_closed.ctypes.data,
                       closed.ctypes.data, actions.ctypes.data, n_actions.ctypes.data) == 0
    return dict(valid=int(valid[0]), cost=float(cost[0]), expanded=int(expanded[0]), n_closed=int(n_closed[0]),
                closed=closed[: n_closed[0]].copy(), actions=actions[: n_actions[0]].copy())


def assert_matches_cpu(r, q, ref, yaw):
    assert (int(r["valid"][q]), int(r["expanded"][q]), int(r["n_closed"][q])) == (ref["valid"], ref["expanded"],
                                                                                 ref["n_closed"]), q
    assert np.array_equal(r["closed"][q], ref["closed"]) and np.array_equal(r["actions"][q], ref["actions"]), q
    if not ref["valid"]:
        assert np.isinf(r["cost"][q])
    elif yaw:
        assert abs(r["cost"][q] - ref["cost"]) <= 1e-12 * abs(ref["cost"]), q
    else:
        assert np.float64(r["cost"][q]).tobytes() == np.float64(ref["cost"]).tobytes(), q


# ---- the two GPU paths -----------------------------------------------------------------------------------
def both_paths(args, starts, goals, **kw):
    out = {}
    for path in ("device_cost_terms", "lockstep"):
        s = P.BatchPlanner(args, path=path)
        try:
            out[path] = s.plan_detail(starts, goals, **kw)
        finally:
            s.close()
    assert out["device_cost_terms"][1]["path"] == "device_cost_terms" and out["lockstep"][1]["path"] == "lockstep"
    return out["device_cost_terms"], out["lockstep"]


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


def as_dict(d):
    r, _, acts, closed = d
    return dict(valid=r["valid"], cost=r["cost"], expanded=r["expanded"], n_closed=r["n_closed"], actions=acts,
                closed=closed)


# ---- small maps and plans ---------------------------------------------------------------------------------
def small_world(dim, seed=3):
    """A box map with a potential field: values <= 0 (including -1) free, 1..99 cost, >= 100 block."""
    rng = np.random.default_rng(seed)
    mdim = (48, 40) if dim == 2 else (20, 18, 16)
    res = 0.25
    origin = tuple(-m * res / 2 for m in mdim)
    shape = tuple(reversed(mdim))
    grid = np.zeros(shape, np.int8)
    for _ in range(6 if dim == 2 else 5):
        lo = [rng.integers(0, s - 4) for s in shape]
        sl = tuple(slice(a, a + int(rng.integers(2, 5))) for a in lo)
        grid[sl] = 100
    pot = rng.integers(-1, 60, size=shape).astype(np.int8)
    pot[rng.random(shape) < 0.01] = 100
    pot[grid == 100] = 100
    return dict(grid=grid.reshape(-1), pot=pot.reshape(-1), mdim=mdim, origin=origin, res=res, shape=shape)


def control_set(dim, order, yaw):
    u = {1: 1.0, 2: 1.0, 3: 2.0, 4: 4.0}[order]
    import scenarios as S

    return S.control_set(u, 3, dim, yaw_rates=(-0.5, 0.0, 0.5) if yaw else None)


def queries(w, dim, n, seed, yaw):
    rng = np.random.default_rng(seed)
    free = np.argwhere(w["grid"].reshape(w["shape"]) == 0)
    S = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
    G = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
    for q in range(n):
        a = free[rng.integers(len(free))]
        d = np.sum(np.abs(free - a), 1)
        near = free[(d > 2) & (d < 10)]
        b = near[rng.integers(len(near))] if len(near) else a
        for W, cell in ((S, a), (G, b)):
            W["pos"][q, :dim] = (np.asarray(cell[::-1], float) + 0.5) * w["res"] + np.asarray(w["origin"])
        if yaw:
            # start yaws near +-pi and elsewhere
            S["yaw"][q] = [np.pi - 1e-3, -np.pi + 1e-3, 3.1, -3.1, 0.0, 1.0][q % 6]
            G["yaw"][q] = rng.uniform(-np.pi, np.pi)
    return S, G


def case_params(case, yaw):
    """(potential on, gradient weight, region on, wyaw, yaw_max) of a matrix case."""
    p = dict(pot=True, grad=0.0, region=False, wyaw=1.0, yaw_max=-1.0)
    if case == "pot_grad":
        p["grad"] = 0.3
    elif case == "pot_region":
        p["region"] = True
    elif case == "wyaw":
        p.update(pot=False, wyaw=1.0)
    elif case == "wyaw0_yawmax":
        p.update(pot=False, wyaw=0.0, yaw_max=0.7)
    elif case == "yaw_pot":
        p.update(wyaw=1.0, yaw_max=0.9, grad=0.2)
    return p


def env_for(w, dim, control, U, p, region=None):
    from motion_primitive_library_b200 import MapUtil, env_map

    mu = MapUtil()
    mu.setMap(w["origin"], w["mdim"], w["grid"], w["res"])
    e = env_map(mu, device=0)
    e.set_control(control)
    e.set_u(U)
    e.set_dt(1.0)
    e.set_w(10.0)
    e.set_wyaw(p["wyaw"])
    e.set_v_max(2.0)
    e.set_a_max(2.0 if control & 15 >= 0x07 else -1.0)
    e.set_j_max(3.0 if control & 15 == 0x0F else -1.0)
    e.set_yaw_max(p["yaw_max"])
    if p["pot"]:
        e.set_potential_weight(0.5)
        e.set_gradient_weight(p["grad"])
        e.set_potential_map(w["pot"])
    if region is not None:
        e.set_search_region(region)
    return e


def oracle_for(w, dim, control, U, p, region=None):
    return ob.OracleEnv(dim, control, U, w["grid"], w["mdim"], w["origin"], w["res"], T=1.0, w=10.0, wyaw=p["wyaw"],
                        v_max=2.0, a_max=2.0 if control & 15 >= 0x07 else -1.0,
                        j_max=3.0 if control & 15 == 0x0F else -1.0, yaw_max=p["yaw_max"],
                        potential=w["pot"] if p["pot"] else None, potential_weight=0.5, gradient_weight=p["grad"],
                        region=region)


def args_for(w, dim, control, U, p, max_num, eps):
    return pb.make_args(dim, control, w["grid"], w["mdim"], w["origin"], w["res"], U, start=dict(pos=[0.0] * dim),
                        goal=dict(pos=[0.0] * dim), T=1.0, w=10.0, wyaw=p["wyaw"], v_max=2.0,
                        a_max=2.0 if control & 15 >= 0x07 else -1.0, j_max=3.0 if control & 15 == 0x0F else -1.0,
                        yaw_max=p["yaw_max"], max_num=max_num, eps=eps,
                        potential=w["pot"] if p["pot"] else None, potential_weight=0.5, gradient_weight=p["grad"])


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("dim,order,yaw", MATRIX, ids=[f"{d}d-{o}-{'yaw' if y else 'noyaw'}" for d, o, y in MATRIX])
def test_matrix(sbkc, dim, order, yaw, case):
    control = ORDERS[order] | (YAW_BIT if yaw else 0)
    U = control_set(dim, ORDER_OF[order], yaw)
    p = case_params(case, yaw)
    w = small_world(dim)
    nq, mx, eps = 8, 40 if dim == 3 else 60, 2.0
    S, G = queries(w, dim, nq, seed=11 + dim, yaw=yaw)
    if p["region"]:
        # a search region (tunnel): the raw entry point, against the CPU bookkeeping on every query.  The
        # lock-step loop cannot take this plan: the batch session's arguments (mplh_plan_args) carry no region
        region = np.ones(w["shape"], np.uint8)
        region.reshape(-1)[: w["grid"].size // 3] = 0
        region = region.reshape(-1)
        e = env_for(w, dim, control, U, p, region=region)
        e._sync_params()  # the parameters, the field and the tunnel reach the device before the count
        n0 = e.launch_count()
        r = e.plan_batch_cost_terms(S, G, eps=eps, max_expand=mx)
        assert e.launch_count() == n0 + 1
        e.close()
        env = oracle_for(w, dim, control, U, p, region=region)
    else:
        d, l = both_paths(args_for(w, dim, control, U, p, mx, eps), S, G)
        assert_same(d, l)
        r = as_dict(d)
        env = oracle_for(w, dim, control, U, p)
    for q in range(nq):
        ref = run_sbkc(sbkc, env, S[q], G[q], eps, mx)
        assert_matches_cpu(r, q, ref, yaw)


# ---- potential semantics ----------------------------------------------------------------------------------
def test_potential_values_and_start_under_field(sbkc):
    dim, control = 2, ORDERS["ACC"]
    U = control_set(dim, 2, False)
    p = case_params("pot", False)
    w = small_world(dim, seed=9)
    pot = w["pot"].reshape(w["shape"]).copy()
    S, G = queries(w, dim, 6, seed=2, yaw=False)
    # query 0's start cell is free in the grid but blocked (>= 100) in the field: the start test reads the grid,
    # so the search starts, and every primitive leaving it is blocked by the field's first sample
    cell = ((S["pos"][0, :dim] - np.asarray(w["origin"])) / w["res"]).astype(int)
    pot[cell[1], cell[0]] = 100
    pot[0, 0] = -1
    w["pot"] = pot.reshape(-1)
    e = env_for(w, dim, control, U, p)
    r = e.plan_batch_cost_terms(S, G, eps=1.0, max_expand=60)
    e.close()
    env = oracle_for(w, dim, control, U, p)
    for q in range(len(S)):
        assert_matches_cpu(r, q, run_sbkc(sbkc, env, S[q], G[q], 1.0, 60), False)
    assert r["expanded"][0] >= 1  # started: the start test reads the grid, not the field
    d, l = both_paths(args_for(w, dim, control, U, p, 60, 1.0), S, G)
    assert_same(d, l)


def test_goal_ray_reads_the_grid_not_the_field(sbkc):
    # The goal lies 6 cells along x from the start, within tol_pos, on grid-free cells; the field is 100 on the
    # cells between them.  The walkRay test of is_goal reads the grid, so the start is already a goal: valid,
    # no expansion, cost 0.  With the field installed as the grid (mplx_update_potential_map) the same ray is
    # blocked and the search has to run.
    dim, control = 2, ORDERS["ACC"]
    U = control_set(dim, 2, False)
    p = case_params("pot", False)
    w = small_world(dim, seed=9)
    grid = w["grid"].reshape(w["shape"])
    rows = [y for y in range(2, w["shape"][0] - 2) if (grid[y - 1:y + 2, 2:12] == 0).all()]
    y = rows[0]
    pot = w["pot"].reshape(w["shape"]).copy()
    pot[y, 2:12] = 0
    pot[y - 1:y + 2, 4:10] = 100  # between the start (x = 3) and the goal (x = 9)
    w["pot"] = pot.reshape(-1)
    S, G = np.zeros(2, P.WAYPOINT_DTYPE), np.zeros(2, P.WAYPOINT_DTYPE)
    for W, x in ((S, 3), (G, 9)):
        W["pos"][:, 0] = (x + 0.5) * w["res"] + w["origin"][0]
        W["pos"][:, 1] = (y + 0.5) * w["res"] + w["origin"][1]
    G["pos"][1, 1] += w["res"]  # query 1: the same ray one row up
    tol = 1.6  # 6 cells of 0.25 m = 1.5 m
    e = env_for(w, dim, control, U, p)
    r = e.plan_batch_cost_terms(S, G, eps=1.0, max_expand=60, tol_pos=tol)
    e.close()
    assert (r["valid"] == 1).all() and (r["expanded"] == 0).all() and (r["cost"] == 0).all()
    env = oracle_for(w, dim, control, U, p)
    for q in range(2):
        assert_matches_cpu(r, q, run_sbkc(sbkc, env, S[q], G[q], 1.0, 60, tol_pos=tol), False)
    # the counterfactual: the field as the grid blocks the ray, so neither start is a goal
    wf = dict(w, grid=w["pot"])
    e = env_for(wf, dim, control, U, p)
    rf = e.plan_batch_cost_terms(S, G, eps=1.0, max_expand=60, tol_pos=tol)
    e.close()
    assert (rf["expanded"] > 0).all()
    envf = oracle_for(wf, dim, control, U, p)
    for q in range(2):
        assert_matches_cpu(rf, q, run_sbkc(sbkc, envf, S[q], G[q], 1.0, 60, tol_pos=tol), False)


def test_field_installed_both_ways():
    # mplx_update_potential_map: the grid becomes the field; mplx_set_potential with that field keeps the
    # occupancy grid.  Both must match the lock-step loop under the same installation.
    from motion_primitive_library_b200 import MapUtil, env_map

    c = fixtures.corridor()
    mu = MapUtil()
    mu.setMap(c["origin"], c["dim"], c["grid"], c["res"])
    e = env_map(mu, device=0)
    e.set_potential_weight(0.5)
    e.set_gradient_weight(0.0)
    field = e.update_potential_map((1.0, 1.0, 0.0)).copy()
    e.close()
    rng = np.random.default_rng(4)
    free = np.argwhere(field.reshape(199, 799) < 100)
    pick = free[rng.choice(len(free), 32, replace=False)]
    pts = np.stack([(pick[:, 1] + 0.5) * c["res"] + c["origin"][0], (pick[:, 0] + 0.5) * c["res"] + c["origin"][1]], 1)
    S, G = np.zeros(16, P.WAYPOINT_DTYPE), np.zeros(16, P.WAYPOINT_DTYPE)
    S["pos"][:, :2], G["pos"][:, :2] = pts[:16], pts[16:]
    G["pos"][:, :2] = S["pos"][:, :2] + np.clip(G["pos"][:, :2] - S["pos"][:, :2], -3, 3)
    outs = {}
    for name, grid in (("update", field), ("set", c["grid"])):
        args = pb.make_args(2, ORDERS["ACC"], grid, c["dim"], c["origin"], c["res"], fixtures.U_2d(),
                            start=dict(pos=c["start"]), goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, max_num=300,
                            potential=field, potential_weight=0.5)
        d, l = both_paths(args, S, G)
        assert_same(d, l)
        outs[name] = d
    assert outs["update"][0]["valid"].sum() > 0


# ---- yaw ----------------------------------------------------------------------------------------------------
def test_yaw_tolerance_pure_yaw_rates_and_start_is_goal(sbkc):
    dim, control = 2, ORDERS["ACC"] | YAW_BIT
    # pure yaw-rate primitives at rest keep the position: intrinsic cost only
    U = np.array([[0.0, 0.0, -0.5], [0.0, 0.0, 0.5], [0.5, 0.0, 0.0], [0.0, 0.5, 0.5], [-0.5, 0.0, -0.5]])
    p = case_params("wyaw", True)
    w = small_world(dim, seed=5)
    S, G = queries(w, dim, 6, seed=3, yaw=True)
    G["pos"][0] = S["pos"][0]  # same position, other yaw: only yaw primitives reach it under tol_yaw
    G["yaw"][0] = S["yaw"][0] - 1.0 if S["yaw"][0] > 0 else S["yaw"][0] + 1.0
    G[1] = S[1]  # start == goal
    e = env_for(w, dim, control, U, p)
    env = oracle_for(w, dim, control, U, p)
    for tol_yaw in (-1.0, 0.3, 0.0):
        r = e.plan_batch_cost_terms(S, G, eps=1.0, max_expand=50, tol_yaw=tol_yaw)
        for q in range(len(S)):
            assert_matches_cpu(r, q, run_sbkc(sbkc, env, S[q], G[q], 1.0, 50, tol_yaw=tol_yaw), True)
        assert r["valid"][1] == 1 and r["expanded"][1] == 0 and r["cost"][1] == 0
        if tol_yaw == 0.3:
            assert r["valid"][0] == 1 and r["expanded"][0] > 1
    e.close()


# ---- launches, refusals, sizing ------------------------------------------------------------------------------
def _raw(lib, h, nq, max_expand):
    S = np.zeros(nq, P.WAYPOINT_DTYPE)
    o = dict(valid=np.full(nq, 7, np.int32), cost=np.full(nq, 7.0), expanded=np.full(nq, 7, np.int32),
             n_closed=np.full(nq, 7, np.int32), aoff=np.full(nq + 1, 7, np.int64),
             acts=np.full(max(1, nq * max(max_expand, 1)), 7, np.int32), coff=np.full(nq + 1, 7, np.int64),
             keys=np.full(max(1, nq * max(max_expand, 1)), 7, np.uint64))
    out = abi.BatchOut(o["valid"].ctypes.data, o["cost"].ctypes.data, o["expanded"].ctypes.data, o["n_closed"].ctypes.data,
                       o["aoff"].ctypes.data, o["acts"].ctypes.data, o["acts"].size, o["coff"].ctypes.data,
                       o["keys"].ctypes.data, o["keys"].size, 7, 7, 7.0)
    rc = lib.mplx_plan_batch_cost_terms(h, S.ctypes.data, S.ctypes.data, None, nq, 1.0, max_expand, 0.5, -1.0, -1.0,
                                        -1.0, C.byref(out))
    o["meta"] = (out.slots, out.arena_bytes, out.seconds)
    return rc, o


def _untouched(o):
    return all((v == 7).all() for k, v in o.items() if k != "meta") and o["meta"] == (7, 7, 7.0)


def test_refusals_fits_and_one_launch_per_call():
    lib = abi.load()
    h = C.c_void_p()
    assert lib.mplx_create(2, 0, C.byref(h)) == abi.MPLX_OK
    rc, o = _raw(lib, h, 3, 50)
    assert rc == abi.MPLX_ERR_ARG and _untouched(o)
    assert lib.mplx_plan_batch_cost_terms_fits(h, 3, 50, 1, None, None) == abi.MPLX_ERR_ARG
    lib.mplx_destroy(h)

    w = small_world(2)
    p = case_params("yaw_pot", True)
    control = ORDERS["ACC"] | YAW_BIT
    many = np.array([[0.01 * i, 0.0, 0.0] for i in range(257)])
    for U, mx in ((many, 50), (control_set(2, 2, True), 0), (control_set(2, 2, True), -2)):
        e = env_for(w, 2, control, U, p)
        e._sync_params()
        n0 = e.launch_count()
        rc, o = _raw(lib, e.handle, 3, mx)
        assert rc == abi.MPLX_ERR_ARG and _untouched(o), (len(U), mx)
        assert e.launch_count() == n0
        e.close()
    e = env_for(w, 2, control, control_set(2, 2, True), p)
    S, G = queries(w, 2, 5, seed=1, yaw=True)
    e._sync_params()
    n0 = e.launch_count()
    before = e.plan_batch_cost_terms(S, G, max_expand=100)
    assert e.launch_count() == n0 + 1
    n1 = e.launch_count()
    slots, nbytes = C.c_int32(-1), C.c_int64(-1)
    assert lib.mplx_plan_batch_cost_terms_fits(e.handle, 3, 10 ** 9, 0, C.byref(slots), C.byref(nbytes)) == abi.MPLX_ERR_ALLOC
    assert (slots.value, nbytes.value) == (-1, -1)
    rc, o = _raw(lib, e.handle, 1, 10 ** 7)
    assert rc == abi.MPLX_ERR_ALLOC and _untouched(o) and e.launch_count() == n1
    assert lib.mplx_plan_batch_cost_terms_fits(e.handle, 5, 100, 1, C.byref(slots), C.byref(nbytes)) == abi.MPLX_OK
    assert slots.value == before["slots"] and nbytes.value == before["arena_bytes"]
    # the occupancy entry point still refuses the plan
    with pytest.raises(abi.MplxError) as ex:
        e.plan_batch(S, G, max_expand=100)
    assert ex.value.code == abi.MPLX_ERR_ARG
    after = e.plan_batch_cost_terms(S, G, max_expand=100)
    for f in ("valid", "cost", "expanded", "n_closed"):
        assert np.array_equal(before[f], after[f])
    e.close()


# ---- MultiQueryPlanner path choice --------------------------------------------------------------------------
def test_auto_threshold_device_contract_and_memory_fallback():
    w = small_world(2)
    p = case_params("pot", False)
    control = ORDERS["ACC"]
    U = control_set(2, 2, False)
    S, G = queries(w, 2, 40, seed=6, yaw=False)
    k = COST_TERMS_MIN_QUERIES
    args = args_for(w, 2, control, U, p, 60, 1.0)
    auto = P.BatchPlanner(args)
    dev = P.BatchPlanner(args, path="device")
    lck = P.BatchPlanner(args, path="lockstep")
    try:
        _, t = auto.plan(S[: k - 1], G[: k - 1])
        assert t["path"] == "lockstep"
        r_auto, t = auto.plan(S[:k], G[:k])
        assert t["path"] == "device_cost_terms"
        r_l, _ = lck.plan(S[:k], G[:k])
        assert np.array_equal(r_auto, r_l) and r_auto["cost"].tobytes() == r_l["cost"].tobytes()
        # DEVICE keeps its contract: the occupancy search only, so a cost-term plan runs lock-step
        _, t = dev.plan(S, G)
        assert t["path"] == "lockstep"
    finally:
        auto.close()
        dev.close()
        lck.close()
    # a worst-case arena beyond any budget (1 + max_num*|U| states): AUTO falls back to lock-step, which gives
    # what it gave before, and the forced path fails
    c = fixtures.corridor()
    Sc = np.zeros(k, P.WAYPOINT_DTYPE)
    Gc = np.zeros(k, P.WAYPOINT_DTYPE)
    Sc["pos"][:, :2], Gc["pos"][:, :2] = c["start"][:2], c["goal"][:2]
    big = pb.make_args(2, control, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                       goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, max_num=10 ** 7,
                       potential=np.zeros(c["grid"].size, np.int8))
    auto = P.BatchPlanner(big)
    lck = P.BatchPlanner(big, path="lockstep")
    try:
        res, t = auto.plan(Sc, Gc)
        assert t["path"] == "lockstep" and res["valid"].all()
        ref, _ = lck.plan(Sc, Gc)
        assert np.array_equal(res, ref) and res["cost"].tobytes() == ref["cost"].tobytes()
    finally:
        auto.close()
        lck.close()
    forced = P.BatchPlanner(args, path="device_cost_terms")
    try:
        with pytest.raises(RuntimeError, match="budget"):
            forced.plan(S[:2], G[:2], max_num=10 ** 7)
        _, t = forced.plan(S[:2], G[:2])
        assert t["path"] == "device_cost_terms"
    finally:
        forced.close()
    # occupancy plans under AUTO still take mplx_plan_batch
    occ = args_for(w, 2, control, U, dict(p, pot=False), 60, 1.0)
    a = P.BatchPlanner(occ)
    try:
        _, t = a.plan(S[:k], G[:k])
        assert t["path"] == "device"
    finally:
        a.close()


def test_occupancy_plans_equal_through_both_entry_points():
    w = small_world(3)
    p = dict(case_params("pot", False), pot=False)
    for order in ("ACC", "JRK"):
        control = ORDERS[order]
        U = control_set(3, {"ACC": 2, "JRK": 3}[order], False)
        S, G = queries(w, 3, 16, seed=8, yaw=False)
        args = args_for(w, 3, control, U, p, 40, 2.0)
        outs = {}
        for path in ("device", "device_cost_terms"):
            s = P.BatchPlanner(args, path=path)
            try:
                outs[path] = s.plan_detail(S, G)
                assert outs[path][1]["path"] == path
            finally:
                s.close()
        assert_same(outs["device_cost_terms"], outs["device"])


# ---- one ctx across occupancy and cost-term searches ---------------------------------------------------------
def test_one_ctx_alternating_searches_equals_fresh_ctx():
    w = small_world(2, seed=7)
    control = ORDERS["ACC"]
    U = control_set(2, 2, False)
    S, G = queries(w, 2, 10, seed=9, yaw=False)
    region = np.ones(w["grid"].size, np.uint8)
    region[: w["grid"].size // 4] = 0
    cells = np.argwhere(w["grid"].reshape(w["shape"]) == 0)[:20]

    def fresh(pot_w, grad_w, pot, with_region, edited, cost_terms, mx):
        from motion_primitive_library_b200 import MapUtil, env_map

        grid = w["grid"].reshape(w["shape"]).copy()
        if edited:
            grid[cells[:, 0], cells[:, 1]] = 100
        mu = MapUtil()
        mu.setMap(w["origin"], w["mdim"], grid.reshape(-1), w["res"])
        e = env_map(mu, device=0)
        e.set_control(control)
        e.set_u(U)
        e.set_dt(1.0)
        e.set_w(10.0)
        e.set_v_max(2.0)
        if pot:
            e.set_potential_weight(pot_w)
            e.set_gradient_weight(grad_w)
            e.set_potential_map(w["pot"])
        if with_region:
            e.set_search_region(region)
        r = (e.plan_batch_cost_terms if cost_terms else e.plan_batch)(S, G, max_expand=mx)
        e.close()
        return r

    from motion_primitive_library_b200 import MapUtil, env_map

    mu = MapUtil()
    mu.setMap(w["origin"], w["mdim"], w["grid"].copy(), w["res"])  # update_cells edits this grid in place
    e = env_map(mu, device=0)
    e.set_control(control)
    e.set_u(U)
    e.set_dt(1.0)
    e.set_w(10.0)
    e.set_v_max(2.0)
    script = []
    script.append(((0.5, 0.0, False, False, False, False, 60), e.plan_batch(S, G, max_expand=60)))
    e.set_potential_weight(0.5)
    e.set_gradient_weight(0.0)
    e.set_potential_map(w["pot"])
    script.append(((0.5, 0.0, True, False, False, True, 60), e.plan_batch_cost_terms(S, G, max_expand=60)))
    e.set_potential_weight(0.8)
    e.set_gradient_weight(0.25)
    script.append(((0.8, 0.25, True, False, False, True, 30), e.plan_batch_cost_terms(S, G, max_expand=30)))
    e.update_cells(cells[:, ::-1], np.full(len(cells), 100, np.int8))  # (x, y) cells; the field is kept
    script.append(((0.8, 0.25, True, False, True, True, 60), e.plan_batch_cost_terms(S, G, max_expand=60)))
    e.set_search_region(region)
    script.append(((0.8, 0.25, True, True, True, True, 80), e.plan_batch_cost_terms(S, G, max_expand=80)))
    e.close()
    for key, r in script:
        f = fresh(*key)
        for fld in ("valid", "expanded", "n_closed"):
            assert np.array_equal(r[fld], f[fld]), (key, fld)
        assert r["cost"].tobytes() == f["cost"].tobytes(), key
        assert all(np.array_equal(a, b) for a, b in zip(r["actions"], f["actions"])), key
        assert all(np.array_equal(a, b) for a, b in zip(r["closed"], f["closed"])), key


# ---- the reference's configurations on the corridor ----------------------------------------------------------
def corridor_queries(c, grid, nq, seed):
    rng = np.random.default_rng(seed)
    free = np.argwhere(grid.reshape(199, 799) == 0)
    S, G = np.zeros(nq, P.WAYPOINT_DTYPE), np.zeros(nq, P.WAYPOINT_DTYPE)
    a = free[rng.choice(len(free), nq, replace=False)]
    for q in range(nq):
        d = np.abs(free - a[q]).max(1)
        near = free[(d > 8) & (d < 30)]
        b = near[rng.integers(len(near))]
        S["pos"][q, :2] = (a[q][::-1] + 0.5) * c["res"] + np.asarray(c["origin"][:2])
        G["pos"][q, :2] = (b[::-1] + 0.5) * c["res"] + np.asarray(c["origin"][:2])
    S[0]["pos"][:2], G[0]["pos"][:2] = c["start"][:2], c["goal"][:2]
    return S, G


CORRIDOR_CONFIGS = ("distance_map_planner_2d", "planner_2d_with_yaw", "distance_map_planner_2d_with_yaw")


def corridor_config(name):
    """One of the reference's corridor tests as a 16-query batch: (args, starts, goals, field).  The field is the
    reference's own MapPlanner::updatePotentialMap (radius 1; the reference overwrites its map with it, so it is
    both the grid and the potential map), recorded under tests/golden/reference; None without one."""
    c = fixtures.corridor()
    yaw = "yaw" in name
    control = ORDERS["ACC"] | (YAW_BIT if yaw else 0)
    U = fixtures.U_2d_yaw() if yaw else fixtures.U_2d()
    grid, pot = c["grid"], None
    if "distance_map" in name:
        a0 = pb.make_args(2, control, c["grid"], c["dim"], c["origin"], c["res"], U, start=dict(pos=c["start"]),
                          goal=dict(pos=c["goal"]))
        grid = pot = pb.reference_potential_map(a0, (1.0, 1.0), c["grid"].size, record_all=True)
    kw = dict(v_max=1.0, a_max=1.0, max_num=400, eps=1.0, yaw_max=0.7 if yaw else -1.0, potential=pot,
              potential_weight=0.5)
    args = pb.make_args(2, control, grid, c["dim"], c["origin"], c["res"], U, start=dict(pos=c["start"]),
                        goal=dict(pos=c["goal"]), **kw)
    S, G = corridor_queries(c, grid, 16, seed=21)
    return args, S, G, pot


@pytest.mark.parametrize("name", CORRIDOR_CONFIGS)
def test_reference_configurations_on_corridor_under_auto(sbkc, name):
    import test_search_cost_inputs_oracle_vs_ref as ref_pin
    from motion_primitive_library_b200 import MapUtil, env_map

    c = fixtures.corridor()
    yaw = "yaw" in name
    args, S, G, pot = corridor_config(name)
    # the reference planner's result of every query (recorded where oracle/_ref is not built)
    refs = [ref_pin.plan_reference(ref_pin.query_args(args, S, G, q, 2)) for q in range(len(S))]
    if pot is not None:
        # the device builds the same field (mplx_update_potential_map)
        mu = MapUtil()
        mu.setMap(c["origin"], c["dim"], c["grid"], c["res"])
        e = env_map(mu, device=0)
        e.set_potential_weight(0.5)
        e.set_gradient_weight(0.0)
        same_array(e.update_potential_map((1.0, 1.0, 0.0)).copy(), pot, "field")
        e.close()
    s = P.BatchPlanner(args)
    try:
        d = s.plan_detail(S, G)
    finally:
        s.close()
    assert d[1]["path"] == "device_cost_terms"
    l = P.BatchPlanner(args, path="lockstep")
    try:
        assert_same(d, l.plan_detail(S, G))
    finally:
        l.close()
    assert d[0]["valid"].sum() > 0
    r = as_dict(d)
    for q in range(len(S)):
        mine = dict(valid=r["valid"][q], cost=r["cost"][q], expanded=r["expanded"][q], n_closed=r["n_closed"][q],
                    closed=r["closed"][q], actions=r["actions"][q])
        ref_pin.same_as_reference(mine, refs[q], (name, q), yaw_cost_tol=1e-12 if yaw else None)
    control = args.control
    U = fixtures.U_2d_yaw() if yaw else fixtures.U_2d()
    grid = c["grid"] if pot is None else pot
    env = ob.OracleEnv(2, control, U, grid, c["dim"], c["origin"], c["res"], v_max=1.0, a_max=1.0,
                       yaw_max=0.7 if yaw else -1.0, potential=pot, potential_weight=0.5)
    for q in range(len(S)):
        assert_matches_cpu(r, q, run_sbkc(sbkc, env, S[q], G[q], 1.0, 400), yaw)


# ---- the named shape ------------------------------------------------------------------------------------------
def test_cfg4_512_64_queries_equal_lockstep():
    import cfg5_bench
    import scenarios as Sc
    from motion_primitive_library_b200 import MapUtil, env_map

    sc = Sc.cfg4()
    mu = MapUtil()
    mu.setMap(sc.origin, sc.dim_cells, sc.grid(), sc.res)
    e = env_map(mu, device=0)
    e.set_potential_weight(sc.potential_weight)
    e.set_gradient_weight(sc.gradient_weight)
    field = e.update_potential_map(sc.potential_radius).copy()
    e.close()
    q = cfg5_bench.make_queries(sc, 64, 20.0)
    args = pb.make_args(3, sc.control, field, sc.dim_cells, sc.origin, sc.res, sc.U,
                        start=dict(pos=q["start"]["pos"][0]), goal=dict(pos=q["goal"]["pos"][0]), v_max=sc.v_max,
                        yaw_max=sc.yaw_max, wyaw=sc.wyaw, T=sc.T, w=sc.w, max_num=1000, eps=2.0, potential=field,
                        potential_weight=sc.potential_weight, gradient_weight=sc.gradient_weight)
    d, l = both_paths(args, q["start"], q["goal"])
    assert_same(d, l)
    assert d[0]["valid"].sum() > 0
