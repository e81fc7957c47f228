"""Per-query tunnels in the device searches (mplx_set_batch_regions).

  - Tunnel build: each query's tunnel, read back one byte per voxel, equals mplx_set_search_region_path's region of
    the same points, byte for byte.
  - Search results: each query of a tunnelled batch gives what the device search of that query alone gives with its
    tunnel installed ctx-wide (valid, cost bits, expansions, closed keys, actions, recorded trajectory), on every
    search instantiation and entry point; on a sample of queries also what the search bookkeeping driven by the
    oracle env gives with that tunnel as its search region.
  - Batch structure, the ctx-wide region, map edits, refusals and launch counts."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import oracle_bindings as ob
from motion_primitive_library_b200 import MapUtil, abi, env_map

pytestmark = pytest.mark.gpu
HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
ORDERS = {"VEL": 0x01, "ACC": 0x03, "JRK": 0x07, "SNP": 0x0F}
ORDER_OF = {"VEL": 1, "ACC": 2, "JRK": 3, "SNP": 4}
YAW_BIT = 0x10
WAYPOINT = abi.WAYPOINT_DTYPE


@pytest.fixture(scope="module")
def sbkc(tmp_path_factory):
    so = tmp_path_factory.mktemp("sbkc_tun") / "libsbkc.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(so),
                           str(HERE / "search_bookkeeping_cost_host.cpp"), str(ROOT / "oracle" / "mpl_oracle.cpp")])
    L = C.CDLL(str(so))
    vp = C.c_void_p
    L.sbkc_plan.argtypes = [C.POINTER(ob.OrcEnv), vp, vp, C.c_double, C.c_int, C.c_double, C.c_double, C.c_double,
                            C.c_double, vp, vp, vp, vp, vp, vp, vp]
    L.sbkc_plan.restype = C.c_int
    return L


def run_sbkc(L, env, start, goal, eps, max_expand):
    s = np.zeros(1, dtype=ob.WAYPOINT_DTYPE)
    g = np.zeros(1, dtype=ob.WAYPOINT_DTYPE)
    s[0], g[0] = start, goal
    valid, expanded, n_closed, n_actions = (np.zeros(1, np.int32) for _ in range(4))
    cost = np.zeros(1)
    closed = np.zeros(max_expand, np.uint64)
    actions = np.zeros(max_expand, np.int32)
    assert L.sbkc_plan(C.byref(env.e), s.ctypes.data, g.ctypes.data, eps, max_expand, 0.5, -1.0, -1.0, -1.0,
                       valid.ctypes.data, cost.ctypes.data, expanded.ctypes.data, n_closed.ctypes.data,
                       closed.ctypes.data, actions.ctypes.data, n_actions.ctypes.data) == 0
    return dict(valid=int(valid[0]), cost=float(cost[0]), expanded=int(expanded[0]), n_closed=int(n_closed[0]),
                closed=closed[: n_closed[0]].copy(), actions=actions[: n_actions[0]].copy())


# ---- worlds, plans and tunnels ---------------------------------------------------------------------------------
def world(dim, seed=3):
    """A box map with a potential field: values <= 0 free, 1..99 cost, >= 100 block.  The sizes are not multiples
    of the brick edge, so tunnels reach partial bricks at the far edges."""
    rng = np.random.default_rng(seed)
    mdim = (45, 38) if dim == 2 else (20, 19, 13)
    res = 0.25
    origin = tuple(-m * res / 2 for m in mdim)
    shape = tuple(reversed(mdim))
    grid = np.zeros(shape, np.int8)
    for _ in range(6 if dim == 2 else 5):
        lo = [rng.integers(0, s - 4) for s in shape]
        grid[tuple(slice(a, a + int(rng.integers(2, 5))) for a in lo)] = 100
    pot = rng.integers(-1, 60, size=shape).astype(np.int8)
    pot[grid == 100] = 100
    return dict(grid=grid.reshape(-1), pot=pot.reshape(-1), mdim=mdim, origin=origin, res=res, shape=shape)


def control_set(dim, order, yaw):
    import scenarios as S

    return S.control_set({1: 1.0, 2: 1.0, 3: 2.0, 4: 4.0}[order], 3, dim, yaw_rates=(-0.5, 0.0, 0.5) if yaw else None)


def queries(w, dim, n, seed, yaw):
    rng = np.random.default_rng(seed)
    free = np.argwhere(w["grid"].reshape(w["shape"]) == 0)
    S = np.zeros(n, dtype=WAYPOINT)
    G = np.zeros(n, dtype=WAYPOINT)
    for q in range(n):
        a = free[rng.integers(len(free))]
        d = np.sum(np.abs(free - a), 1)
        near = free[(d > 2) & (d < 10)]
        b = near[rng.integers(len(near))] if len(near) else a
        for W, cell in ((S, a), (G, b)):
            W["pos"][q, :dim] = (np.asarray(cell[::-1], float) + 0.5) * w["res"] + np.asarray(w["origin"])
        if yaw:
            S["yaw"][q] = rng.uniform(-np.pi, np.pi)
            G["yaw"][q] = rng.uniform(-np.pi, np.pi)
    return S, G


def routes(S, G, dim, seed=0):
    """Each query's route: start -> a point off the straight line -> goal; every fourth only its start (a tunnel
    that may shut the goal out)."""
    rng = np.random.default_rng(seed)
    out = []
    for q in range(len(S)):
        a, b = S["pos"][q, :dim], G["pos"][q, :dim]
        if q % 4 == 3:
            out.append(a[None, :].copy())
        else:
            out.append(np.stack([a, (a + b) / 2 + rng.uniform(-0.5, 0.5, dim), b]))
    return out


def make_env(w, dim, control, U, pot=False, wyaw=1.0):
    mu = MapUtil()
    mu.setMap(w["origin"], w["mdim"], w["grid"], w["res"])
    e = env_map(mu, device=0)
    e.set_control(control)
    e.set_u(U)
    e.set_dt(1.0)
    e.set_w(10.0)
    e.set_wyaw(wyaw)
    e.set_v_max(2.0)
    e.set_a_max(2.0 if control & 15 >= 0x07 else -1.0)
    e.set_j_max(3.0 if control & 15 == 0x0F else -1.0)
    if pot:
        e.set_potential_weight(0.5)
        e.set_gradient_weight(0.2)
        e.set_potential_map(w["pot"])
    e._sync_params()
    return e


def make_oracle(w, dim, control, U, pot, region, wyaw=1.0):
    return ob.OracleEnv(dim, control, U, w["grid"], w["mdim"], w["origin"], w["res"], T=1.0, w=10.0, wyaw=wyaw,
                        v_max=2.0, a_max=2.0 if control & 15 >= 0x07 else -1.0,
                        j_max=3.0 if control & 15 == 0x0F else -1.0, potential=w["pot"] if pot else None,
                        potential_weight=0.5, gradient_weight=0.2, region=region)


def search(e, entry, S, G, mx, eps=2.0, traj=True, **kw):
    if entry == "batch":
        return e.plan_batch(S, G, eps=eps, max_expand=mx, trajectories=traj)
    if entry == "cost_terms":
        return e.plan_batch_cost_terms(S, G, eps=eps, max_expand=mx, trajectories=traj)
    return e.plan_batch_grow(S, G, eps=eps, max_expand=mx, cost_terms=entry == "grow_cost", trajectories=traj, **kw)


def same_query(a, qa, b, qb, traj=True):
    for f in ("valid", "expanded", "n_closed"):
        assert int(a[f][qa]) == int(b[f][qb]), (f, qa)
    assert np.float64(a["cost"][qa]).tobytes() == np.float64(b["cost"][qb]).tobytes(), qa
    assert np.array_equal(a["actions"][qa], b["actions"][qb]), qa
    assert np.array_equal(a["closed"][qa], b["closed"][qb]), qa
    if traj and "trajectories" in a and "trajectories" in b:
        ta, tb = a["trajectories"][qa], b["trajectories"][qb]
        assert ta["nodes"].tobytes() == tb["nodes"].tobytes(), qa
        assert ta["coeff"].tobytes() == tb["coeff"].tobytes(), qa


def alone(e, entry, S, G, paths, radius, dense, q, mx, **kw):
    """Query q searched by itself with its tunnel installed ctx-wide."""
    e.set_batch_regions([], radius)
    region = e.set_search_region_path(paths[q], radius, dense)
    r = search(e, entry, S[q:q + 1], G[q:q + 1], mx, **kw)
    return r, region


# ---- tunnel build ------------------------------------------------------------------------------------------------
def build_paths(w, dim):
    """Paths that leave the map, run along its edge, cross brick boundaries, have one point or repeat points."""
    lo = np.asarray(w["origin"], float)
    hi = lo + np.asarray(w["mdim"], float) * w["res"]
    mid = (lo + hi) / 2
    e = w["res"] * 0.5
    paths = [
        np.stack([mid, hi + 1.0]),                                        # leaves the map
        np.stack([lo - 2.0, mid]),                                        # enters it from outside
        np.stack([lo + e, np.r_[hi[0] - e, lo[1:] + e]]),                 # along the low edge
        np.stack([lo + e, hi - e]),                                       # the diagonal: many brick boundaries
        mid[None, :],                                                     # one point
        np.stack([mid, mid, mid + 0.3, mid + 0.3, mid]),                  # repeated points
        np.stack([lo + 8 * w["res"] - 0.01, lo + 8 * w["res"] + 0.01]),   # across one brick corner
        (hi + 3.0)[None, :],                                              # one point outside the map
    ]
    rng = np.random.default_rng(dim)
    for _ in range(6):
        paths.append(rng.uniform(lo - 0.5, hi + 0.5, size=(int(rng.integers(2, 7)), dim)))
    return paths


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("dense", [False, True])
@pytest.mark.parametrize("radius", ["zero", "aniso", "wide"])
def test_tunnel_build_equals_region_path(dim, dense, radius):
    w = world(dim)
    rad = {"zero": [0.0] * dim, "aniso": [0.3, 0.8, 0.1][:dim], "wide": [1.2] * dim}[radius]
    e = make_env(w, dim, ORDERS["ACC"], control_set(dim, 2, False))
    paths = build_paths(w, dim)
    e.set_batch_regions(paths, rad, dense)
    info = e.batch_regions_info()
    assert info["n_q"] == len(paths) and info["bytes"] > 0
    words = 16 if dim == 3 else 2
    assert info["bytes"] == info["n_bricks"] * (8 + 4 * words) + (len(paths) + 1) * 8
    got = [e.read_batch_region(q) for q in range(len(paths))]
    for q, p in enumerate(paths):
        want = e.set_search_region_path(p, rad, dense)
        assert np.array_equal(got[q], want), q
    assert sum(int(g.any()) for g in got) >= len(paths) // 2
    e.close()


def test_set_call_launches_do_not_depend_on_the_query_count():
    dim = 3
    w = world(dim)
    e = make_env(w, dim, ORDERS["ACC"], control_set(dim, 2, False))
    paths = build_paths(w, dim)
    counts = []
    for n in (1, 3, len(paths)):
        n0 = e.launch_count()
        e.set_batch_regions(paths[:n], [0.5] * dim, False)
        counts.append(e.launch_count() - n0)
    many = [p for _ in range(40) for p in paths]
    n0 = e.launch_count()
    e.set_batch_regions(many, [0.5] * dim, False)
    counts.append(e.launch_count() - n0)
    assert len(set(counts)) == 1 and counts[0] > 0, counts
    n0 = e.launch_count()
    e.set_batch_regions([], [0.5] * dim)
    assert e.launch_count() == n0 and e.batch_regions_info()["n_q"] == 0
    e.close()


# ---- search results ------------------------------------------------------------------------------------------------
MATRIX = [(dim, o, kind) for dim in (2, 3) for o in ORDERS for kind in ("occ", "cost", "yaw")]


@pytest.mark.parametrize("dim,order,kind", MATRIX, ids=[f"{d}d-{o}-{k}" for d, o, k in MATRIX])
def test_each_query_searches_in_its_tunnel(sbkc, dim, order, kind):
    yaw = kind == "yaw"
    control = ORDERS[order] | (YAW_BIT if yaw else 0)
    U = control_set(dim, ORDER_OF[order], yaw)
    w = world(dim)
    pot = kind == "cost"
    nq, mx = 8, 40 if dim == 3 else 60
    S, G = queries(w, dim, nq, seed=11 + dim, yaw=yaw)
    paths = routes(S, G, dim, seed=dim)
    radius, dense = [0.3, 0.55, 0.3][:dim], False
    entries = ("batch", "cost_terms", "grow") if kind == "occ" else ("cost_terms", "grow_cost")
    e = make_env(w, dim, control, U, pot=pot)
    batch = {}
    for entry in entries:
        e.set_batch_regions(paths, radius, dense)
        # recording on for the one-round entry points, off for the growing search: both kernel variants run
        batch[entry] = search(e, entry, S, G, mx, traj=entry not in ("grow", "grow_cost"))
    regions = {}
    for entry in entries:
        for q in range(nq):
            r, regions[q] = alone(e, entry, S, G, paths, radius, dense, q, mx, traj=True)
            same_query(batch[entry], q, r, 0)
    e.close()
    if order != "SNP":  # SNP's plans reach no goal within these caps and tunnels
        assert batch[entries[0]]["valid"].sum() > 0
    for q in (0, 3, 5):
        env = make_oracle(w, dim, control, U, pot, regions[q])
        ref = run_sbkc(sbkc, env, S[q], G[q], 2.0, mx)
        r = batch[entries[0]]
        assert (int(r["valid"][q]), int(r["expanded"][q]), int(r["n_closed"][q])) == (
            ref["valid"], ref["expanded"], ref["n_closed"]), q
        assert np.array_equal(r["closed"][q], ref["closed"]) and np.array_equal(r["actions"][q], ref["actions"]), q
        if ref["valid"] and yaw:
            assert abs(r["cost"][q] - ref["cost"]) <= 1e-12 * abs(ref["cost"]), q
        elif ref["valid"]:
            assert np.float64(r["cost"][q]).tobytes() == np.float64(ref["cost"]).tobytes(), q


@pytest.mark.parametrize("dim,cost_terms", [(2, False), (3, True)])
def test_grow_reruns_with_small_arenas_and_pool(dim, cost_terms):
    control = ORDERS["ACC"]
    U = control_set(dim, 2, False)
    w = world(dim)
    nq, mx = 12, 40 if dim == 3 else 60
    S, G = queries(w, dim, nq, seed=5 + dim, yaw=False)
    paths = routes(S, G, dim, seed=7)
    e = make_env(w, dim, control, U, pot=cost_terms)
    e.set_batch_regions(paths, [0.55] * dim, False)
    ref = search(e, "cost_terms" if cost_terms else "batch", S, G, mx)
    g = e.plan_batch_grow(S, G, eps=2.0, max_expand=mx, cost_terms=cost_terms, first_cap=8, pool_bytes=64,
                          trajectories=True, traj_room_bytes=4 * WAYPOINT.itemsize)
    assert g["reruns"] > 0 and g["rounds"] > 1 and g["searched"].all()
    for q in range(nq):
        same_query(g, q, ref, q)
    e.close()


# ---- batch structure ------------------------------------------------------------------------------------------------
def test_shuffled_and_split_batches_give_the_same_results():
    dim = 2
    w = world(dim)
    U = control_set(dim, 2, False)
    nq, mx = 16, 60
    S, G = queries(w, dim, nq, seed=21, yaw=False)
    paths = routes(S, G, dim, seed=3)
    rad = [0.55, 0.3]
    e = make_env(w, dim, ORDERS["ACC"], U)
    e.set_batch_regions(paths, rad)
    full = search(e, "batch", S, G, mx)
    perm = np.random.default_rng(2).permutation(nq)
    e.set_batch_regions([paths[i] for i in perm], rad)
    shuf = search(e, "batch", S[perm], G[perm], mx)
    for i, q in enumerate(perm):
        same_query(shuf, i, full, q)
    for part in (np.arange(0, 5), np.arange(5, nq)):
        e.set_batch_regions([paths[i] for i in part], rad)
        r = search(e, "batch", S[part], G[part], mx)
        for i, q in enumerate(part):
            same_query(r, i, full, q)
    e.close()


def test_tunnel_that_shuts_in_the_start_fails_as_the_host_fails(sbkc):
    dim = 2
    w = world(dim)
    U = control_set(dim, 2, False)
    S, G = queries(w, dim, 32, seed=8, yaw=False)
    apart = np.flatnonzero(np.linalg.norm(S["pos"] - G["pos"], axis=1) > 1.0)[:4]  # no start is already a goal
    S, G = S[apart], G[apart]
    far = np.asarray(w["origin"]) + 0.1
    paths = [far[None, :]] * 2 + routes(S[2:], G[2:], dim)[:2]
    e = make_env(w, dim, ORDERS["ACC"], U)
    e.set_batch_regions(paths, [0.3, 0.3])
    r = search(e, "batch", S, G, 60)
    region = e.read_batch_region(0)
    e.close()
    assert (r["valid"][:2] == 0).all()
    env = make_oracle(w, dim, ORDERS["ACC"], U, False, region)
    for q in range(2):
        ref = run_sbkc(sbkc, env, S[q], G[q], 2.0, 60)
        assert ref["valid"] == 0
        assert (int(r["expanded"][q]), int(r["n_closed"][q])) == (ref["expanded"], ref["n_closed"])
        assert np.array_equal(r["closed"][q], ref["closed"])


# ---- the ctx-wide region and map edits ------------------------------------------------------------------------------
def test_tunnels_win_over_the_ctx_region_and_clearing_restores_it():
    dim = 3
    w = world(dim)
    U = control_set(dim, 2, False)
    nq, mx = 10, 40
    S, G = queries(w, dim, nq, seed=31, yaw=False)
    paths = routes(S, G, dim, seed=4)
    rad = [0.3, 0.55, 0.3]
    e = make_env(w, dim, ORDERS["ACC"], U)
    e.set_batch_regions(paths, rad)
    tunnels_only = search(e, "cost_terms", S, G, mx)
    e.set_batch_regions([], rad)
    plain = search(e, "cost_terms", S, G, mx)
    ctx = np.ones(w["grid"].size, np.uint8)
    ctx[: w["grid"].size // 3] = 0
    e.set_search_region(ctx)
    with_ctx = search(e, "cost_terms", S, G, mx)
    e.set_batch_regions(paths, rad)
    both = search(e, "cost_terms", S, G, mx)
    for q in range(nq):
        same_query(both, q, tunnels_only, q)
    e.set_batch_regions([], rad)
    after = search(e, "cost_terms", S, G, mx)
    for q in range(nq):
        same_query(after, q, with_ctx, q)
    e.set_search_region(None)
    again = search(e, "cost_terms", S, G, mx)
    for q in range(nq):
        same_query(again, q, plain, q)
    e.close()


def test_set_map_drops_the_tunnels_and_update_cells_keeps_them():
    dim = 2
    w = world(dim)
    U = control_set(dim, 2, False)
    nq, mx = 8, 60
    S, G = queries(w, dim, nq, seed=41, yaw=False)
    paths = routes(S, G, dim, seed=5)
    e = make_env(w, dim, ORDERS["ACC"], U)
    e.set_batch_regions(paths, [0.3, 0.3])
    before = search(e, "batch", S, G, mx)
    info = e.batch_regions_info()
    idx = np.flatnonzero(w["grid"] == 0)[:5]
    e.update_cells(idx, np.zeros(5, np.int8))  # the same values: the map does not change
    assert e.batch_regions_info() == info
    kept = search(e, "batch", S, G, mx)
    for q in range(nq):
        same_query(kept, q, before, q)
    e.upload_map()
    assert e.batch_regions_info()["n_q"] == 0
    untunnelled = search(e, "batch", S[:3], G[:3], mx)  # any query count again
    e.set_batch_regions([], [0.3, 0.3])
    ref = search(e, "batch", S[:3], G[:3], mx)
    for q in range(3):
        same_query(untunnelled, q, ref, q)
    e.close()


# ---- refusals ------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing_and_launch_nothing():
    lib = abi.load()
    h = C.c_void_p()
    abi.check(lib.mplx_create(2, 0, C.byref(h)))
    off = np.array([0, 2], np.int64)
    pts = np.zeros(4)
    rad = np.array([0.5, 0.5])
    assert lib.mplx_set_batch_regions(h, 1, off.ctypes.data, pts.ctypes.data, rad.ctypes.data, 0) == abi.MPLX_ERR_ARG
    lib.mplx_destroy(h)

    dim = 2
    w = world(dim)
    e = make_env(w, dim, ORDERS["ACC"], control_set(dim, 2, False))
    S, G = queries(w, dim, 4, seed=1, yaw=False)
    paths = routes(S, G, dim)
    e.set_batch_regions(paths, rad)
    info = e.batch_regions_info()
    regions = [e.read_batch_region(q) for q in range(4)]
    h = e.handle
    pts = np.ascontiguousarray(np.concatenate(paths))
    good = np.zeros(5, np.int64)
    good[1:] = np.cumsum([len(p) for p in paths])
    bad_start = good + 1
    decreasing = good.copy()
    decreasing[2] = decreasing[1] - 1
    empty = good.copy()
    empty[2] = empty[1]
    calls = [
        (-1, good.ctypes.data, pts.ctypes.data, rad.ctypes.data),
        (4, None, pts.ctypes.data, rad.ctypes.data),
        (4, good.ctypes.data, None, rad.ctypes.data),
        (4, good.ctypes.data, pts.ctypes.data, None),
        (4, bad_start.ctypes.data, pts.ctypes.data, rad.ctypes.data),
        (4, decreasing.ctypes.data, pts.ctypes.data, rad.ctypes.data),
        (4, empty.ctypes.data, pts.ctypes.data, rad.ctypes.data),
    ]
    for args in calls:
        n0 = e.launch_count()
        assert lib.mplx_set_batch_regions(h, *args, 0) == abi.MPLX_ERR_ARG, args
        assert e.launch_count() == n0
        assert e.batch_regions_info() == info
    for q in range(4):
        assert np.array_equal(e.read_batch_region(q), regions[q])
    out = np.zeros(w["grid"].size, np.uint8)
    for q in (-1, 4):
        assert lib.mplx_read_batch_region(h, q, out.ctypes.data) == abi.MPLX_ERR_ARG
    # a search call with another query count is refused before any launch
    n0 = e.launch_count()
    for fn in (e.plan_batch, e.plan_batch_cost_terms, e.plan_batch_grow):
        with pytest.raises(abi.MplxError) as ex:
            fn(S[:3], G[:3], max_expand=20)
        assert ex.value.code == abi.MPLX_ERR_ARG
    slots, ab = C.c_int32(), C.c_int64()
    assert lib.mplx_plan_batch_fits(h, 3, 20, 1, C.byref(slots), C.byref(ab)) == abi.MPLX_ERR_ARG
    assert lib.mplx_plan_batch_fits(h, 4, 20, 1, C.byref(slots), C.byref(ab)) == abi.MPLX_OK
    assert e.launch_count() == n0
    assert e.batch_regions_info() == info
    e.close()


# ---- planner paths -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["occ", "cost"])
def test_every_planner_path_gives_the_same_results(kind):
    from motion_primitive_library_b200 import planner as P

    dim, order = 2, "ACC"
    control = ORDERS[order]
    U = control_set(dim, ORDER_OF[order], False)
    w = world(dim)
    pot = kind == "cost"
    nq, mx = 16, 60
    S, G = queries(w, dim, nq, seed=51, yaw=False)
    paths = routes(S, G, dim, seed=9)
    rad = [0.55, 0.3]
    e = make_env(w, dim, control, U, pot=pot)
    e.set_batch_regions(paths, rad)
    ref = search(e, "cost_terms", S, G, mx)
    e.close()
    args = P.make_args(dim, control, w["grid"], w["mdim"], w["origin"], w["res"], U, start=dict(pos=[0.0] * dim),
                       goal=dict(pos=[0.0] * dim), T=1.0, w=10.0, wyaw=1.0, v_max=2.0, max_num=mx, eps=2.0,
                       potential=w["pot"] if pot else None, potential_weight=0.5, gradient_weight=0.2)
    ran = {}
    for path in ("auto", "lockstep", "device", "device_cost_terms", "device_grow", "grow_fallback"):
        s = P.BatchPlanner(args, path="device_grow" if path == "grow_fallback" else path)
        try:
            if path == "grow_fallback":
                s.set_grow_caps(2, 12)  # queries that need more than 12 records go through the lock-step loop
            s.set_search_regions(paths, rad)
            res, tot, acts, closed, trajs = s.plan_detail(S, G, trajectories=True)
            with pytest.raises(RuntimeError):
                s.plan_detail(S[:3], G[:3])  # one path per query
            s.set_search_regions([], rad)
            plain = s.plan_detail(S, G)[0]
        finally:
            s.close()
        ran[path] = tot
        got = dict(valid=res["valid"], cost=res["cost"], expanded=res["expanded"], n_closed=res["n_closed"],
                   actions=acts, closed=closed, trajectories=trajs)
        for q in range(nq):
            same_query(got, q, ref, q)
        assert any(int(plain["expanded"][q]) != int(res["expanded"][q]) for q in range(nq))
    assert ran["lockstep"]["path"] == "lockstep"
    assert ran["auto"]["path"] == ("device_cost_terms" if pot else "device")
    assert ran["device_grow"]["path"] == "device_grow" and ran["grow_fallback"]["grow_lockstep"] > 0
    assert ran["device"]["path"] == ("lockstep" if pot else "device")
