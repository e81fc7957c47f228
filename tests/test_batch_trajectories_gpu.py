"""The planned trajectories of the batched device searches (mplx_set_batch_trajectories,
mplx_plan_batch_trajectories; env_map.plan_batch*(..., trajectories=True)).

Every query's trajectory is compared bit for bit across the device searches (mplx_plan_batch, mplx_plan_batch_cost_terms,
mplx_plan_batch_grow), across MultiQueryPlanner's four paths (BatchPlanner.plan_detail(trajectories=True): lockstep,
device, device_cost_terms, device_grow, and the growing search's lock-step fallback) and with the single-query host
planner on the CPU oracle env (planner_bindings.trajectory_oracle: its recovered Trajectory's waypoints and sample
rows), on every search instantiation; on non-dyadic JRK plans against the host planner and against a replay of the
action ids; with the reference's own trajectory on the corridor and one 3-D JRK plan; and under reruns (tiny arenas,
a tiny trajectory room)."""
import ctypes as C

import numpy as np
import pytest

import fixtures
import planner_bindings as pb
from motion_primitive_library_b200 import MapUtil, TrajSolverBatch, abi, env_map
from motion_primitive_library_b200 import planner as P
from reference_record import same_array
from test_device_search_cost_terms_gpu import case_params, control_set, env_for, queries, small_world

pytestmark = pytest.mark.gpu
ORDERS = {"VEL": 0x01, "ACC": 0x03, "JRK": 0x07, "SNP": 0x0F}
ORDER_OF = {"VEL": 1, "ACC": 2, "JRK": 3, "SNP": 4}
YAW_BIT = 0x10
N_SAMPLES = 24


def same_traj(a, b, what):
    assert len(a) == len(b), what
    for q, (x, y) in enumerate(zip(a, b)):
        assert x.keys() == y.keys(), (what, q)
        for k in x:
            same_array(np.ascontiguousarray(x[k]).view(np.uint8), np.ascontiguousarray(y[k]).view(np.uint8),
                       (what, q, k), bits=True)


def check_layout(r, dim, control, U, T):
    """Each trajectory's own structure: n_actions + 1 nodes (none without a segment), seg_t = T, and the
    coefficients Primitive(nodes[j], U[actions[j]], T) holds."""
    o = control & 15
    for q, t in enumerate(r["trajectories"]):
        a = r["actions"][q]
        n = len(a)
        assert len(t["nodes"]) == (n + 1 if n else 0) and len(t["seg_t"]) == n and t["coeff"].shape == (n, dim + 1, 6)
        assert np.all(t["seg_t"] == T)
        for j in range(n):
            w, u, c = t["nodes"][j], U[a[j]], np.zeros((dim + 1, 6))
            for i in range(dim):
                if o == 0x0F:
                    c[i, 1:] = (u[i], w["jrk"][i], w["acc"][i], w["vel"][i], w["pos"][i])
                elif o == 0x07:
                    c[i, 2:] = (u[i], w["acc"][i], w["vel"][i], w["pos"][i])
                elif o == 0x03:
                    c[i, 3:] = (u[i], w["vel"][i], w["pos"][i])
                else:
                    c[i, 4:] = (u[i], w["pos"][i])
            if control & YAW_BIT:
                c[dim, 4:] = (u[dim], w["yaw"])
            assert c.tobytes() == t["coeff"][j].tobytes(), (q, j)
        if n == 0:
            assert not np.any(t["samples"])


def host_trajectory_equal(args, S, G, r, dim, order, n_samples=N_SAMPLES):
    """Each query against the single-query host planner on the oracle env: validity, the waypoints' derivatives
    the primitives start from, and the sample rows bit for bit."""
    for q in range(len(S)):
        args.start.pos[:dim] = S["pos"][q, :dim]
        args.goal.pos[:dim] = G["pos"][q, :dim]
        args.start.yaw, args.goal.yaw = float(S["yaw"][q]), float(G["yaw"][q])
        h = pb.trajectory_oracle(args, n_samples)
        t = r["trajectories"][q]
        n = len(r["actions"][q])
        assert h["valid"] == int(r["valid"][q]) and h["n_actions"] == n, q
        if n == 0:
            continue
        assert h["segments"] == n
        wp = h["waypoints"]
        for k, f in enumerate(("pos", "vel", "acc", "jrk")[:order]):
            assert np.array_equal(wp[:n, k * dim:(k + 1) * dim], t["nodes"][f][:n, :dim]), (q, f)
        assert h["commands"].tobytes() == t["samples"].tobytes(), q


MATRIX = [(dim, o) for dim in (2, 3) for o in ORDERS]
CASES = ("occ", "pot", "pot_grad", "yaw", "region")


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("dim,order", MATRIX, ids=[f"{d}d-{o}" for d, o in MATRIX])
def test_paths_and_host_planner(dim, order, case):
    yaw = case == "yaw"
    control = ORDERS[order] | (YAW_BIT if yaw else 0)
    if order == "SNP":
        # a snap of 2 rather than the shared set's 4, whose first step already passes the jerk limit of 3
        import scenarios as SC

        U = SC.control_set(2.0, 3, dim, yaw_rates=(-0.5, 0.0, 0.5) if yaw else None)
    else:
        U = control_set(dim, ORDER_OF[order], yaw)
    p = case_params({"occ": "wyaw", "yaw": "wyaw", "region": "pot_region"}.get(case, case), yaw)
    w = small_world(dim)
    nq, mx, eps = 8, 40 if dim == 3 else 60, 2.0
    S, G = queries(w, dim, nq, seed=11 + dim, yaw=yaw)
    region = None
    if case == "region":
        region = np.ones(w["shape"], np.uint8)
        region.reshape(-1)[: w["grid"].size // 3] = 0
        region = region.reshape(-1)
    e = env_for(w, dim, control, U, p, region=region)
    kw = dict(eps=eps, max_expand=mx, trajectories=True, n_samples=N_SAMPLES)
    runs = {"cost_terms": e.plan_batch_cost_terms(S, G, **kw),
            "grow": e.plan_batch_grow(S, G, cost_terms=True, **kw)}
    if case == "occ":
        runs["device"] = e.plan_batch(S, G, **kw)
        runs["grow_occ"] = e.plan_batch_grow(S, G, **kw)
    e.close()
    base = runs["cost_terms"]
    # the tunnel, and in 3-D the 81 SNP x yaw primitives within 40 expansions, leave plans without a trajectory
    if case != "region" and not (dim == 3 and order == "SNP" and yaw):
        assert any(len(a) for a in base["actions"])
    for name, r in runs.items():
        for q in range(nq):
            assert np.array_equal(r["actions"][q], base["actions"][q]), (name, q)
        same_traj(r["trajectories"], base["trajectories"], name)
    check_layout(base, dim, control, U, 1.0)
    if case != "region":  # the batch session's arguments carry no search region
        from test_device_search_cost_terms_gpu import args_for

        args = args_for(w, dim, control, U, p, mx, eps)
        paths = ["lockstep", "device_cost_terms", "device_grow"] + (["device"] if case == "occ" else [])
        for path in paths:
            r = planner_trajectories(args, S, G, path)
            same_traj(r, base["trajectories"], path)
        host_trajectory_equal(args, S, G, base, dim, ORDER_OF[order])


def planner_trajectories(args, S, G, path, grow_caps=None):
    """MultiQueryPlanner's trajectories on one path (BatchPlanner.plan_detail(trajectories=True)), checked to have
    run there."""
    bp = P.BatchPlanner(args, path=path)
    try:
        if grow_caps:
            bp.set_grow_caps(*grow_caps)
        res, tot, acts, _, trajs = bp.plan_detail(S, G, closed=False, trajectories=True, n_samples=N_SAMPLES)
        # the session's next plan no longer collects them
        again = bp.plan_detail(S, G, closed=False)
    finally:
        bp.close()
    assert tot["path"] == path and len(again) == 4
    for q, t in enumerate(trajs):
        assert len(t["seg_t"]) == len(acts[q])
    if grow_caps:
        assert tot["grow_lockstep"] > 0
    return trajs


def test_grow_lockstep_fallback_merges_trajectories():
    w = small_world(2, seed=4)
    U = control_set(2, 2, False)
    p = case_params("wyaw", False)
    from test_device_search_cost_terms_gpu import args_for

    args = args_for(w, 2, ORDERS["ACC"], U, p, 60, 2.0)
    S, G = queries(w, 2, 16, seed=4, yaw=False)
    lock = planner_trajectories(args, S, G, "lockstep")
    grow = planner_trajectories(args, S, G, "device_grow", grow_caps=(3, 12))
    assert any(len(t["seg_t"]) for t in lock)
    same_traj(grow, lock, "device_grow with lock-step fallback")


# ---- non-dyadic plans: the stored coordinates against the host and against a replay of the actions ---------------
FIELDS = ("pos", "vel", "acc", "jrk", "yaw")


@pytest.mark.parametrize("dim", [2, 3])
def test_non_dyadic_jrk_nodes_are_the_hosts(dim, capsys):
    """JRK at T = 0.7 (not a power of two), U = {-1.3, 0, 1.3}^dim and starts 0.013 off the cell centres.  Every
    query's recorded nodes and samples must be the host planner's bit for bit.  The replay of the action ids from the
    start (each step the device expansion's own successor, the arithmetic the search runs) is compared with the
    recorded nodes and the queries where it differs are counted; on these inputs every replay has matched the
    recorded nodes (0 differing queries on an H100), so the replay check reports rather than requires a difference:
    that the nodes are the search's is shown by their equality with the host planner's stored coordinates."""
    import scenarios as SC

    T = 0.7
    w = small_world(dim, seed=21)
    U = SC.control_set(1.3, 3, dim)
    p = case_params("wyaw", False)
    e = env_for(w, dim, ORDERS["JRK"], U, p)
    e.set_dt(T)
    nq = 48 if dim == 2 else 24
    S, G = queries(w, dim, nq, seed=5, yaw=False)
    S["pos"][:, :dim] += 0.013
    mx = 300 if dim == 2 else 120
    r = e.plan_batch(S, G, eps=2.0, max_expand=mx, trajectories=True, n_samples=N_SAMPLES)
    qs = [q for q in range(nq) if len(r["actions"][q])]
    assert len(qs) >= nq // 3
    cur = np.array([r["trajectories"][q]["nodes"][0] for q in qs])
    differs = set()
    for k in range(max(len(r["actions"][q]) for q in qs)):
        live = [i for i, q in enumerate(qs) if k < len(r["actions"][q])]
        ex = e.expand(cur[live], want=("succ", "action"))
        for j, i in enumerate(live):
            q = qs[i]
            succ, _, act = ex.node(j)
            hit = np.nonzero(act == r["actions"][q][k])[0]
            if not len(hit):  # the replayed state no longer has the action
                differs.add(q)
                continue
            nxt = succ[hit[0]]
            rec = r["trajectories"][q]["nodes"][k + 1]
            if any(nxt[f].tobytes() != rec[f].tobytes() for f in FIELDS):
                differs.add(q)
            cur[i] = nxt
    e.close()
    args = pb.make_args(dim, ORDERS["JRK"], w["grid"], w["mdim"], w["origin"], w["res"], U, start=dict(pos=[0] * dim),
                        goal=dict(pos=[0] * dim), T=T, w=10.0, v_max=2.0, a_max=2.0, max_num=mx, eps=2.0)
    host_trajectory_equal(args, S, G, r, dim, 3)
    with capsys.disabled():
        print(f"\n[{dim}-D JRK, T = {T}] replay of the actions differs from the recorded nodes on {len(differs)} of "
              f"{len(qs)} trajectories")


# ---- the reference's own trajectory -------------------------------------------------------------------------
def corridor_env(control, U):
    c = fixtures.corridor()
    mu = MapUtil()
    mu.setMap(c["origin"], c["dim"], c["grid"], c["res"])
    e = env_map(mu, device=0)
    e.set_control(control)
    e.set_u(U)
    e.set_dt(1.0)
    e.set_w(10.0)
    e.set_v_max(1.0)
    e.set_a_max(1.0)
    return c, e


@pytest.mark.parametrize("control", [0x01, 0x03])
def test_corridor_matches_the_reference(control):
    U = fixtures.U_2d() * (2.0 if control == 0x01 else 1.0)
    c = fixtures.corridor()
    args = pb.make_args(2, control, c["grid"], c["dim"], c["origin"], c["res"], U, start=dict(pos=c["start"]),
                        goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0, max_num=2000)
    ref = pb.trajectory_reference(args, N_SAMPLES)
    _, e = corridor_env(control, U)
    S = np.zeros(1, dtype=P.WAYPOINT_DTYPE)
    G = np.zeros(1, dtype=P.WAYPOINT_DTYPE)
    S["pos"][0, :2], G["pos"][0, :2] = c["start"], c["goal"]
    r = e.plan_batch(S, G, eps=1.0, max_expand=2000, trajectories=True, n_samples=N_SAMPLES)
    e.close()
    t = r["trajectories"][0]
    assert ref["valid"] == 1 and int(r["valid"][0]) == 1 and ref["segments"] == len(t["seg_t"])
    same_array(ref["commands"], t["samples"], "samples", bits=True)
    n = len(t["seg_t"])
    same_array(ref["waypoints"][:n, :2], t["nodes"]["pos"][:n, :2], "waypoints")


def test_3d_jrk_matches_the_reference():
    import scenarios as SC

    sc = SC.scaled(SC.cfg3(), 32)
    U = SC.control_set(1.0, 3, 3)
    nodes = sc.frontier(2, seed=7, max_steps=0)
    s, g = nodes["pos"][0], nodes["pos"][1]
    args = pb.make_args(3, 0x07, sc.grid(), sc.dim_cells, sc.origin, sc.res, U, start=dict(pos=s), goal=dict(pos=g),
                        T=sc.T, w=sc.w, v_max=sc.v_max, a_max=sc.a_max, eps=2.0, max_num=400)
    ref = pb.trajectory_reference(args, N_SAMPLES)
    mu = MapUtil()
    mu.setMap(sc.origin, sc.dim_cells, sc.grid(), sc.res)
    e = env_map(mu, device=0)
    e.set_control(0x07)
    e.set_u(U)
    e.set_dt(sc.T)
    e.set_w(sc.w)
    e.set_v_max(sc.v_max)
    e.set_a_max(sc.a_max)
    S = np.zeros(1, dtype=P.WAYPOINT_DTYPE)
    G = np.zeros(1, dtype=P.WAYPOINT_DTYPE)
    S["pos"][0], G["pos"][0] = s, g
    r = e.plan_batch(S, G, eps=2.0, max_expand=400, trajectories=True, n_samples=N_SAMPLES)
    e.close()
    t = r["trajectories"][0]
    assert int(r["valid"][0]) == ref["valid"] and ref["segments"] == len(t["seg_t"])
    same_array(ref["commands"], t["samples"], "samples", bits=True)


# ---- reruns, the ABI contract and the feed-through ------------------------------------------------------------
def occ_setup(n=24, seed=4):
    dim = 2
    w = small_world(dim, seed=seed)
    U = control_set(dim, 2, False)
    e = env_for(w, dim, ORDERS["ACC"], U, case_params("wyaw", False))
    S, G = queries(w, dim, n, seed=seed, yaw=False)
    return w, U, e, S, G


def test_results_do_not_depend_on_room_or_arenas():
    _, _, e, S, G = occ_setup()
    kw = dict(eps=2.0, max_expand=60, trajectories=True, n_samples=N_SAMPLES)
    base = e.plan_batch(S, G, **kw)
    e._sync_params()
    n0 = e.launch_count()
    tiny = e.plan_batch(S, G, traj_room_bytes=112, **kw)
    # a room of one waypoint: every query with a trajectory needs a round of its own
    assert e.launch_count() - n0 > 2
    grow = e.plan_batch_grow(S, G, first_cap=3, max_cap=200, pool_bytes=64, traj_room_bytes=300, **kw)
    assert grow["reruns"] > 0
    for r in (tiny, grow):
        for q in range(len(S)):
            if "searched" in r and not r["searched"][q]:
                assert len(r["trajectories"][q]["nodes"]) == 0
                continue
            assert np.array_equal(r["actions"][q], base["actions"][q])
            same_traj([r["trajectories"][q]], [base["trajectories"][q]], q)
    e.close()


def test_recording_off_keeps_one_launch_and_on_is_one_round():
    _, _, e, S, G = occ_setup()
    e._sync_params()
    n0 = e.launch_count()
    off = e.plan_batch(S, G, eps=2.0, max_expand=60)
    assert e.launch_count() == n0 + 1
    n1 = e.launch_count()
    on = e.plan_batch(S, G, eps=2.0, max_expand=60, trajectories=True)
    # one search launch, then mplx_plan_batch_trajectories' two
    assert e.launch_count() == n1 + 3
    for q in range(len(S)):
        assert np.array_equal(off["actions"][q], on["actions"][q]) and off["cost"][q] == on["cost"][q]
    e.close()


def test_abi_contract():
    w, U, e, S, G = occ_setup(n=12)
    lib, h = e._lib, e._h
    dim = 2
    out = abi.BatchTrajOut()
    offset = np.full(len(S) + 1, -5, np.int64)
    nodes = np.zeros(4096, dtype=P.WAYPOINT_DTYPE)
    seg_t, coeff = np.zeros(4096), np.zeros((4096, dim + 1, 6))
    samples = np.zeros((len(S), 9, 4 * dim + 3))

    def call(n_samples=0, cap=4096, with_samples=False, **drop):
        o = abi.BatchTrajOut(offset.ctypes.data, nodes.ctypes.data, seg_t.ctypes.data, coeff.ctypes.data,
                             samples.ctypes.data if with_samples else None, cap, -3, 0.0)
        for k in drop:
            setattr(o, k, None)
        n0 = e.launch_count()
        rc = lib.mplx_plan_batch_trajectories(h, n_samples, C.byref(o))
        return rc, o, e.launch_count() - n0

    # no search call yet: refused, nothing written
    rc, o, nl = call()
    assert rc == abi.MPLX_ERR_ARG and nl == 0 and o.total == -3 and np.all(offset == -5)
    # the last search ran without recording
    e.plan_batch(S, G, eps=2.0, max_expand=60)
    rc, o, nl = call()
    assert rc == abi.MPLX_ERR_ARG and nl == 0 and np.all(offset == -5)
    r = e.plan_batch(S, G, eps=2.0, max_expand=60, trajectories=True)
    need = sum(len(a) + 1 for a in r["actions"] if len(a))
    assert need > 0
    for bad in (dict(n_samples=-1), dict(n_samples=0, with_samples=True), dict(offset=1), dict(nodes=1),
                dict(seg_t=1), dict(coeff=1)):
        kw = {k: v for k, v in bad.items() if k in ("n_samples", "with_samples")}
        drop = {k: v for k, v in bad.items() if k not in kw}
        rc, o, nl = call(**kw, **drop)
        assert rc == abi.MPLX_ERR_ARG and nl == 0 and o.total == -3 and np.all(offset == -5), bad
    # capacity: too small fills offset and total, then fails
    rc, o, nl = call(cap=need - 1)
    assert rc == abi.MPLX_ERR_ARG and nl == 0 and o.total == need and offset[-1] == need
    # a constant launch count whatever the batch
    rc, o, nl = call(cap=need)
    assert rc == 0 and nl == 2
    rc, o, nl = call(n_samples=8, with_samples=True)
    assert rc == 0 and nl == 3
    first = nodes[:need].copy()
    # a second search replaces what the ctx kept
    r2 = e.plan_batch(G, S, eps=2.0, max_expand=60, trajectories=True)
    need2 = sum(len(a) + 1 for a in r2["actions"] if len(a))
    rc, o, nl = call()
    assert rc == 0 and o.total == need2 and nl == 2
    assert not (need2 == need and nodes[:need].tobytes() == first.tobytes())
    single = e.plan_batch(S[:1], G[:1], eps=2.0, max_expand=60, trajectories=True)
    rc, o, nl = call()
    assert rc == 0 and nl == 2 and o.total == sum(len(a) + 1 for a in single["actions"] if len(a))
    e.close()


def test_feed_through_check_and_scale():
    w, U, e, S, G = occ_setup(n=16)
    r = e.plan_batch(S, G, eps=2.0, max_expand=60, trajectories=True, n_samples=N_SAMPLES)
    trajs = r["trajectories"]
    dev, _ = e.traverse_trajectories(trajs, ORDERS["ACC"])
    host = P.traj_check(2, w["grid"], w["mdim"], w["origin"], w["res"], trajs, ORDERS["ACC"], v_max=2.0)
    for q in range(len(S)):
        assert dev[q]["status"] == int(host["status"][q])
        assert np.float64(dev[q]["cost"]).tobytes() == np.float64(host["cost"][q]).tobytes(), q
    tsb = TrajSolverBatch(2, device=0)
    scaled, _ = tsb.scale(trajs, abi.TRAJ_SCALE, ri=0.5, rf=0.5)
    for q, s in enumerate(scaled):
        assert s["status"] == (1 if len(trajs[q]["seg_t"]) else 0), q
    tsb.close()
    e.close()
