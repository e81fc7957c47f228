"""The device search (mplx_plan_batch, csrc/mplx_search.cu + mplx_search.cuh) on every instantiation, control-set
width, bookkeeping edge and cross-call arena state.

Every query is compared with the host planner on the CPU oracle env (planner_bindings.plan_oracle: the host
A* and the CPU expansion, no code shared with the search kernel) and with the forced lock-step loop of
MultiQueryPlanner.  The bar: validity, expansions, n_closed, the action sequence and the sorted closed keys
equal, the cost equal bit for bit.  Every device call shows that the device search ran: BatchPlanner reports
path "device", and the raw mplx_plan_batch call adds exactly one launch to its ctx.

tests/test_search_inputs_oracle_vs_ref.py pins the oracle planner against the reference planner on the same
input classes.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import planner_bindings as pb
from motion_primitive_library_b200 import abi
from motion_primitive_library_b200 import planner as P

pytestmark = pytest.mark.gpu

VEL, ACC, JRK, SNP = 0x01, 0x03, 0x07, 0x0F
ORDER = {VEL: 1, ACC: 2, JRK: 3, SNP: 4}
NAME = {VEL: "VEL", ACC: "ACC", JRK: "JRK", SNP: "SNP"}
THREADS = 256                   # kThreads: the widest control set the device search takes
SEARCH_BUDGET = 8 << 30         # kSearchArenaBudget
WAYPOINT_BYTES = 14 * 8         # mplx_waypoint
SSTATE_BYTES = WAYPOINT_BYTES + 2 * 8 + 8 + 4 * 4
SPRED_BYTES = 4 * 4 + 8
SHEAP_BYTES = 8 + 2 * 4
SSLOT_BYTES = 8 + 2 * 4
WIDTHS = (1, 2, 31, 32, 33, 64, 65, 243, 255, 256)


# ---- restatements of the launcher and the sizing rules ------------------------------------------------
def search_instantiation(dim, control):
    """mplx_plan_batch (csrc/mplx_search.cu): the search_kernel<DIM, ORD> a plan runs, from control & 15."""
    order = ORDER.get(control & 15)
    if order is None:
        raise ValueError(f"control {control:#x} has no search kernel")
    return dim, order


def block_of(nU):
    """The search kernel's block: nU rounded up to a whole warp."""
    return ((nU + 31) // 32) * 32


def ballot_words(nU):
    """Shared words of the validity ballot (vbits)."""
    return (nU + 31) // 32


def round256(x):
    return (x + 255) & ~255


def layout_for(max_expand, nU):
    """layout_for (csrc/mplx_search.cuh): the worst-case arena of one query."""
    cap = 1 + max_expand * nU
    tab = 1
    while tab < 2 * cap:
        tab <<= 1
    st, pr, hp = round256(cap * SSTATE_BYTES), round256(cap * SPRED_BYTES), round256(cap * SHEAP_BYTES)
    return dict(cap=cap, tab=tab, off_pred=st, off_heap=st + pr, off_tab=st + pr + hp,
                bytes=st + pr + hp + tab * SSLOT_BYTES)


def results_bytes(n_q, max_expand, with_closed):
    """size_batch: the per-query arrays (start, goal, start-is-free flag, five int32 results and the query list,
    the cost, the pool offset) and the result pool (every query's worst case: max_expand closed keys when asked
    for, max_expand int32 action ids two to a uint64) a call holds next to its arenas."""
    pool_units = n_q * ((max_expand if with_closed else 0) + (max_expand + 1) // 2)
    return n_q * (2 * WAYPOINT_BYTES + 1 + 6 * 4 + 8 + 8) + 8 * pool_units


class ArenaModel:
    """The reserve/clear rule of mplx_plan_batch for one ctx: which branch a call with `slots` slots of
    `arena_bytes` bytes takes."""

    def __init__(self):
        self.cap = self.cleared = self.layout = 0

    def call(self, slots, arena_bytes):
        need = slots * arena_bytes
        taken = set()
        if self.cap < need:
            self.cap, self.cleared = need, 0
            taken.add("realloc")
        if self.layout != arena_bytes or self.cleared < need:
            taken.add("clear-layout" if self.layout != arena_bytes else "clear-more-slots")
            self.layout, self.cleared = arena_bytes, need
        else:
            taken.add("epochs-continue")
        return taken


# ---- inputs ------------------------------------------------------------------------------------------
class Scene:
    """One plan's map, controls and limits, with the per-call search parameters."""

    def __init__(self, dim, control, U, grid, mdim, origin, res, T=1.0, w=10.0, v_max=-1.0, a_max=-1.0, j_max=-1.0,
                 eps=1.0, max_expand=150, tol_pos=0.5, tol_vel=-1.0, tol_acc=-1.0):
        self.dim, self.control = dim, control
        self.U = np.ascontiguousarray(U, dtype=np.float64)
        self.grid = np.ascontiguousarray(grid, dtype=np.int8).reshape(-1)
        self.mdim, self.origin, self.res = tuple(int(m) for m in mdim), tuple(float(o) for o in origin), float(res)
        self.T, self.w, self.v_max, self.a_max, self.j_max = T, w, v_max, a_max, j_max
        self.search = dict(eps=eps, max_expand=max_expand, tol_pos=tol_pos, tol_vel=tol_vel, tol_acc=tol_acc)

    @property
    def nU(self):
        return self.U.shape[0]

    def with_(self, **kw):
        s = Scene(self.dim, self.control, self.U, self.grid, self.mdim, self.origin, self.res, self.T, self.w,
                  self.v_max, self.a_max, self.j_max, **self.search)
        for k, v in kw.items():
            if k in s.search:
                s.search[k] = v
            else:
                setattr(s, k, v)
        return s

    def args(self, start=None, goal=None):
        sp = lambda x: {} if x is None else {f: x[f][: self.dim] for f in ("pos", "vel", "acc", "jrk")}
        s = self.search
        return pb.make_args(self.dim, self.control, self.grid, self.mdim, self.origin, self.res, self.U, start=sp(start),
                            goal=sp(goal), T=self.T, w=self.w, v_max=self.v_max, a_max=self.a_max, j_max=self.j_max,
                            eps=s["eps"], max_num=s["max_expand"], tol_pos=s["tol_pos"], tol_vel=s["tol_vel"],
                            tol_acc=s["tol_acc"])

    def env(self):
        from motion_primitive_library_b200 import MapUtil, env_map

        mu = MapUtil()
        mu.setMap(self.origin, self.mdim, self.grid.copy(), self.res)
        e = env_map(mu, device=0)
        e.set_control(self.control)
        e.set_u(self.U)
        e.set_dt(self.T)
        e.set_w(self.w)
        e.set_v_max(self.v_max)
        e.set_a_max(self.a_max)
        e.set_j_max(self.j_max)
        e._sync_params()
        return e

    def oracle_env(self):
        import oracle_bindings as ob

        return ob.OracleEnv(self.dim, self.control, self.U, self.grid, self.mdim, self.origin, self.res, T=self.T,
                            w=self.w, v_max=self.v_max, a_max=self.a_max, j_max=self.j_max)

    def cell(self, pos):
        """MapUtil::floatToInt: round half away from zero of (p - origin)/res - 0.5."""
        x = (np.asarray(pos, dtype=np.float64)[: self.dim] - np.asarray(self.origin[: self.dim])) / self.res - 0.5
        a = np.abs(x)
        r = np.floor(a)
        r = r + (a - r >= 0.5)
        return np.copysign(r, x).astype(np.int64)

    def value(self, pos):
        """The grid value at pos, or None outside the map."""
        c = self.cell(pos)
        if (c < 0).any() or (c >= np.asarray(self.mdim[: self.dim])).any():
            return None
        i = c[0] + self.mdim[0] * c[1] + (self.mdim[0] * self.mdim[1] * c[2] if self.dim == 3 else 0)
        return int(self.grid[i])

    def is_free(self, pos):
        v = self.value(pos)
        return v is not None and 0 <= v < 100

    def centre(self, cell):
        return np.asarray(self.origin[: self.dim]) + (np.asarray(cell, dtype=np.float64) + 0.5) * self.res

    def free_cells(self, margin=3):
        shape = self.mdim[: self.dim][::-1]
        g = self.grid.reshape(shape)
        cells = np.argwhere(g == 0)[:, ::-1]  # x first
        inner = ((cells >= margin) & (cells < np.asarray(self.mdim[: self.dim]) - margin)).all(1)
        return cells[inner]


def voxel_grid(mdim, seed, boxes=None, occupied=0.02, unknown=0.03):
    """Random boxes of occupied cells plus scattered occupied and unknown (-1) cells, x fastest."""
    rng = np.random.default_rng(seed)
    shape = tuple(mdim[::-1])
    g = np.zeros(shape, np.int8)
    for _ in range(boxes if boxes is not None else 6 * len(mdim)):
        lo = [int(rng.integers(0, s - 4)) for s in shape]
        size = [int(rng.integers(2, 7)) for _ in shape]
        g[tuple(slice(l, l + z) for l, z in zip(lo, size))] = 100
    r = rng.random(shape)
    g[r < occupied] = 100
    g[(r >= occupied) & (r < occupied + unknown)] = -1
    return g.reshape(-1)


MAP3 = dict(mdim=(48, 44, 40), origin=(-2.0, 1.0, -0.5), res=0.25)
MAP2 = dict(mdim=(96, 80), origin=(-3.0, 2.0), res=0.25)


def base_scene(dim, control, U=None, seed=1, **kw):
    m = MAP3 if dim == 3 else MAP2
    if U is None:
        U = product_set(*[u_values(control)] * dim)
    lim = dict(v_max=2.0, a_max=2.0, j_max=4.0)
    lim.update(kw)
    return Scene(dim, control, U, voxel_grid(m["mdim"], seed), m["mdim"], m["origin"], m["res"], **lim)


def product_set(*axes):
    grids = np.meshgrid(*[np.asarray(a, dtype=np.float64) for a in axes], indexing="ij")
    return np.ascontiguousarray(np.stack([g.reshape(-1) for g in grids], axis=1))


def u_values(control):
    return {VEL: (-1.0, 0.0, 1.0), ACC: (-1.0, 0.0, 1.0), JRK: (-2.0, 0.0, 2.0), SNP: (-4.0, 0.0, 4.0)}[control & 15]


def wps(pts, dim):
    w = np.zeros(len(pts), dtype=P.WAYPOINT_DTYPE)
    w["pos"][:, :dim] = np.asarray(pts, dtype=np.float64).reshape(len(pts), dim)
    return w


def random_queries(scene, n, seed, near=(0.75, 2.5), far_every=4):
    """Starts on free cell centres; goals near the start (most), or at a random free cell far away."""
    rng = np.random.default_rng(seed)
    cells = scene.free_cells()
    hi = np.asarray(scene.origin[: scene.dim]) + np.asarray(scene.mdim[: scene.dim]) * scene.res
    S, G = [], []
    for k in range(n):
        s = scene.centre(cells[rng.integers(len(cells))])
        if k % far_every == far_every - 1:
            g = scene.centre(cells[rng.integers(len(cells))])
        else:
            d = rng.normal(size=scene.dim)
            g = s + d / np.linalg.norm(d) * rng.uniform(*near)
            g = np.clip(np.round(g / 0.25) * 0.25, np.asarray(scene.origin[: scene.dim]) + 0.5, hi - 0.5)
        S.append(s)
        G.append(g)
    return wps(S, scene.dim), wps(G, scene.dim)


# ---- runs --------------------------------------------------------------------------------------------
def oracle_run(scene, S, G):
    """The host planner on the CPU oracle env, one query at a time."""
    return [pb.plan_oracle(scene.args(S[q], G[q])) for q in range(len(S))]


def device_run(env, scene, S, G, start_free=None, closed=True):
    """mplx_plan_batch on env's ctx: exactly one launch."""
    n0 = env.launch_count()
    s = scene.search
    r = env.plan_batch(S, G, eps=s["eps"], max_expand=s["max_expand"], tol_pos=s["tol_pos"], tol_vel=s["tol_vel"],
                       tol_acc=s["tol_acc"], start_free=start_free, closed=closed)
    assert env.launch_count() == n0 + (1 if len(S) else 0)
    return r


def batch_run(scene, S, G, path):
    s = P.BatchPlanner(scene.args(), path=path)
    try:
        res, tot, acts, closed = s.plan_detail(S, G)
    finally:
        s.close()
    assert tot["path"] == path
    return dict(valid=res["valid"], cost=res["cost"], expanded=res["expanded"], n_closed=res["n_closed"], actions=acts,
                closed=closed)


def same_results(a, b, what, closed=True):
    for f in ("valid", "expanded", "n_closed"):
        assert np.array_equal(a[f], b[f]), (what, f)
    assert np.asarray(a["cost"], np.float64).tobytes() == np.asarray(b["cost"], np.float64).tobytes(), what
    for q in range(len(a["valid"])):
        assert np.array_equal(a["actions"][q], b["actions"][q]), (what, "actions", q)
        if closed:
            assert np.array_equal(a["closed"][q], b["closed"][q]), (what, "closed", q)


def same_as_oracle(d, orc):
    for q, o in enumerate(orc):
        got = (int(d["valid"][q]), int(d["expanded"][q]), int(d["n_closed"][q]))
        assert got == (o["valid"], o["expanded"], o["n_closed"]), (q, got, o)
        assert np.array_equal(d["actions"][q], o["actions"]), q
        assert np.array_equal(d["closed"][q], np.sort(o["closed"])), q
        if o["valid"]:
            assert np.float64(d["cost"][q]).tobytes() == np.float64(o["cost"]).tobytes(), (q, d["cost"][q], o["cost"])
        else:
            # no trajectory: the batch planners report +inf; MapPlanner::plan leaves its cost at 0 when the
            # start is not free (the reference leaves it unset)
            assert np.isinf(d["cost"][q]), q


def check(scene, S, G):
    """The device search through BatchPlanner (start_free from the host map) and through the raw ABI with
    start_free NULL (the device grid decides) and from the host, the lock-step loop and the oracle planner,
    all equal.  Returns the device results."""
    d = batch_run(scene, S, G, "device")
    same_results(d, batch_run(scene, S, G, "lockstep"), "lockstep")
    env = scene.env()
    try:
        same_results(d, device_run(env, scene, S, G), "raw, start_free NULL")
        sf = np.array([scene.is_free(S["pos"][q]) for q in range(len(S))], np.uint8)
        same_results(d, device_run(env, scene, S, G, start_free=sf), "raw, start_free from the host")
    finally:
        env.close()
    same_as_oracle(d, oracle_run(scene, S, G))
    return d


# ---- instantiations ----------------------------------------------------------------------------------
MATRIX = [(dim, control) for dim in (2, 3) for control in (VEL, ACC, JRK, SNP)]
# per control: eps, max_expand, T, goal distances (m).  SNP moves slowly: a shorter T, nearer goals.
MATRIX_SEARCH = {VEL: (1.0, 100, 1.0, (1.0, 3.0)), ACC: (1.0, 100, 1.0, (1.0, 3.0)), JRK: (2.0, 150, 1.0, (1.0, 3.0)),
                 SNP: (2.0, 150, 0.5, (0.3, 1.0))}


def matrix_case(dim, control):
    eps, mx, T, near = MATRIX_SEARCH[control]
    sc = base_scene(dim, control, seed=10 * dim + ORDER[control], eps=eps, max_expand=mx, T=T)
    S, G = random_queries(sc, 12, seed=dim * 100 + control, near=near, far_every=3)
    return sc, S, G


def test_matrix_reaches_every_instantiation():
    reached = {search_instantiation(dim, control) for dim, control in MATRIX}
    assert reached == {(d, o) for d in (2, 3) for o in (1, 2, 3, 4)}
    with pytest.raises(ValueError):
        search_instantiation(3, 0x00)
    # the widths reach both ends of the ballot: one word (nU 1..32) up to all eight (nU 225..256)
    assert {ballot_words(n) for n in WIDTHS} == {1, 2, 3, 8}
    assert {block_of(n) for n in WIDTHS} == {32, 64, 96, 256}
    print("search instantiations:", sorted(reached), "widths:", WIDTHS)


@pytest.mark.parametrize("dim,control", MATRIX, ids=[f"{d}d-{NAME[c]}" for d, c in MATRIX])
def test_instantiation_matrix(dim, control):
    sc, S, G = matrix_case(dim, control)
    assert (sc.grid == -1).any() and (sc.grid == 100).any()
    d = check(sc, S, G)
    assert d["valid"].any(), "no query of this instantiation reached its goal"
    assert (d["expanded"] == sc.search["max_expand"]).any(), "no query ended at max_expand"


# ---- control-set widths ------------------------------------------------------------------------------
def width_set(nU, kind, dim, seed):
    """A control set of exactly nU rows: a product of per-axis value lists, or random rows."""
    if kind == "product":
        per_axis = {1: (1, 1, 1), 2: (2, 1, 1), 32: (2, 4, 4) if dim == 3 else (4, 8), 33: (3, 11),
                    64: (4, 4, 4) if dim == 3 else (8, 8), 65: (5, 13), 243: (3, 9, 9) if dim == 3 else (9, 27),
                    255: (3, 5, 17), 256: (4, 8, 8) if dim == 3 else (16, 16)}[nU][:dim]
        per_axis = per_axis + (1,) * (dim - len(per_axis))
        # outer axes within [-1, 1], the innermost (fastest-varying) axis out to 1.5: under v_max = 1 every
        # run of 32 control ids holds primitives that pass and primitives that fail
        axes = [np.linspace(-1.5 if k == dim - 1 else -1.0, 1.5 if k == dim - 1 else 1.0, m) if m > 2
                else np.array([-1.0, 0.75][:m] if m == 2 else [0.5]) for k, m in enumerate(per_axis)]
        U = product_set(*axes)
    else:
        rng = np.random.default_rng(seed)
        U = np.round(rng.uniform(-1.5, 1.5, (nU, dim)) * 8) / 8
    assert U.shape == (nU, dim)
    return U


WIDTH_CASES = [(1, "product", 3), (1, "random", 2), (2, "product", 2), (2, "random", 3), (31, "random", 2),
               (31, "random", 3), (32, "product", 2), (32, "product", 3), (33, "product", 2), (33, "random", 3),
               (64, "product", 3), (64, "random", 2), (65, "product", 2), (65, "random", 3), (243, "product", 3),
               (243, "random", 2), (255, "product", 3), (255, "random", 2), (256, "product", 2), (256, "product", 3),
               (256, "random", 3)]


def width_scene(nU, kind, dim):
    U = width_set(nU, kind, dim, seed=nU * 10 + dim)
    mx = 60 if nU > 100 else 120
    # from rest, v_max = 1 fails every primitive with a control component beyond 1: gaps in every ballot word
    return base_scene(dim, ACC, U=U, seed=nU + dim, v_max=1.0, a_max=1.2, eps=2.0, max_expand=mx)


def sparse_ballot_words(scene, S):
    """The ballot words (32 control ids each, the last one partial) that the oracle's expansion of the starts
    and of their successors leaves sparse: some node emits a non-empty strict subset of the word's ids, or,
    for a word of one id, some node emits it while another does not."""
    nU = scene.nU
    orc = scene.oracle_env()
    e = orc.expand(S)
    succ = np.concatenate([e["succ"][i * nU: i * nU + e["count"][i]] for i in range(len(S))])
    nodes = np.concatenate([S, succ])
    e = orc.expand(nodes)
    emitted = np.zeros((len(nodes), nU), bool)
    for i in range(len(nodes)):
        emitted[i, e["action"][i * nU: i * nU + e["count"][i]]] = True
    sparse = []
    for w in range(ballot_words(nU)):
        word = emitted[:, 32 * w: min(32 * w + 32, nU)]
        some = word.any(1)
        if word.shape[1] > 1 and (some & ~word.all(1)).any():
            sparse.append(w)
        elif word.shape[1] == 1 and some.any() and not some.all():
            sparse.append(w)
    return sparse


@pytest.mark.parametrize("nU,kind,dim", WIDTH_CASES, ids=[f"{n}-{k}-{d}d" for n, k, d in WIDTH_CASES])
def test_control_set_widths(nU, kind, dim):
    sc = width_scene(nU, kind, dim)
    S, G = random_queries(sc, 8, seed=nU + 7 * dim, near=(1.5, 3.0))
    d = check(sc, S, G)
    assert (d["expanded"] > 0).any()
    if nU > 2:
        # every ballot word, the later ones included, holds emitted and rejected primitives of one node
        assert sparse_ballot_words(sc, S) == list(range(ballot_words(nU)))


def test_width_257_refused_and_auto_takes_the_lockstep_path():
    sc = width_scene(256, "random", 3)
    sc = sc.with_(U=np.vstack([sc.U, [[0.0, 0.0, 0.25]]]))
    assert sc.nU == THREADS + 1
    S, G = random_queries(sc, 16, seed=3, near=(0.5, 1.0))
    env = sc.env()
    try:
        n0 = env.launch_count()
        with pytest.raises(abi.MplxError) as ex:
            env.plan_batch(S, G, max_expand=20)
        assert ex.value.code == abi.MPLX_ERR_ARG and env.launch_count() == n0
        assert env._lib.mplx_plan_batch_fits(env.handle, 16, 20, 1, None, None) == abi.MPLX_ERR_ARG
    finally:
        env.close()
    sc = sc.with_(max_expand=20)
    s = P.BatchPlanner(sc.args())
    try:
        res, tot = s.plan(S, G)
        assert tot["path"] == "lockstep"
    finally:
        s.close()
    orc = oracle_run(sc, S, G)
    assert [int(v) for v in res["valid"]] == [o["valid"] for o in orc]
    assert [int(v) for v in res["expanded"]] == [o["expanded"] for o in orc]


# ---- bookkeeping edges -------------------------------------------------------------------------------
def edge_scene(**kw):
    return base_scene(3, ACC, seed=31, **kw)


def eps_case(eps):
    """16 random queries, and four that re-open a closed state at eps 2 or 5 (the re-opened state is
    expanded twice but closed once)."""
    sc = edge_scene(eps=eps, w=1.0, max_expand=200)
    S, G = random_queries(sc, 16, seed=41, near=(2.0, 5.0), far_every=2)
    S2, G2 = random_queries(sc, 214, seed=99, near=(2.0, 5.0), far_every=2)
    pick = [25, 213, 11, 17]
    return sc, np.concatenate([S, S2[pick]]), np.concatenate([G, G2[pick]])


@pytest.mark.parametrize("eps", [0.0, 1.0, 2.0, 5.0])
def test_eps_values(eps):
    sc, S, G = eps_case(eps)
    d = check(sc, S, G)
    if eps > 1:
        assert (d["expanded"] > d["n_closed"]).any(), "no closed state was re-opened"


def heur(scene, pos, goal):
    """get_heur for a non-goal key, as the search computes it (w * linf / v_max)."""
    m = 0.0
    for k in range(scene.dim):
        x = abs(pos[k] - goal[k])
        m = x if m < x else m
    return scene.w * m / scene.v_max if scene.v_max > 0 else scene.w * m


def tie_at_second_pop(scene, S, G, q):
    """After the start's expansion, the open states of least f share it with different g: the heap's g
    tie-break decides the second pop."""
    e = scene.oracle_env().expand(S[q:q + 1])
    n = int(e["count"][0])
    cost, succ = e["cost"][:n], e["succ"][:n]
    fin = np.isfinite(cost)
    eps = scene.search["eps"]
    f = np.array([c + eps * heur(scene, s["pos"], G["pos"][q]) for c, s in zip(cost[fin], succ[fin])])
    g = cost[fin]
    if not len(f):
        return False
    tied = f == f.min()
    # successors that share a position are one state: keep distinct keys only
    keys = e["key"][:n][fin][tied]
    return len(set(g[tied].tolist())) > 1 and len(set(keys.tolist())) > 1


def tie_case():
    # ACC from rest, T = 1: one more unit of control on an axis adds 1 to the edge cost (J = |u|^2 T) and
    # moves 0.5 m nearer the goal, which lowers eps*h = eps*w*linf/v_max by exactly 1 with eps = w = v_max = 2.
    # So from a cell centre, the successors towards a diagonal goal share the least f with different g.
    sc = edge_scene(eps=2.0, w=2.0, v_max=2.0, tol_pos=0.25)
    cells = sc.free_cells(margin=10)
    rng = np.random.default_rng(5)
    pick = cells[rng.choice(len(cells), 12, replace=False)]
    S = wps([sc.centre(c) for c in pick], 3)
    off = np.array([[2.0, 2.0, 0], [-2.0, 2.0, 0], [2.0, 0, -2.0], [0, -2.0, -2.0], [1.5, 1.5, 1.5], [2.0, -2.0, 2.0]])
    G = wps([S["pos"][q] + off[q % len(off)] for q in range(len(S))], 3)
    return sc, S, G


def test_equal_f_ties_on_lattice_aligned_starts():
    sc, S, G = tie_case()
    ties = [q for q in range(len(S)) if sc.is_free(S["pos"][q]) and tie_at_second_pop(sc, S, G, q)]
    assert len(ties) >= 6, "too few starts whose second pop is decided by the g tie-break"
    for mx in (2, 3, 150):
        check(sc.with_(max_expand=mx), S, G)


def cap_case():
    """Queries for max_expand = 1, and the first that pops its goal after more than two expansions."""
    sc = edge_scene(eps=2.0, max_expand=150)
    S, G = random_queries(sc, 16, seed=43, near=(1.0, 2.0), far_every=100)
    full = oracle_run(sc, S, G)
    k = [q for q, o in enumerate(full) if o["valid"] and o["expanded"] > 2]
    assert k, "no query needs more than two expansions"
    return sc, S, G, k[0], full[k[0]]["expanded"]


def test_max_expand_one_and_goal_popped_at_the_cap():
    sc, S, G, q, cap = cap_case()
    d1 = check(sc.with_(max_expand=1), S, G)
    assert (d1["expanded"] <= 1).all() and (d1["expanded"] == 1).any()
    Sq, Gq = S[q:q + 1].copy(), G[q:q + 1].copy()
    at = check(sc.with_(max_expand=cap), Sq, Gq)
    # the goal is tested before the cap: the query that pops its goal at expansion `cap` succeeds
    assert at["valid"][0] == 1 and at["expanded"][0] == cap
    below = check(sc.with_(max_expand=cap - 1), Sq, Gq)
    assert below["expanded"][0] == cap - 1


def ray_blocked(scene, a, b):
    """ray_clear (mplx_search.cuh, MapUtil::walkRay with is_goal's visitor) restated: False when an
    occupied cell lies on the ray."""
    span = [b[k] - a[k] for k in range(scene.dim)]
    m = 0.0
    for k in range(scene.dim):
        x = abs(span[k] / scene.res)
        m = x if m < x else m
    steps = int(m / 0.8)
    inc = [span[k] * (1.0 / steps) for k in range(scene.dim)] if steps else [0.0] * scene.dim
    for i in range(1, steps):
        p = [a[k] + inc[k] * float(i) for k in range(scene.dim)]
        v = scene.value(p)
        if v is None:
            return False
        if v == 100:
            return True
    return False


def wall_scene():
    """The edge map with a wall across x at cells 20..21, in y 10..33, every z."""
    sc = edge_scene(eps=2.0, max_expand=150)
    g = sc.grid.reshape(sc.mdim[::-1]).copy()
    g[:, 10:34, 20:22] = 100
    g[:, 10:34, 14:20] = 0
    g[:, 10:34, 22:28] = 0
    return sc.with_(grid=g.reshape(-1))


def goal_class_case():
    """Goals outside the map, on occupied cells, and behind a wall within tol_pos (2 m) of the start."""
    sc = wall_scene().with_(tol_pos=2.0)
    lo = np.asarray(sc.origin)
    hi = lo + np.asarray(sc.mdim) * sc.res
    rng = np.random.default_rng(7)
    S, G, kinds = [], [], []
    free = sc.free_cells(margin=4)
    for k in range(4):
        # outside the map: beyond each face, near a start close to it
        s = sc.centre(free[np.argmin(free[:, k % 3])] if k < 3 else free[np.argmax(free[:, 0])])
        g = s.copy()
        g[k % 3] = lo[k % 3] - 0.4 if k < 3 else hi[0] + 0.4
        S.append(s), G.append(g), kinds.append("outside")
    occ = np.argwhere(sc.grid.reshape(sc.mdim[::-1]) == 100)[:, ::-1]
    occ = occ[((occ >= 4) & (occ < np.asarray(sc.mdim) - 4)).all(1)]
    for c in occ[rng.choice(len(occ), 4, replace=False)]:
        g = sc.centre(c)
        near = free[np.argmin(np.abs(free - c).sum(1) + 1000 * (np.abs(free - c).sum(1) < 3))]
        S.append(sc.centre(near)), G.append(g), kinds.append("occupied")
    for y, z in ((14, 8), (20, 20), (28, 30)):
        # start at x cell 17, goal at x cell 24: within tol_pos 2.0, but the wall at x 20..21 is between
        S.append(sc.centre([17, y, z])), G.append(sc.centre([24, y, z])), kinds.append("ray")
    return sc, wps(S, 3), wps(G, 3), kinds


def tol_pos_zero_case():
    """tol_pos = 0: only a state exactly on the goal position is a goal.  One and two ACC primitives from
    rest end exactly on these goals: a = (1, 1, 0), then a = (0, -1, 0)."""
    sc = wall_scene().with_(tol_pos=0.0)
    S, G = random_queries(sc, 8, seed=9, near=(1.0, 1.5), far_every=100)
    G["pos"] = S["pos"] + np.where(np.arange(8)[:, None] % 2 == 0, [0.5, 0.5, 0.0], [1.5, 1.0, 0.0])
    return sc, S, G


def test_goal_classes():
    sc, S, G, kinds = goal_class_case()
    for q, kind in enumerate(kinds):
        if kind == "outside":
            assert sc.value(G["pos"][q]) is None
        elif kind == "occupied":
            assert sc.value(G["pos"][q]) == 100
        else:
            assert sc.is_free(S["pos"][q]) and ray_blocked(sc, S["pos"][q], G["pos"][q])
    d = check(sc, S, G)
    ray = [q for q, k in enumerate(kinds) if k == "ray"]
    # the start is within tol_pos of the goal, so only the walkRay test kept it from being a goal
    assert all(d["expanded"][q] > 0 for q in ray)
    assert d["valid"][[q for q, k in enumerate(kinds) if k == "occupied"]].any()
    sc0, S0, G0 = tol_pos_zero_case()
    d0 = check(sc0, S0, G0)
    assert d0["valid"].any()
    for q in np.nonzero(d0["valid"])[0]:
        assert d0["expanded"][q] > 1


TOLERANCES = [dict(tol_vel=0.5), dict(tol_vel=1.0, tol_acc=0.5), dict(tol_vel=0.0, tol_acc=0.0)]


def tolerance_case():
    sc = edge_scene(eps=2.0, max_expand=150)
    S, G = random_queries(sc, 16, seed=47, near=(1.0, 2.5))
    return sc, S, G


@pytest.mark.parametrize("tol", TOLERANCES)
def test_velocity_and_acceleration_tolerances(tol):
    sc, S, G = tolerance_case()
    plain = oracle_run(sc, S, G)
    d = check(sc.with_(**tol), S, G)
    # the tolerances changed what some query did
    assert any(d["expanded"][q] != plain[q]["expanded"] or d["valid"][q] != plain[q]["valid"] for q in range(len(S)))


def start_class_case():
    """Free starts, starts on occupied, unknown and outside cells, and starts that are their goal."""
    sc = edge_scene(eps=2.0, max_expand=100)
    S, G = random_queries(sc, 12, seed=53, near=(1.0, 2.0))
    grid = sc.grid.reshape(sc.mdim[::-1])
    occ = np.argwhere(grid == 100)[:, ::-1][:2]
    unk = np.argwhere(grid == -1)[:, ::-1][:2]
    extra_s = [sc.centre(c) for c in occ] + [sc.centre(c) for c in unk] + \
              [np.array([-2.6, 3.0, 1.0]), np.array([0.0, 1.0 + 44 * 0.25 + 0.1, 2.0])]
    extra_g = [S["pos"][k] for k in range(len(extra_s))]
    S = np.concatenate([S, wps(extra_s, 3), S[:2]])
    G = np.concatenate([G, wps(extra_g, 3), S[:2]])  # the last two: start == goal
    kinds = ["free"] * 12 + ["occupied"] * 2 + ["unknown"] * 2 + ["outside"] * 2 + ["goal"] * 2
    return sc, S, G, kinds


def test_start_classes_and_start_free_from_the_host():
    sc, S, G, kinds = start_class_case()
    d = check(sc, S, G)
    for q, k in enumerate(kinds):
        if k in ("occupied", "unknown", "outside"):
            assert not sc.is_free(S["pos"][q])
            assert (d["valid"][q], d["expanded"][q], d["n_closed"][q]) == (0, 0, 0)
        elif k == "goal":
            assert (d["valid"][q], d["expanded"][q], d["cost"][q], len(d["actions"][q])) == (1, 0, 0.0, 0)
    assert sc.value(S["pos"][14]) == -1 and sc.value(S["pos"][16]) is None


# ---- cross-call arena state --------------------------------------------------------------------------
def test_cross_call_arena_state():
    """One ctx through a scripted sequence of calls, each compared bit for bit with the same call on a fresh
    ctx.  The script takes every branch of the arena's reserve/clear rule (ArenaModel)."""
    sc = base_scene(3, ACC, seed=61, v_max=2.0, a_max=2.0, eps=2.0, max_expand=150)
    U27 = sc.U
    U_alt = U27[::-1].copy()  # same width, other action ids: the keys of the successors are the same
    U_wide = product_set(np.linspace(-1, 1, 5), np.linspace(-1, 1, 5), (-1.0, 1.0))
    big_mx = 12000
    S_long, G_long = random_queries(sc, 8, seed=62, near=(6.0, 8.0), far_every=2)
    S_short, G_short = random_queries(sc, 12, seed=63, near=(0.5, 1.5), far_every=100)

    env = sc.env()
    # how many slots the big layout gets, to give its calls more queries than slots
    slots_big = C.c_int32(0)
    assert env._lib.mplx_plan_batch_fits(env.handle, 4096, big_mx, 1, C.byref(slots_big), None) == abi.MPLX_OK
    n_big = min(int(slots_big.value) + 48, 600)
    rng = np.random.default_rng(64)
    pick = rng.integers(0, 12, n_big)
    S_big = np.concatenate([S_long, S_short[pick[8:]]])[:n_big]
    G_big = np.concatenate([G_long, G_short[pick[8:]]])[:n_big]

    region = np.ones(sc.grid.size, np.uint8)
    region.reshape(sc.mdim[::-1])[:, :, :20] = 0
    cells = np.array([[x, y, z] for x in (24, 25) for y in range(8, 36) for z in range(0, 40, 3)], np.int32)

    # (name, U, max_expand, starts, goals, closed, action before the call)
    script = [
        ("small layout", U27, 150, S_short[:4], G_short[:4], True, None),
        ("growth: re-allocation", U27, big_mx, S_big, G_big, True, None),
        ("smaller layout inside the arena", U27, 150, S_short[:6], G_short[:6], True, None),
        ("same layout, more slots", U27, 150, S_short, G_short, True, None),
        ("same layout, fewer slots", U27, 150, S_short[:5], G_short[:5], True, None),
        ("n_q = 0", U27, 150, S_short[:0], G_short[:0], True, None),
        ("n_q = 1", U27, 150, S_short[7:8], G_short[7:8], True, None),
        ("closed keys off", U27, 150, S_short[:9], G_short[:9], False, None),
        ("closed keys on again", U27, 150, S_short[2:9], G_short[2:9], True, None),
        ("set_u: same nU, other order", U_alt, 150, S_short[:8], G_short[:8], True, "set_u"),
        ("after update_cells", U_alt, 150, S_short[:10], G_short[:10], True, "update_cells"),
        ("after expand", U_alt, 150, S_short[3:11], G_short[3:11], True, "expand"),
        ("after set_search_region", U_alt, 150, S_short, G_short, True, "set_search_region"),
        ("set_u: other nU", U_wide, 100, S_short, G_short, True, "set_u"),
        # The step that guards the clear.  The arena past the small layouts' cleared bytes still holds the big
        # layout's key table from the second call, entries with epochs 1..n_big at the offsets this call
        # reads.  The epochs restarted at 1 with the clear of "set_u: other nU", so without this call's clear
        # those stale entries would carry live epochs.  After the other layout changes the stale bytes are
        # state records of another layout, whose words almost never equal a live epoch.
        ("return to the big layout", U27, big_mx, S_big, G_big, False, "set_u"),
    ]
    model = ArenaModel()
    branches = {}
    grid = sc.grid.copy()
    reg = None
    n_over_slots = 0
    try:
        for name, U, mx, S, G, closed, action in script:
            if action == "set_u":
                env.set_u(U)
                env._sync_params()
            elif action == "update_cells":
                env.update_cells(cells, np.full(len(cells), 100, np.int8))
                g3 = grid.reshape(sc.mdim[::-1])
                g3[cells[:, 2], cells[:, 1], cells[:, 0]] = 100
            elif action == "expand":
                env.expand(S_short[:4])
            elif action == "set_search_region":
                env.set_search_region(region)
                reg = region
            call = sc.with_(U=U, grid=grid, max_expand=mx)
            r = device_run(env, call, S, G, closed=closed)
            fresh = call.env()
            try:
                if reg is not None:
                    fresh.set_search_region(reg)
                f = device_run(fresh, call, S, G, closed=closed)
            finally:
                fresh.close()
            same_results(r, f, name, closed=closed)
            if len(S):
                assert r["arena_bytes"] == layout_for(mx, len(U))["bytes"], name
                assert 1 <= r["slots"] <= len(S), name
                taken = model.call(r["slots"], r["arena_bytes"])
                for b in taken:
                    branches.setdefault(b, []).append(name)
                n_over_slots += len(S) > r["slots"]
                # several epochs per slot: the queries of very different lengths were taken out of order
                if mx == big_mx:
                    assert len(S) > r["slots"] and r["expanded"].max() > 10 * max(1, int(np.median(r["expanded"])))
            else:
                assert (r["slots"], r["arena_bytes"]) == (0, 0)
    finally:
        env.close()
    print("arena branches:", branches)
    assert branches.get("realloc", [])[:2] == ["small layout", "growth: re-allocation"]
    assert "smaller layout inside the arena" in branches["clear-layout"]
    assert "return to the big layout" in branches["clear-layout"]
    assert "same layout, more slots" in branches["clear-more-slots"]
    assert "realloc" not in {b for b, names in branches.items() if "same layout, more slots" in names}
    assert "same layout, fewer slots" in branches["epochs-continue"]
    assert "set_u: same nU, other order" in branches["epochs-continue"]
    assert "set_u: other nU" in branches["clear-layout"]
    assert n_over_slots >= 2


# ---- sizing contract ---------------------------------------------------------------------------------
@pytest.mark.parametrize("dim,control,nU,mx", [(2, ACC, 9, 150), (3, JRK, 27, 1000), (3, ACC, 256, 200),
                                               (2, VEL, 1, 50), (3, SNP, 65, 333)])
def test_sizing_contract(dim, control, nU, mx):
    import torch

    U = width_set(nU, "random", dim, seed=nU) if nU not in (9, 27) else product_set(*[u_values(control)] * dim)
    sc = base_scene(dim, control, U=U, seed=71, max_expand=mx)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    # an upper bound of the resident CTAs: 2048 threads and 32 blocks per SM
    resident_max = min(32, 2048 // block_of(nU)) * sm
    S, G = random_queries(sc, 40, seed=72, near=(0.5, 1.0), far_every=100)
    env = sc.env()
    try:
        for n_q, with_closed in ((1, 1), (40, 1), (40, 0), (5000, 1), (0, 0)):
            slots, nbytes = C.c_int32(-1), C.c_int64(-1)
            assert env._lib.mplx_plan_batch_fits(env.handle, n_q, mx, with_closed, C.byref(slots), C.byref(nbytes)) == 0
            L = layout_for(mx, nU)
            assert nbytes.value == L["bytes"]
            assert 1 <= slots.value <= min(max(n_q, 1), resident_max)
            assert slots.value * L["bytes"] + results_bytes(n_q, mx, with_closed) <= SEARCH_BUDGET
            if 0 < n_q <= len(S):
                r = device_run(env, sc, S[:n_q], G[:n_q], closed=bool(with_closed))
                assert (r["slots"], r["arena_bytes"]) == (slots.value, nbytes.value)
        # one arena larger than the budget: refused, whatever the free memory
        big = -(-SEARCH_BUDGET // (nU * (SSTATE_BYTES + SPRED_BYTES + SHEAP_BYTES)))
        assert layout_for(big, nU)["bytes"] > SEARCH_BUDGET
        assert env._lib.mplx_plan_batch_fits(env.handle, 1, big, 0, None, None) == abi.MPLX_ERR_ALLOC
    finally:
        env.close()
