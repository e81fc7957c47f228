"""mplx_expand_packed (csrc/mplx_packed.cu: pack_kernel behind the expansion kernels, four buffer sets over three
streams) against the CPU oracle, record for record: every selection of {state, cost, action, key}, every
<Dim, control> layout of the state record, control sets that take one, two and many trips of the warp loop, the
chunk geometry around the pipeline's depth, and the capacity refusal with the call that follows it.

Bars: counts, offsets, states, keys, actions and the costs of occupancy plans bit for bit; costs of plans with a
yaw or potential term 1e-12 relative with the same +inf pattern.  The raw ABI is called directly so that every
array carries guard words past `capacity`."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

import oracle_bindings as ob
from test_expand_parity_gpu import gpu_env

pytestmark = pytest.mark.gpu

VEL, ACC, JRK, SNP, YAW = 0x01, 0x03, 0x07, 0x0F, 0x10
FIELDS = ("state", "cost", "action", "key")
DTYPES = dict(state=np.float64, cost=np.float64, action=np.uint16, key=np.uint64)
GUARD = 64                     # guard elements past the capacity of every array
FXN_MIN_SLOTS = 64 * 256       # the occupancy pair expand_fxn_kernel + fx_resolve_kernel runs from this many slots
ALL = frozenset(FIELDS)


# ---- plans and nodes -----------------------------------------------------------------------------------
def plan(dim, control, cells=40, res=0.2, U=None, seed=5, **kw):
    from scenarios import Scenario, control_set

    yaw = bool(control & YAW)
    if U is None:
        U = control_set(4.0 if (control & 15) == SNP else 1.0, 3, dim, yaw_rates=(-0.4, 0.0, 0.4) if yaw else None)
    kw.setdefault("v_max", 2.5)
    return Scenario(f"packed{dim}d_{control:x}", (cells,) * dim, res, tuple(-cells * res / 2 for _ in range(dim)), control,
                    U, n_boxes=max(2, cells // 5), edge_m=(4 * res, 10 * res), seed=seed, a_max=3.0, j_max=6.0,
                    yaw_max=0.9 if yaw else -1.0, wyaw=1.5, **kw)


def hand_nodes(sc, n, seed=0):
    """Lattice states of every order inside the map (the frontier generator serves ACC and JRK only)."""
    rng = np.random.default_rng(seed)
    D, half = sc.Dim, sc.dim_cells[0] * sc.res / 2
    nodes = np.zeros(n, dtype=ob.WAYPOINT_DTYPE)
    nodes["pos"][:, :D] = np.round(rng.uniform(-half * 0.9, half * 0.9, (n, D)) / 0.05) * 0.05
    nodes["vel"][:, :D] = rng.integers(-4, 5, (n, D)) * 0.5
    nodes["acc"][:, :D] = rng.integers(-4, 5, (n, D)) * 0.5
    nodes["jrk"][:, :D] = rng.integers(-3, 4, (n, D)) * 1.0
    nodes["yaw"] = rng.integers(-7, 8, n) * 0.4
    nodes["t"] = rng.integers(0, 5, n) * 1.0
    return nodes


def occupied_nodes(sc, n, seed=0):
    """Nodes at rest in the centre of occupied cells: every successor they emit costs +inf."""
    rng = np.random.default_rng(seed)
    D = sc.Dim
    occ = np.flatnonzero(sc.grid() > 0)
    idx = occ[rng.integers(0, occ.size, n)]
    cells = np.stack(np.unravel_index(idx, sc.dim_cells[::-1])[::-1], axis=1)
    nodes = np.zeros(n, dtype=ob.WAYPOINT_DTYPE)
    nodes["pos"][:, :D] = (cells + 0.5) * sc.res + np.asarray(sc.origin)
    return nodes


def too_fast_nodes(sc, n):
    """Nodes beyond v_max by more than any control recovers: no successor is emitted (count = 0)."""
    nodes = np.zeros(n, dtype=ob.WAYPOINT_DTYPE)
    nodes["vel"][:, :sc.Dim] = 40.0
    return nodes


def oracle(sc, nodes):
    return ob.OracleEnv.from_scenario(sc).expand(nodes, nthreads=16, lattice=False)


# ---- the call and its check ------------------------------------------------------------------------------
def packed_call(env, nodes, fields=ALL, drop_inf=False, capacity=None, pinned=False):
    """mplx_expand_packed through the raw ABI with the arrays of `fields` only, each GUARD elements longer than
    `capacity` and pre-filled with a pattern.  Returns (status, result dict)."""
    from motion_primitive_library_b200 import abi

    env._sync_params()
    nodes = np.ascontiguousarray(nodes, dtype=ob.WAYPOINT_DTYPE).reshape(-1)
    n, nU = nodes.size, env.U_.shape[0]
    nstate = env.Dim * bin(env.control & 15).count("1") + (1 if env.control & YAW else 0)
    cap = n * nU if capacity is None else capacity
    alloc = env._pinned_empty if pinned else (lambda m, dt: np.empty(m, dtype=dt))
    b = dict(count=alloc(n + GUARD, np.int32), offset=alloc(n + GUARD, np.int64))
    for f in FIELDS:
        if f in fields:
            b[f] = alloc((cap + GUARD) * (nstate if f == "state" else 1), DTYPES[f])
    for a in b.values():
        a.view(np.uint8)[:] = 0xA5
    out = abi.PackedOut(abi.ptr(b["count"]), abi.ptr(b["offset"]), abi.ptr(b.get("state")), abi.ptr(b.get("cost")),
                        abi.ptr(b.get("action")), abi.ptr(b.get("key")), cap, -7, -7)
    rc = env._lib.mplx_expand_packed(env.handle, nodes.ctypes.data, n, abi.PACK_DROP_INF if drop_inf else 0, C.byref(out))
    return rc, dict(b, n=n, cap=cap, total=int(out.total), nstate=int(out.nstate), nstate_expected=nstate)


def guards_intact(p):
    """Nothing past `capacity` records (count / offset: past n nodes) was written."""
    for name, a in p.items():
        if not isinstance(a, np.ndarray):
            continue
        used = p["n"] if name in ("count", "offset") else p["cap"] * (p["nstate_expected"] if name == "state" else 1)
        assert (a[used:].view(np.uint8) == 0xA5).all(), f"{name}: written past its capacity"


def chunk_nodes(n, nU):
    """Nodes per pipeline chunk (mplx_packed.cu): 2^MPLX_PACK_CHUNK_LOG2 slots (default 21, clamped to 10..26)."""
    log2 = min(26, max(10, int(os.environ.get("MPLX_PACK_CHUNK_LOG2", "21"))))
    return min(n, max(1, (1 << log2) // nU)) if n else 1


def expected_records(sc, orc, nodes, drop_inf):
    nU, D = orc["nU"], sc.Dim
    keep = np.arange(nU)[None, :] < orc["count"][:, None]
    if drop_inf:
        keep &= ~np.isinf(orc["cost"].reshape(-1, nU))
    sel = np.flatnonzero(keep.reshape(-1))
    names = ["pos", "vel", "acc", "jrk"][: bin(sc.control & 15).count("1")]
    state = np.concatenate([orc["succ"][f][sel][:, :D] for f in names] +
                           ([orc["succ"]["yaw"][sel][:, None]] if sc.control & YAW else []), axis=1)
    return keep, sel, np.ascontiguousarray(state)


def check_packed(env, sc, orc, nodes, fields=ALL, drop_inf=False, pinned=False, capacity=None, exact_cost=True):
    """One call, compared with the oracle for exactly the requested fields."""
    rc, p = packed_call(env, nodes, fields, drop_inf, capacity, pinned)
    assert rc == 0, env._lib.mplx_last_error()
    guards_intact(p)
    n, nU = len(nodes), orc["nU"]
    keep, sel, exp_state = expected_records(sc, orc, nodes, drop_inf)
    count, offset = p["count"][:n], p["offset"][:n]
    np.testing.assert_array_equal(count, keep.sum(1))
    assert p["total"] == sel.size and p["nstate"] == exp_state.shape[1] == p["nstate_expected"]
    # the segments tile [0, total), and the records of chunk k lie behind those of chunk k - 1
    nz = np.flatnonzero(count > 0)
    by_offset = nz[np.argsort(offset[nz], kind="stable")]
    np.testing.assert_array_equal(offset[by_offset], np.concatenate([[0], np.cumsum(count[by_offset])[:-1]]))
    ch = chunk_nodes(n, nU)
    bases = np.concatenate([[0], np.cumsum(np.add.reduceat(count, np.arange(0, n, ch)))]) if n else np.zeros(1, np.int64)
    k_of = np.arange(n) // ch
    assert ((offset[nz] >= bases[k_of[nz]]) & (offset[nz] + count[nz] <= bases[k_of[nz] + 1])).all()
    idx = (np.repeat(offset, count) + np.arange(sel.size) - np.repeat(np.cumsum(count) - count, count)).astype(np.int64)
    if "state" in fields:
        got = p["state"][: p["cap"] * p["nstate"]].reshape(-1, p["nstate"])[idx]
        assert got.tobytes() == exp_state.tobytes(), "state"
        # the reconstruction rule of include/mplx.h: state fields from the record, the first derivative above the
        # state order = 0 + U[action], higher ones 0, yaw 0 without a yaw control, t = parent.t + dt
        D, nf = sc.Dim, bin(sc.control & 15).count("1")
        full = np.zeros(sel.size, dtype=ob.WAYPOINT_DTYPE)
        act = orc["action"][sel].astype(np.int64)
        for f_i, name in enumerate(["pos", "vel", "acc", "jrk"]):
            if f_i < nf:
                full[name][:, :D] = got[:, f_i * D:(f_i + 1) * D]
            elif f_i == nf:
                full[name][:, :D] = 0.0 + sc.U[act][:, :D]
        if sc.control & YAW:
            full["yaw"] = got[:, nf * D]
        full["t"] = nodes["t"][np.repeat(np.arange(n), count)] + sc.T
        assert full.tobytes() == orc["succ"][sel].tobytes(), "reconstructed waypoint"
    if "action" in fields:
        np.testing.assert_array_equal(p["action"][idx], orc["action"][sel].astype(np.uint16))
    if "key" in fields:
        np.testing.assert_array_equal(p["key"][idx], orc["key"][sel])
    if "cost" in fields:
        g, o = p["cost"][idx], orc["cost"][sel]
        if exact_cost:
            assert g.tobytes() == o.tobytes(), "cost"
        else:
            np.testing.assert_array_equal(np.isinf(g), np.isinf(o))
            np.testing.assert_allclose(g[~np.isinf(o)], o[~np.isinf(o)], rtol=1e-12, atol=0)
    return p


class chunk_log2:
    """MPLX_PACK_CHUNK_LOG2 for the block, the environment restored after it."""

    def __init__(self, v):
        self.v = v

    def __enter__(self):
        self.old = os.environ.get("MPLX_PACK_CHUNK_LOG2")
        os.environ["MPLX_PACK_CHUNK_LOG2"] = str(self.v)

    def __exit__(self, *a):
        if self.old is None:
            os.environ.pop("MPLX_PACK_CHUNK_LOG2", None)
        else:
            os.environ["MPLX_PACK_CHUNK_LOG2"] = self.old


SUBSETS = [frozenset(s) for r in range(5) for s in itertools.combinations(FIELDS, r)]


# ---- 1. field selections ---------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["occupancy", "cost_terms"])
def test_every_field_selection(which):
    """All 16 subsets of {state, cost, action, key}, +inf successors kept and dropped, on one ctx."""
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 64) if which == "occupancy" else S.scaled(S.cfg4(), 48)
    nodes = sc.frontier(2500 if which == "occupancy" else 900, seed=12)
    orc = oracle(sc, nodes)
    assert np.isinf(orc["cost"]).any() and (orc["count"] < sc.nU).any()
    env = gpu_env(sc)
    assert len(SUBSETS) == 16
    for fields in SUBSETS:
        for drop in (False, True):
            check_packed(env, sc, orc, nodes, fields, drop, exact_cost=which == "occupancy")


def test_keys_only_stream_runs_the_occupancy_pair_without_successor_records():
    """The product's default stream: state = cost = NULL, so the expansion runs with succ == NULL.  A chunk of at
    least 64 * 256 slots takes expand_fxn_kernel + fx_resolve_kernel + pack_kernel (3 launches), a smaller one the
    single expansion kernel + pack_kernel (2)."""
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 64)
    env = gpu_env(sc)
    for n in (FXN_MIN_SLOTS // 27 + 1, FXN_MIN_SLOTS // 27 - 1, 40):
        nodes = sc.frontier(n, seed=n)
        orc = oracle(sc, nodes)
        for fields in (frozenset({"key", "action"}), frozenset({"key"}), ALL):
            env._sync_params()
            before = env.launch_count()
            check_packed(env, sc, orc, nodes, fields, drop_inf=True, pinned=True)
            assert env.launch_count() - before == (3 if n * 27 >= FXN_MIN_SLOTS else 2), (n, sorted(fields))


# ---- 2. the state record of every plan -------------------------------------------------------------------
@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("control", [VEL, ACC, JRK, SNP, VEL | YAW, ACC | YAW, JRK | YAW, SNP | YAW])
def test_state_record_layout(dim, control):
    sc = plan(dim, control)
    nodes = hand_nodes(sc, 1200, seed=control * 4 + dim)
    orc = oracle(sc, nodes)
    env = gpu_env(sc)
    order = bin(control & 15).count("1")
    for fields in (ALL, frozenset({"state"})):
        p = check_packed(env, sc, orc, nodes, fields, drop_inf=False, exact_cost=not control & YAW)
        assert p["nstate"] == dim * order + (1 if control & YAW else 0)
    check_packed(env, sc, orc, nodes, ALL, drop_inf=True, exact_cost=not control & YAW)
    assert 0 < (~np.isinf(orc["cost"])).sum() and orc["count"].sum() > nodes.size


# ---- 3. width of the control set --------------------------------------------------------------------------
@pytest.mark.parametrize("nU", [1, 31, 32, 33, 64, 65, 125, 343])
def test_control_set_width(nU):
    """One, exactly one, and several trips of pack_kernel's warp loop (`written` carried between trips); 343 > 256
    primitives per node runs the literal kernel.  Some nodes emit nothing, some only +inf successors."""
    from scenarios import control_set

    U = np.random.default_rng(nU).permutation(control_set(1.5, 7, 3))[:nU]
    sc = plan(3, ACC, cells=48, U=np.ascontiguousarray(U), v_max=3.0)
    nodes = np.concatenate([hand_nodes(sc, 700, seed=nU), too_fast_nodes(sc, 3), occupied_nodes(sc, 40, seed=nU),
                            hand_nodes(sc, 200, seed=nU + 1), too_fast_nodes(sc, 1)])
    orc = oracle(sc, nodes)
    cost = orc["cost"].reshape(-1, nU)
    emitted = np.arange(nU)[None, :] < orc["count"][:, None]
    assert (orc["count"] == 0).sum() >= 4 and (orc["count"] == nU).any()
    assert ((orc["count"] > 0) & (np.isinf(cost) | ~emitted).all(1)).any(), "a node whose successors are all +inf"
    if nU > 32:
        assert ((np.isinf(cost) & emitted)[:, :32].any(1) & (~np.isinf(cost) & emitted)[:, 32:].any(1)).any()
    env = gpu_env(sc)
    for drop in (False, True):
        check_packed(env, sc, orc, nodes, ALL, drop)
        check_packed(env, sc, orc, nodes, frozenset({"key", "cost"}), drop)


# ---- 4. chunk geometry ----------------------------------------------------------------------------------
def test_chunk_geometry_around_the_pipeline_depth():
    """Chunks of 2^10 slots = 37 nodes of 27 primitives.  Two chunks are queued before the host waits for a count
    and four buffer sets cycle: 1..5 and 9 chunks, k * chunk +- 1 nodes, a tail of one node, and a chunk in the
    middle whose nodes all stand in obstacles (nothing kept under drop_inf)."""
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 64)
    env = gpu_env(sc)
    pool = sc.frontier(37 * 9 + 1, seed=31)
    with chunk_log2(10):
        ch = chunk_nodes(10 ** 6, 27)
        assert ch == 37
        sizes = [ch * k for k in (1, 2, 3, 4, 5, 9)] + [ch - 1, ch + 1, 2 * ch - 1, 2 * ch + 1, 4 * ch + 1, 5 * ch - 1, 9 * ch + 1]
        for n in sizes:
            nodes = pool[:n]
            orc = oracle(sc, nodes)
            for fields, drop in ((ALL, True), (frozenset({"key", "action"}), False)):
                check_packed(env, sc, orc, nodes, fields, drop, pinned=n % 2 == 0)
        for k_empty, nchunks in ((1, 3), (2, 6), (0, 5), (5, 6)):
            nodes = pool[: ch * nchunks].copy()
            nodes[k_empty * ch:(k_empty + 1) * ch] = occupied_nodes(sc, ch, seed=k_empty)
            orc = oracle(sc, nodes)
            keep, _, _ = expected_records(sc, orc, nodes, True)
            per_chunk = keep.sum(1).reshape(nchunks, ch).sum(1)
            assert per_chunk[k_empty] == 0 and (np.delete(per_chunk, k_empty) > 0).all()
            check_packed(env, sc, orc, nodes, ALL, True)
            check_packed(env, sc, orc, nodes, ALL, False)
    assert "MPLX_PACK_CHUNK_LOG2" not in os.environ
    # the default chunk (2^21 slots): one chunk, then one and a bit
    nodes = sc.frontier(300, seed=2)
    check_packed(env, sc, oracle(sc, nodes), nodes, ALL, True)


# ---- 5. capacity ----------------------------------------------------------------------------------------
def test_capacity_refusal_and_the_call_after_it():
    """capacity == total is served; one record short is refused with MPLX_ERR_ARG whichever chunk overflows (first,
    middle, last), nothing past the capacity is written — the refused call waits for its queued copies before it
    returns — and the same ctx then serves a correct call."""
    from motion_primitive_library_b200 import abi
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 64)
    env = gpu_env(sc)
    with chunk_log2(10):
        ch = chunk_nodes(10 ** 6, 27)
        nodes = sc.frontier(ch * 7 + 5, seed=41)
        orc = oracle(sc, nodes)
        for drop in (True, False):
            keep, sel, _ = expected_records(sc, orc, nodes, drop)
            cum = np.cumsum(np.add.reduceat(keep.sum(1), np.arange(0, nodes.size, ch)))
            total = int(cum[-1])
            check_packed(env, sc, orc, nodes, ALL, drop, capacity=total)
            for k in (0, 3, len(cum) - 1):
                for fields, pinned in ((ALL, False), (frozenset({"key"}), True)):
                    rc, p = packed_call(env, nodes, fields, drop, capacity=int(cum[k]) - 1, pinned=pinned)
                    assert rc == abi.MPLX_ERR_ARG and b"capacity" in env._lib.mplx_last_error(), (k, drop)
                    assert p["total"] == 0
                    guards_intact(p)
                    p2 = check_packed(env, sc, orc, nodes, fields, drop, capacity=total, pinned=pinned)
                    guards_intact(p)  # the refused call's arrays: still nothing behind their capacity
                    assert p2["total"] == total
        # capacity 0 with records to write, and a single-chunk refusal
        rc, p = packed_call(env, nodes[:5], ALL, False, capacity=0)
        assert rc == abi.MPLX_ERR_ARG
        guards_intact(p)
    rc, p = packed_call(env, nodes, ALL, False, capacity=int(orc["count"].sum()) - 1)
    assert rc == abi.MPLX_ERR_ARG
    guards_intact(p)
    check_packed(env, sc, orc, nodes, ALL, False)
    check_packed(gpu_env(sc), sc, orc, nodes, ALL, False)  # a fresh ctx agrees with the same oracle records


def test_required_arrays_and_empty_batch():
    from motion_primitive_library_b200 import abi
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 64)
    env = gpu_env(sc)
    env._sync_params()
    nodes = sc.frontier(10, seed=1)
    count, offset = np.zeros(10, np.int32), np.zeros(10, np.int64)
    for cnt, off in ((None, offset), (count, None)):
        out = abi.PackedOut(abi.ptr(cnt), abi.ptr(off), None, None, None, None, 270, 0, 0)
        assert env._lib.mplx_expand_packed(env.handle, nodes.ctypes.data, 10, 0, C.byref(out)) == abi.MPLX_ERR_ARG
    out = abi.PackedOut(abi.ptr(count), abi.ptr(offset), None, None, None, None, 270, 0, 0)
    assert env._lib.mplx_expand_packed(env.handle, None, 10, 0, C.byref(out)) == abi.MPLX_ERR_ARG
    rc, p = packed_call(env, nodes[:0], ALL)
    assert rc == 0 and p["total"] == 0 and p["nstate"] == 6
    guards_intact(p)


# ---- 6. one ctx, alternating selections and host memory kinds ----------------------------------------------
def test_alternating_selections_on_one_ctx():
    """The staging buffers are reserved per selection and kept: a keys-only call, then one with states, a larger
    batch, pinned and pageable arrays in turn — each equal to the oracle, as a fresh ctx is."""
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 64)
    env = gpu_env(sc)
    big, small = sc.frontier(4000, seed=51), sc.frontier(150, seed=52)
    ob_, os_ = oracle(sc, big), oracle(sc, small)
    seq = ((small, os_, frozenset({"key"}), True), (big, ob_, ALL, False), (small, os_, frozenset({"state"}), True),
           (big, ob_, frozenset({"key", "action"}), True), (small, os_, ALL, False), (big, ob_, frozenset(), False),
           (big, ob_, frozenset({"state", "cost"}), True), (small, os_, frozenset({"cost", "key"}), False))
    with chunk_log2(14):
        for i, (nodes, orc, fields, pinned) in enumerate(seq):
            check_packed(env, sc, orc, nodes, fields, drop_inf=i % 2 == 0, pinned=pinned)
