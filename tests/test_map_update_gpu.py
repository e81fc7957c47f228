"""Sparse map updates on the device (mplx_update_cells) and the layers above them: after any sequence of
updates the device grid, occupancy words and occ2 pairs are bit-identical to one mplx_set_map of the
final grid, and every query that reads them answers as after a full upload, while the potential map
and the search region set before the updates stay in effect.  The LPA* session's BLOCK / CLEAR steps
and a BatchPlanner session replan through the sparse path."""
import ctypes as C

import numpy as np
import pytest

import fixtures
import planner_bindings as pb
from test_lpastar_vs_ref import integrate_cells, same_session, voxel_session_args

pytestmark = pytest.mark.gpu
ACC = 0x03


def make_env(grid, dims, origin=None, res=0.1):
    from motion_primitive_library_b200 import MapUtil, env_map

    mu = MapUtil()
    mu.setMap(origin if origin is not None else (0.0,) * len(dims), dims, np.array(grid, dtype=np.int8), res)
    return env_map(mu)


def apply(ref, idx, vals):
    """numpy restatement: grid[idx[k]] = vals[k] in array order"""
    idx = np.asarray(idx, dtype=np.int64).reshape(-1)
    vals = np.asarray(vals, dtype=np.int8).reshape(-1)
    u, first = np.unique(idx[::-1], return_index=True)
    ref[u] = vals[::-1][first]


def assert_device_state(env, final, dims):
    fresh = make_env(final, dims)
    got, want = env.read_map(), fresh.read_map()
    for name, g, w in zip(("grid", "occ", "occ2"), got, want):
        assert g.tobytes() == w.tobytes(), name
    assert got[0].tobytes() == final.tobytes()
    fresh.close()


def edge_indices(dims):
    """every voxel on a face (incl. row ends and plane ends) and every voxel of the last, partial word"""
    nvox = int(np.prod(dims))
    ii = np.arange(nvox, dtype=np.int64)
    x, y = ii % dims[0], (ii // dims[0]) % dims[1]
    on = (x == 0) | (x == dims[0] - 1) | (y == 0) | (y == dims[1] - 1)
    if len(dims) == 3:
        z = ii // (dims[0] * dims[1])
        on |= (z == 0) | (z == dims[2] - 1)
    on[(nvox // 32) * 32:] = True
    return ii[on]


VALUES = np.array([100, 0, -1, 1, 37, 99, 100, 100], dtype=np.int8)  # occupied / free / unknown / potential values


def update_sequence(env, ref, rng, n_random):
    nvox = ref.size
    edges = edge_indices(tuple(int(d) for d in env.map_util_.dim))
    # one call: the boundary voxels, random voxels and duplicates within the call
    idx = np.concatenate([edges, rng.integers(0, nvox, n_random), edges[rng.integers(0, edges.size, 50)]])
    rng.shuffle(idx)
    vals = VALUES[rng.integers(0, VALUES.size, idx.size)]
    env.update_cells(idx, vals)
    apply(ref, idx, vals)
    env.update_cells(np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int8))  # n = 0
    for k in (0, nvox - 1, int(edges[len(edges) // 2])):  # n = 1
        env.update_cells([k], [100])
        apply(ref, [k], [100])
    for _ in range(200):  # many small calls, duplicates across calls
        m = int(rng.integers(1, 6))
        idx = np.concatenate([rng.integers(0, nvox, m), edges[rng.integers(0, edges.size, 2)]])
        vals = VALUES[rng.integers(0, VALUES.size, idx.size)]
        env.update_cells(idx, vals)
        apply(ref, idx, vals)


@pytest.mark.parametrize("case", ["corridor", "odd3d"])
def test_device_state_bitwise(case):
    rng = np.random.default_rng(7)
    if case == "corridor":
        c = fixtures.corridor()
        dims, grid = tuple(int(d) for d in c["dim"]), c["grid"]
    else:
        dims = (37, 29, 23)
        assert np.prod(dims) % 32 != 0
        grid = np.where(rng.random(int(np.prod(dims))) < 0.1, 100, 0).astype(np.int8)
    env = make_env(grid, dims)
    ref = np.array(grid, dtype=np.int8).reshape(-1)
    update_sequence(env, ref, rng, 2000)
    np.testing.assert_array_equal(env.map_util_.map, ref)  # the Python MapUtil was edited in place too
    assert_device_state(env, ref, dims)
    # a full upload after updates, then more updates
    env.upload_map()
    update_sequence(env, ref, rng, 100)
    assert_device_state(env, ref, dims)


def test_device_state_bitwise_headline_map():
    import scenarios as S

    sc = S.cfg_headline()
    dims = tuple(int(d) for d in sc.dim_cells)
    env = make_env(sc.grid(), dims, sc.origin, sc.res)
    ref = np.array(sc.grid(), dtype=np.int8).reshape(-1)
    rng = np.random.default_rng(9)
    idx = rng.integers(0, ref.size, 100_000)
    vals = VALUES[rng.integers(0, VALUES.size, idx.size)]
    env.update_cells(idx, vals)  # unsorted: the radix-sort path
    apply(ref, idx, vals)
    box = (np.arange(40)[:, None, None] * dims[0] * dims[1] + np.arange(40)[None, :, None] * dims[0]
           + np.arange(40)[None, None, :] + 200 * (1 + dims[0] + dims[0] * dims[1])).reshape(-1)
    env.update_cells(box, np.full(box.size, 100, dtype=np.int8))  # in index order: the presorted path
    apply(ref, box, np.full(box.size, 100, dtype=np.int8))
    for k in (0, ref.size - 1):
        env.update_cells([k], [100])
        apply(ref, [k], [100])
    assert_device_state(env, ref, dims)


def _headline64():
    import scenarios as S

    return S.scaled(S.cfg_headline(), 64)


def _configured(sc, grid, pot, region):
    from motion_primitive_library_b200 import MapUtil, env_map

    mu = MapUtil()
    mu.setMap(sc.origin, sc.dim_cells, np.array(grid, dtype=np.int8), sc.res)
    e = env_map(mu)
    e.set_control(sc.control)
    e.set_u(sc.U)
    e.set_v_max(sc.v_max)
    e.set_a_max(sc.a_max)
    if pot is not None:
        e.set_potential_weight(0.5)
        e.set_potential_map(pot)
    e.set_search_region(region)
    return e


def _same_expansion(a, b):
    assert a.count.tobytes() == b.count.tobytes()
    for f in ("succ", "cost", "action", "key"):
        assert getattr(a, f).tobytes() == getattr(b, f).tobytes(), f


def _by_node(p, field):
    """records of a packed result in node order"""
    cnt = p["count"].astype(np.int64)
    start = np.repeat(p["offset"].astype(np.int64), cnt)
    within = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    return p[field][start + within]


@pytest.mark.parametrize("with_potential", [True, False])
def test_queries_after_updates_match_full_upload(with_potential):
    """env_map.update_cells (the Python mirror) with a potential map and a tunnel installed first: every
    kernel, the packed stream and both edge queries answer exactly as an env built from the final grid with
    the same potential map and tunnel."""
    import oracle_bindings as ob
    from test_edges_oracle_vs_ref import edges_of

    sc = _headline64()
    rng = np.random.default_rng(21)
    grid = np.array(sc.grid(), dtype=np.int8).reshape(-1)
    pot = np.where(grid == 100, 100, rng.integers(0, 60, grid.size)).astype(np.int8) if with_potential else None
    region = (rng.random(grid.size) < 0.97).astype(np.uint8)
    env = _configured(sc, grid, pot, region)
    nodes = sc.frontier(3000, seed=12)
    before = env.expand(nodes)
    # walls through the frontier's cells, clearings and random edits
    cells = np.floor((nodes["pos"] - np.asarray(sc.origin)) / sc.res).astype(np.int64)
    cells = np.clip(cells, 0, np.asarray(sc.dim_cells) - 1)[:400]
    idx = cells[:, 0] + sc.dim_cells[0] * cells[:, 1] + sc.dim_cells[0] * sc.dim_cells[1] * cells[:, 2]
    idx = np.concatenate([idx, rng.integers(0, grid.size, 3000)])
    vals = np.where(rng.random(idx.size) < 0.6, 100, 0).astype(np.int8)
    env.update_cells(idx, vals)
    env.update_cells(cells[:50], np.zeros(50, dtype=np.int8))  # cell coordinates; clears some of the walls
    final = env.map_util_.map.copy()
    assert (final != grid).sum() > 1000
    fresh = _configured(sc, final, pot, region)
    for which in range(6):
        env.set_kernel(which)
        fresh.set_kernel(which)
        _same_expansion(env.expand(nodes), fresh.expand(nodes))
    env.set_kernel(0)
    fresh.set_kernel(0)
    after = env.expand(nodes)
    if with_potential:
        # with a potential map the sample test reads it instead of the grid (env_map.h:104-121): the kept
        # potential map still decides every cost
        _same_expansion(after, before)
    else:
        assert after.cost.tobytes() != before.cost.tobytes()  # the updates reached the expansion
    for drop in (False, True):
        pa, pf = env.expand_packed(nodes, drop_inf=drop), fresh.expand_packed(nodes, drop_inf=drop)
        assert pa["total"] == pf["total"] and pa["count"].tobytes() == pf["count"].tobytes()
        for f in ("state", "cost", "action", "key"):  # a node's records sit where an atomicAdd put them
            assert _by_node(pa, f).tobytes() == _by_node(pf, f).tobytes(), f
    orc = ob.OracleEnv.from_scenario(sc)
    parents, actions, _ = edges_of(orc, nodes[:500], rng, extra=500)
    fa, ca = env.is_free_edges(parents, actions)
    ff, cf = fresh.is_free_edges(parents, actions)
    assert fa.tobytes() == ff.tobytes() and ca.tobytes() == cf.tobytes()
    ea, ef = env.edge_cells(parents, actions, table=True), fresh.edge_cells(parents, actions, table=True)
    for x, y in zip(ea, ef):
        assert x.tobytes() == y.tobytes()
    assert_device_state(env, final, tuple(int(d) for d in sc.dim_cells))


def test_invalid_updates_rejected_with_nothing_applied():
    from motion_primitive_library_b200 import abi

    dims = (37, 29, 23)
    rng = np.random.default_rng(3)
    grid = np.where(rng.random(int(np.prod(dims))) < 0.2, 100, 0).astype(np.int8)
    env = make_env(grid, dims)
    lib, h = abi.load(), env.handle
    state = env.read_map()
    nvox = grid.size
    vals = np.full(4, 100, dtype=np.int8)
    for bad in ([1, 2, nvox, 3], [1, -1, 2, 3], [0, 1, 2, 2 ** 31 - 1]):
        idx = np.array(bad + [0] * (4 - len(bad)), dtype=np.int32)
        assert lib.mplx_update_cells(h, idx.ctypes.data, vals.ctypes.data, 4) == abi.MPLX_ERR_ARG
    idx = np.array([1, 2, 3, 4], dtype=np.int32)
    assert lib.mplx_update_cells(h, idx.ctypes.data, vals.ctypes.data, -1) == abi.MPLX_ERR_ARG
    assert lib.mplx_update_cells(h, None, vals.ctypes.data, 4) == abi.MPLX_ERR_ARG
    assert lib.mplx_update_cells(h, idx.ctypes.data, None, 4) == abi.MPLX_ERR_ARG
    assert b"outside" in lib.mplx_last_error() or b"null" in lib.mplx_last_error()
    for a, b in zip(env.read_map(), state):
        assert a.tobytes() == b.tobytes()
    with pytest.raises(ValueError):
        env.update_cells(np.array([[0, 0, 0], [37, 0, 0]]), [100, 100])  # cells: x == nx is outside
    assert lib.mplx_update_cells(h, idx.ctypes.data, vals.ctypes.data, 0) == abi.MPLX_OK
    for a, b in zip(env.read_map(), state):
        assert a.tobytes() == b.tobytes()


def test_lpa_session_128_many_block_clear_steps():
    """BLOCK / CLEAR now reach the device as sparse updates: the GPU session must match the CPU oracle env
    (which reads the MapUtil directly) after every step, over many edits on a 128^3 map."""
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 128)
    a = voxel_session_args(sc, 1, 3000)
    first = pb.lpa_oracle(a, [("plan",)])[0]
    assert first["valid"] == 1
    cells = integrate_cells(sc.control, sc.U, [a.start.pos[k] for k in range(3)], first["actions"], sc.origin, sc.res)
    script = [("plan",), ("link",)]
    for frac in (0.25, 0.5, 0.75, 0.5):
        c = cells[int(frac * (len(cells) - 1))]
        wall = np.array([c + (0, dy, dz) for dy in range(-3, 4) for dz in range(-3, 4)], dtype=np.int32)  # across x
        script += [("block", wall), ("plan",), ("link",), ("clear", wall), ("plan",)]
    script += [("block", cells[1:-1]), ("plan",), ("clear", cells[1:-1]), ("plan",)]
    orc = pb.lpa_oracle(a, script)
    assert orc[1]["n_linked"] > 100
    same_session(pb.lpa_session(a, script), orc)


def test_batch_planner_replans_after_update_cells():
    from motion_primitive_library_b200 import planner as P

    sc = _headline64()
    nodes = sc.frontier(48, seed=5, max_steps=0)
    starts, goals = nodes[:24].copy(), nodes[24:].copy()
    base = dict(v_max=sc.v_max, a_max=sc.a_max, max_num=1500)
    grid = np.array(sc.grid(), dtype=np.int8).reshape(-1)
    args = P.make_args(3, ACC, grid, sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=starts["pos"][0]),
                       goal=dict(pos=goals["pos"][0]), **base)
    bp = P.BatchPlanner(args)
    r0, _ = bp.plan(starts, goals)
    assert r0["valid"].sum() > 4
    # walls through the midpoints of the first queries' start-goal segments
    dims = np.asarray(sc.dim_cells)
    mids = np.floor(((starts["pos"] + goals["pos"]) / 2 - np.asarray(sc.origin)) / sc.res).astype(int)[:8]
    wall = np.array([m + (dx, dy, dz) for m in mids for dx in range(-3, 4) for dy in range(-3, 4) for dz in range(-3, 4)])
    wall = wall[((wall >= 0) & (wall < dims)).all(1)].astype(np.int32)
    bp.update_cells(wall, np.full(len(wall), 100, dtype=np.int8))
    r1, _ = bp.plan(starts, goals)
    assert bp.map_uploads() == (1, 1)  # the session's first upload, then one sparse update
    bp.close()
    edited = grid.copy()
    edited[wall[:, 0] + dims[0] * wall[:, 1] + dims[0] * dims[1] * wall[:, 2]] = 100
    a2 = P.make_args(3, ACC, edited, sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=starts["pos"][0]),
                     goal=dict(pos=goals["pos"][0]), **base)
    r2, _ = P.plan_batch(a2, starts, goals)
    assert r1.tobytes() == r2.tobytes()
    assert r1.tobytes() != r0.tobytes()  # the walls changed some query's search
