"""mplx_edges_is_free / mplx_edges_cells (csrc/mplx_edges.cu) on constructed edges for every branch, every
<Dim, order> instantiation with and without a yaw control and a search region, launch geometry and buffer reuse.

Witnesses.  Constructed ACC edges (tests/test_edges_inputs_oracle_vs_ref.py): the oracle, pinned there to the
reference for is_free and the intrinsic cost, and the plain-numpy walk for the cells.  Random edges of the other
instantiations: the oracle (pinned to the reference by tests/test_edges_oracle_vs_ref.py and, for the walk,
tests/test_lpastar_vs_ref.py).  Edges beyond 2^20 samples and NaN / infinite velocities: the contract of
include/mplx.h only — not free, no cells.  Everything bit for bit."""
import ctypes as C

import numpy as np
import pytest

import oracle_bindings as ob
import test_edges_inputs_oracle_vs_ref as K
from test_edges_oracle_vs_ref import edges_of

pytestmark = pytest.mark.gpu
VEL, ACC, JRK, SNP, YAW = 0x01, 0x03, 0x07, 0x0F, 0x10


def gpu_of(orc):
    """A libmplx env with the parameters, map and region of an OracleEnv."""
    from motion_primitive_library_b200 import MapUtil, env_map

    e, dim = orc.e, int(orc.e.dim)
    mu = MapUtil()
    mu.setMap(tuple(e.origin)[:dim], tuple(e.mdim)[:dim], orc.grid.copy(), e.res)
    env = env_map(mu)
    env.set_control(int(e.control))
    env.set_u(orc.U)
    env.set_dt(e.T)
    env.set_w(e.w)
    env.set_wyaw(e.wyaw)
    env.set_v_max(e.v_max)
    env.set_a_max(e.a_max)
    env.set_j_max(e.j_max)
    env.set_yaw_max(e.yaw_max)
    if orc.region is not None:
        env.set_search_region(orc.region)
    return env


def table_of(orc, off, cells):
    """The inverted table from the cell lists: (getIndex with int32 wrap-around, edge) sorted by voxel, stably."""
    dims = np.asarray(tuple(orc.e.mdim)[: int(orc.e.dim)], dtype=np.int64)
    strides = np.concatenate([[1], np.cumprod(dims[:-1])])
    ids = (cells.astype(np.int64) * strides).sum(1).astype(np.int32)
    owner = np.repeat(np.arange(off.size - 1, dtype=np.int32), np.diff(off))
    order = np.argsort(ids, kind="stable")
    return ids[order], owner[order]


def check(env, orc, parents, actions):
    """Both queries against the oracle, with the launches each adds: is_free 1; cells 2 when it stops at the
    count (nothing to write), 3 when it writes."""
    env._sync_params()
    before = env.launch_count()
    fg, cg = env.is_free_edges(parents, actions)
    assert env.launch_count() - before == (1 if parents.size else 0)
    fo, co = orc.edges_is_free(parents, actions)
    np.testing.assert_array_equal(fg, fo)
    assert cg.tobytes() == co.tobytes()
    oo, oc = orc.edges_cells(parents, actions)
    before = env.launch_count()
    go, gc, tv, te = env.edge_cells(parents, actions, table=True)
    np.testing.assert_array_equal(go, oo)
    np.testing.assert_array_equal(gc, oc)
    ev, ee = table_of(orc, oo, oc)
    np.testing.assert_array_equal(tv, ev)
    np.testing.assert_array_equal(te, ee)
    writes = 3 if oc.shape[0] else 2
    retried = oc.shape[0] > max(1, 8 * parents.size)  # env.edge_cells sizes its arrays from a first, refused call
    assert env.launch_count() - before == (writes + (2 if retried else 0) if parents.size else 0)
    return fo, oo, oc, tv


# ---- 1. constructed edges -------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("with_region", [False, True])
def test_constructed_edges(dim, with_region):
    names, parents, actions = K.batch(dim)
    orc = K.oracle_env(dim, K.region_of(dim) if with_region else None)
    env = gpu_of(orc)
    fo, off, cells, tv = check(env, orc, parents, actions)
    U = K.controls(dim)
    for i, name in enumerate(names):  # the third witness: the plain-numpy walk
        assert cells[off[i]:off[i + 1]].tolist() == K.walk_acc(dim, parents[i], U[actions[i]])[0], name
    assert (tv < -1).any(), "the table holds negative voxel ids"
    assert (np.diff(tv.astype(np.int64)) >= 0).all()
    # each edge alone: a batch of one gives what the batch gave
    for i in (0, names.index("first_index_minus_one"), names.index("negative_indices")):
        f1, _ = env.is_free_edges(parents[i:i + 1], actions[i:i + 1])
        o1, c1 = env.edge_cells(parents[i:i + 1], actions[i:i + 1])
        assert f1[0] == fo[i] and c1.tolist() == cells[off[i]:off[i + 1]].tolist()


@pytest.mark.parametrize("dim", [2, 3])
def test_edges_beyond_the_sample_limit_follow_the_contract(dim):
    """n > kEdgeNMax, NaN and infinite velocities: not free, no cells (no CPU witness walks them).  n == kEdgeNMax
    is the largest edge served: the oracle walks its 2^20 + 1 samples."""
    orc = K.oracle_env(dim)
    env = gpu_of(orc)
    parents, actions = K.contract_only(dim)
    free, cost = env.is_free_edges(parents, actions)
    assert not free.any()
    off, cells = env.edge_cells(parents, actions)
    assert off.tolist() == [0] * (parents.size + 1) and cells.shape == (0, dim)
    # mixed with ordinary edges they take no room and shift nothing
    names, p2, a2 = K.batch(dim)
    mixed_p, mixed_a = np.concatenate([p2[:3], parents, p2[3:]]), np.concatenate([a2[:3], actions, a2[3:]])
    keep = np.r_[0:3, 3 + parents.size:mixed_p.size]
    f, _ = env.is_free_edges(mixed_p, mixed_a)
    fo, _ = orc.edges_is_free(p2, a2)
    np.testing.assert_array_equal(f[keep], fo)
    assert not f[3:3 + parents.size].any()
    off, cells = env.edge_cells(mixed_p, mixed_a)
    oo, oc = orc.edges_cells(p2, a2)
    np.testing.assert_array_equal(np.diff(off)[keep], np.diff(oo))
    assert (np.diff(off)[3:3 + parents.size] == 0).all() and cells.tolist() == oc.tolist()
    if dim == 2:
        p1, a1 = K.largest_served(dim)
        fo, oo, oc, _ = check(env, orc, p1, a1)
        assert not fo[0] and oc.shape[0] > K.EDGE_N_MAX // 2


# ---- 2. instantiations -------------------------------------------------------------------------------------
def interior_extremum_edge(dim, control, U):
    """A JRK / SNP edge whose speed peaks inside (0, T): v = 1, a = 0.5, jerk -1 => |v| is 1.125 at t = 0.5 and 1
    at both ends, so the interior extremum decides n."""
    w = np.zeros((), dtype=ob.WAYPOINT_DTYPE)
    w["vel"][0], w["acc"][0] = 1.0, 0.5
    if control & 15 == SNP:
        w["jrk"][0] = -1.0
        u = [0.0] * dim
    else:
        u = [-1.0] + [0.0] * (dim - 1)
    rows = np.flatnonzero((U[:, :dim] == np.asarray(u)).all(1))
    return w, int(rows[0])


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("control", [VEL, ACC, JRK, SNP, VEL | YAW, ACC | YAW, JRK | YAW, SNP | YAW])
@pytest.mark.parametrize("with_region", [False, True])
def test_every_instantiation(dim, control, with_region):
    """<2|3, VEL|ACC|JRK|SNP> with and without a yaw rate in U (udim = Dim + 1) and a region, on a map whose rows
    start mid-word."""
    from scenarios import box_map, control_set
    from test_oracle_vs_ref import random_nodes

    yaw = bool(control & YAW)
    rng = np.random.default_rng(300 + control * 4 + dim * 2 + with_region)
    u_max = 4.0 if control & 15 == SNP else 1.0
    U = control_set(u_max, 3, dim, yaw_rates=(-0.4, 0.0, 0.4) if yaw else None)
    assert U.shape[1] == dim + yaw
    dims, res = ((37, 41), 0.2) if dim == 2 else ((37, 41, 35), 0.2)
    origin = tuple(-d * res / 2 for d in dims)
    grid = box_map(dims, res, origin, 6, (0.6, 1.6), seed=3)
    region = (rng.random(int(np.prod(dims))) < 0.97).astype(np.uint8) if with_region else None
    orc = ob.OracleEnv(dim, control, U, grid, dims, origin, res, T=1.0, w=10.0, wyaw=1.5, v_max=2.5, a_max=3.0, j_max=6.0,
                       yaw_max=0.9 if yaw else -1.0, region=region)
    nodes = random_nodes(rng, 300, dim, 35 * res / 2, yaw=yaw)
    parents, actions, _ = edges_of(orc, nodes, rng, extra=300)
    if control & 15 in (JRK, SNP):
        w, a = interior_extremum_edge(dim, control, U)
        ends = max(abs(w["vel"][0]), abs(w["vel"][0] + w["acc"][0] - 0.5))
        peak = ob.lib().orc_max_vel(C.byref(orc.e), w.reshape(1).ctypes.data, a, 0)
        assert abs(peak - 1.125) < 1e-12 and ends == 1.0 and np.ceil(peak / res) > np.ceil(ends / res)
        parents, actions = np.concatenate([parents, w.reshape(1)]), np.concatenate([actions, [a]]).astype(np.int32)
    env = gpu_of(orc)
    fo, off, cells, _ = check(env, orc, parents, actions)
    assert 0 < fo.sum() < fo.size and cells.shape[0] > parents.size


# ---- 3. geometry, capacity, reuse ----------------------------------------------------------------------
def test_batch_sizes_capacity_and_raw_abi():
    """1, 127, 128, 129 and 4097 edges (CTAs of 128), a capacity of exactly `total`, out_cost = NULL, one table
    pointer without the other, action ids -1 and |U|."""
    from motion_primitive_library_b200 import abi
    import scenarios as S

    sc = S.scaled(S.cfg_headline(), 64)
    orc = ob.OracleEnv.from_scenario(sc)
    env = gpu_of(orc)
    rng = np.random.default_rng(5)
    parents, actions, _ = edges_of(orc, sc.frontier(400, seed=3), rng, extra=200)
    assert parents.size >= 4097
    lib, h = env._lib, env.handle
    for n in (1, 127, 128, 129, 4097):
        p, a = np.ascontiguousarray(parents[:n]), np.ascontiguousarray(actions[:n])
        fo, oo, oc, _ = check(env, orc, p, a)
        # out_cost = NULL
        free = np.full(n + 8, 0xA5, dtype=np.uint8)
        abi.check(lib.mplx_edges_is_free(h, p.ctypes.data, a.ctypes.data, n, free.ctypes.data, None))
        np.testing.assert_array_equal(free[:n], fo)
        assert (free[n:] == 0xA5).all()
        # capacity exactly total, one less, and zero
        total = int(oo[-1])
        off, tot = np.zeros(n + 1, np.int64), C.c_int64(0)
        cells = np.full((total + 8, 3), -7, dtype=np.int32)
        before = env.launch_count()
        abi.check(lib.mplx_edges_cells(h, p.ctypes.data, a.ctypes.data, n, off.ctypes.data, cells.ctypes.data, total,
                                       C.byref(tot), None, None))
        assert env.launch_count() - before == 3 and tot.value == total
        np.testing.assert_array_equal(cells[:total], oc)
        assert (cells[total:] == -7).all()
        for cap in (total - 1, 0):
            off[:] = -1
            cells[:] = -7
            before = env.launch_count()
            rc = lib.mplx_edges_cells(h, p.ctypes.data, a.ctypes.data, n, off.ctypes.data, cells.ctypes.data, cap,
                                      C.byref(tot), None, None)
            assert rc == abi.MPLX_ERR_ARG and tot.value == total and env.launch_count() - before == 2
            np.testing.assert_array_equal(off, oo)
            assert (cells == -7).all()
    p, a = np.ascontiguousarray(parents[:50]), np.ascontiguousarray(actions[:50])
    off, tot, buf = np.zeros(51, np.int64), C.c_int64(0), np.zeros(4000, np.int32)
    for tv, te in ((buf.ctypes.data, None), (None, buf.ctypes.data)):
        assert lib.mplx_edges_cells(h, p.ctypes.data, a.ctypes.data, 50, off.ctypes.data, buf.ctypes.data, 1000,
                                    C.byref(tot), tv, te) == abi.MPLX_ERR_ARG
    for bad in (-1, sc.nU):
        a2 = a.copy()
        a2[49] = bad
        before = env.launch_count()
        with pytest.raises(abi.MplxError) as e:
            env.is_free_edges(p, a2)
        assert e.value.code == abi.MPLX_ERR_ARG and "edge 49" in str(e.value)
        with pytest.raises(abi.MplxError):
            env.edge_cells(p, a2)
        assert env.launch_count() == before
    check(env, orc, p, a)  # the ctx serves a correct call after the refusals


def test_buffer_reuse_big_small_bigger():
    """The ctx keeps its edge buffers: a large call, a small one and a larger one each equal a fresh ctx's."""
    import scenarios as S

    sc = S.scaled(S.cfg3(), 64)
    orc = ob.OracleEnv.from_scenario(sc)
    parents, actions, _ = edges_of(orc, sc.frontier(200, seed=4), np.random.default_rng(6), extra=500)
    assert parents.size > 9000
    env = gpu_of(orc)
    for lo, hi in ((0, 6000), (6000, 6007), (100, parents.size), (0, 0), (5, 6)):
        p, a = np.ascontiguousarray(parents[lo:hi]), np.ascontiguousarray(actions[lo:hi])
        check(env, orc, p, a)
        fresh = gpu_of(orc)
        assert fresh.is_free_edges(p, a)[0].tobytes() == env.is_free_edges(p, a)[0].tobytes()
        for x, y in zip(fresh.edge_cells(p, a, table=True), env.edge_cells(p, a, table=True)):
            assert x.tobytes() == y.tobytes()


def test_far_corner_of_a_512_cube():
    """Voxel indices near 2^27: edges in the last cells of a 512^3 map, some leaving it."""
    from scenarios import control_set

    n = 512
    grid = np.zeros(n ** 3, dtype=np.int8)
    g3 = grid.reshape(n, n, n)
    g3[-6:-4, -9:-3, -30:-2] = 100
    res, origin = 0.1, (-25.6,) * 3
    orc = ob.OracleEnv(3, ACC, control_set(1.0, 3, 3), grid, (n,) * 3, origin, res, T=1.0, w=10.0, v_max=3.0)
    rng = np.random.default_rng(7)
    m = 600
    parents = np.zeros(m, dtype=ob.WAYPOINT_DTYPE)
    parents["pos"][:, :3] = 25.6 - rng.random((m, 3)) * 3.0
    parents["vel"][:, :3] = rng.integers(-2, 3, (m, 3)) * 1.0
    actions = rng.integers(0, 27, m).astype(np.int32)
    env = gpu_of(orc)
    fo, off, cells, tv = check(env, orc, parents, actions)
    assert 0 < fo.sum() < fo.size and tv.max() > 2 ** 27 - 2 ** 19
