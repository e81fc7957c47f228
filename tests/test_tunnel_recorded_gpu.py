"""Tunnels built on the device from the paths the last search call recorded (mplx_set_batch_regions_recorded).

  - Every tunnel, read back one byte per voxel, equals mplx_set_search_region_path's region of that query's recorded
    node positions (batch_trajectories), or of its host points, byte for byte: 2-D and 3-D, dense and not, recordings
    of mplx_plan_batch, _cost_terms and _grow (one whose records span several rounds' rooms), selections that are
    subsets, permutations and repeats and that mix host points in, paths that leave the map part-way through a
    segment and segments of 0 and 1 steps.
  - Refusals change nothing and launch nothing; the launch count does not depend on the query count.
The expected regions come from mplx_set_search_region_path, which runs the same walk (search::segment_cells) on the
host; tests/test_segment_cells_cpu.py pins that walk to the per-segment loop it replaced, so the two together hold
the device trace to the original one."""
import ctypes as C

import numpy as np
import pytest

from motion_primitive_library_b200 import abi
from test_device_search_tunnels_gpu import ORDERS, build_paths, control_set, make_env, queries, world

pytestmark = pytest.mark.gpu
WAYPOINT = abi.WAYPOINT_DTYPE


def record(e, entry, S, G, mx, dim):
    if entry == "batch":
        return e.plan_batch(S, G, eps=2.0, max_expand=mx, trajectories=True)
    if entry == "cost_terms":
        return e.plan_batch_cost_terms(S, G, eps=2.0, max_expand=mx, trajectories=True)
    # small arenas, pool and room: the records span several rounds' rooms
    r = e.plan_batch_grow(S, G, eps=2.0, max_expand=mx, cost_terms=dim == 3, first_cap=8, pool_bytes=64,
                          trajectories=True, traj_room_bytes=4 * WAYPOINT.itemsize)
    assert r["rounds"] > 1
    return r


def short_steps(w, dim):
    """Host paths whose segments take 0 and 1 samples (max_diff 0, 1 and 2) and one that leaves the map."""
    res = w["res"]
    a = np.asarray(w["origin"], float) + 3.3 * res
    one = np.zeros(dim)
    one[0] = 0.8 * res * 1.5
    return [np.stack([a, a + 0.3 * res, a + 0.3 * res + one, a + 0.3 * res + 2 * one]),
            np.stack([a, a - 10.0 * res * np.ones(dim)])]


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("dense", [False, True])
@pytest.mark.parametrize("entry", ["batch", "cost_terms", "grow"])
def test_recorded_tunnel_equals_region_path(dim, dense, entry):
    w = world(dim)
    e = make_env(w, dim, ORDERS["ACC"], control_set(dim, 2, False), pot=entry == "cost_terms")
    nq, mx = 14, 40 if dim == 3 else 60
    S, G = queries(w, dim, nq, seed=61 + dim, yaw=False)
    r = record(e, entry, S, G, mx, dim)
    nodes = [t["nodes"]["pos"][:, :dim].copy() for t in r["trajectories"]]
    have = [q for q in range(nq) if len(nodes[q])]
    assert len(have) >= 4, have
    rng = np.random.default_rng(dim + 7 * int(dense))
    host = build_paths(w, dim) + short_steps(w, dim)
    rad = [0.3, 0.55, 0.3][:dim]
    sel = [
        np.array(have, np.int32),                                   # every recorded path
        np.array(have[1::2], np.int32),                             # a subset
        rng.permutation(np.array(have, np.int32)),                  # a permutation
        np.array([have[0]] * 3 + [have[-1]] * 2, np.int32),         # repeats
    ]
    mixed = []
    for j in range(len(have) + len(host)):
        mixed.append(have[j // 2] if j % 2 == 0 and j // 2 < len(have) else -1)
    sel.append(np.array(mixed, np.int32))
    for from_ in sel:
        paths = [host[j % len(host)] if f < 0 else np.zeros((0, dim)) for j, f in enumerate(from_)]
        e.set_batch_regions_recorded(from_, rad, dense, paths=paths if (from_ < 0).any() else None)
        info = e.batch_regions_info()
        assert info["n_q"] == len(from_)
        got = [e.read_batch_region(j) for j in range(len(from_))]
        for j, f in enumerate(from_):
            want = e.set_search_region_path(nodes[f] if f >= 0 else paths[j], rad, dense)
            assert np.array_equal(got[j], want), (j, int(f))
    # the same tunnels from the host points through mplx_set_batch_regions
    e.set_batch_regions([nodes[q] for q in have], rad, dense)
    host_built = [e.read_batch_region(j) for j in range(len(have))]
    e.set_batch_regions_recorded(np.array(have, np.int32), rad, dense)
    for j in range(len(have)):
        assert np.array_equal(e.read_batch_region(j), host_built[j]), j
    e.close()


def test_launches_do_not_depend_on_the_query_count():
    dim = 2
    w = world(dim)
    e = make_env(w, dim, ORDERS["ACC"], control_set(dim, 2, False))
    S, G = queries(w, dim, 16, seed=71, yaw=False)
    r = e.plan_batch(S, G, eps=2.0, max_expand=60, trajectories=True)
    have = [q for q in range(16) if len(r["trajectories"][q]["nodes"])]
    counts = []
    for n in (1, 3, 40):
        from_ = np.array([have[j % len(have)] for j in range(n)], np.int32)
        n0 = e.launch_count()
        e.set_batch_regions_recorded(from_, [0.5, 0.5])
        counts.append(e.launch_count() - n0)
    assert len(set(counts)) == 1 and counts[0] > 0, counts
    n0 = e.launch_count()
    e.set_batch_regions_recorded(np.zeros(0, np.int32), [0.5, 0.5])
    assert e.launch_count() == n0 and e.batch_regions_info()["n_q"] == 0
    e.close()


def test_refusals_change_nothing_and_launch_nothing():
    dim = 2
    w = world(dim)
    e = make_env(w, dim, ORDERS["ACC"], control_set(dim, 2, False))
    lib, h = e._lib, e.handle
    S, G = queries(w, dim, 6, seed=81, yaw=False)
    S[5] = G[5]  # start already a goal: no recorded path
    rad = np.array([0.5, 0.5])
    pts = np.ascontiguousarray(np.concatenate([S["pos"][:2, :dim], G["pos"][:2, :dim]]))
    off = np.array([0, 2, 4], np.int64)

    def refused(n_q, from_, o, p, r):
        n0 = e.launch_count()
        info = e.batch_regions_info()
        before = [e.read_batch_region(q) for q in range(info["n_q"])]
        rc = lib.mplx_set_batch_regions_recorded(h, n_q, abi.ptr(from_), abi.ptr(o), abi.ptr(p), abi.ptr(r), 0)
        assert rc == abi.MPLX_ERR_ARG
        assert e.launch_count() == n0 and e.batch_regions_info() == info
        for q, b in enumerate(before):
            assert np.array_equal(e.read_batch_region(q), b)

    ok = np.array([0, 1], np.int32)
    refused(2, ok, None, None, rad)                            # no search call yet
    e.plan_batch(S, G, eps=2.0, max_expand=60, trajectories=False)
    refused(2, ok, None, None, rad)                            # the last call ran without recording
    r = e.plan_batch(S, G, eps=2.0, max_expand=60, trajectories=True)
    e.set_batch_regions([S["pos"][q, :dim][None, :] for q in range(6)], rad)  # tunnels the refusals must keep
    assert len(r["trajectories"][5]["nodes"]) == 0
    have = [q for q in range(5) if len(r["trajectories"][q]["nodes"])]
    none = [q for q in range(6) if not len(r["trajectories"][q]["nodes"])]
    assert have and none
    refused(2, np.array([have[0], 6], np.int32), None, None, rad)       # outside the last call's queries
    refused(2, np.array([have[0], none[0]], np.int32), None, None, rad)  # a query without a recorded path
    refused(2, np.array([have[0], -1], np.int32), None, None, rad)       # a host-points query without points
    refused(2, np.array([have[0], -1], np.int32), off, None, rad)
    refused(2, np.array([have[0], -1], np.int32), np.array([0, 2, 2], np.int64), pts, rad)  # no points for query 1
    refused(2, np.array([have[0], -1], np.int32), np.array([1, 2, 4], np.int64), pts, rad)  # pt_offset[0] != 0
    refused(2, None, None, None, rad)                                    # NULL from
    refused(2, ok, None, None, None)                                     # NULL radius
    refused(-1, ok, None, None, rad)
    # a mixed call with valid arguments is accepted
    e.set_batch_regions_recorded(np.array([have[0], -1], np.int32), rad, paths=[np.zeros((0, dim)), pts[2:]])
    assert e.batch_regions_info()["n_q"] == 2
    e.close()
    # a ctx without a map
    h2 = C.c_void_p()
    abi.check(lib.mplx_create(2, 0, C.byref(h2)))
    assert lib.mplx_set_batch_regions_recorded(h2, 2, ok.ctypes.data, None, None, rad.ctypes.data, 0) == \
        abi.MPLX_ERR_ARG
    lib.mplx_destroy(h2)
