"""The batched searches' trajectories on the CPU: the device trace-back's state chain (search::finish in
mplx_search.cuh, compiled by g++) against the host planner's recoverTraj best_child_ on scripted search graphs;
the ctypes mirror of mplx_batch_traj_out against the header; and the new entry points refusing without a GPU."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent
K_GOAL, K_TRIVIAL, K_FAILED = 3, 2, 4


@pytest.fixture(scope="module")
def btj(tmp_path_factory):
    so = tmp_path_factory.mktemp("btj") / "libbtj.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-pthread", "-fPIC", "-shared", "-o",
                           str(so), str(HERE / "batch_traj_host.cpp")])
    L = C.CDLL(str(so))
    vp = C.c_void_p
    L.btj_trace.argtypes = [C.c_int, vp, vp, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_uint64, C.c_int,
                            vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.btj_trace.restype = C.c_int
    return L


def trace(L, g, preds, status, cur, start=0, cap=64):
    """Scripted graph: states 0..n-1 with g[i] and key 1000 + i; preds: (to, from, action, cost) in record order.
    Returns (device, host) dicts."""
    g = np.asarray(g, np.float64)
    n = len(g)
    key = np.arange(1000, 1000 + n, dtype=np.uint64)
    P = np.array(preds, dtype=np.float64).reshape(-1, 4)
    to, node, act = (np.ascontiguousarray(P[:, k], np.int32) for k in range(3))
    cost = np.ascontiguousarray(P[:, 3])
    dc, dna = np.zeros(1), np.zeros(1, np.int32)
    dact, dchain = np.zeros(max(cap, 1), np.int32), np.zeros(cap + 3, np.int32)
    hf, hna, hn = (np.zeros(1, np.int32) for _ in range(3))
    hact, hchain = np.zeros(n + 2, np.int32), np.zeros(n + 2, np.int32)
    assert L.btj_trace(n, g.ctypes.data, key.ctypes.data, len(P), to.ctypes.data, node.ctypes.data, act.ctypes.data,
                       cost.ctypes.data, status, cur, int(key[start]), cap, dc.ctypes.data, dna.ctypes.data,
                       dact.ctypes.data, dchain.ctypes.data, hf.ctypes.data, hna.ctypes.data, hact.ctypes.data,
                       hchain.ctypes.data, hn.ctypes.data) == 0
    na = int(dna[0])
    dev = dict(cost=float(dc[0]), n_actions=na, actions=dact[:max(na, 0)].copy(), chain=dchain[:na + 1].copy(),
               raw_chain=dchain.copy())
    host = dict(found=int(hf[0]), actions=hact[:hna[0]].copy(), chain=hchain[:hn[0]].copy())
    return dev, host


def check_same(dev, host):
    assert host["found"] == 1
    assert dev["n_actions"] == len(host["actions"])
    assert np.array_equal(dev["actions"], host["actions"])
    assert len(dev["chain"]) == dev["n_actions"] + 1
    assert np.array_equal(dev["chain"], host["chain"])


def test_chain_follows_the_best_predecessor_not_the_creator(btj):
    # 0 = start; 1 and 2 reached from 0; 3 first created from 1 (its stored coordinates are 1's successor's), but
    # its best predecessor is 2; 4 = goal from 3
    g = [0.0, 1.0, 0.5, 1.5, 2.5]
    preds = [(1, 0, 0, 1.0), (2, 0, 1, 0.5), (3, 1, 2, 1.0), (3, 2, 3, 1.0), (4, 3, 4, 1.0)]
    dev, host = trace(btj, g, preds, K_GOAL, 4)
    check_same(dev, host)
    assert list(dev["chain"]) == [0, 2, 3, 4]
    assert list(dev["actions"]) == [1, 3, 4]
    assert dev["cost"] == 2.5


def test_equal_g_plus_cost_tie_takes_the_larger_g(btj):
    # state 3 has two predecessors with g + cost = 2.0: 1 (g 0.5, cost 1.5) recorded first, 2 (g 1.0, cost 1.0)
    g = [0.0, 0.5, 1.0, 2.0]
    preds = [(1, 0, 0, 0.5), (2, 0, 1, 1.0), (3, 1, 5, 1.5), (3, 2, 6, 1.0)]
    dev, host = trace(btj, g, preds, K_GOAL, 3)
    check_same(dev, host)
    assert list(dev["chain"]) == [0, 2, 3]
    # and the first one wins when its g is the larger
    g2 = [0.0, 1.0, 0.5, 2.0]
    preds2 = [(1, 0, 0, 1.0), (2, 0, 1, 0.5), (3, 1, 5, 1.0), (3, 2, 6, 1.5)]
    dev, host = trace(btj, g2, preds2, K_GOAL, 3)
    check_same(dev, host)
    assert list(dev["chain"]) == [0, 1, 3]


def test_longer_chain_with_revisited_states(btj):
    rng = np.random.default_rng(5)
    n = 40
    g = np.sort(rng.uniform(0, 10, n))
    g[0] = 0.0
    preds = []
    for i in range(1, n):
        for _ in range(int(rng.integers(1, 4))):
            j = int(rng.integers(0, i))
            preds.append((i, j, int(rng.integers(0, 27)), float(rng.choice([g[i] - g[j], g[i] - g[j] + 0.25]))))
    dev, host = trace(btj, g, preds, K_GOAL, n - 1)
    check_same(dev, host)
    assert dev["chain"][0] == 0 and dev["chain"][-1] == n - 1


def test_start_already_a_goal_and_failed_search(btj):
    dev, _ = trace(btj, [0.0], [], K_TRIVIAL, 0)
    assert dev["n_actions"] == 0 and dev["cost"] == 0.0
    dev, _ = trace(btj, [0.0, 1.0], [(1, 0, 0, 1.0)], K_FAILED, 1)
    assert dev["n_actions"] == 0 and np.isinf(dev["cost"])
    # a chain that never reaches the start: no trajectory, as recoverTraj finds none
    dev, host = trace(btj, [0.0, 1.0, 2.0], [(2, 1, 0, 1.0)], K_GOAL, 2)
    assert host["found"] == 0 and dev["n_actions"] == 0 and np.isinf(dev["cost"])


def test_action_buffer_too_small(btj):
    g = [0.0, 1.0, 2.0, 3.0, 4.0]
    preds = [(k + 1, k, k, 1.0) for k in range(4)]
    dev, host = trace(btj, g, preds, K_GOAL, 4, cap=2)
    assert host["found"] == 1 and len(host["actions"]) == 4
    assert dev["n_actions"] == -1
    # the chain keeps to its cap + 1 entries
    assert list(dev["raw_chain"][3:]) == [-7, -7]
    dev, host = trace(btj, g, preds, K_GOAL, 4, cap=4)
    check_same(dev, host)


def _header_struct(name):
    text = (ROOT / "include" / "mplx.h").read_text()
    end = text.index("} " + name + ";")
    body = text[text.rindex("typedef struct {", 0, end) + len("typedef struct {"):end]
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return [(t.strip(), f.strip()) for t, f in re.findall(r"([\w\s\*]+?[\s\*])(\w+);", body)]


def test_batch_traj_out_mirror_matches_header():
    from motion_primitive_library_b200 import abi

    fields = _header_struct("mplx_batch_traj_out")
    assert [f for _, f in fields] == [f for f, _ in abi.BatchTrajOut._fields_]
    sizes = {"int64_t": 8, "double": 8}
    off = 0
    for (t, f), (mf, _) in zip(fields, abi.BatchTrajOut._fields_):
        size = 8 if "*" in t else sizes[t]
        off = (off + size - 1) // size * size
        assert getattr(abi.BatchTrajOut, mf).offset == off, f
        off += size
    assert C.sizeof(abi.BatchTrajOut) == off


def test_entry_points_exported():
    from motion_primitive_library_b200 import abi

    assert "mplx_set_batch_trajectories" in abi.EXPORTED_SYMBOLS
    assert "mplx_plan_batch_trajectories" in abi.EXPORTED_SYMBOLS


def test_entry_points_refuse_without_a_ctx():
    from motion_primitive_library_b200 import abi

    lib = abi.load()
    out = abi.BatchTrajOut()
    assert lib.mplx_set_batch_trajectories(None, 1, 0) == abi.MPLX_ERR_ARG
    assert lib.mplx_plan_batch_trajectories(None, 0, C.byref(out)) == abi.MPLX_ERR_ARG


def test_batch_session_entry_points_refuse_without_a_session():
    from motion_primitive_library_b200 import planner as P

    lib = P._lib()
    total = C.c_int64(-3)
    off = np.full(2, -5, np.int64)
    assert lib.mplh_batch_set_trajectories(None, 1) == 1
    assert lib.mplh_batch_trajectories(None, 0, off.ctypes.data, None, None, None, None, 0, C.byref(total)) == 1
    assert total.value == -3 and np.all(off == -5)
