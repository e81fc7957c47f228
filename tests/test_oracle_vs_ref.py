"""Pins the oracle: the restatement (oracle/mpl_oracle.cpp) against the REFERENCE's own
env_map<Dim>::get_succ, compiled unmodified from the reference's include/ with the Eigen/Boost
stand-ins of oracle/shim (oracle/_ref/libmplref.so, built by `make -C oracle ref`), or against its
recorded results where oracle/_ref is not built (tests/reference_record.py).

Both run on the CPU with the same flags, so everything must agree BIT FOR BIT: successor
waypoints, edge costs (including the potential / yaw-alignment sums), action ids, hash keys."""
import numpy as np
import pytest

import fixtures
import oracle_bindings as ob
from reference_record import same_array

VEL, ACC, JRK, SNP, VELxYAW, ACCxYAW, JRKxYAW, SNPxYAW = 0x01, 0x03, 0x07, 0x0F, 0x11, 0x13, 0x17, 0x1F


def assert_bit_equal(o, r):
    same_array(o["count"], r["count"], "count")
    o, r = ob.emitted(o), ob.emitted(r)
    same_array(o["action"], r["action"], "action")
    same_array(o["succ"], r["succ"], "succ", bits=True)
    same_array(o["cost"], r["cost"], "cost", bits=True)
    same_array(o["key"], r["key"], "key")
    return int(o["count"].sum())


def random_nodes(rng, n, dim, half, vstep=0.5, yaw=True):
    nodes = np.zeros(n, dtype=ob.WAYPOINT_DTYPE)
    nodes["pos"][:, :dim] = np.round(rng.uniform(-half * 0.95, half * 0.95, (n, dim)) / 0.05) * 0.05
    nodes["vel"][:, :dim] = rng.integers(-4, 5, (n, dim)) * vstep
    nodes["acc"][:, :dim] = rng.integers(-4, 5, (n, dim)) * 0.5
    nodes["jrk"][:, :dim] = rng.integers(-3, 4, (n, dim)) * 1.0
    if yaw:
        nodes["yaw"] = rng.integers(-7, 8, n) * 0.4
    nodes["t"] = rng.integers(0, 5, n) * 1.0
    # a few off-lattice states too
    nodes["pos"][::7, :dim] += rng.uniform(-0.03, 0.03, (len(nodes[::7]), dim))
    nodes["vel"][::11, :dim] += rng.uniform(-0.2, 0.2, (len(nodes[::11]), dim))
    return nodes


def test_reference_build_info():
    info = ob.ref_info()
    assert "unmodified" in info and "env_map.h" in info


def test_corridor_reference_test_config_first_expansions():
    """config 1 (test/test_planner_2d.cpp) — also re-checks the SURVEY §10 table on the reference itself."""
    c = fixtures.corridor()
    env = ob.OracleEnv(2, ACC, fixtures.U_2d(), c["grid"], c["dim"], c["origin"], c["res"], T=1.0, w=10.0, v_max=1.0,
                       a_max=1.0)
    start = np.zeros(1, dtype=ob.WAYPOINT_DTYPE)
    start["pos"][0, :2] = c["start"]
    r = ob.ref_expand(env, start)
    assert list(r["action"][: r["count"][0]]) == [0, 1, 2, 3, 5, 6, 7, 8]
    assert list(r["cost"][:8]) == [10.5, 10.25, 10.5, 10.25, 10.25, 10.5, 10.25, 10.5]
    front = start
    total = 0
    for _ in range(6):
        o = env.expand(front, nthreads=4)
        total += assert_bit_equal(o, ob.ref_expand(env, front, nthreads=4))
        valid = (np.arange(o["nU"])[None, :] < o["count"][:, None]).reshape(-1) & ~np.isinf(o["cost"])
        _, uniq = np.unique(o["key"][valid], return_index=True)
        front = o["succ"][valid][np.sort(uniq)]
    assert total > 3000


@pytest.mark.parametrize("control,dim", [(VEL, 2), (ACC, 2), (JRK, 2), (SNP, 2), (VELxYAW, 2), (ACCxYAW, 2),
                                         (JRKxYAW, 2), (SNPxYAW, 2), (VEL, 3), (ACC, 3), (JRK, 3), (SNP, 3),
                                         (ACCxYAW, 3), (JRKxYAW, 3), (SNPxYAW, 3)])
def test_all_controls_random_states(control, dim):
    from scenarios import Scenario, control_set

    rng = np.random.default_rng(control * 10 + dim)
    yaw = bool(control & 16)
    U = control_set(1.0 if (control & 15) < SNP else 4.0, 3, dim, yaw_rates=(-0.4, 0.0, 0.4) if yaw else None)
    cells, res = 40, 0.2
    sc = Scenario("x", (cells,) * dim, res, tuple(-cells * res / 2 for _ in range(dim)), control, U, n_boxes=8,
                  edge_m=(0.6, 1.8), seed=3, v_max=2.5, a_max=3.0, j_max=6.0, yaw_max=0.9 if yaw else -1.0, wyaw=1.5)
    env = ob.OracleEnv.from_scenario(sc)
    nodes = random_nodes(rng, 700, dim, cells * res / 2, yaw=yaw)
    n = assert_bit_equal(env.expand(nodes, nthreads=4), ob.ref_expand(env, nodes, nthreads=4))
    assert n > 500


def test_potential_gradient_and_region():
    import scenarios as S

    sc = S.scaled(S.cfg4(), 48)
    sc.gradient_weight = 0.3
    rng = np.random.default_rng(1)
    region = (rng.random(48 ** 3) < 0.9).astype(np.uint8)
    env = ob.OracleEnv.from_scenario(sc, region=region)
    nodes = sc.frontier(600, seed=4)
    assert assert_bit_equal(env.expand(nodes, nthreads=4), ob.ref_expand(env, nodes, nthreads=4)) > 1000


def test_unlimited_dynamics_and_large_sample_counts():
    """limits <= 0 are 'unlimited' (env_base.h:380-386); fast nodes give n up to ~200 samples."""
    from scenarios import Scenario, control_set

    sc = Scenario("x", (64, 64, 64), 0.05, (-1.6, -1.6, -1.6), ACC, control_set(1.0, 3, 3), n_boxes=6,
                  edge_m=(0.2, 0.6), seed=5)
    env = ob.OracleEnv.from_scenario(sc)
    rng = np.random.default_rng(2)
    nodes = np.zeros(300, dtype=ob.WAYPOINT_DTYPE)
    nodes["pos"][:, :3] = np.round(rng.uniform(-1.2, 1.2, (300, 3)) / 0.05) * 0.05
    nodes["vel"][:, :3] = rng.integers(-9, 10, (300, 3)) * 1.0
    assert assert_bit_equal(env.expand(nodes), ob.ref_expand(env, nodes)) > 3000


def test_headline_workload_sample():
    import scenarios as S

    for sc, n in ((S.scaled(S.cfg_headline(), 96), 1500), (S.scaled(S.cfg3(), 96), 400), (S.scaled(S.cfg2(), 64), 800)):
        env = ob.OracleEnv.from_scenario(sc)
        nodes = sc.frontier(n, seed=6)
        assert assert_bit_equal(env.expand(nodes, nthreads=4), ob.ref_expand(env, nodes, nthreads=4)) > n
