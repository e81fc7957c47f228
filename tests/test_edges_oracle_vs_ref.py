"""Pins the oracle's stored-edge queries against the REFERENCE's own env_map::is_free(pr) and
calculate_intrinsic_cost(pr) (oracle/_ref, unmodified headers): bit-for-bit on the CPU."""
import numpy as np
import pytest

import oracle_bindings as ob
from reference_record import same_array

VEL, ACC, JRK, SNP, ACCxYAW = 0x01, 0x03, 0x07, 0x0F, 0x13


def edges_of(env, nodes, rng, extra=400):
    """Stored edges as LPA* keeps them: every emitted successor (finite AND +inf) of `nodes`,
    plus random (node, action) pairs — including ones get_succ would have rejected."""
    o = env.expand(nodes, nthreads=4)
    nU = o["nU"]
    valid = (np.arange(nU)[None, :] < o["count"][:, None]).reshape(-1)
    parent_idx = np.repeat(np.arange(nodes.size), nU)[valid]
    parents = np.concatenate([nodes[parent_idx], nodes[rng.integers(0, nodes.size, extra)]])
    actions = np.concatenate([o["action"][valid], rng.integers(0, nU, extra).astype(np.int32)])
    return parents, actions, o["cost"][valid]


@pytest.mark.parametrize("control,dim", [(VEL, 2), (ACC, 2), (JRK, 2), (SNP, 2), (ACCxYAW, 2), (VEL, 3), (ACC, 3),
                                         (JRK, 3), (SNP, 3)])
def test_is_free_and_cost_match_reference(control, dim):
    from scenarios import Scenario, control_set
    from test_oracle_vs_ref import random_nodes

    rng = np.random.default_rng(100 + control * 10 + dim)
    yaw = bool(control & 16)
    U = control_set(1.0 if (control & 15) < SNP else 4.0, 3, dim, yaw_rates=(-0.4, 0.0, 0.4) if yaw else None)
    cells, res = 40, 0.2
    sc = Scenario("x", (cells,) * dim, res, tuple(-cells * res / 2 for _ in range(dim)), control, U, n_boxes=8,
                  edge_m=(0.6, 1.8), seed=3, v_max=2.5, a_max=3.0, j_max=6.0, yaw_max=0.9 if yaw else -1.0, wyaw=1.5)
    region = (rng.random(cells ** dim) < 0.97).astype(np.uint8) if dim == 2 else None
    env = ob.OracleEnv.from_scenario(sc, region=region)
    nodes = random_nodes(rng, 300, dim, cells * res / 2, yaw=yaw)
    parents, actions, _ = edges_of(env, nodes, rng)
    fo, co = env.edges_is_free(parents, actions)
    fr, cr = ob.ref_edges_is_free(env, parents, actions)
    same_array(fo, fr, "free")
    same_array(co, cr, "cost", bits=True)
    assert 0 < fo.sum() < fo.size


def test_empty_map_edges_free_unless_they_leave_the_map():
    """On an empty map an edge is free iff all n+1 samples stay inside; is_free also samples t = T
    exactly (Primitive::sample), which traverse_primitive's running sum may not."""
    from scenarios import control_set

    grid = np.zeros(32 ** 3, dtype=np.int8)
    env = ob.OracleEnv(3, ACC, control_set(1.0, 3, 3), grid, (32, 32, 32), (-4.0, -4.0, -4.0), 0.25, T=1.0, w=10.0,
                       v_max=3.0)
    rng = np.random.default_rng(0)
    nodes = np.zeros(200, dtype=ob.WAYPOINT_DTYPE)
    nodes["pos"][:, :3] = np.round(rng.uniform(-3.9, 3.9, (200, 3)) / 0.25) * 0.25
    nodes["vel"][:, :3] = rng.integers(-2, 3, (200, 3)) * 1.0
    parents, actions, cost = edges_of(env, nodes, rng, extra=0)
    free, _ = env.edges_is_free(parents, actions)
    fr, _ = ob.ref_edges_is_free(env, parents, actions)
    same_array(free, fr, "free")
    end = parents["pos"][:, :3] + parents["vel"][:, :3] + 0.5 * env.U[actions]
    leaves = np.any((end < -4.0) | (end >= 4.0), axis=1)
    assert not np.any(free[leaves])          # the t = T sample is outside
    assert free.sum() > 0 and leaves.sum() > 0
