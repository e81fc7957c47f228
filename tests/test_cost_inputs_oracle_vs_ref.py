"""Pins the oracle against the reference (bit for bit) on the input classes of tests/test_cost_paths_gpu.py
before the GPU tests rely on it: int8 potential values of every class (negative, 1..99, 100..127) over grids
that disagree with them, the gradient term in 2-D and 3-D, planar speeds straddling the 1e-5 of the yaw
term, yaws at +-pi, sample loops past the 128-row table with potential and yaw, and is_free(pr) with a
potential map installed.  The reference's results are recorded under tests/golden/reference
(tests/reference_record.py), so these run without oracle/_ref too."""
import numpy as np
import pytest

import oracle_bindings as ob
import test_cost_paths_gpu as cp
import test_fx_paths_gpu as fx
from reference_record import same_array
from test_fx_inputs_oracle_vs_ref import assert_bit_equal

NTHREADS = 8


@pytest.mark.parametrize("grid_kind", ["free", "occupied", "unknown"])
@pytest.mark.parametrize("dim,control", [(3, cp.ACC), (2, cp.JRK)])
def test_potential_classes(dim, control, grid_kind):
    nodes = cp.pclass_nodes(cp.pclass_case(dim, control, "free"), n=120)
    for value in (-128, -1, 0, 1, 50, 99, 100, 101, 127):
        for gw in ((0.0, 0.3) if value <= 0 else (0.0,)):
            o = assert_bit_equal(cp.pclass_case(dim, control, grid_kind, value, gw=gw), nodes)
            assert np.isinf(o["cost"]).any() == (value >= 100)


def test_uniform_random_int8_potential():
    rng = np.random.default_rng(41)
    m = cp.PCLASS_MAP[3]
    size = int(np.prod(m["mdim"]))
    case = cp.Case(3, cp.ACC, fx.product_set(*[fx.u_values(cp.ACC)] * 3), m["mdim"], m["origin"], 0.25,
                   grid=cp.random_grid(rng, size), potential=rng.integers(-128, 128, size).astype(np.int8), pw=0.21,
                   v_max=2.5)
    o = assert_bit_equal(case, cp.random_nodes(rng, 300, case, 8, 24))
    assert np.isinf(o["cost"]).any() and np.isfinite(o["cost"]).any()


@pytest.mark.parametrize("dim,control,config", [(3, cp.ACC, "P"), (2, cp.SNP, "P"), (3, cp.JRK, "PG"),
                                                (2, cp.ACC, "PG"), (3, cp.VEL, "PG"), (2, cp.VEL, "PR"),
                                                (3, cp.ACC | cp.YAW, "Y"), (2, cp.JRK | cp.YAW, "Y0")])
def test_matrix_inputs(dim, control, config):
    """Potential over an independent grid (occupied, unknown and free voxels under every potential class),
    the gradient term in 2-D and 3-D, the region, and yaw plans."""
    for loop in cp.LOOPS:
        case = cp.matrix_case(dim, control, config, loop, seed=7 * dim + control)
        o = assert_bit_equal(case, cp.matrix_nodes(case, 7 * dim + control)[:150])
        assert np.isfinite(o["cost"]).any()


def test_yaw_norm_straddle_inputs():
    case = cp.yaw_edge_case(3)
    v = cp.straddle_vectors()
    rng = np.random.default_rng(5)
    nodes = cp.random_nodes(rng, v.shape[0] * 2, case, 28, 36)
    nodes["vel"][:, :2] = np.repeat(v, 2, axis=0)
    nodes["yaw"] = np.arctan2(nodes["vel"][:, 1], nodes["vel"][:, 0]) + np.pi / 2
    assert_bit_equal(case, nodes)


def test_yaw_at_pi_inputs():
    pi = np.pi
    yaws = np.array([pi, np.nextafter(pi, 4), np.nextafter(pi, 3), -pi, np.nextafter(-pi, -4), np.nextafter(-pi, -3)])
    for yaw_max in (-1.0, 0.9):
        case = cp.yaw_edge_case(2)
        case.yaw_max = yaw_max
        nodes = cp.random_nodes(np.random.default_rng(13), yaws.size * 20, case, 28, 36)
        nodes["yaw"] = np.repeat(yaws, 20)
        assert_bit_equal(case, nodes)


@pytest.mark.parametrize("yaw", [False, True])
def test_past_the_sample_table_inputs(yaw):
    case, nodes = cp.beyond_cost_case(yaw)
    o = assert_bit_equal(case, nodes[::5])
    assert np.isfinite(o["cost"]).any()


@pytest.mark.parametrize("dim,control", [(3, cp.ACC), (2, cp.ACC | cp.YAW)])
def test_is_free_with_a_potential(dim, control):
    """is_free(pr) reads the grid and the region only: the reference's answer with a potential that
    disagrees with the grid installed."""
    from test_edges_oracle_vs_ref import edges_of

    rng = np.random.default_rng(3 + dim)
    case = cp.edges_case(dim, control, rng)
    orc = case.oracle()
    parents, actions, _ = edges_of(orc, cp.matrix_nodes(case, 23)[:100], rng, extra=200)
    fo, co = orc.edges_is_free(parents, actions)
    fr, cr = ob.ref_edges_is_free(orc, parents, actions)
    same_array(fo, fr, "free")
    same_array(co, cr, "cost", bits=True)
    assert 0 < fo.sum() < fo.size
