"""Pins the oracle against the reference (bit for bit) on the input classes of tests/test_fx_paths_gpu.py
before the GPU tests rely on it: starts on cell boundaries next to obstacles, the overflow sites, maps
across and far beyond the 2^17-cell range gate, sample counts around the 128-row table, trajectories
gliding along a boundary plane, successors at the parent's position, and garbage, NaN and signed zeros
in the fields a control does not read.  The reference's results are recorded under
tests/golden/reference (tests/reference_record.py), so these run without oracle/_ref too."""
import numpy as np
import pytest

import oracle_bindings as ob
import test_fx_paths_gpu as fx
from reference_record import same_array

NTHREADS = 8


def assert_bit_equal(case, nodes):
    env = case.oracle()
    o = env.expand(nodes, nthreads=NTHREADS, lattice=False)
    r = ob.ref_expand(env, nodes, nthreads=NTHREADS)
    same_array(o["count"], r["count"], "count")
    o, r = ob.emitted(o), ob.emitted(r)
    same_array(o["action"], r["action"], "action")
    same_array(o["succ"], r["succ"], "succ", bits=True)
    same_array(o["cost"], r["cost"], "cost", bits=True)
    same_array(o["key"], r["key"], "key")
    return o


def test_instantiation_inputs():
    for dim, control, region in ((2, fx.JRK, True), (2, fx.VEL, False), (3, fx.SNP, True), (3, fx.ACC, False)):
        seed = 100 * dim + 10 * control + region
        case = fx.matrix_case(dim, control, region, seed)
        o = assert_bit_equal(case, fx.matrix_nodes(case, seed)[:700])
        assert np.isinf(o["cost"]).any() and np.isfinite(o["cost"]).any()


@pytest.mark.parametrize("res", [0.1, 0.15, 0.3])
def test_boundary_starts(res):
    case, nodes = fx.boundary_case(res, seed=int(res * 1000))
    o = assert_bit_equal(case, nodes[:600])
    assert np.isfinite(o["cost"]).sum() > 1000


def test_boundary_starts_2d():
    case, nodes = fx.boundary_case(0.15, seed=3, dim=2, n=2003)
    assert_bit_equal(case, nodes[:1000])


@pytest.mark.parametrize("with_region", [True, False])
def test_overflow_sites(with_region):
    case, nodes, site, holed, away = fx.overflow_case(with_region, n=2000)
    o = assert_bit_equal(case, nodes)
    assert np.isinf(o["cost"]).any() and np.isfinite(o["cost"]).any()


def test_range_gate_inputs():
    case, nodes = fx.gate_case(0.15, (-1, 1, -1), seed=22)
    gq = fx.gate_quantity(nodes, case)
    assert (gq < fx.FX_RANGE).any() and (gq > fx.FX_RANGE).any()
    assert_bit_equal(case, nodes[::2])


@pytest.mark.parametrize("far_log2,res", [(24, 0.05), (27, 0.05)])
def test_far_map_inputs(far_log2, res):
    case, nodes = fx.gate_case(res, (1, -1, -1) if far_log2 % 2 else (-1, 1, 1), seed=far_log2, far=2.0 ** far_log2)
    o = assert_bit_equal(case, nodes[::2])
    assert np.isfinite(o["cost"]).sum() > 1000


def test_sample_table_edge_inputs():
    case, nodes = fx.beyond_case()
    assert_bit_equal(case, nodes[::3])


def test_boundary_plane_glide_inputs():
    case, nodes, _ = fx.full_case()
    assert_bit_equal(case, nodes[::3])


def test_same_position_inputs():
    case, nodes, kind = fx.same_case()
    o = assert_bit_equal(case, nodes[:400])
    assert np.isfinite(o["cost"]).any()


@pytest.mark.parametrize("dim,control", [(2, fx.VEL), (2, fx.ACC), (3, fx.ACC), (3, fx.JRK), (2, fx.SNP)])
def test_ignored_fields_and_signed_zeros(dim, control):
    case, nodes = fx.contract_case(dim, control, seed=10 * dim + control)
    assert_bit_equal(case, nodes[:600])
