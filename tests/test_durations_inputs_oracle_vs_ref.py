"""Pins the oracle and the host planner against the reference (bit for bit) at primitive durations T != 1, on the
input classes of tests/test_durations_gpu.py, before the GPU tests rely on them: the instantiation matrix, the
ceiling, last-sample and stationary-point edges, the yaw verdicts, sample counts past the 128-row table and
clamped at 5, stored edges and searches.  Two restatements independent of both: the sample loop in Python
doubles, which must run n + 1 times for some n each input reaches, and the end states and J in exact rationals.
The reference's results are recorded under tests/golden/reference (tests/reference_record.py), so these run
without oracle/_ref too."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

import oracle_bindings as ob
import test_cost_paths_gpu as cp
import test_durations_gpu as du
import test_fx_paths_gpu as fx
from test_fx_inputs_oracle_vs_ref import assert_bit_equal
from test_search_inputs_oracle_vs_ref import same_as_reference

ALL_T = du.DURATIONS + (du.T_LONG, du.T_SHORT)


# ---- the restatements ---------------------------------------------------------------------------------------
def test_sample_loop_runs_n_plus_one_times_at_every_duration():
    """`for (t = 0; t < T; t += T/n)` in Python doubles equals the oracle's loop, and at each non-dyadic T it runs
    n + 1 times for some n in the range the inputs reach (5 to 60, and past 128 at T_LONG)."""
    for T in ALL_T:
        for n in range(1, 200):
            assert du.loop_count(T, n) == ob.lib().orc_sample_count(T, n), (T, n)
    for T in (0.7, 1.3, du.T_LONG):
        extra = du.n_plus_one(T, 5, 60)
        print(f"T={T}: n in [5, 60] with n + 1 samples: {extra}")
        assert len(extra) >= 3, T
    assert du.n_plus_one(du.T_LONG, du.N_TABLE + 1, 160)
    # the clamp: n = 5 at T_SHORT, whose loop runs 5 or 6 times
    assert du.sample_n(6.0, du.T_SHORT, 0.15) == 5


@pytest.mark.parametrize("T", du.DURATIONS)
@pytest.mark.parametrize("control", [fx.VEL, fx.ACC, fx.JRK, fx.SNP], ids=["vel", "acc", "jrk", "snp"])
def test_oracle_end_states_and_J_are_exact(control, T):
    """The oracle's successors and the costs of its free primitives (occupancy planning: J + w*T) within
    EXACT_RTOL of exact rational arithmetic: the Taylor polynomial at T with the control as top derivative."""
    case, nodes = du.matrix_case(3, control, T, False)
    nodes = nodes[:300]
    o = case.oracle().expand(nodes, nthreads=8)
    from motion_primitive_library_b200.env import Expansion

    g = Expansion(case.nU, o["count"], o["succ"], o["cost"], o["action"], o["key"], None)
    assert du.check_exact(case, nodes, g, n_check=600) >= 400


def test_exact_restatement_sees_a_wrong_power_of_T():
    """The bound of check_exact rejects a successor computed with T^3 in place of T^4 (the SNP snap term)."""
    case, nodes = du.matrix_case(3, fx.SNP, 1.3, False)
    node, u = nodes[0], case.U[0]
    st, sc, _ = du.exact_end_state(node, u, fx.SNP, 3, 1.3)
    wrong = st["pos"][0] - Fraction(float(u[0])) * (Fraction(1.3) ** 4 - Fraction(1.3) ** 3) / 24
    assert abs(wrong - st["pos"][0]) > du.EXACT_RTOL * sc["pos"][0]


# ---- the oracle against the reference -----------------------------------------------------------------------
@pytest.mark.parametrize("T", ALL_T)
def test_instantiation_inputs(T):
    for dim, control in ((2, fx.JRK), (3, fx.SNP), (2, fx.VEL), (3, fx.ACC)):
        case, nodes = du.matrix_case(dim, control, T, T in (0.7, 2.0))
        o = assert_bit_equal(case, nodes[:500])
        assert np.isfinite(o["cost"]).any()


@pytest.mark.parametrize("dim,control,config,T", du.COST_MATRIX,
                         ids=[f"{cp.matrix_id((d, c, cfg, 'long'))}-T{T}" for d, c, cfg, T in du.COST_MATRIX])
def test_cost_inputs(dim, control, config, T):
    seed = 7 * dim + control + int(T * 10)
    case = du.at_duration(cp.matrix_case(dim, control, config, "long", seed), T)
    assert_bit_equal(case, cp.matrix_nodes(case, seed)[:150])


@pytest.mark.parametrize("yaw", [False, True])
def test_cost_past_the_table_inputs(yaw):
    case, nodes = cp.beyond_cost_case(yaw, seed=73)
    case.T = 1.3
    assert_bit_equal(case, nodes[::4])


@pytest.mark.parametrize("T", [0.7, 1.3])
def test_ceiling_inputs(T):
    case, nodes = du.ceiling_case(T, seed=int(T * 10))
    o = case.oracle().expand(nodes, nthreads=8)
    up, down, fp_only = du.ceiling_classes(case, nodes, o)
    print(f"T={T}: decimal integer with FP64 above {up}, below {down}; FP64 integer only {fp_only}")
    assert (down if T == 0.7 else up) > 100
    assert_bit_equal(case, nodes[::3])


@pytest.mark.parametrize("T", [0.7, 1.3, 2.0])
def test_last_sample_inputs(T):
    case, nodes, blocked = du.last_sample_case(T, seed=int(T * 10))
    assert blocked > 300
    assert_bit_equal(case, nodes[::3])


@pytest.mark.parametrize("control,T", [(fx.JRK, 2.0), (fx.JRK, 0.7), (fx.SNP, 1.3), (fx.SNP, 0.5)],
                         ids=["jrk-T2.0", "jrk-T0.7", "snp-T1.3", "snp-T0.5"])
def test_stationary_point_inputs(control, T):
    case, nodes = du.roots_case(control, T, seed=int(T * 10) + control)
    o = assert_bit_equal(case, nodes[::3])
    decided = du.root_decides(case, nodes)
    print(f"{du.NAME[control]} T={T}: {decided} primitives decided by a stationary point between 1 and T")
    assert decided > 200 and np.asarray(o["count"]).sum() > 0


@pytest.mark.parametrize("control,T", [(fx.VEL | cp.YAW, 2.0), (fx.ACC | cp.YAW, 0.5)], ids=["velyaw-T2.0", "accyaw-T0.5"])
def test_yaw_verdict_inputs(control, T):
    case, nodes = du.yaw_case(control, T, seed=int(T * 10) + control)
    assert du.yaw_verdicts_differ(case, nodes) > 300
    assert_bit_equal(case, nodes[::3])


@pytest.mark.parametrize("T", [du.T_LONG, du.T_SHORT])
def test_table_and_clamp_inputs(T):
    from scenarios import box_map

    res = 0.1 if T == du.T_LONG else 0.15
    mdim, origin = (200, 72, 56), (-9.9731, -3.6113, -2.8117)
    grid = box_map(mdim, res, origin, n_boxes=40, edge_m=(0.3, 1.0), seed=11)
    case = fx.Case(3, fx.ACC, fx.product_set(*[fx.u_values(fx.ACC)] * 3), mdim, origin, res, grid=grid, T=T)
    rng = np.random.default_rng(12)
    nodes = fx.random_nodes(rng, 1001, case, (60, 20, 16), (140, 52, 40), centred=True)
    nodes["vel"][:, 0] = rng.choice([-5.5, -4.0, -2.5, 0.5, 2.5, 4.0, 5.5], nodes.size)
    assert_bit_equal(case, nodes[::3])


@pytest.mark.parametrize("T", [0.7, 2.0])
@pytest.mark.parametrize("dim,control", [(3, fx.ACC), (2, fx.JRK), (3, fx.SNP | cp.YAW)],
                         ids=["3d-acc", "2d-jrk", "3d-snpyaw"])
def test_edges_is_free_inputs(dim, control, T):
    from reference_record import same_array

    orc, parents, actions = du.edges_case(dim, control, T)
    fo, co = orc.edges_is_free(parents, actions)
    fr, cr = ob.ref_edges_is_free(orc, parents, actions)
    same_array(fo, fr, "free")
    same_array(co, cr, "cost", bits=True)
    assert 0 < fo.sum() < fo.size


def walk(orc, parent, u):
    """getLinkedNodes' walk (map_planner.cpp:135-151) of a 3-D ACC edge in Python doubles: n = ceil(max_v*T/res)
    with no lower bound, n + 1 samples at i*(T/n), p = u/2 t t + v t + p0, one entry per change of getIndex."""
    e = orc.e
    T, res = e.T, e.res
    max_v = max(max(abs(float(parent["vel"][k])), abs(float(u[k]) * T + float(parent["vel"][k]))) for k in range(3))
    n = math.ceil(max_v * T / res)
    dt = T / n
    cells, prev = [], -1
    for i in range(n + 1):
        t = i * dt
        pn = [int(fx.ref_cell(float(u[k]) / 2 * t * t + float(parent["vel"][k]) * t + float(parent["pos"][k]),
                              e.origin[k], res)) for k in range(3)]
        idx = pn[0] + e.mdim[0] * pn[1] + e.mdim[0] * e.mdim[1] * pn[2]
        if idx != prev:
            cells.append(pn)
            prev = idx
    return cells


@pytest.mark.parametrize("T", [0.7, 2.0])
def test_edges_cells_inputs(T):
    """The oracle's cell walk of 3-D ACC edges against `walk`."""
    orc, parents, actions = du.edges_case(3, fx.ACC, T)
    moving = np.abs(parents["vel"][:, :3]).sum(1) + np.abs(orc.U[actions]).sum(1) > 0
    parents, actions = parents[moving][:400], actions[moving][:400]
    off, cells = orc.edges_cells(parents, actions)
    for i in range(parents.size):
        assert cells[off[i]:off[i + 1]].tolist() == walk(orc, parents[i], orc.U[actions[i]]), i


@pytest.mark.parametrize("dim,control,T", du.SEARCH_CASES, ids=[f"{d}d-{du.NAME[c]}-T{T}" for d, c, T in du.SEARCH_CASES])
def test_search_inputs(dim, control, T):
    sc, S, G = du.search_case(dim, control, T)
    same_as_reference(sc, S, G)
