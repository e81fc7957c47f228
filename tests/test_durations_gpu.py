"""The expansion kernels, the stored-edge queries and the device searches at primitive durations T != 1.

Every primitive lasts T (set_dt).  At T = 1, T, T*T and T*T*T*T are equal, so a wrong power of T, a dropped
factor of T or a literal 1.0 where T belongs leaves every result unchanged.  The cases here run the kernels at
T in DURATIONS, at a T whose sample counts pass the 128-row sample-time table (T_LONG) and at a T whose n clamps
at 5 (T_SHORT), against the CPU oracle: successors and keys bit for bit, costs exact (1e-12 relative where a yaw
term is summed).  tests/test_durations_inputs_oracle_vs_ref.py pins the oracle against the reference on the same
inputs and checks it against the exact rationals of `exact_end_state`.

  matrix      expand_fxn_kernel / expand_fx_kernel / register / literal on every <dim, order>, map and region;
              the cost-summing kernels (potential, gradient, yaw), the dealing kernel over several rounds and
              past the table
  ceiling     starts whose max_v*T/res is an integer in exact arithmetic but not in FP64, and the reverse
  last        sample loops that run n + 1 times (t < T on a running sum of T/n), the last sample in an obstacle;
              sample counts from the statistics against the oracle's
  roots       max_vel / max_acc stationary points between 1 and T that decide the v_max / a_max verdict; yaw
              controls whose yaw_max verdict at T differs from the one at 1
  plans       the unchecked fixed-point loop at T = 1 turning into the checked one at T = 2; primitives past the
              table taking the literal loop; starts at the faces of the map
  edges       mplx_edges_is_free / mplx_edges_cells
  searches    mplx_plan_batch, _cost_terms, _grow and the recorded trajectories against the host planner
  live        T changed on a context that already holds a map, a region and tables
  exact       emitted successors and free costs against exact rational arithmetic
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np
import pytest

import oracle_bindings as ob
import test_cost_paths_gpu as cp
import test_fx_paths_gpu as fx
from parity import assert_expansion_equal

pytestmark = pytest.mark.gpu

VEL, ACC, JRK, SNP, YAW = fx.VEL, fx.ACC, fx.JRK, fx.SNP, cp.YAW
NAME = {VEL: "vel", ACC: "acc", JRK: "jrk", SNP: "snp"}
DURATIONS = (0.5, 0.7, 1.3, 2.0)
T_LONG = 2.6    # with res 0.1 and speeds up to 6 m/s: n up to 156, past the 128-row table
T_SHORT = 0.05  # with res 0.15 and speeds up to 3 m/s: ceil(max_v*T/res) <= 1, n = 5
N_TABLE = fx.N_TABLE
EXACT_RTOL = 1e-13
NTHREADS = fx.NTHREADS


# ---- restatements ---------------------------------------------------------------------------------------
def loop_count(T, n):
    """Samples of the reference's loop `for (t = 0; t < T; t += T/n)` (env_map.h:90-132), in doubles: n or n + 1."""
    k, t, dt = 0, 0.0, T / n
    while t < T:
        k += 1
        t += dt
    return k


def sample_n(max_v, T, res):
    """n = max(5, ceil(max_v*T/res)) in doubles, as traverse_primitive computes it."""
    return max(5, math.ceil(max_v * T / res))


def n_plus_one(T, lo, hi):
    """The n in [lo, hi] whose loop runs n + 1 times at T."""
    return [n for n in range(lo, hi + 1) if loop_count(T, n) == n + 1]


FACT = (1, 1, 2, 6, 24)


def exact_end_state(node, u, control, dim, T):
    """(pos, vel, acc, jrk) at t = T as Fractions: the Taylor polynomial of order ORDER[control] with the control
    as its top derivative, and J = sum over axes of u^2 T.  Also the sum of the terms' magnitudes per field, the
    scale of the bound."""
    order = fx.ORDER[control & 15]
    T = Fraction(T)
    out = {f: [] for f in fx.FIELDS}
    scale = {f: [] for f in fx.FIELDS}
    for k in range(dim):
        d = [Fraction(float(node[f][k])) for f in fx.FIELDS[:order]] + [Fraction(float(u[k]))]
        for i, f in enumerate(fx.FIELDS):
            terms = [d[i + m] * T ** m / FACT[m] for m in range(order + 1 - i)] if i <= order else []
            out[f].append(sum(terms, Fraction(0)))
            scale[f].append(sum((abs(x) for x in terms), Fraction(0)))
    J = sum((Fraction(float(u[k])) ** 2 * T for k in range(dim)), Fraction(0))
    return out, scale, J


def check_exact(case, nodes, g, n_check=400, seed=0):
    """Emitted successors (pos/vel/acc/jrk, t) and the costs of free primitives, J + w*T, against exact rationals
    within EXACT_RTOL of the sum of the terms' magnitudes.  Returns the number of slots checked."""
    nU = case.nU
    em = np.flatnonzero(np.arange(nU)[None, :] < g.count[:, None])
    rng = np.random.default_rng(seed)
    pick = rng.choice(em, min(n_check, em.size), replace=False)
    order = fx.ORDER[case.control & 15]
    checked = 0
    for s in pick:
        node = nodes[s // nU]
        u = case.U[g.action[s]]
        st, sc, J = exact_end_state(node, u, case.control, case.dim, case.T)
        for i, f in enumerate(fx.FIELDS[:order]):
            for k in range(case.dim):
                got = Fraction(float(g.succ[s][f][k]))
                assert abs(got - st[f][k]) <= EXACT_RTOL * max(sc[f][k], Fraction(1, 1 << 40)), (s, f, k)
        assert float(g.succ[s]["t"]) == float(node["t"]) + case.T
        c = float(g.cost[s])
        if np.isfinite(c) and getattr(case, "potential", None) is None and not case.control & YAW:
            want = J + Fraction(case.w) * Fraction(case.T)
            assert abs(Fraction(c) - want) <= EXACT_RTOL * max(want, Fraction(1)), (s, c, float(want))
        checked += 1
    return checked


# ---- 1. instantiation matrix ----------------------------------------------------------------------------
def at_duration(case, T):
    """The case at duration T; for T > 1 the limits grow with T (v, a by T^2, j by T), so that a similar share
    of the primitives stays valid."""
    case.T = T
    if T > 1:
        case.v_max, case.a_max, case.j_max = case.v_max * T * T, case.a_max * T * T, case.j_max * T
    return case


def matrix_case(dim, control, T, with_region):
    seed = 100 * dim + 10 * control + with_region + int(T * 10)
    case = at_duration(fx.matrix_case(dim, control, with_region, seed), T)
    return case, fx.matrix_nodes(case, seed)


MATRIX = [(d, c, T) for d in (2, 3) for c in (VEL, ACC, JRK, SNP) for T in DURATIONS]


@pytest.mark.parametrize("dim,control,T", MATRIX, ids=[f"{d}d-{NAME[c]}-T{T}" for d, c, T in MATRIX])
def test_fixed_point_instantiations(dim, control, T):
    """Kernels 1, 2, 5 and 0 (expand_fxn_kernel + fx_resolve_kernel, from the launch count), map or region;
    kernels 0 and 5 also against exact rationals."""
    with_region = T in (0.7, 2.0)
    case, nodes = matrix_case(dim, control, T, with_region)
    orc, env = fx.run_kernels(case, nodes)
    st = fx.emitted_mask(orc)
    assert st.sum() > nodes.size and np.isinf(orc["cost"][st]).any() and np.isfinite(orc["cost"][st]).any()
    for k in (0, 5):
        env.set_kernel(k)
        assert check_exact(case, nodes, env.expand(nodes, want=fx.WANT), n_check=150, seed=k) > 0


COST_MATRIX = [(d, c, cfg, T) for T in (0.7, 2.0) for d, c, cfg in ((3, ACC, "P"), (2, JRK, "PG"), (2, SNP, "PR"),
                                                                    (2, VEL | YAW, "Y"), (3, ACC | YAW, "Y"),
                                                                    (3, JRK | YAW, "Y0"))]


@pytest.mark.parametrize("dim,control,config,T", COST_MATRIX,
                         ids=[f"{cp.matrix_id((d, c, cfg, 'long'))}-T{T}" for d, c, cfg, T in COST_MATRIX])
def test_cost_instantiations(dim, control, config, T):
    seed = 7 * dim + control + int(T * 10)
    case = at_duration(cp.matrix_case(dim, control, config, "long", seed), T)
    nodes = cp.matrix_nodes(case, seed)
    orc, _ = cp.run_cost_kernels(case, nodes, label=f"T={T} {config}")
    st = fx.emitted_mask(orc)
    assert st.sum() > nodes.size and np.isfinite(orc["cost"][st]).any()


@pytest.mark.parametrize("mix,T", [("mixed", 0.7), ("mixed-vel", 2.0)])
def test_multi_round_dealing(mix, T):
    sms = cp.sm_count()
    case = cp.deal_case(mix, seed=90 + int(T * 10))
    case.T = T
    npb = cp.THREADS // case.nU
    n = cp.deal_batch(2, sms, npb)
    nodes = cp.deal_nodes(case, n, mix, seed=95)
    rounds = cp.launches_of(case, 4, n, False, sms)[1]
    assert rounds >= 2
    orc = cp.check_deal(case, nodes, rounds, cp.NO_SUCC)
    em = fx.emitted_mask(orc)
    assert em.sum() > n and np.isfinite(orc["cost"][em]).any() and np.isinf(orc["cost"][em]).any()


@pytest.mark.parametrize("yaw", [False, True], ids=["potential", "potential-gradient-yaw"])
def test_cost_kernels_past_the_table(yaw):
    """The dealing, register and literal kernels with primitives on both sides of the 128-row table at T = 1.3."""
    case, nodes = cp.beyond_cost_case(yaw, seed=73)
    case.T = 1.3
    orc, _ = cp.run_cost_kernels(case, nodes, kernels=(1, 2, 4), label=f"T=1.3 past the table yaw={yaw}")
    em = fx.emitted_mask(orc) & ~fx.same_mask(orc, nodes, 3)
    n = fx.sample_counts(cp.position_part(case), nodes, orc)[em]
    assert (n > N_TABLE).sum() > 200 and (n <= N_TABLE).sum() > 200
    assert np.isfinite(orc["cost"][em][n > N_TABLE]).sum() > 50


# ---- 2. ceiling edges -----------------------------------------------------------------------------------
CEIL_RES = {0.7: 0.1, 1.3: 0.15}  # FP64's max_v*T/res falls below the exact integer at 0.7, above it at 1.3


def ceiling_case(T, seed=3, n=1201):
    """3-D ACC starts whose x velocity is a two-decimal multiple of 0.05 m/s and y, z velocities 0: for the
    primitives that keep x in front, max_v*T/res is an integer in exact decimal arithmetic that FP64 misses."""
    from scenarios import box_map

    res = CEIL_RES[T]
    mdim, origin = (80, 64, 48), (-3.9713, -3.1117, -2.3791)
    grid = box_map(mdim, res, origin, n_boxes=14, edge_m=(3 * res, 9 * res), seed=seed)
    case = fx.Case(3, ACC, fx.product_set(*[fx.u_values(ACC)] * 3), mdim, origin, res, grid=grid, T=T)
    rng = np.random.default_rng(seed)
    nodes = fx.random_nodes(rng, n, case, (20, 16, 12), (60, 48, 36), centred=True)
    nodes["vel"][:, 0] = np.round(rng.integers(-60, 61, n) * 0.05, 2)
    nodes["vel"][:, 1:3] = 0.0
    return case, nodes


def ceiling_classes(case, nodes, orc):
    """Per emitted slot: q = fl(fl(max_v*T)/res) against the decimal value of max_v*T/res.  `up`: the decimal
    value is an integer and q is above it (ceil gives one more); `down`: integer, q below; `fp_only`: q an
    integer, the decimal value not."""
    nU = case.nU
    em = fx.emitted_mask(orc)
    parent = np.repeat(np.arange(nodes.size), nU)[em]
    u = case.U[orc["action"][em]]
    v0 = nodes["vel"][parent]
    up = down = fp_only = 0
    for i in range(parent.size):
        mv = max(max(abs(float(v0[i, k])), abs(float(v0[i, k]) + float(u[i, k]) * case.T)) for k in range(3))
        q = mv * case.T / case.res
        dec = Fraction(repr(mv)) * Fraction(repr(case.T)) / Fraction(repr(case.res))
        if dec.denominator == 1:
            up += q > dec
            down += q < dec
        elif q == math.floor(q):
            fp_only += 1
    return up, down, fp_only


@pytest.mark.parametrize("T", [0.7, 1.3])
def test_ceiling_edges(T):
    case, nodes = ceiling_case(T, seed=int(T * 10))
    orc, env = fx.run_kernels(case, nodes)
    up, down, fp_only = ceiling_classes(case, nodes, orc)
    print(f"[ceiling] T={T}: decimal integer, FP64 above {up}, below {down}; FP64 integer only {fp_only}")
    assert (down if T == 0.7 else up) > 100
    t = case.oracle().timed(nodes, nthreads=NTHREADS)
    env.enable_stats(True)
    for k in (2, 5, 0):
        env.set_kernel(k)
        env.expand(nodes, want=fx.NO_SUCC)
        assert env.last_stats() == (t["samples"], t["successors"]), k


# ---- 3. the last sample -------------------------------------------------------------------------------------
LAST_RES = 0.15


def last_sample_case(T, seed=5, n=1201):
    """3-D ACC nodes at cell centres moving along x (y, z at rest) with |v| chosen so that the u = 0 primitive's
    loop runs n + 1 times; the cell of its last sample (t just below T, position p0 + v*T up to rounding) is
    occupied when no earlier sample of that primitive lies in it."""
    mdim, origin = (120, 40, 40), (-8.9917, -3.0113, -2.9771)
    case = fx.Case(3, ACC, fx.product_set(*[fx.u_values(ACC)] * 3), mdim, origin, LAST_RES, T=T)
    rng = np.random.default_rng(seed)
    speeds = [v for v in np.arange(0.05, 3.0, 0.05) if loop_count(T, sample_n(v, T, LAST_RES)) ==
              sample_n(v, T, LAST_RES) + 1]
    assert len(speeds) > 5, (T, speeds)
    nodes = np.zeros(n, dtype=ob.WAYPOINT_DTYPE)
    o = np.asarray(origin)
    cells = np.stack([rng.integers(30, 90, n), rng.integers(8, 32, n), rng.integers(8, 32, n)], 1)
    nodes["pos"][:, :3] = o + (cells + 0.5) * LAST_RES
    nodes["vel"][:, 0] = rng.choice(speeds, n) * rng.choice([-1.0, 1.0], n)
    blocked = 0
    for i in range(n):
        p0, v = nodes["pos"][i, :3].copy(), float(nodes["vel"][i, 0])
        nn = sample_n(abs(v), T, LAST_RES)
        t, dt, xs = 0.0, T / nn, []
        while t < T:
            xs.append(int(fx.ref_cell(v * t + p0[0], o[0], LAST_RES)))
            t += dt
        if xs[-1] not in xs[:-1] and i % 3:
            c = (xs[-1], cells[i, 1], cells[i, 2])
            case.grid[case.index(c)] = 100
            blocked += 1
    return case, nodes, blocked


@pytest.mark.parametrize("T", [0.7, 1.3, 2.0])
def test_last_sample_in_an_obstacle(T):
    case, nodes, blocked = last_sample_case(T, seed=int(T * 10))
    assert blocked > 300
    orc, env = fx.run_kernels(case, nodes)
    # the u = 0 primitive of a node with a blocked last cell: inf, though its first n samples are free
    zero = int(np.flatnonzero((case.U == 0).all(1))[0])
    nU = case.nU
    em = fx.emitted_mask(orc).reshape(-1, nU)
    act = orc["action"].reshape(-1, nU)
    cost = orc["cost"].reshape(-1, nU)
    inf_zero = sum(bool(np.isinf(cost[i][em[i] & (act[i] == zero)]).any()) for i in range(nodes.size))
    assert inf_zero > 200, inf_zero
    t = case.oracle().timed(nodes, nthreads=NTHREADS)
    env.enable_stats(True)
    for k in (2, 4, 0):
        env.set_kernel(k)
        env.expand(nodes, want=fx.NO_SUCC)
        assert env.last_stats() == (t["samples"], t["successors"]), k


# ---- 4. stationary points between 1 and T -------------------------------------------------------------
def roots_case(control, T, seed=7, n=1001):
    """JRK (SNP) nodes whose x velocity (acceleration) under the control u = -s*um on x and 0 on y, z is
    stationary at r between 1 and T (JRK: a0 + u r = 0; SNP: j0 + u r = 0) with |v(r)| = lim + d/2 and the
    largest value at 0 and T at most lim - d/2, d = um/2 (T - r)^2: the v_max (a_max) verdict is the root's.  A
    quarter of the nodes have |v(r)| = lim - d/2 instead (valid either way).  y and z are at rest."""
    mdim, origin, res = (64, 64, 48), (-4.7913, -4.8117, -3.5971), 0.15
    U = fx.product_set(*[fx.u_values(control)] * 3)
    um = fx.u_values(control)[2]
    lim = 2.5 if T > 1 else 1.4
    case = fx.Case(3, control, U, mdim, origin, res, T=T, v_max=lim if control == JRK else -1.0,
                   a_max=lim if control == SNP else -1.0)
    rng = np.random.default_rng(seed)
    nodes = fx.random_nodes(rng, n, case, 16, np.asarray(mdim) - 16, centred=True)
    for f in fx.FIELDS[1:]:
        nodes[f][:, :3] = 0.0
    lo, hi = min(1.0, T), max(1.0, T)
    r = rng.uniform(lo + 0.05 * (hi - lo), hi - 0.05 * (hi - lo), n)
    s = rng.choice([-1.0, 1.0], n)
    d = um / 2 * (T - r) ** 2
    peak = np.where(np.arange(n) % 4 == 3, lim - d / 2, lim + d / 2)
    low, high = ("vel", "acc") if control == JRK else ("acc", "jrk")
    nodes[high][:, 0] = s * um * r
    nodes[low][:, 0] = s * (peak - um * r * r / 2)
    return case, nodes


def root_decides(case, nodes):
    """Slots whose v_max (JRK) or a_max (SNP) verdict changes when the stationary points are taken from (0, 1)
    in place of (0, T): a restatement of max_vel / max_acc with the bound of the root test moved."""
    T, lim = case.T, (case.v_max if case.control == JRK else case.a_max)
    low, high = ("vel", "acc") if case.control == JRK else ("acc", "jrk")
    decided = 0
    for i in range(nodes.size):
        for u in case.U:
            real = moved = 0.0
            for k in range(3):
                c0, c1, c2 = float(nodes[low][i, k]), float(nodes[high][i, k]), float(u[k])
                f = lambda t: abs(c0 + c1 * t + c2 / 2 * t * t)
                r = -c1 / c2 if c2 != 0 else -1.0
                ends = max(f(0.0), f(T))
                real = max(real, ends, f(r) if 0 < r < T else 0.0)
                moved = max(moved, ends, f(r) if 0 < r < 1.0 else 0.0)
            decided += (real > lim) != (moved > lim)
    return decided


@pytest.mark.parametrize("control,T", [(JRK, 2.0), (JRK, 0.7), (SNP, 1.3), (SNP, 0.5)],
                         ids=["jrk-T2.0", "jrk-T0.7", "snp-T1.3", "snp-T0.5"])
def test_stationary_points_between_1_and_T(control, T):
    case, nodes = roots_case(control, T, seed=int(T * 10) + control)
    orc, _ = fx.run_kernels(case, nodes, kernels=(1, 2, 5, 0))
    decided = root_decides(case, nodes)
    print(f"[roots] {NAME[control]} T={T}: {decided} primitives whose verdict a root in the gap decides")
    assert decided > 200
    em = fx.emitted_mask(orc)
    assert 0 < em.sum() < nodes.size * case.nU


def yaw_case(control, T, seed=9, n=1501):
    """VEL|YAW and ACC|YAW with yaw_max 0.6: a primitive is valid when its velocity and yaw at t = 0 and t = T lie
    within yaw_max of each other."""
    dim, res = 2, 0.2
    mdim, origin = (120, 100), (-11.9731, -9.9917)
    U = fx.product_set(*[fx.u_values(control & 15)] * dim, (-0.6, -0.3, 0.0, 0.3, 0.6))
    case = cp.Case(dim, control, U, mdim, origin, res, pw=0.1, wyaw=1.5, yaw_max=0.6, T=T)
    rng = np.random.default_rng(seed)
    nodes = cp.random_nodes(rng, n, case, 20, np.asarray(mdim) - 20, centred=True)
    v = nodes["vel"][:, :2] if control & 15 == ACC else rng.choice([-1.0, 1.0], (n, 2))
    nodes["yaw"] = np.arctan2(v[:, 1], v[:, 0]) + rng.uniform(-0.55, 0.55, n)
    return case, nodes


def yaw_verdicts_differ(case, nodes):
    """Slots whose yaw_max verdict with the end state at T differs from the one with the end state at 1."""
    n = 0
    for i in range(nodes.size):
        for u in case.U:
            ok = []
            for t in (case.T, 1.0):
                if case.control & 15 == VEL:
                    vx, vy = u[0], u[1]
                else:
                    vx, vy = nodes["vel"][i, 0] + u[0] * t, nodes["vel"][i, 1] + u[1] * t
                y = nodes["yaw"][i] + u[2] * t
                nv = math.hypot(vx, vy)
                ok.append(nv == 0 or (vx * math.cos(y) + vy * math.sin(y)) / nv >= math.cos(case.yaw_max))
            n += ok[0] != ok[1]
    return n


@pytest.mark.parametrize("control,T", [(VEL | YAW, 2.0), (ACC | YAW, 0.5)], ids=["velyaw-T2.0", "accyaw-T0.5"])
def test_yaw_verdict_at_T(control, T):
    case, nodes = yaw_case(control, T, seed=int(T * 10) + control)
    differ = yaw_verdicts_differ(case, nodes)
    print(f"[yaw] control {control:#x} T={T}: {differ} primitives whose yaw_max verdict differs at t = T and t = 1")
    assert differ > 300
    cp.run_cost_kernels(case, nodes, label=f"yaw_max T={T}")


# ---- 5. plan switches ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [3, 2])
def test_duration_switches_the_fixed_point_loop(dim):
    """v_max 4.2, res 0.15: maxn 29 at T = 1 (unchecked loop: 29 + 2 <= 32 guard cells) and 57 at T = 2 (checked);
    starts at the faces, so samples reach the guard band and beyond."""
    import test_fx_guard_gpu as fg

    v_max = 4.2
    assert fg.maxn(v_max, T=1.0) + 2 <= fg.GUARD < fg.maxn(v_max, T=2.0) + 2
    for T in (1.0, 2.0):
        rng = np.random.default_rng(40 + dim)
        case = fg.case_for(dim, v_max, fg.face_grid(fg.MAPS[dim]["mdim"], dim, rng, 0.02))
        case.T = T
        nodes = fg.edge_nodes(rng, fg.n_nodes(dim), dim, (0.5, 1.5, 3.0, 4.0))
        orc, env = fx.run_kernels(case, nodes, kernels=fg.KERNELS)
        em = fx.emitted_mask(orc)
        assert np.isinf(orc["cost"][em]).sum() > 1000 and np.isfinite(orc["cost"][em]).sum() > 100
        if T == 2.0:
            env.set_kernel(5)
            check_exact(case, nodes, env.expand(nodes, want=fx.WANT), n_check=100)


@pytest.mark.parametrize("T", [T_LONG, T_SHORT])
def test_sample_counts_past_the_table_and_clamped(T):
    """T_LONG: unbounded speeds up to 6 m/s at res 0.1 put some primitives past the 128-row table (literal loop)
    and keep others on it; T_SHORT: every n is the clamp 5."""
    from scenarios import box_map

    res = 0.1 if T == T_LONG else 0.15
    mdim, origin = (200, 72, 56), (-9.9731, -3.6113, -2.8117)
    grid = box_map(mdim, res, origin, n_boxes=40, edge_m=(0.3, 1.0), seed=11)
    case = fx.Case(3, ACC, fx.product_set(*[fx.u_values(ACC)] * 3), mdim, origin, res, grid=grid, T=T)
    rng = np.random.default_rng(12)
    nodes = fx.random_nodes(rng, 1001, case, (60, 20, 16), (140, 52, 40), centred=True)
    nodes["vel"][:, 0] = rng.choice([-5.5, -4.0, -2.5, 0.5, 2.5, 4.0, 5.5], nodes.size)
    orc, env = fx.run_kernels(case, nodes)
    em = fx.emitted_mask(orc) & ~fx.same_mask(orc, nodes, 3)
    n = fx.sample_counts(case, nodes, orc)[em]
    if T == T_LONG:
        print(f"[table] T={T}: {(n > N_TABLE).sum()} primitives past the table, {(n <= N_TABLE).sum()} on it")
        assert (n > N_TABLE).sum() > 500 and (n <= N_TABLE).sum() > 500
        assert np.isinf(orc["cost"][em][n > N_TABLE]).any() and np.isfinite(orc["cost"][em][n > N_TABLE]).any()
    else:
        assert (n == 5).all() and np.ceil(6.0 * T / res) < 5
    env.set_kernel(0)
    check_exact(case, nodes, env.expand(nodes, want=fx.WANT), n_check=150)


# ---- 6. edges and searches ------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [0.7, 2.0])
@pytest.mark.parametrize("dim,control", [(3, ACC), (2, JRK), (3, SNP | YAW)], ids=["3d-acc", "2d-jrk", "3d-snpyaw"])
def test_edges(dim, control, T):
    import test_edges_paths_gpu as ep

    orc, parents, actions = edges_case(dim, control, T)
    env = ep.gpu_of(orc)
    fo, off, cells, _ = ep.check(env, orc, parents, actions)
    assert 0 < fo.sum() < fo.size and cells.shape[0] > parents.size


def edges_case(dim, control, T, seed=13):
    """Stored edges (test_edges_oracle_vs_ref.edges_of) at T on a box map, with and without a yaw column."""
    from scenarios import box_map, control_set
    from test_edges_oracle_vs_ref import edges_of
    from test_oracle_vs_ref import random_nodes

    yaw = bool(control & YAW)
    rng = np.random.default_rng(seed + dim + control + int(T * 10))
    U = control_set(4.0 if control & 15 == SNP else 1.0, 3, dim, yaw_rates=(-0.4, 0.0, 0.4) if yaw else None)
    dims = (41, 37) if dim == 2 else (41, 37, 29)
    res = 0.2
    origin = tuple(-d * res / 2 + 0.0137 for d in dims)
    grid = box_map(dims, res, origin, 7, (0.6, 1.6), seed=seed)
    orc = ob.OracleEnv(dim, control, U, grid, dims, origin, res, T=T, w=10.0, wyaw=1.5, v_max=2.5, a_max=3.0,
                       j_max=6.0, yaw_max=0.9 if yaw else -1.0)
    nodes = random_nodes(rng, 300, dim, 25 * res / 2, yaw=yaw)
    parents, actions, _ = edges_of(orc, nodes, rng, extra=300)
    return orc, parents, actions


SEARCH_CASES = [(2, ACC, 0.5), (3, JRK, 0.5), (2, JRK, 0.7), (3, ACC, 0.7)]


def search_case(dim, control, T):
    import test_device_search_paths_gpu as ds

    sc = ds.base_scene(dim, control, seed=20 * dim + control, eps=2.0, max_expand=150, T=T)
    S, G = ds.random_queries(sc, 12, seed=dim * 10 + control + int(T * 10), near=(1.0, 2.5), far_every=3)
    return sc, S, G


@pytest.mark.parametrize("dim,control,T", SEARCH_CASES, ids=[f"{d}d-{NAME[c]}-T{T}" for d, c, T in SEARCH_CASES])
def test_searches(dim, control, T):
    """mplx_plan_batch (BatchPlanner, raw ABI, lock-step) against the host planner on the oracle env;
    _cost_terms and _grow equal to it; the recorded trajectories hold seg_t = T and the host's nodes."""
    import test_batch_trajectories_gpu as bt
    import test_device_search_paths_gpu as ds

    sc, S, G = search_case(dim, control, T)
    d = ds.check(sc, S, G)
    assert d["valid"].any()
    s = sc.search
    env = sc.env()
    try:
        kw = dict(eps=s["eps"], tol_pos=s["tol_pos"], tol_vel=s["tol_vel"], tol_acc=s["tol_acc"])
        r = env.plan_batch(S, G, max_expand=s["max_expand"], trajectories=True, n_samples=bt.N_SAMPLES, **kw)
        ds.same_results(d, r, "plan_batch with trajectories")
        ds.same_results(d, env.plan_batch_cost_terms(S, G, max_expand=s["max_expand"], **kw), "cost_terms")
        g = env.plan_batch_grow(S, G, max_expand=s["max_expand"], **kw)
        ds.same_results(d, g, "grow")
        bt.check_layout(r, dim, control, sc.U, T)
        host = bt.planner_trajectories(sc.args(), S, G, "lockstep")
        bt.same_traj([{k: t[k] for k in host[q]} for q, t in enumerate(r["trajectories"])], host, "device vs host")
    finally:
        env.close()


# ---- 7. T changed on a live context -----------------------------------------------------------------------
@pytest.mark.parametrize("via", ["set_params", "set_dt"])
def test_duration_changes_on_a_live_context(via):
    """One context with a map and a search region resident and both kernels run: T through 1 -> 0.7 -> 2.0 -> 1,
    by mplx_set_params on the ctx or by the Python env's set_dt (re-sent before the next call); after each
    change kernels 0 and 5 give what a fresh context gives, byte for byte, and what the oracle gives."""
    from motion_primitive_library_b200 import abi

    case, nodes = matrix_case(3, SNP, 1.0, True)
    env = case.gpu()
    for k in (0, 5):
        env.set_kernel(k)
        env.expand(nodes, want=fx.WANT)
    for T in (0.7, 2.0, 1.0):
        case.T = T
        if via == "set_dt":
            env.set_dt(T)
        else:
            env.dt_ = T
            abi.check(env._lib.mplx_set_params(env.handle, env.control, T, env.w_, env.wyaw_, env.v_max_, env.a_max_,
                                               env.j_max_, env.yaw_max_, env.U_.ctypes.data, *env.U_.shape))
        fresh = case.gpu()
        orc = case.oracle().expand(nodes, nthreads=NTHREADS)
        for k in (0, 5):
            env.set_kernel(k)
            fresh.set_kernel(k)
            a, b = env.expand(nodes, want=fx.WANT), fresh.expand(nodes, want=fx.WANT)
            assert a.count.tobytes() == b.count.tobytes(), (T, k)
            sel = fx.emitted_mask(orc)
            for f in fx.WANT:
                assert getattr(a, f)[sel].tobytes() == getattr(b, f)[sel].tobytes(), (T, k, f)
            assert_expansion_equal(a, orc, exact_cost=True)
        fresh.close()
    env.close()
