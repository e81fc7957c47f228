"""The cost-summing expansion kernels (potential field, gradient, yaw) on every instantiation.

Plans with a potential map, a gradient weight or a yaw control sum a cost term per sample in
traverse_primitive (env_map.h:90-132) and run the literal kernel (1), the register kernel (2), the flat
kernel (3) or the dealing kernel (4); auto (0) picks the dealing kernel for batches of at least two
rounds' worth of CTAs and the register kernel below that (csrc/mplx_kernels.cu, launch_expand).

Cost bars (DESIGN.md §4.4):
  no yaw term (no yaw control, or wyaw <= 0)  kernels 1, 2, 4 and 0 add dt*(pot_w*pv + grad_w*|v|) in
                                              sample order, as the reference does: bit for bit.  The flat
                                              kernel sums with atomicAdd in varying order: 1e-12 relative.
  yaw term                                    the device's sincos, the YawRot recurrence, (v.cs + v.sn)/|v|
                                              and c + (pot + yaw) instead of two additions: 1e-12 relative.
                                              Kernels 2 and 4 run the same arithmetic per sample in the
                                              same order: bitwise equal to each other.
Every case prints its largest relative cost deviation from the oracle.  tests/test_cost_inputs_oracle_vs_ref.py
pins the oracle against the reference on the same input classes.
"""
from __future__ import annotations

import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import pytest

import oracle_bindings as ob
import test_fx_paths_gpu as fx
from parity import assert_expansion_equal
from reference_record import same_array

pytestmark = pytest.mark.gpu

VEL, ACC, JRK, SNP = fx.VEL, fx.ACC, fx.JRK, fx.SNP
YAW = 0x10
ORDER = fx.ORDER
WANT, NO_SUCC = fx.WANT, fx.NO_SUCC
KERNELS = (1, 2, 3, 4, 0)
THREADS = 256        # kThreads
N_TABLE = 128        # kNMax
MAX_ROUNDS = 8       # kDealMaxRounds
NTHREADS = fx.NTHREADS
YAW_RTOL = 1e-12
FLAT_RTOL = 1e-12


# ---- inputs ------------------------------------------------------------------------------------------
class Case(fx.Case):
    """fx.Case plus the cost terms: potential map and weights, wyaw and yaw_max."""

    def __init__(self, dim, control, U, mdim, origin, res, potential=None, pw=0.1, gw=0.0, wyaw=1.0, yaw_max=-1.0,
                 **kw):
        super().__init__(dim, control, U, mdim, origin, res, **kw)
        self.potential = None if potential is None else np.ascontiguousarray(potential, np.int8).reshape(-1)
        self.pw, self.gw, self.wyaw, self.yaw_max = float(pw), float(gw), float(wyaw), float(yaw_max)

    @property
    def yaw(self):
        return bool(self.control & YAW)

    @property
    def yaw_term(self):
        """Whether traverse_primitive adds the yaw-alignment term (env_map.h:122)."""
        return self.yaw and self.wyaw > 0

    def oracle(self):
        return ob.OracleEnv(self.dim, self.control, self.U, self.grid, self.mdim, self.origin, self.res, T=self.T,
                            w=self.w, wyaw=self.wyaw, v_max=self.v_max, a_max=self.a_max, j_max=self.j_max,
                            yaw_max=self.yaw_max, potential=self.potential, potential_weight=self.pw,
                            gradient_weight=self.gw, region=self.region)

    def gpu(self):
        e = super().gpu()
        e.set_wyaw(self.wyaw)
        e.set_yaw_max(self.yaw_max)
        e.potential_weight_, e.gradient_weight_ = self.pw, self.gw
        if self.potential is not None:
            e.set_potential_map(self.potential)
        return e


def maxn_of(control, v_max, T, res):
    """refresh_params (csrc/mplx_api.cu): the largest n a validated primitive can have.  VEL and v_max <= 0
    are unbounded (the whole table)."""
    if (control & 15) == VEL or not v_max > 0:
        return N_TABLE
    nb = math.ceil(v_max * T / res)
    return max(5, nb) if nb < N_TABLE else N_TABLE


def launcher(kernel, dim, control, nU, pot, gw, maxn, n_nodes, lat, sms):
    """The expansion kernel launch_expand / launch_t / launch_expand_deal pick on the cost path (a potential
    map or a yaw control) for one launch of n_nodes nodes: (instantiation, rounds).  The instantiation is
    (kernel, DIM, ORD, YAW, VEL, UNR, LAT), None where the kernel has no such template parameter."""
    yaw = bool(control & YAW)
    assert pot or yaw, "not a cost-path plan"
    order = ORDER[control & 15]
    nv = yaw or (pot and gw != 0.0)                       # need_vel: velocities are evaluated per sample
    heavy = (control & 15) >= JRK or yaw or pot           # always true here
    if kernel == 5:
        kernel = 0                                        # the fixed-point kernel does not apply: auto
    deal = kernel == 4 or (kernel == 0 and heavy and n_nodes * nU >= 2 * THREADS * sms * 4 * 8)
    if deal and nU <= THREADS:
        npb = THREADS // nU
        ctas1 = -(-n_nodes // npb)
        rounds = min(max(ctas1 // (sms * 4 * 8), 1), MAX_ROUNDS)
        unr = 2 if (maxn <= 15 or nv) else 4
        return ("deal", dim, order, yaw, nv, unr, lat), rounds
    if nU > THREADS or kernel == 1:
        return ("literal", dim, order, yaw, None, None, None), None
    if kernel == 3:
        return ("flat", dim, order, yaw, None, None, None), None
    short = maxn <= 15
    if nv:
        unr = 2 if short else 4
    else:
        unr = 2 if short else (4 if lat else 8)
    return ("register", dim, order, yaw, nv, unr, lat), None


def launches_of(case, kernel, n_nodes, lat, sms):
    """launcher() for a Case, over the chunks mplx_expand stages (fx.launches_expected)."""
    maxn = maxn_of(case.control, case.v_max, case.T, case.res)
    return launcher(kernel, case.dim, case.control, case.nU, case.potential is not None, case.gw, maxn, n_nodes,
                    lat, sms)


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def yaw_set(control, dim, rates=(-0.5, 0.0, 0.5)):
    """Product control set with a yaw-rate column for yaw plans (udim = Dim + 1)."""
    axes = [fx.u_values(control & 15)] * dim
    return fx.product_set(*axes, rates) if control & YAW else fx.product_set(*axes)


def potential_field(rng, size, p_free=0.1, p_block=0.03):
    """int8 potential over every class: mostly 1..99 (adds cost), some <= 0 (free, including -1 and -128),
    some 100..127 (blocks)."""
    pot = rng.integers(1, 100, size)
    r = rng.random(size)
    free = r < p_free
    pot[free] = rng.choice([-128, -77, -1, 0], free.sum())
    block = r > 1 - p_block
    pot[block] = rng.integers(100, 128, block.sum())
    return pot.astype(np.int8)


def random_grid(rng, size):
    """Occupancy independent of the potential: free, occupied and unknown voxels."""
    return rng.choice(np.array([0, 100, -1], np.int8), size, p=[0.7, 0.2, 0.1])


def position_part(case):
    """The Case as fx's node helpers read it: control without the yaw bit, U without the yaw column."""
    return SimpleNamespace(dim=case.dim, control=case.control & 15, origin=case.origin, res=case.res, T=case.T,
                           U=case.U[:, :case.dim], nU=case.nU)


def random_nodes(rng, n, case, lo, hi, centred=False):
    """fx.random_nodes, with a random yaw in [-pi, pi] for yaw plans."""
    nodes = fx.random_nodes(rng, n, position_part(case), lo, hi, centred=centred)
    if case.yaw:
        nodes["yaw"] = rng.uniform(-np.pi, np.pi, n)
    return nodes


# ---- checks ------------------------------------------------------------------------------------------
def rel_dev(g, o):
    fin = ~np.isinf(o)
    if not fin.any():
        return 0.0
    return float(np.max(np.abs(g[fin] - o[fin]) / np.abs(o[fin])))


def check_costs(case, kernel, g, orc, label=""):
    """Everything but the cost bit for bit; the cost to the bar of this kernel and plan.  Returns the largest
    relative deviation of the cost from the oracle."""
    exact = not case.yaw_term and kernel != 3
    assert_expansion_equal(g, orc, exact_cost=exact)
    if g.cost is None:
        return 0.0
    sel = fx.emitted_mask(orc)
    dev = rel_dev(g.cost[sel], orc["cost"][sel])
    assert dev <= (FLAT_RTOL if kernel == 3 else YAW_RTOL), (label, kernel, dev)
    return dev


def run_cost_kernels(case, nodes, wants=(WANT, NO_SUCC), kernels=KERNELS, env=None, orc=None, label=""):
    """Every kernel with every output set against the oracle at its bar; kernels 2, 4 and 0 bitwise equal
    to each other with a yaw term; one launch per call.  Prints the largest relative deviation."""
    if orc is None:
        orc = case.oracle().expand(nodes, nthreads=NTHREADS)
    env = case.gpu() if env is None else env
    devs, costs = {}, {}
    sel = fx.emitted_mask(orc)
    for k in kernels:
        env.set_kernel(k)
        env._sync_params()
        for want in wants:
            before = env.launch_count()
            g = env.expand(nodes, want=want)
            assert env.launch_count() - before == fx.launches_expected(k, nodes.size, case.nU, fxn_allowed=False)
            devs[k] = max(devs.get(k, 0.0), check_costs(case, k, g, orc, label))
            if g.cost is not None:
                costs.setdefault(k, []).append(g.cost[sel].copy())
    for k in (4, 0):
        if 2 in costs and k in costs:
            for a, b in zip(costs[2], costs[k]):
                same_array(a, b, f"{label} cost: kernel 2 vs {k}", bits=True)
    fx.check_reference(case, nodes, orc)
    print(f"[cost] {label}: max relative cost deviation per kernel {devs}")
    return orc, env


# ---- 1. instantiation matrix ----------------------------------------------------------------------------
CONFIGS_PLAIN = ("P", "PG", "PR")
CONFIGS_YAW = ("Y", "Y0")
MODES = [(d, c) for d in (2, 3) for c in (VEL, ACC, JRK, SNP)]
LOOPS = ("short", "long")


def matrix_params(dim, control, config, loop):
    """Plan parameters of one matrix case (no arrays): short loops have maxn <= 15 except for VEL, which is
    never bounded."""
    res, v_max = (0.25, 2.5) if loop == "short" else (0.1, 3.0)
    p = dict(res=res, v_max=v_max, a_max=3.0, j_max=6.0, pot=config in ("P", "PG", "PR"), gw=0.3 if config == "PG" else 0.0,
             region=config == "PR", wyaw=1.5 if config == "Y" else 0.0, yaw_max=0.9 if config == "Y0" else -1.0)
    p["maxn"] = maxn_of(control, v_max, 1.0, res)
    return p


def matrix_case(dim, control, config, loop, seed, wyaw=None):
    from scenarios import box_map

    p = matrix_params(dim, control, config, loop)
    res = p["res"]
    mdim = ((160, 120) if dim == 2 else (80, 64, 48)) if loop == "long" else ((96, 80) if dim == 2 else (48, 40, 32))
    origin = (-7.9137, -6.0411, -2.3893)[:dim]
    rng = np.random.default_rng(seed)
    size = int(np.prod(mdim))
    if p["pot"]:
        grid = random_grid(rng, size)
        potential = potential_field(rng, size)
    else:
        grid = box_map(mdim, res, origin, n_boxes=12, edge_m=(2 * res, 5 * res), seed=seed)
        grid[rng.random(size) < 0.02] = 100
        potential = None
    region = (rng.random(size) < 0.9).astype(np.uint8) if p["region"] else None
    return Case(dim, control, yaw_set(control, dim), mdim, origin, res, grid=grid, region=region, potential=potential,
                pw=0.1, gw=p["gw"], wyaw=p["wyaw"] if wyaw is None else wyaw, yaw_max=p["yaw_max"],
                v_max=p["v_max"], a_max=p["a_max"], j_max=p["j_max"])


def matrix_nodes(case, seed):
    n = 400 if case.dim == 2 else 200
    lo = np.asarray(case.mdim) // 2 - np.asarray(case.mdim) // 6
    hi = np.asarray(case.mdim) // 2 + np.asarray(case.mdim) // 6
    return random_nodes(np.random.default_rng(seed + 1), n, case, lo, hi)


MATRIX = [(d, c | y, cfg, loop) for d, c in MODES for y, cfgs in ((0, CONFIGS_PLAIN), (YAW, CONFIGS_YAW))
          for cfg in cfgs for loop in LOOPS]


def matrix_id(p):
    d, c, cfg, loop = p
    name = {VEL: "vel", ACC: "acc", JRK: "jrk", SNP: "snp"}[c & 15] + ("yaw" if c & YAW else "")
    return f"{d}d-{name}-{cfg}-{loop}"


@pytest.mark.parametrize("dim,control,config,loop", MATRIX, ids=[matrix_id(p) for p in MATRIX])
def test_cost_instantiations(dim, control, config, loop):
    seed = 1000 * dim + 10 * control + 100 * MATRIX.index((dim, control, config, loop))
    for wyaw in ((0.0, -1.0) if config == "Y0" else (None,)):
        case = matrix_case(dim, control, config, loop, seed, wyaw=wyaw)
        nodes = matrix_nodes(case, seed)
        orc, _ = run_cost_kernels(case, nodes, label=f"{matrix_id((dim, control, config, loop))} wyaw={case.wyaw}")
        st = fx.emitted_mask(orc)
        cost = orc["cost"][st]
        assert st.sum() > nodes.size and np.isfinite(cost).any()
        if config != "Y0":
            assert np.isinf(cost).any()


def instantiations(dims=(2, 3), sms=132):
    """Every instantiation the cost path can launch, from launcher() over all plan classes, kernels and
    output sets (rounds aside)."""
    out = set()
    for dim in dims:
        for c in (VEL, ACC, JRK, SNP):
            for yaw in (0, YAW):
                for pot, gw in ((True, 0.0), (True, 0.3), (False, 0.0)):
                    if not pot and not yaw:
                        continue
                    for maxn in (10, 30, N_TABLE):
                        if (c == VEL) and maxn != N_TABLE:
                            continue
                        for lat in (True, False):
                            for k in (1, 2, 3, 4):
                                out.add(launcher(k, dim, c | yaw, 27, pot, gw, maxn, 100, lat, sms)[0])
    return out


def test_launcher_restatement_reaches_every_instantiation():
    """The matrix above reaches every instantiation the cost path has: register kernel need_vel x UNR 2/4/8
    x LAT, dealing kernel need_vel x UNR 2/4 x LAT, the flat and the literal kernel, each for Dim 2/3 x
    VEL/ACC/JRK/SNP x yaw/no yaw."""
    sms = sm_count()
    reached = set()
    for dim, control, config, loop in MATRIX:
        p = matrix_params(dim, control, config, loop)
        nU = yaw_set(control, dim).shape[0]
        n = 400 if dim == 2 else 200
        for k in KERNELS:
            for want in (WANT, NO_SUCC):
                inst, rounds = launcher(k, dim, control, nU, p["pot"], p["gw"], p["maxn"], n, "lattice" in want, sms)
                assert rounds in (None, 1)
                reached.add(inst)
    universe = instantiations(sms=sms)
    assert reached == universe, sorted(universe - reached, key=str)
    # the counts the docstring names
    reg = {i for i in universe if i[0] == "register"}
    deal = {i for i in universe if i[0] == "deal"}
    assert {(i[4], i[5], i[6]) for i in reg} == {(False, 2, False), (False, 2, True), (False, 4, True),
                                                 (False, 8, False), (True, 2, False), (True, 2, True),
                                                 (True, 4, False), (True, 4, True)}
    assert {(i[4], i[5], i[6]) for i in deal} == {(nv, u, lat) for nv in (False, True) for u in (2, 4)
                                                  for lat in (False, True) if not (nv and u == 4)}
    modes = {(i[1], i[2], i[3]) for i in universe}
    assert len(modes) == 16
    for name in ("register", "deal", "flat", "literal"):
        assert {(i[1], i[2], i[3]) for i in universe if i[0] == name} == modes, name
    # VEL always gets the whole table (mplx_api.cu, refresh_params)
    assert maxn_of(VEL, 2.5, 1.0, 0.25) == N_TABLE and maxn_of(ACC, 2.5, 1.0, 0.25) == 10
    assert maxn_of(ACC, -1.0, 1.0, 0.25) == N_TABLE and maxn_of(ACC, 1.0, 1.0, 0.25) == 5


# ---- 2. potential classes: answers without the oracle ---------------------------------------------------
PCLASS_MAP = {3: dict(mdim=(64, 64, 64), origin=(-3.2071, -3.1933, -3.1811), res=0.1),
              2: dict(mdim=(96, 96), origin=(-4.8113, -4.7919), res=0.1)}


def pclass_case(dim, control, grid_kind, value=None, gw=0.0):
    m = PCLASS_MAP[dim]
    size = int(np.prod(m["mdim"]))
    grid = np.full(size, {"free": 0, "occupied": 100, "unknown": -1}[grid_kind], np.int8)
    pot = None if value is None else np.full(size, value, np.int8)
    return Case(dim, control, fx.product_set(*[fx.u_values(control)] * dim), m["mdim"], m["origin"], m["res"],
                grid=grid, potential=pot, pw=0.37, gw=gw, v_max=2.5, a_max=3.0, j_max=6.0)


def pclass_nodes(case, seed=31, n=300):
    """Nodes within 0.6 m of the map centre: no primitive leaves the map (travel <= 2.5 m, map >= 4.8 m)."""
    c = np.asarray(case.mdim) // 2
    return random_nodes(np.random.default_rng(seed), n, case, c - 6, c + 6)


def sample_iterations(case, nodes, orc):
    """(n, iterations of the sample loop) per emitted slot: n = max(5, ceil(max_v*T/res)) (env_map.h:95)."""
    env = case.oracle()
    nU = case.nU
    parent = np.repeat(np.arange(nodes.size), nU)
    em = fx.emitted_mask(orc)
    n = np.zeros(em.size, np.int64)
    for s in np.nonzero(em)[0]:
        mv = max(ob.lib().orc_max_vel(C.byref(env.e), nodes[parent[s]:parent[s] + 1].ctypes.data, int(orc["action"][s]),
                                      a) for a in range(case.dim))
        n[s] = max(5, math.ceil(mv * case.T / case.res))
    it = np.zeros_like(n)
    for v in np.unique(n[em]):
        it[n == v] = ob.lib().orc_sample_count(case.T, int(v))
    return n, it


@pytest.mark.parametrize("value", [-128, -1, 0, 1, 50, 99, 100, 101, 127])
@pytest.mark.parametrize("dim,control", [(3, ACC), (2, JRK)])
def test_potential_classes(dim, control, value):
    """A potential that is `value` everywhere, over all-free, all-occupied and all-unknown grids: the
    answer depends on the signed potential alone (env_map.h:113-121), never on the grid."""
    free = pclass_case(dim, control, "free")
    nodes = pclass_nodes(free)
    env0 = free.gpu()
    ref = env0.expand(nodes, want=NO_SUCC)
    intrinsic = ref.cost
    orc0 = free.oracle().expand(nodes, nthreads=NTHREADS, lattice=False)
    em = fx.emitted_mask(orc0)
    assert np.isfinite(intrinsic[em]).all() and em.sum() > nodes.size
    same = fx.same_mask(orc0, nodes, dim)
    expected = intrinsic.copy()
    if 0 < value < 100:
        n, it = sample_iterations(free, nodes, orc0)
        dt = free.T / n[em & ~same]
        term = dt * (0.37 * value)
        c = np.zeros_like(term)
        for k in range(int(it.max())):
            live = k < it[em & ~same]
            c[live] = c[live] + term[live]
        expected[em & ~same] = c + intrinsic[em & ~same]
    elif value >= 100:
        expected[em & ~same] = np.inf
    for kind in ("free", "occupied", "unknown"):
        for gw in ((0.0, 0.3) if value <= 0 else (0.0,)):
            case = pclass_case(dim, control, kind, value, gw=gw)
            env = case.gpu()
            for k in KERNELS:
                env.set_kernel(k)
                g = env.expand(nodes, want=NO_SUCC)
                np.testing.assert_array_equal(g.count, orc0["count"])
                assert g.cost[em].tobytes() == expected[em].tobytes(), (kind, gw, k)
            if value >= 100:
                assert np.isfinite(g.cost[same]).all() and np.isinf(g.cost[em & ~same]).all()


def test_uniform_random_int8_potential():
    """Uniformly random int8 potential over an independent random grid, short loops."""
    rng = np.random.default_rng(41)
    m = PCLASS_MAP[3]
    size = int(np.prod(m["mdim"]))
    case = Case(3, ACC, fx.product_set(*[fx.u_values(ACC)] * 3), m["mdim"], m["origin"], 0.25,
                grid=random_grid(rng, size), potential=rng.integers(-128, 128, size).astype(np.int8), pw=0.21,
                gw=0.0, v_max=2.5)
    nodes = random_nodes(rng, 400, case, 8, 24)
    orc, _ = run_cost_kernels(case, nodes, label="uniform int8")
    cost = orc["cost"][fx.emitted_mask(orc)]
    assert np.isinf(cost).any() and np.isfinite(cost).any()


# ---- 3. multi-round dealing through mplx_expand_device -----------------------------------------------------
def oracle_expand(case, nodes, lattice=False, chunk=1 << 14):
    """OracleEnv.expand without the successor records (they would not fit in memory at these sizes): count,
    cost, action, key and, if asked for, the lattice ints, in chunks."""
    env = case.oracle()
    n, nU = nodes.size, env.nU
    out = dict(count=np.zeros(n, np.int32), cost=np.zeros(n * nU), action=np.zeros(n * nU, np.int32),
               key=np.zeros(n * nU, np.uint64), succ=None, nU=nU,
               lattice=np.zeros((n * nU, ob.LATTICE_MAX), np.int32) if lattice else None)
    scratch = np.zeros(chunk * nU, dtype=ob.WAYPOINT_DTYPE)
    for lo in range(0, n, chunk):
        part = np.ascontiguousarray(nodes[lo:lo + chunk])
        m, s = part.size, lo * nU
        ob.lib().orc_expand_batch(C.byref(env.e), part.ctypes.data, m, scratch.ctypes.data,
                                  out["cost"][s:].ctypes.data, out["action"][s:].ctypes.data,
                                  out["key"][s:].ctypes.data, out["lattice"][s:].ctypes.data if lattice else None,
                                  out["count"][lo:].ctypes.data, NTHREADS)
    return out


def deal_U(rng, nU=128, lo=0.25):
    """nU = 128: two nodes per CTA fill all 256 lanes, so a CTA whose primitives all need sampling fills its
    ticket queue exactly.  No control is zero on every axis (no successor is its parent)."""
    U = np.round(rng.uniform(-1.0, 1.0, (nU, 3)) * 8) / 8
    U[np.abs(U).max(1) < lo, 0] = 0.5
    return U


def deal_case(mix, seed):
    """3-D ACC, potential, 128 controls.  mix: the ticket classes the CTAs' queues hold."""
    rng = np.random.default_rng(seed)
    mdim = (96, 96, 64)
    origin = (-11.9731, -12.0313, -8.0177)
    size = int(np.prod(mdim))
    res, v_max, gw = {"mixed": (0.25, 2.0, 0.0), "mixed-vel": (0.25, 2.0, 0.3), "mixed-unr4": (0.2, 3.2, 0.0),
                      "long": (0.25, 1.25, 0.0), "short": (0.1, -1.0, 0.0), "none": (0.25, 0.01, 0.0)}[mix]
    grid = random_grid(rng, size)
    pot = potential_field(rng, size, p_block=0.01)
    return Case(3, ACC, deal_U(rng), mdim, origin, res, grid=grid, potential=pot, pw=0.1, gw=gw, v_max=v_max)


def deal_nodes(case, n, mix, seed):
    rng = np.random.default_rng(seed)
    c = np.asarray(case.mdim) // 2
    nodes = random_nodes(rng, n, case, c - 10, c + 10)
    if mix in ("long", "short", "none"):
        nodes["vel"] = 0.0      # max_v = max |u| <= 1: every primitive long (maxn 5) / short (maxn 128) / rejected
    return nodes


def deal_batch(rounds, sms, npb):
    """A node count for which the auto rule gives `rounds` rounds (capped ones: at least that many) and that
    is not a multiple of npb * rounds, so some CTA's later rounds hold no node."""
    per = sms * 4 * 8
    ctas1 = rounds * per + per // 2 + 1
    n = ctas1 * npb - 1
    assert n % (npb * min(rounds, MAX_ROUNDS)) != 0
    return n


def check_deal(case, nodes, rounds, want, kernels=(4, 0)):
    """mplx_expand_device with each kernel in `kernels`, which must be the dealing kernel with `rounds` rounds:
    against the oracle at the kernel's bar, and bitwise against the register kernel on the same buffers."""
    sms = sm_count()
    lat = "lattice" in want
    for k in kernels:
        inst, r = launches_of(case, k, nodes.size, lat, sms)
        assert inst[0] == "deal" and r == rounds, (k, inst, r)
    if "succ" in want:
        orc = case.oracle().expand(nodes, nthreads=NTHREADS, lattice=lat)
    else:
        orc = oracle_expand(case, nodes, lattice=lat)
    sel = fx.emitted_mask(orc)
    env = case.gpu()
    env.set_kernel(2)
    g2 = fx.expand_device(env, nodes, want)
    devs = {2: check_costs(case, 2, g2, orc, f"register, {rounds} rounds' batch")}
    for k in kernels:
        env.set_kernel(k)
        g = fx.expand_device(env, nodes, want)
        devs[k] = check_costs(case, k, g, orc, f"deal {rounds} rounds")
        same_array(g.cost[sel], g2.cost[sel], f"cost: kernel {k} vs kernel 2", bits=True)
    print(f"[cost] dealing kernel, {rounds} rounds, {nodes.size} nodes: max relative cost deviation {devs}")
    return orc


@pytest.mark.parametrize("rounds,mix", [(1, "mixed"), (2, "mixed-vel"), (3, "mixed-unr4"), (2, "long"),
                                        (2, "short"), (3, "none")])
def test_multi_round_dealing(rounds, mix):
    sms = sm_count()
    case = deal_case(mix, seed=50 + rounds)
    npb = THREADS // case.nU
    n = deal_batch(rounds, sms, npb)
    nodes = deal_nodes(case, n, mix, seed=60 + rounds)
    want = WANT if rounds == 1 else (("cost", "action", "key", "lattice") if mix == "mixed-vel" else NO_SUCC)
    kernels = (4,) if rounds == 1 else (4, 0)   # below two rounds' worth of CTAs auto is the register kernel
    assert launches_of(case, 0, n, "lattice" in want, sms)[0][0] == ("register" if rounds == 1 else "deal")
    orc = check_deal(case, nodes, rounds, want, kernels=kernels)
    inst = launches_of(case, 4, n, "lattice" in want, sms)[0]
    em = fx.emitted_mask(orc)
    counts = orc["count"]
    maxn = maxn_of(case.control, case.v_max, case.T, case.res)
    n_long = (5 + maxn) // 2
    if mix == "none":
        assert counts.sum() == 0
    else:
        assert em.sum() > n and np.isfinite(orc["cost"][em]).any() and np.isinf(orc["cost"][em]).any()
    if mix in ("long", "short"):
        # every primitive emitted and sampled: each full CTA's queue is exactly full (q_long + q_short == cap)
        assert (counts == case.nU).all()
        if mix == "long":
            assert maxn == 5 and n_long == 5
        else:
            assert maxn == N_TABLE and n_long == 66
            vmax = np.abs(case.U).max()
            assert math.ceil(vmax * case.T / case.res) < n_long
    assert inst[5] == (4 if mix in ("mixed-unr4", "short") else 2)
    if mix in ("mixed", "mixed-vel"):
        assert (counts < case.nU).any() and (counts == case.nU).any()   # some queues partly, some fully filled


def test_cfg4_kernel_choice_eight_rounds():
    """cfg4's own launch: ACC x YAW, 81 controls, potential, no lattice, auto -> dealing kernel with the
    8-round cap (the floor of the CTA count over SMs x 32 is 9), on a scaled map."""
    from scenarios import cfg4, scaled

    sms = sm_count()
    sc = scaled(cfg4(), 96)
    case = Case(3, sc.control, sc.U, sc.dim_cells, sc.origin, sc.res, grid=sc.grid(), potential=sc.potential(),
                pw=sc.potential_weight, gw=sc.gradient_weight, wyaw=sc.wyaw, yaw_max=sc.yaw_max, v_max=sc.v_max,
                T=sc.T, w=sc.w)
    npb = THREADS // case.nU
    n = deal_batch(9, sms, npb)
    nodes = sc.frontier(n, seed=5)
    inst, rounds = launches_of(case, 0, n, False, sms)
    assert inst == ("deal", 3, 2, True, True, 2, False) and rounds == MAX_ROUNDS
    assert -(-n // npb) // (sms * 32) == 9
    check_deal(case, nodes, MAX_ROUNDS, NO_SUCC, kernels=(0, 4))


# ---- 4. past the sample-time table --------------------------------------------------------------------
def beyond_cost_case(yaw, seed=71, n=700):
    """v_max <= 0, res = 1/32 and x velocities around 4 m/s: n = 32*max_v reaches 128, 129 and beyond.  The
    potential seldom blocks, so most samples add cost; with yaw, YawRot runs for more than 128 steps."""
    res = 1.0 / 32
    mdim = (400, 48, 48)
    origin = (-6.2519, -0.7371, -0.7613)
    rng = np.random.default_rng(seed)
    size = int(np.prod(mdim))
    control = ACC | (YAW if yaw else 0)
    case = Case(3, control, yaw_set(control, 3), mdim, origin, res, grid=random_grid(rng, size),
                potential=potential_field(rng, size, p_free=0.2, p_block=0.002), pw=0.05, gw=0.3 if yaw else 0.0,
                wyaw=1.5)
    nodes = random_nodes(rng, n, case, (190, 16, 16), (210, 32, 32), centred=True)
    nodes["vel"][:, 0] = rng.choice([3.0, 4.0, 4.03125, -3.0, -4.0, -4.03125, 3.5, -4.5], n)
    nodes["vel"][:, 1:3] = rng.integers(-2, 3, (n, 2)) * 0.25
    nodes["yaw"] = rng.uniform(-np.pi, np.pi, n)
    return case, nodes


@pytest.mark.parametrize("yaw", [False, True], ids=["potential", "potential-gradient-yaw"])
def test_past_the_sample_table(yaw):
    case, nodes = beyond_cost_case(yaw)
    orc, _ = run_cost_kernels(case, nodes, kernels=(1, 2, 3, 4), label=f"beyond table yaw={yaw}")
    em = fx.emitted_mask(orc) & ~fx.same_mask(orc, nodes, 3)
    n = fx.sample_counts(position_part(case), nodes, orc)[em]
    cost = orc["cost"][em]
    assert (n > N_TABLE).sum() > 200 and (n <= N_TABLE).sum() > 200
    assert np.isfinite(cost[n > N_TABLE]).sum() > 50


# ---- 5. yaw edges -----------------------------------------------------------------------------------
def yaw_edge_case(dim=3, wyaw=1.5):
    control = ACC | YAW
    mdim = (64, 64, 64)[:dim]
    origin = (-3.2071, -3.1933, -3.1811)[:dim]
    return Case(dim, control, yaw_set(control, dim), mdim, origin, 0.1, wyaw=wyaw, v_max=-1.0)


def straddle_vectors():
    """Planar velocities whose norm is the double 1e-5, its neighbours, and vectors (a, b) whose
    sqrt(a^2 + b^2) rounds to exactly 1e-5."""
    e = 1e-5
    out = [(e, 0.0), (0.0, e), (-e, 0.0), (np.nextafter(e, 1), 0.0), (np.nextafter(e, 0), 0.0),
           (0.0, -np.nextafter(e, 1)), (0.0, np.nextafter(e, 0))]
    rng = np.random.default_rng(3)
    found = 0
    while found < 24:
        th = rng.uniform(-np.pi, np.pi)
        a, b = e * np.cos(th), e * np.sin(th)
        nn = np.sqrt(a * a + b * b)
        if nn == e:
            out.append((a, b))
            found += 1
            # the neighbours of a that take the norm across 1e-5
            for a2 in (np.nextafter(a, np.inf), np.nextafter(a, -np.inf)):
                if np.sqrt(a2 * a2 + b * b) != e:
                    out.append((a2, b))
    v = np.asarray(out)
    norms = np.sqrt(v[:, 0] ** 2 + v[:, 1] ** 2)
    assert (norms == e).sum() >= 20 and (norms > e).any() and (norms < e).any()
    return v


def test_yaw_norm_straddle():
    """sqrt(v0^2 + v1^2) > 1e-5 decides the yaw term.  Controls with no planar part keep the planar velocity
    of the start at every sample (0*t + v0 == v0); the node's yaw is at right angles to it, so a yaw term
    that is added or left out where it should not be moves the cost by ~wyaw*dt."""
    case = yaw_edge_case(3)
    v = straddle_vectors()
    reps = 8
    n = v.shape[0] * reps
    rng = np.random.default_rng(5)
    nodes = random_nodes(rng, n, case, 28, 36)
    nodes["vel"][:, :2] = np.repeat(v, reps, axis=0)
    nodes["vel"][:, 2] = rng.integers(-2, 3, n) * 0.5
    nodes["yaw"] = np.arctan2(nodes["vel"][:, 1], nodes["vel"][:, 0]) + np.pi / 2
    orc, _ = run_cost_kernels(case, nodes, label="yaw 1e-5 straddle")
    # the term must have made a difference: same nodes, no yaw term
    off = yaw_edge_case(3, wyaw=0.0).oracle().expand(nodes, nthreads=NTHREADS)
    nU = case.nU
    planar0 = (case.U[:, :2] == 0).all(1)
    em = fx.emitted_mask(orc).reshape(n, nU) & planar0[orc["action"].reshape(n, nU)]
    above = np.repeat(np.sqrt(v[:, 0] ** 2 + v[:, 1] ** 2) > 1e-5, reps)
    diff = orc["cost"].reshape(n, nU) != off["cost"].reshape(n, nU)
    assert diff[above[:, None] & em].all() and not diff[~above[:, None] & em].any()


def test_yaw_z_only_motion():
    """3-D nodes moving only along z: zero planar velocity at sample 0 for every control and at every sample
    for the controls without a planar part."""
    case = yaw_edge_case(3)
    rng = np.random.default_rng(9)
    n = 300
    nodes = random_nodes(rng, n, case, 28, 36)
    nodes["vel"][:, :2] = 0.0
    nodes["acc"] = 0.0
    nodes["vel"][:, 2] = rng.choice([-1.5, -0.5, 0.5, 1.5], n)
    nodes["yaw"] = rng.uniform(-np.pi, np.pi, n)
    run_cost_kernels(case, nodes, label="yaw z-only")


def test_yaw_at_pi():
    """Node yaws at +-pi (as the double M_PI) and their neighbours, with yaw rates that cross it."""
    case = yaw_edge_case(2)
    pi = np.pi
    yaws = np.array([pi, np.nextafter(pi, 4), np.nextafter(pi, 3), -pi, np.nextafter(-pi, -4), np.nextafter(-pi, -3),
                     pi - 0.5, -pi + 0.5])
    rng = np.random.default_rng(13)
    reps = 60
    nodes = random_nodes(rng, yaws.size * reps, case, 28, 36)
    nodes["yaw"] = np.repeat(yaws, reps)
    run_cost_kernels(case, nodes, label="yaw at pi")
    # and with yaw_max on the same nodes (validate_yaw at the endpoints)
    case.yaw_max = 0.9
    run_cost_kernels(case, nodes, label="yaw at pi, yaw_max 0.9")


# ---- 6. edge queries with a potential map installed -----------------------------------------------------
def edges_case(dim, control, rng):
    """A box-map grid (plus the search region in 2-D) and a potential that disagrees with it: occupied voxels
    that the potential calls free, free voxels that it blocks."""
    from scenarios import box_map

    case = matrix_case(dim, control, "Y" if control & YAW else "P", "short", 23)
    size = case.grid.size
    case.grid = box_map(case.mdim, case.res, case.origin, n_boxes=12, edge_m=(2 * case.res, 5 * case.res), seed=29)
    if dim == 2:
        case.region = (rng.random(size) < 0.97).astype(np.uint8)
    occ = case.grid == 100
    pot = potential_field(rng, size)
    pot[occ] = rng.choice([-128, -1, 0, 5], occ.sum())
    pot[~occ & (rng.random(size) < 0.1)] = 100
    case.potential = pot
    return case


@pytest.mark.parametrize("dim,control", [(3, ACC), (2, JRK), (2, ACC | YAW)])
def test_edges_ignore_the_potential(dim, control):
    """is_free(pr) tests occupancy and the search region, never the potential (env_map.h:60-76): the edge
    queries with a potential that disagrees with the grid equal the oracle and the same queries without it,
    bit for bit."""
    from test_edges_oracle_vs_ref import edges_of

    rng = np.random.default_rng(17 + dim + control)
    case = edges_case(dim, control, rng)
    nodes = matrix_nodes(case, 23)[:150]
    orc = case.oracle()
    parents, actions, _ = edges_of(orc, nodes, rng, extra=300)
    fo, co = orc.edges_is_free(parents, actions)
    oo, oc = orc.edges_cells(parents, actions)
    with_pot = case.gpu()
    bare = Case(case.dim, case.control, case.U, case.mdim, case.origin, case.res, grid=case.grid, region=case.region,
                wyaw=case.wyaw, yaw_max=case.yaw_max, v_max=case.v_max, a_max=case.a_max, j_max=case.j_max).gpu()
    results = []
    for env in (with_pot, bare):
        f, c = env.is_free_edges(parents, actions)
        off, cells = env.edge_cells(parents, actions)
        np.testing.assert_array_equal(f, fo)
        assert c.tobytes() == co.tobytes()
        np.testing.assert_array_equal(off, oo)
        np.testing.assert_array_equal(cells, oc)
        results.append((f.tobytes(), c.tobytes(), off.tobytes(), cells.tobytes()))
    assert results[0] == results[1]
    assert 0 < fo.sum() < fo.size
    # the potential decides differently from the grid on some of these edges
    o = orc.expand(nodes, nthreads=NTHREADS, lattice=False)
    if not case.yaw:
        em = fx.emitted_mask(o)
        assert (np.isinf(o["cost"][em]) != ~fo[:em.sum()].astype(bool)).any()


# ---- 7. small related checks ------------------------------------------------------------------------
@pytest.mark.parametrize("config", ["PG", "Y"])
def test_stats_counters_on_the_cost_path(config):
    control = ACC | (YAW if config == "Y" else 0)
    case = matrix_case(3, control, config, "long", 77)
    nodes = matrix_nodes(case, 77)
    t = case.oracle().timed(nodes, nthreads=NTHREADS)
    env = case.gpu()
    env.enable_stats(True)
    for k in (2, 3, 4):
        env.set_kernel(k)
        env.expand(nodes, want=NO_SUCC)
        assert env.last_stats() == (t["samples"], t["successors"]), k
    assert t["samples"] > t["successors"] > 0


def test_setter_transitions():
    """Install a potential, change its weights through mplx_set_potential_weights, remove it, remove the
    region: after each step every kernel gives what a freshly built env gives, bit for bit."""
    from motion_primitive_library_b200 import abi

    base = matrix_case(3, ACC, "PR", "long", 91)
    nodes = matrix_nodes(base, 91)
    env = Case(base.dim, base.control, base.U, base.mdim, base.origin, base.res, grid=base.grid, region=base.region,
               v_max=base.v_max).gpu()

    def fresh(pot, pw, gw, region):
        return Case(base.dim, base.control, base.U, base.mdim, base.origin, base.res, grid=base.grid, region=region,
                    potential=pot, pw=pw, gw=gw, v_max=base.v_max)

    def same_as(ref_case, label):
        ref_env = ref_case.gpu()
        orc = ref_case.oracle().expand(nodes, nthreads=NTHREADS)
        for k in (1, 2, 3, 4, 0):
            env.set_kernel(k)
            ref_env.set_kernel(k)
            a = env.expand(nodes, want=WANT)
            b = ref_env.expand(nodes, want=WANT)
            np.testing.assert_array_equal(a.count, b.count)
            sel = fx.emitted_mask(orc)
            if k == 3 and ref_case.potential is not None:
                assert rel_dev(a.cost[sel], b.cost[sel]) <= FLAT_RTOL, (label, k)
            else:
                assert a.cost[sel].tobytes() == b.cost[sel].tobytes(), (label, k)
            assert a.succ[sel].tobytes() == b.succ[sel].tobytes() and a.key[sel].tobytes() == b.key[sel].tobytes()
            check_costs(ref_case, k, a, orc, label)

    env.potential_weight_, env.gradient_weight_ = 0.1, 0.0
    env.set_potential_map(base.potential)
    same_as(fresh(base.potential, 0.1, 0.0, base.region), "potential installed")
    abi.check(env._lib.mplx_set_potential_weights(env.handle, 0.7, 0.3))
    same_as(fresh(base.potential, 0.7, 0.3, base.region), "weights changed")
    env.gradient_weight_, env.potential_weight_ = 0.3, 0.7
    env.set_potential_map(None)
    same_as(fresh(None, 0.7, 0.3, base.region), "potential removed")
    env.set_search_region(None)
    same_as(fresh(None, 0.7, 0.3, None), "region removed")

