"""The fixed-point expansion kernels on every instantiation and fall-back path.

Occupancy planning (no potential map, no yaw control) runs expand_fxn_kernel + fx_resolve_kernel for
batches of at least 64*256 primitive slots and expand_fx_kernel below that (csrc/mplx_kernels.cu,
launch_expand).  Both decide a sample's cell in fixed point: a sample is CERTAIN, or UNCERTAIN with all
its candidate cells free, or AMBIGUOUS and re-decided with the exact FP64 chain (DESIGN.md §4.2).  On top
of that come the paths that leave the fixed-point loop:

  queue full  a segment of the ambiguity queue is full: the primitive runs the literal loop (verdict 3)
  literal     (|p0| + |origin|)/res >= 2^17 on some axis: beyond the range of the error bound
  beyond      n > 128: beyond the sample-time table
  full        an ambiguous sample at index >= 64: the resolve step re-walks every sample
  same        curr.pos == tn.pos: intrinsic cost only, no traversal (env_map.h:163)

Every case compares kernels 1 (literal loop), 2 (register), 5 (expand_fx_kernel) and 0 (auto, which is
expand_fxn_kernel for the large batches here) bit for bit with the CPU oracle, and with the reference where
oracle/_ref is built, and shows from launch counts and from its own construction that the path it is
about ran.  tests/test_fx_inputs_oracle_vs_ref.py pins the oracle on the same inputs.
"""
from __future__ import annotations

import numpy as np
import pytest

import oracle_bindings as ob
from parity import assert_expansion_equal
from reference_record import same_array

pytestmark = pytest.mark.gpu

VEL, ACC, JRK, SNP = 0x01, 0x03, 0x07, 0x0F
ORDER = {VEL: 1, ACC: 2, JRK: 3, SNP: 4}
FIELDS = ("pos", "vel", "acc", "jrk")
WANT = ("succ", "cost", "action", "key", "lattice")
NO_SUCC = ("cost", "action", "key")  # succ == NULL and no lattice: the LAT=false instantiations
KERNELS = (1, 2, 5, 0)
THREADS = 256                     # primitives per CTA (kThreads)
FXN_MIN_SLOTS = 64 * THREADS      # fxn_supported: n_nodes * |U| >= 64 * kThreads
STAGE_SLOTS = 1 << 20             # mplx_expand stages (1 << 20) // |U| nodes per launch
ZERO_COPY_SLOTS = 4096            # ... and runs batches of <= 4096 slots as one zero-copy launch
FX_RANGE = 2.0 ** 17              # kFxRange (csrc/mplx_fx.cuh)
N_TABLE = 128                     # kNMax: rows of the sample-time table
SEGMENTS = 64                     # kFxSegments
NTHREADS = 16                     # oracle threads

# ---- inputs ------------------------------------------------------------------------------------------
class Case:
    """One plan: the parameters of an env and its map, for the oracle, the reference and libmplx."""

    def __init__(self, dim, control, U, mdim, origin, res, grid=None, region=None, T=1.0, w=10.0, v_max=-1.0,
                 a_max=-1.0, j_max=-1.0):
        self.dim, self.control = dim, control
        self.U = np.ascontiguousarray(U, dtype=np.float64)
        self.mdim, self.origin, self.res = tuple(int(m) for m in mdim), tuple(float(o) for o in origin), float(res)
        self.grid = np.zeros(int(np.prod(self.mdim)), np.int8) if grid is None else np.ascontiguousarray(grid, np.int8)
        self.region = region
        self.T, self.w, self.v_max, self.a_max, self.j_max = T, w, v_max, a_max, j_max

    @property
    def nU(self):
        return self.U.shape[0]

    def oracle(self):
        return ob.OracleEnv(self.dim, self.control, self.U, self.grid, self.mdim, self.origin, self.res, T=self.T,
                            w=self.w, v_max=self.v_max, a_max=self.a_max, j_max=self.j_max, region=self.region)

    def gpu(self):
        from motion_primitive_library_b200 import MapUtil, env_map

        mu = MapUtil()
        mu.setMap(self.origin, self.mdim, self.grid, self.res)
        e = env_map(mu)
        e.set_control(self.control)
        e.set_u(self.U)
        e.set_dt(self.T)
        e.set_w(self.w)
        e.set_v_max(self.v_max)
        e.set_a_max(self.a_max)
        e.set_j_max(self.j_max)
        if self.region is not None:
            e.set_search_region(self.region)
        return e

    def index(self, cells):
        cells = np.asarray(cells, dtype=np.int64).reshape(-1, self.dim)
        idx = cells[:, 0] + self.mdim[0] * cells[:, 1]
        if self.dim == 3:
            idx = idx + self.mdim[0] * self.mdim[1] * cells[:, 2]
        return idx

def product_set(*axes):
    """U = axes[0] x axes[1] (x axes[2]), first axis outermost, values kept bit for bit (-0.0 stays)."""
    grids = np.meshgrid(*[np.asarray(a, dtype=np.float64) for a in axes], indexing="ij")
    return np.ascontiguousarray(np.stack([g.reshape(-1) for g in grids], axis=1))

def u_values(control):
    """Three values of the control per axis (SNP/JRK larger, as their users set them)."""
    return {VEL: (-1.0, 0.0, 1.0), ACC: (-1.0, 0.0, 1.0), JRK: (-2.0, 0.0, 2.0), SNP: (-4.0, 0.0, 4.0)}[control]

def ref_cell(p, origin, res):
    """MapUtil::floatToInt (map_util.h): std::round((p - origin)/res - 0.5), half away from zero, exactly."""
    x = (np.asarray(p, dtype=np.float64) - origin) / res - 0.5
    a = np.abs(x)
    r = np.floor(a)
    r = r + (a - r >= 0.5)
    return np.copysign(r, x).astype(np.int64)

def boundary(origin, res, k):
    """The coordinate of the cell boundary k: origin + k*res, as a user's lattice puts it."""
    return origin + np.asarray(k, dtype=np.float64) * res

def random_nodes(rng, n, case, lo_cells, hi_cells, steps=(0.5, 0.5, 1.0), centred=False):
    """Nodes with positions in the cell box [lo, hi) (cell centres or 0.05 m-lattice points) and lattice
    derivatives; the fields the control does not read are zero."""
    nodes = np.zeros(n, dtype=ob.WAYPOINT_DTYPE)
    d, order = case.dim, ORDER[case.control]
    cells = rng.integers(lo_cells, hi_cells, (n, d))
    o = np.asarray(case.origin[:d])
    if centred:
        nodes["pos"][:, :d] = o + (cells + 0.5) * case.res
    else:
        nodes["pos"][:, :d] = o + np.round((cells + rng.random((n, d))) * case.res / 0.05) * 0.05
    for f in range(1, order):
        nodes[FIELDS[f]][:, :d] = rng.integers(-3, 4, (n, d)) * steps[f - 1]
    nodes["t"] = rng.integers(0, 5, n) * 1.0
    return nodes

# ---- runs --------------------------------------------------------------------------------------------
def launches_expected(kernel, n, nU, fxn_allowed=True):
    """Launches mplx_expand adds for a batch of n nodes: one per staged chunk, two where the chunk runs
    expand_fxn_kernel + fx_resolve_kernel (csrc/mplx_api.cu)."""
    if n * nU <= ZERO_COPY_SLOTS:
        chunks = [n]
    else:
        c = max(1, STAGE_SLOTS // nU)
        chunks = [min(c, n - off) for off in range(0, n, c)]
    return sum(2 if kernel == 0 and fxn_allowed and m * nU >= FXN_MIN_SLOTS else 1 for m in chunks)

def check_reference(case, nodes, orc):
    """Where oracle/_ref is built: the reference itself on the same nodes, bit for bit."""
    if not ob.ref_available():
        return
    r = ob.ref_expand(case.oracle(), nodes, nthreads=NTHREADS)
    same_array(orc["count"], r["count"], "count")
    o, r = ob.emitted(orc), ob.emitted(r)
    for name in ("action", "key"):
        same_array(o[name], r[name], name)
    for name in ("succ", "cost"):
        same_array(o[name], r[name], name, bits=True)

def run_kernels(case, nodes, wants=(WANT, NO_SUCC), kernels=KERNELS, env=None, orc=None, fxn=True):
    """Every kernel in `kernels` with every output set in `wants` against the oracle, costs exact; the
    launch count of each call must be the one of its path (kernel 0: expand_fxn_kernel where fxn)."""
    if orc is None:
        orc = case.oracle().expand(nodes, nthreads=NTHREADS)
    env = case.gpu() if env is None else env
    for k in kernels:
        env.set_kernel(k)
        env._sync_params()
        for want in wants:
            before = env.launch_count()
            g = env.expand(nodes, want=want)
            assert env.launch_count() - before == launches_expected(k, nodes.size, case.nU, fxn), (k, want)
            assert_expansion_equal(g, orc, exact_cost=True)
    check_reference(case, nodes, orc)
    return orc, env

def emitted_mask(orc):
    return (np.arange(orc["nU"])[None, :] < orc["count"][:, None]).reshape(-1)

def same_mask(orc, nodes, dim):
    """Emitted slots whose successor has the parent's position, bit for bit (env_map.h:163)."""
    nU = orc["nU"]
    parent = np.repeat(np.arange(nodes.size), nU)
    a = orc["succ"]["pos"][:, :dim].view(np.uint64)
    b = nodes["pos"][parent][:, :dim].view(np.uint64)
    return emitted_mask(orc) & (a == b).all(1)

def expand_device(env, nodes, want, succ_misalign=0):
    """mplx_expand_device with torch device buffers; the succ buffer starts `succ_misalign` bytes past a
    256-byte aligned address."""
    import ctypes as C

    import torch

    from motion_primitive_library_b200 import abi

    env._sync_params()
    n, nU = nodes.size, env.U_.shape[0]
    dev = torch.device("cuda", 0)
    d_nodes = torch.from_numpy(nodes.view(np.uint8).copy()).to(dev)
    rec = ob.WAYPOINT_DTYPE.itemsize
    bufs = dict(count=torch.empty(n * 4, dtype=torch.uint8, device=dev))
    sizes = dict(succ=rec, cost=8, action=4, key=8, lattice=4 * ob.LATTICE_MAX)
    for name in want:
        extra = succ_misalign if name == "succ" else 0
        bufs[name] = torch.empty(n * nU * sizes[name] + extra, dtype=torch.uint8, device=dev)[extra:]
    if "succ" in bufs:
        assert bufs["succ"].data_ptr() % 16 == succ_misalign % 16
    out = abi.SuccOut(*[bufs[k].data_ptr() if k in bufs else None
                        for k in ("count", "succ", "cost", "action", "key", "lattice")])
    abi.check(env._lib.mplx_expand_device(env.handle, d_nodes.data_ptr(), n, C.byref(out), None))
    abi.check(env._lib.mplx_sync(env.handle))
    host = {k: v.cpu().numpy() for k, v in bufs.items()}
    from motion_primitive_library_b200.env import Expansion

    return Expansion(nU, host["count"].view(np.int32),
                     host["succ"].view(ob.WAYPOINT_DTYPE) if "succ" in host else None,
                     host["cost"].view(np.float64) if "cost" in host else None,
                     host["action"].view(np.int32) if "action" in host else None,
                     host["key"].view(np.uint64) if "key" in host else None,
                     host["lattice"].view(np.int32).reshape(-1, ob.LATTICE_MAX) if "lattice" in host else None)

# ---- 1. instantiation matrix of expand_fxn_kernel ------------------------------------------------------
MAP2 = dict(mdim=(211, 97), origin=(-31.1337, -14.2791), res=0.3)
MAP3 = dict(mdim=(61, 37, 29), origin=(-4.3711, -2.7093, -1.9318), res=0.15)

def matrix_case(dim, control, with_region, seed):
    from scenarios import box_map

    m = MAP2 if dim == 2 else MAP3
    res = m["res"]
    grid = box_map(m["mdim"], res, m["origin"], n_boxes=12 if dim == 2 else 10, edge_m=(3 * res, 10 * res), seed=seed)
    rng = np.random.default_rng(seed)
    region = (rng.random(grid.size) < 0.8).astype(np.uint8) if with_region else None
    U = product_set(*[u_values(control)] * dim)
    return Case(dim, control, U, m["mdim"], m["origin"], res, grid=grid, region=region, v_max=2.5, a_max=3.0,
                j_max=6.0)

def matrix_nodes(case, seed):
    # >= 16384 slots, node count not a multiple of the nodes per CTA (28 for |U| = 9, 9 for |U| = 27)
    n = 2003 if case.dim == 2 else 701
    npb = THREADS // case.nU
    assert n * case.nU >= FXN_MIN_SLOTS and n % npb != 0
    return random_nodes(np.random.default_rng(seed + 1), n, case, 2, np.asarray(case.mdim) - 2)

@pytest.mark.parametrize("with_region", [False, True], ids=["map", "region"])
@pytest.mark.parametrize("control", [VEL, ACC, JRK, SNP], ids=["vel", "acc", "jrk", "snp"])
@pytest.mark.parametrize("dim", [2, 3])
def test_fxn_instantiations(dim, control, with_region):
    seed = 100 * dim + 10 * control + with_region
    case = matrix_case(dim, control, with_region, seed)
    nodes = matrix_nodes(case, seed)
    npb, order = THREADS // case.nU, ORDER[control]
    if npb * dim * order > 64:
        # the node-hash loop past the first 64 (node, field) ids of the CTA runs (mplx_fxn.cu, phase A0)
        assert (dim, control) in ((2, ACC), (2, JRK), (2, SNP), (3, JRK), (3, SNP))
    orc, _ = run_kernels(case, nodes)
    st = emitted_mask(orc)
    assert st.sum() > nodes.size and np.isinf(orc["cost"][st]).any() and np.isfinite(orc["cost"][st]).any()

def test_fxn_device_buffers_unaligned_succ():
    """mplx_expand_device with a succ buffer that is 8- but not 16-byte aligned: the per-lane stores of
    store_waypoint instead of the bulk copies."""
    case = matrix_case(3, ACC, False, 7)
    nodes = matrix_nodes(case, 7)
    orc = case.oracle().expand(nodes, nthreads=NTHREADS)
    env = case.gpu()
    env._sync_params()
    for misalign in (8, 0):
        before = env.launch_count()
        g = expand_device(env, nodes, WANT, succ_misalign=misalign)
        assert env.launch_count() - before == 2
        assert_expansion_equal(g, orc, exact_cost=True)

def test_fxn_packed_stream_2d_drop_inf():
    """mplx_expand_packed on a 2-D fxn batch, +inf successors dropped."""
    case = matrix_case(2, ACC, False, 11)
    nodes = matrix_nodes(case, 11)
    orc = case.oracle().expand(nodes, nthreads=NTHREADS, lattice=False)
    env = case.gpu()
    p = env.expand_packed(nodes, drop_inf=True)
    nU = case.nU
    keep = (np.arange(nU)[None, :] < orc["count"][:, None]) & ~np.isinf(orc["cost"].reshape(-1, nU))
    np.testing.assert_array_equal(p["count"], keep.sum(1))
    assert p["total"] == int(keep.sum()) and 0 < p["total"] < int(orc["count"].sum())
    sel = np.nonzero(keep.reshape(-1))[0]
    idx = np.concatenate([p["offset"][i] + np.arange(p["count"][i]) for i in range(nodes.size)])
    exp_state = np.concatenate([orc["succ"]["pos"][sel][:, :2], orc["succ"]["vel"][sel][:, :2]], axis=1)
    assert p["state"][idx].tobytes() == np.ascontiguousarray(exp_state).tobytes()
    np.testing.assert_array_equal(p["action"][idx], orc["action"][sel].astype(np.uint16))
    np.testing.assert_array_equal(p["key"][idx], orc["key"][sel])
    np.testing.assert_array_equal(p["cost"][idx], orc["cost"][sel])

# ---- 2. starts on cell boundaries next to obstacles -------------------------------------------------------
def boundary_case(res, seed, dim=3, n=1201):
    """ACC-27 nodes whose positions lie on cell boundaries (origin + k*res) on every axis, zero velocity on
    about half the axes; for each start one voxel across its boundaries is occupied: the one the reference
    puts sample 0 in (blocked) or the one next to it on a boundary axis (free, but a candidate)."""
    mdim = (40, 33, 29) if dim == 3 else (400, 301)
    origin = (-2.9173, -1.3311, -2.0517)[:dim]
    case = Case(dim, ACC, product_set(*[u_values(ACC)] * dim), mdim, origin, res)
    rng = np.random.default_rng(seed)
    k = rng.integers(8, np.asarray(mdim) - 8, (n, dim))
    nodes = np.zeros(n, dtype=ob.WAYPOINT_DTYPE)
    o = np.asarray(origin)
    nodes["pos"][:, :dim] = boundary(o, res, k)
    still = rng.random((n, dim)) < 0.5
    nodes["vel"][:, :dim] = np.where(still, 0.0, rng.integers(-2, 3, (n, dim)) * 0.5)
    c0 = ref_cell(nodes["pos"][:, :dim], o, res)
    # reaching the boundary from the -0 side would not be a lattice start: sample 0 is uncertain on all axes
    y = (nodes["pos"][:, :dim] - o) * (1.0 / res)
    assert (np.abs(y - k) < 1e-9).all()
    other = c0.copy()
    axis = rng.integers(0, dim, n)
    rows = np.arange(n)
    other[rows, axis] = np.where(c0[rows, axis] == k[rows, axis], k[rows, axis] - 1, k[rows, axis])
    blocked = rng.random(n) < 0.3
    occ = np.where(blocked[:, None], c0, other)
    case.grid[case.index(occ)] = 100
    return case, nodes

@pytest.mark.parametrize("res", [0.1, 0.15, 0.25, 0.3])
def test_boundary_starts_next_to_obstacles(res):
    case, nodes = boundary_case(res, seed=int(res * 1000))
    orc, _ = run_kernels(case, nodes)
    # every emitted, finite, not-`same` primitive had an uncertain sample 0 with an occupied candidate cell
    # and no blocked certain sample: it was queued and set free by the exact chain
    live = emitted_mask(orc) & ~same_mask(orc, nodes, case.dim)
    resolved_free = int((live & np.isfinite(orc["cost"])).sum())
    assert resolved_free > 2000, resolved_free
    assert int((live & np.isinf(orc["cost"])).sum()) > 2000

def test_boundary_starts_2d():
    case, nodes = boundary_case(0.15, seed=3, dim=2, n=2003)
    orc, _ = run_kernels(case, nodes)
    live = emitted_mask(orc) & ~same_mask(orc, nodes, 2)
    assert int((live & np.isfinite(orc["cost"])).sum()) > 2000

# ---- 3. queue overflow: the in-kernel literal loop (verdict 3) --------------------------------------------
def queue_capacity(n_prims):
    """FxQueue::reserve (csrc/mplx_internal.h) on a fresh ctx: records for a quarter of the batch's primitives
    plus 64 * 4096, rounded up to a multiple of 64 and split evenly into the 64 segments."""
    cap = ((n_prims // 4 + 64 * 4096 + 63) // 64) * 64
    return cap // SEGMENTS

def overflow_case(with_region, n=60000, seed=5):
    """ACC-27 nodes at `sites`: x on a cell boundary with zero x velocity, y and z at cell centres.  Every
    primitive whose x control is 0 or points away from the reference's sample-0 cell c0 has an uncertain
    sample 0 and, x being monotone, no later sample in c0.  At 4 of 5 sites c0 is blocked: outside the
    search region (with_region) or occupied.  Sites are 8 cells apart in x and x moves at most 0.5 m = 4
    cells, so no primitive reaches another site's blocked voxel."""
    res = 0.15
    mdim = (200, 48, 48)
    origin = (-15.0731, -3.6217, -3.5989)
    case = Case(3, ACC, product_set(*[u_values(ACC)] * 3), mdim, origin, res)
    o = np.asarray(origin)
    xs = np.arange(8, mdim[0] - 8, 8)
    rng = np.random.default_rng(seed)
    site_k = np.stack([xs, rng.integers(16, 32, xs.size), rng.integers(16, 32, xs.size)], 1)
    site_pos = np.stack([boundary(o[0], res, site_k[:, 0]), o[1] + (site_k[:, 1] + 0.5) * res,
                         o[2] + (site_k[:, 2] + 0.5) * res], 1)
    c0 = ref_cell(site_pos, o, res)
    holed = np.arange(xs.size) % 5 != 0
    if with_region:
        case.region = np.ones(case.grid.size, np.uint8)
        case.region[case.index(c0[holed])] = 0
    else:
        case.grid[case.index(c0[holed])] = 100
    site = np.arange(n) % xs.size
    nodes = np.zeros(n, dtype=ob.WAYPOINT_DTYPE)
    nodes["pos"][:, :3] = site_pos[site]
    nodes["vel"][:, 1:3] = rng.integers(-1, 2, (n, 2)) * 0.5
    nodes["t"] = rng.integers(0, 3, n) * 1.0
    # the direction of x that leaves c0: +1 when c0 is the cell below the boundary, else -1
    away = np.where(c0[:, 0] < site_k[:, 0], 1.0, -1.0)
    return case, nodes, site, holed, away

@pytest.mark.parametrize("with_region", [True, False], ids=["region", "map"])
def test_queue_overflow_falls_back_to_the_literal_loop(with_region):
    case, nodes, site, holed, away = overflow_case(with_region)
    nU, n = case.nU, nodes.size
    orc = case.oracle().expand(nodes, nthreads=NTHREADS)
    em = emitted_mask(orc).reshape(n, nU)
    ux = case.U[orc["action"].reshape(n, nU), 0]
    same = same_mask(orc, nodes, 3).reshape(n, nU)
    # queued: sample 0 uncertain, never a blocked certain sample.  With a region every uncertain sample is
    # ambiguous; without one only where a candidate cell (c0 here) is occupied.
    leaves = (ux == 0.0) | (ux == away[site][:, None])
    queued = em & ~same & leaves & (holed[site][:, None] if not with_region else True)
    cost = orc["cost"].reshape(n, nU)
    blocked = queued & np.isinf(cost)
    # construction check: a queued primitive is blocked exactly when its site is holed
    np.testing.assert_array_equal(blocked, queued & holed[site][:, None])
    np.testing.assert_array_equal(np.isfinite(cost[queued & ~holed[site][:, None]]), True)
    # segments: CTA b holds nodes [b*npb, (b+1)*npb) and appends to segment b & 63
    npb = THREADS // nU
    seg = (np.arange(n) // npb) & (SEGMENTS - 1)
    cap = queue_capacity(n * nU)
    q_seg = np.bincount(seg, weights=queued.sum(1), minlength=SEGMENTS)
    b_seg = np.bincount(seg, weights=blocked.sum(1), minlength=SEGMENTS)
    # whatever order the atomics run in, more blocked primitives than places: some blocked one falls back
    assert (q_seg > cap).any() and (b_seg > cap).any(), (cap, q_seg.max(), b_seg.max())
    # a fresh ctx, so the queue is sized for this batch; one launch of expand_fxn_kernel + fx_resolve_kernel
    env = case.gpu()
    env._sync_params()
    before = env.launch_count()
    g = expand_device(env, nodes, WANT)
    assert env.launch_count() - before == 2
    assert_expansion_equal(g, orc, exact_cost=True)
    run_kernels(case, nodes, wants=(NO_SUCC,), env=env, orc=orc)

# ---- 4. the 2^17 range gate ----------------------------------------------------------------------------
def gate_origin(sign, res, cells, offset):
    """An origin whose map [o, o + cells*res] has (|p| + |o|)/res cross 2^17 in its middle."""
    L = cells * res
    if sign > 0:
        return (FX_RANGE * res - L / 2) / 2 + offset
    return -((FX_RANGE * res + L / 2) / 2) + offset

def gate_quantity(nodes, case):
    o = np.abs(np.asarray(case.origin[:case.dim]))
    return ((np.abs(nodes["pos"][:, :case.dim]) + o) * (1.0 / case.res)).max(1)

def gate_case(res, signs, seed, far=None):
    from scenarios import box_map

    mdim = (64, 48, 40)
    if far is None:
        origin = tuple(gate_origin(s, res, m, 0.0137 * (a + 1)) for a, (s, m) in enumerate(zip(signs, mdim)))
    else:
        origin = tuple(s * far * res + 0.0191 * (a + 1) for a, s in enumerate(signs))
    grid = box_map(mdim, res, origin, n_boxes=8, edge_m=(3 * res, 9 * res), seed=seed)
    case = Case(3, ACC, product_set(*[u_values(ACC)] * 3), mdim, origin, res, grid=grid, v_max=2.0)
    rng = np.random.default_rng(seed)
    n = 1001
    nodes = random_nodes(rng, n, case, 4, np.asarray(mdim) - 4, centred=True)
    if far is None:
        # boundary-aligned starts just below the gate, with the voxel across the boundary occupied
        o = np.asarray(origin)
        m = n // 4
        k = np.empty((m, 3), np.int64)
        for a in range(3):
            if o[a] > 0:
                kk = np.floor((FX_RANGE * res - 2 * o[a]) / res).astype(np.int64) - rng.integers(1, 4, m)
            else:
                kk = np.ceil((-2 * o[a] - FX_RANGE * res) / res).astype(np.int64) + rng.integers(1, 4, m)
            k[:, a] = np.clip(kk, 4, mdim[a] - 4)
        nodes["pos"][:m, :3] = boundary(o, res, k)
        nodes["vel"][:m, :3] = np.where(rng.random((m, 3)) < 0.5, 0.0, nodes["vel"][:m, :3])
        c0 = ref_cell(nodes["pos"][:m, :3], o, res)
        other = c0.copy()
        other[:, 0] = np.where(c0[:, 0] == k[:, 0], k[:, 0] - 1, k[:, 0])
        case.grid[case.index(other)] = 100
    return case, nodes

@pytest.mark.parametrize("res,signs", [(0.05, (1, -1, 1)), (0.15, (-1, 1, -1)), (0.1, (-1, -1, 1))])
def test_range_gate_straddled(res, signs):
    case, nodes = gate_case(res, signs, seed=int(res * 100) + signs[0] + 7)
    gq = gate_quantity(nodes, case)
    assert (gq < FX_RANGE - 1).sum() > 100 and (gq > FX_RANGE + 1).sum() > 100
    orc, env = run_kernels(case, nodes)
    # small batches: kernel 0 is expand_fx_kernel (one launch each) with its own gate
    env.set_kernel(0)
    for lo in range(0, nodes.size, 500):
        part = nodes[lo:lo + 500]
        before = env.launch_count()
        g = env.expand(part, want=WANT)
        assert env.launch_count() - before == 1
        sub = {k: (v[lo * case.nU:(lo + part.size) * case.nU] if isinstance(v, np.ndarray) and k != "count" else v)
               for k, v in orc.items()}
        sub["count"] = orc["count"][lo:lo + part.size]
        assert_expansion_equal(g, sub, exact_cost=True)

@pytest.mark.parametrize("far_log2,res", [(24, 0.05), (25, 0.3), (26, 0.15), (27, 0.05)])
def test_far_maps_take_the_literal_loop(far_log2, res):
    case, nodes = gate_case(res, (1, -1, -1) if far_log2 % 2 else (-1, 1, 1), seed=far_log2, far=2.0 ** far_log2)
    assert (gate_quantity(nodes, case) > FX_RANGE).all()
    assert (np.abs(nodes["pos"][:, :3]) * 100 < 2 ** 31 - 1e6).all()  # lattice ids fit int32
    run_kernels(case, nodes)

# ---- 5. beyond the sample-time table in expand_fxn_kernel --------------------------------------------------
def beyond_case(seed=9, n=1001):
    """v_max <= 0, res = 1/32: n = max(5, ceil(max_v*T/res)) = 32*max_v, with x velocities around 4 m/s, so
    that primitives with n = 128 and n = 129 both occur."""
    from scenarios import box_map

    res = 1.0 / 32
    mdim = (400, 48, 48)
    origin = (-6.2519, -0.7371, -0.7613)
    grid = box_map(mdim, res, origin, n_boxes=30, edge_m=(0.2, 0.6), seed=seed)
    case = Case(3, ACC, product_set(*[u_values(ACC)] * 3), mdim, origin, res, grid=grid)
    rng = np.random.default_rng(seed)
    nodes = random_nodes(rng, n, case, (190, 16, 16), (210, 32, 32), centred=True)
    nodes["vel"][:, 0] = rng.choice([3.0, 4.0, 4.03125, -3.0, -4.0, -4.03125, 3.5, -4.5], n)
    nodes["vel"][:, 1:3] = rng.integers(-2, 3, (n, 2)) * 0.25
    return case, nodes

def sample_counts(case, nodes, orc):
    """n per emitted ACC primitive: max(5, ceil(max_v*T/res)), max_v = max over axes of |v| at 0 and T."""
    nU = case.nU
    parent = np.repeat(np.arange(nodes.size), nU)
    u = case.U[orc["action"]]
    v0 = nodes["vel"][parent][:, :case.dim]
    mv = np.maximum(np.abs(v0), np.abs(v0 + u * case.T)).max(1)
    return np.maximum(5, np.ceil(mv * case.T / case.res)).astype(np.int64)

def test_fxn_beyond_the_sample_table():
    case, nodes = beyond_case()
    orc, _ = run_kernels(case, nodes)
    em = emitted_mask(orc) & ~same_mask(orc, nodes, 3)
    n = sample_counts(case, nodes, orc)[em]
    assert (n == N_TABLE).sum() > 50 and (n == N_TABLE + 1).sum() > 50 and (n > N_TABLE + 1).sum() > 50
    assert (n < N_TABLE).sum() > 50
    cost = orc["cost"][em]
    assert np.isinf(cost[n > N_TABLE]).any() and np.isfinite(cost[n > N_TABLE]).any()

# ---- 6. ambiguous samples past bit 63: the full re-walk ------------------------------------------------
WALL = (65, 70)  # x cells of the wall, relative to the start cell

def full_case(seed=13, n=1001):
    """x velocity 3.5 m/s at res 0.05 (n = 70 or 90), z on a cell boundary with zero z velocity: every sample
    of a primitive with z control 0 is uncertain in z.  A wall of voxels at z = c0 (blocked) or the cell
    across the boundary (free) spans x cells [x0 + 65, x0 + 70): with x control 0 or +1 only samples
    k >= 64 reach it."""
    res = 0.05
    mdim = (160, 48, 24)
    origin = (-1.0313, -1.2077, -0.6191)
    case = Case(3, ACC, product_set(*[u_values(ACC)] * 3), mdim, origin, res)
    o = np.asarray(origin)
    rng = np.random.default_rng(seed)
    x0 = 20
    kz = 12
    nodes = np.zeros(n, dtype=ob.WAYPOINT_DTYPE)
    yk = rng.integers(18, 30, n)
    nodes["pos"][:, 0] = o[0] + (x0 + 0.5) * res
    nodes["pos"][:, 1] = o[1] + (yk + 0.5) * res
    nodes["pos"][:, 2] = boundary(o[2], res, kz)
    nodes["vel"][:, 0] = 3.5
    nodes["t"] = rng.integers(0, 3, n) * 1.0
    cz = int(ref_cell(nodes["pos"][0, 2], o[2], res))
    assert (ref_cell(nodes["pos"][:, 2], o[2], res) == cz).all()
    other = kz - 1 if cz == kz else kz
    # two y bands: the wall sits on the blocked side for y < 24 and on the free side above
    gx, gy = np.meshgrid(np.arange(x0 + WALL[0], x0 + WALL[1]), np.arange(0, mdim[1]), indexing="ij")
    gx, gy = gx.reshape(-1), gy.reshape(-1)
    gz = np.where(gy < 24, cz, other)
    case.grid[case.index(np.stack([gx, gy, gz], 1))] = 100
    return case, nodes, x0

def test_fxn_full_rewalk_past_bit_63():
    case, nodes, x0 = full_case()
    orc = case.oracle().expand(nodes, nthreads=NTHREADS)
    n_nodes, nU = nodes.size, case.nU
    em = emitted_mask(orc)
    parent = np.repeat(np.arange(n_nodes), nU)
    u = case.U[orc["action"]]
    glide = em & (u[:, 2] == 0.0) & (u[:, 0] >= 0.0)
    n = sample_counts(case, nodes, orc)
    assert ((n[glide] > 64) & (n[glide] <= N_TABLE)).all()
    # x of samples 0..63 stays a cell short of the wall, and the last sample is a cell inside it or past it
    # (x travel from the start, a cell centre: the wall begins WALL[0] - 0.5 cells away)
    v0 = nodes["vel"][parent][:, 0]
    x_at = lambda t: v0 * t + 0.5 * u[:, 0] * t ** 2
    wall_lo = (WALL[0] - 0.5) * case.res
    assert (x_at(63.0 / n * case.T)[glide] < wall_lo - case.res).all()
    assert (x_at((n - 1.0) / n * case.T)[glide] > wall_lo + case.res).all()
    band = nodes["pos"][parent][:, 1] < case.origin[1] + 24 * case.res
    # primitives that stay in their y band: blocked by a late sample, or set free by the full re-walk
    steady = glide & (u[:, 1] == 0.0)
    assert np.isinf(orc["cost"][steady & band]).all() and np.isfinite(orc["cost"][steady & ~band]).all()
    assert (steady & band).sum() > 500 and (steady & ~band).sum() > 500
    run_kernels(case, nodes, orc=orc)

# ---- 7. curr.pos == tn.pos with tn != curr -----------------------------------------------------------------
def same_case(seed=17, n=1001):
    """ACC nodes with vel = -u*T/2 for some u in U: the primitive of u ends where it started.  Starts in an
    occupied voxel, an unknown (-1) voxel, outside the map, and free."""
    from scenarios import box_map

    res = 0.15
    mdim = (61, 37, 29)
    origin = MAP3["origin"]
    grid = box_map(mdim, res, origin, n_boxes=10, edge_m=(3 * res, 10 * res), seed=seed)
    case = Case(3, ACC, product_set(*[u_values(ACC)] * 3), mdim, origin, res, grid=grid)
    rng = np.random.default_rng(seed)
    nodes = random_nodes(rng, n, case, 3, np.asarray(mdim) - 3, centred=True)
    # positions on a 1/64 m lattice, so that p0 - u/2 + u/2 == p0 whatever order the terms are added in
    nodes["pos"][:, :3] = np.round(nodes["pos"][:, :3] * 64) / 64
    ui = rng.integers(0, case.nU, n)
    ui = np.where(np.abs(case.U[ui]).sum(1) == 0, 0, ui)  # u = 0 gives tn == curr: not emitted
    nodes["vel"][:, :3] = -case.U[ui] * case.T / 2
    kind = np.arange(n) % 4  # 0 occupied, 1 unknown, 2 outside, 3 as drawn
    o = np.asarray(origin)
    cells = ref_cell(nodes["pos"][:, :3], o, res)
    case.grid[case.index(cells[kind == 0])] = 100
    case.grid[case.index(cells[kind == 1])] = -1
    out = kind == 2
    nodes["pos"][out, 0] = np.round((o[0] - (rng.integers(1, 20, out.sum()) + 0.5) * res) * 64) / 64
    return case, nodes, kind

def test_same_position_successors():
    case, nodes, kind = same_case()
    orc, _ = run_kernels(case, nodes)
    same = same_mask(orc, nodes, 3).reshape(nodes.size, -1)
    cost = orc["cost"].reshape(nodes.size, -1)
    for k in (0, 1, 2):
        rows = kind == k
        assert same[rows].sum() == rows.sum(), k  # exactly one per node
        assert np.isfinite(cost[rows][same[rows]]).all(), k
    em = emitted_mask(orc).reshape(nodes.size, -1)
    assert np.isinf(cost[(kind == 0)[:, None] & em & ~same]).all()
    assert np.isinf(cost[(kind == 2)[:, None] & em & ~same]).all()

# ---- 8. the input contract: ignored fields and signed zeros -----------------------------------------------
def contract_case(dim, control, seed=19, n=None, nan=True):
    """Garbage (and NaN) in every field the control does not read, a control set that is the negation of a
    product set (it holds -0.0), one axis holding both +0.0 and -0.0, and nodes with -0.0 fields."""
    from scenarios import box_map

    m = MAP2 if dim == 2 else MAP3
    res = m["res"]
    grid = box_map(m["mdim"], res, m["origin"], n_boxes=10, edge_m=(3 * res, 10 * res), seed=seed)
    vals = u_values(control)
    U = -product_set(*[vals] * dim)
    U[::2, dim - 1] = np.where(U[::2, dim - 1] == 0.0, 0.0, U[::2, dim - 1])  # +0.0 beside -0.0 on the last axis
    assert (np.signbit(U) & (U == 0)).any() and (~np.signbit(U) & (U == 0)).any()
    case = Case(dim, control, U, m["mdim"], m["origin"], res, grid=grid, v_max=2.5, a_max=3.0, j_max=6.0)
    rng = np.random.default_rng(seed)
    n = n or (2003 if dim == 2 else 701)
    nodes = random_nodes(rng, n, case, 2, np.asarray(m["mdim"]) - 2)
    order = ORDER[control]
    # -0.0 in read fields: exact zeros of some nodes become negative zeros
    for f in range(order):
        a = nodes[FIELDS[f]][:, :dim]
        neg = (a == 0.0) & (rng.random(a.shape) < 0.5)
        a[neg] = -0.0
        nodes[FIELDS[f]][:, :dim] = a
    garbage = lambda shape: np.where(rng.random(shape) < 0.2, np.nan if nan else 7.0,
                                     rng.uniform(-1e6, 1e6, shape))
    for f in range(4):
        lo = 0 if f >= order else dim
        if lo < 3:
            nodes[FIELDS[f]][:, lo:] = garbage((n, 3 - lo))
    nodes["yaw"] = garbage(n)
    return case, nodes

@pytest.mark.parametrize("dim,control", [(2, VEL), (2, ACC), (3, ACC), (3, JRK), (2, SNP)])
def test_ignored_fields_and_signed_zeros(dim, control):
    case, nodes = contract_case(dim, control, seed=10 * dim + control)
    orc, _ = run_kernels(case, nodes)
    # the inputs hold -0.0 where they are read; the same nodes with clean ignored fields give the same result
    read = np.concatenate([nodes[f][:, :dim] for f in FIELDS[:ORDER[control]]], 1)
    assert (np.signbit(read) & (read == 0)).any() or control == VEL
    em = emitted_mask(orc)
    clean = np.zeros_like(nodes)
    for f in FIELDS[:ORDER[control]]:
        clean[f][:, :dim] = nodes[f][:, :dim]
    clean["t"] = nodes["t"]
    c = case.oracle().expand(clean, nthreads=NTHREADS)
    same_array(c["count"], orc["count"], "count")
    same_array(c["succ"][em], orc["succ"][em], "succ", bits=True)
    same_array(c["cost"][em], orc["cost"][em], "cost", bits=True)
