"""An independent statement of the two map transforms, and its pin to the REFERENCE on the CPU.

`restate_potential` is MapPlanner::createMask + updatePotentialMap (src/mpl_planner/map_planner.cpp:286-391)
and `restate_region` is MapPlanner::setSearchRegion with MapUtil::rayTrace (map_planner.cpp:46-95,
map_util.h:103-134), written as literally as numpy allows: scatter with max(), the (int8_t) truncation of the
stencil, unknown cells, `map > 0` sources, the exponent, the source range with its clamps.  The libm calls are
the reference's (math.hypot / math.pow per stencil offset).

The case lists below are shared with tests/test_maps_paths_gpu.py, which compares the device with the
restatement bit for bit.  Here every case is compared with the reference itself (oracle/_ref, or its recorded
result), so device = restatement = reference holds case by case.  The exponent reaches the reference through
the driver's subclass (refp_update_potential_map_pow: `pow_` is protected and has no setter)."""
import math

import numpy as np
import pytest

import planner_bindings as pb
from reference_record import reference, same_array

ACC = 0x03
H_MAX = 100  # map_planner.h:104


# ---- the restatement ---------------------------------------------------------------------------------
def c_round(x):
    """std::round: half away from zero."""
    return int(math.copysign(math.floor(abs(x) + 0.5), x))


def float_to_int(pt, origin, res):
    """MapUtil::floatToInt, map_util.h:103-108."""
    return [c_round((p - o) / res - 0.5) for p, o in zip(pt, origin)]


def create_mask(dim, res, radius, pow_):
    """createMask, map_planner.cpp:286-320: [(offset, int8 value)]."""
    rn = math.ceil(radius[0] / res)
    mask = []
    if dim == 2:
        for n0 in range(-rn, rn + 1):
            for n1 in range(-rn, rn + 1):
                if math.hypot(n0, n1) > rn:
                    continue
                h = H_MAX * math.pow(1 - math.hypot(n0, n1) / rn, pow_)
                if h > 1e-3:
                    mask.append(((n0, n1, 0), int(h)))  # (int8_t)h truncates; h <= 100
    else:
        hn = math.ceil(radius[2] / res)
        for n0 in range(-rn, rn + 1):
            for n1 in range(-rn, rn + 1):
                for n2 in range(-hn, hn + 1):
                    if math.hypot(n0, n1) > rn:
                        continue
                    h = H_MAX * math.pow((1 - math.hypot(n0, n1) / rn) * (1 - abs(n2) / hn), pow_)
                    if h > 1e-3:
                        mask.append(((n0, n1, n2), int(h)))
    return mask


def source_box(dims, origin, res, range_, pos):
    """The [coord1, coord2) of updatePotentialMap, map_planner.cpp:327-343: the upper corner is clamped to
    dim - 1 and then used as an exclusive bound."""
    D = len(dims)
    lo, hi = [0] * D, list(dims)
    if range_ is not None and math.sqrt(sum(r * r for r in range_[:D])) > 0:
        lo = float_to_int([pos[k] - range_[k] for k in range(D)], origin, res)
        hi = float_to_int([pos[k] + range_[k] for k in range(D)], origin, res)
        for k in range(D):
            lo[k] = 0 if lo[k] < 0 else (dims[k] - 1 if lo[k] >= dims[k] else lo[k])
            hi[k] = 0 if hi[k] < 0 else (dims[k] - 1 if hi[k] >= dims[k] else hi[k])
    return lo, hi


def restate_potential(grid, dims, origin, res, radius, pow_=1.0, range_=None, pos=None):
    """updatePotentialMap: every cell with map > 0 inside the source box becomes H_MAX and stamps
    dmap = max(dmap, value) through the mask (isOutside cells skipped).  One shifted maximum per mask offset:
    max() commutes, so this is the reference's scatter in another order."""
    D = len(dims)
    nx, ny, nz = (list(dims) + [1])[:3]
    g = np.ascontiguousarray(grid, dtype=np.int8).reshape(nz, ny, nx)
    lo, hi = source_box(dims, origin, res, range_, pos)
    lo, hi = (lo + [0])[:3], (hi + [1])[:3]
    src = np.zeros((nz, ny, nx), dtype=bool)
    box = (slice(lo[2], max(lo[2], hi[2])), slice(lo[1], max(lo[1], hi[1])), slice(lo[0], max(lo[0], hi[0])))
    src[box] = g[box] > 0
    out = g.copy()
    out[src] = H_MAX
    if src.any():
        for (dx, dy, dz), val in create_mask(D, res, radius, pow_):
            if abs(dx) >= nx or abs(dy) >= ny or abs(dz) >= nz:
                continue
            s = src[max(0, -dz):nz - max(0, dz), max(0, -dy):ny - max(0, dy), max(0, -dx):nx - max(0, dx)]
            d = out[max(0, dz):nz - max(0, -dz), max(0, dy):ny - max(0, -dy), max(0, dx):nx - max(0, -dx)]
            np.maximum(d, np.where(s, np.int8(val), np.int8(-128)), out=d)
    return out.reshape(-1)


def ray_trace(p1, p2, dims, origin, res):
    """MapUtil::rayTrace, map_util.h:117-134."""
    D = len(dims)
    diff = [b - a for a, b in zip(p1, p2)]
    max_diff = int(max(abs(d / res) for d in diff) / 0.8)
    pns, prev = [], [-1] * D
    if max_diff < 2:
        return pns  # `for (n = 1; n < max_diff; n++)` does not run; s = 1.0 / max_diff (inf for 0) is unused
    s = 1.0 / max_diff
    step = [d * s for d in diff]
    for n in range(1, max_diff):
        pn = float_to_int([a + st * n for a, st in zip(p1, step)], origin, res)
        if any(c < 0 or c >= m for c, m in zip(pn, dims)):
            break
        if pn != prev:
            pns.append(pn)
        prev = pn
    return pns


def restate_region(path, dims, origin, res, radius, dense=False):
    """setSearchRegion, map_planner.cpp:46-95: one byte per voxel."""
    D = len(dims)
    path = [list(map(float, p)) for p in path]
    ps = []
    if not dense:
        for i in range(1, len(path)):
            ps += ray_trace(path[i - 1], path[i], dims, origin, res)
            ps.append(float_to_int(path[i], origin, res))
    else:
        ps = [float_to_int(p, origin, res) for p in path]
    rn = [math.ceil(radius[k] / res) for k in range(D)] + [0] * (3 - D)
    nx, ny, nz = (list(dims) + [1])[:3]
    reg = np.zeros((nz, ny, nx), dtype=np.uint8)
    for it in ps:
        c = (list(it) + [0])[:3]
        a = [c[k] - rn[k] for k in range(3)]
        b = [c[k] + rn[k] + 1 for k in range(3)]
        if any(b[k] <= 0 or a[k] >= (nx, ny, nz)[k] for k in range(3)):
            continue
        reg[max(0, a[2]):b[2], max(0, a[1]):b[1], max(0, a[0]):b[0]] = 1  # isOutside cells skipped
    return reg.reshape(-1)


# ---- the rank table's limit ----------------------------------------------------------------------------
def distinct_stencil_radii(rn):
    """Distinct values of 1 - hypot(i, j)/rn inside the disc: what mplx_update_potential_map ranks."""
    return len({1 - math.hypot(i, j) / rn for i in range(rn + 1) for j in range(rn + 1) if not math.hypot(i, j) > rn})


def largest_ranked_rn(limit=255):
    """Largest rn whose distinct-value count stays below `limit` while rn + 1 does not."""
    rn = 1
    while distinct_stencil_radii(rn + 1) < limit:
        rn += 1
    assert distinct_stencil_radii(rn) < limit <= distinct_stencil_radii(rn + 1)
    return rn


# ---- the reference with an exponent ------------------------------------------------------------------------
def reference_potential_map_pow(args, radius, pow_, n_cells, range_=None, pos=None):
    """MapPlanner::updatePotentialMap with createMask's exponent set (refp_update_potential_map_pow of
    oracle/ref_planner_driver.cpp).  A reference library built before that symbol existed counts as not built:
    the call is then served by its recording, as on a checkout without the reference sources."""
    import ctypes as C

    def exported():
        try:
            return hasattr(C.CDLL(str(pb.REF_PLANNER)), "refp_update_potential_map_pow")
        except OSError:
            return False

    def live():
        lib = C.CDLL(str(pb.REF_PLANNER))
        out = np.zeros(n_cells, dtype=np.int8)
        rad = np.asarray(radius, dtype=np.float64)
        rng = None if range_ is None else np.asarray(range_, dtype=np.float64)
        p = None if pos is None else np.asarray(pos, dtype=np.float64)
        fn = lib.refp_update_potential_map_pow
        fn.argtypes = [C.POINTER(pb.PlanArgs), C.c_void_p, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
        fn(C.byref(args), rad.ctypes.data, float(pow_), None if rng is None else rng.ctypes.data,
           None if p is None else p.ctypes.data, out.ctypes.data)
        return out

    library = pb.REF_PLANNER if pb.REF_PLANNER.exists() and exported() else pb.REF_PLANNER.with_name("not_built")
    return reference(library, live)


# ---- potential cases -----------------------------------------------------------------------------------
class PCase:
    def __init__(self, name, dims, res, rn, hn=None, pow_=1.0, grid="sparse", range_=None, pos=None, seed=0,
                 origin=None):
        self.name, self.dims, self.res, self.pow_ = name, tuple(dims), res, pow_
        D = len(dims)
        self.origin = tuple(origin) if origin is not None else (-1.0, 0.5, 0.25)[:D]
        # radii that are whole cells of a power-of-two resolution: ceil(radius/res) is rn / hn exactly
        self.radius = (rn * res, rn * res) if D == 2 else (rn * res, rn * res, hn * res)
        self.rn, self.hn = rn, hn
        self.range_, self.pos = range_, pos
        self.kind, self.seed = grid, seed

    def grid(self):
        n = int(np.prod(self.dims))
        rng = np.random.default_rng(1000 + self.seed)
        g = np.zeros(n, dtype=np.int8)
        if self.kind == "sparse":       # 2 % sources of value 100, some unknown cells
            g[rng.random(n) < 0.02] = 100
            g[rng.integers(0, n, max(1, n // 40))] = -1
        elif self.kind == "unknown":    # density 0: nothing to stamp, unknown cells stay
            g[rng.integers(0, n, max(1, n // 10))] = -1
        elif self.kind == "one":        # one source in a map of unknown cells: the (1e-3, 1) ring shows as 0
            g[:] = -1
            g[n // 2] = 37
        elif self.kind == "full":       # density 100 %
            g[:] = rng.integers(1, 100, n)  # below H_MAX: a cell reads 100 only where it was a source
        elif self.kind == "int8":       # every int8 value; 1..127 are sources, -128..0 are not
            g = np.where(rng.random(n) < 0.5, -1, 0).astype(np.int8)
            g[rng.permutation(n)[:256]] = np.arange(-128, 128).astype(np.int8)
        return g

    def ref_args(self, grid=None):
        D = len(self.dims)
        return pb.make_args(D, ACC, self.grid() if grid is None else grid, self.dims, self.origin, self.res,
                            np.zeros((1, D)), start=dict(pos=(0,) * D), goal=dict(pos=(0,) * D))

    def restate(self, grid=None):
        return restate_potential(self.grid() if grid is None else grid, self.dims, self.origin, self.res, self.radius,
                                 self.pow_, self.range_, self.pos)

    def reference(self, grid=None):
        return reference_potential_map_pow(self.ref_args(grid), self.radius, self.pow_, int(np.prod(self.dims)),
                                           self.range_, self.pos)


RN_MAX = largest_ranked_rn()


def potential_cases():
    c = []
    # exponent x dimension (gap 2), on maps whose rows start mid-word
    for p in (0.5, 1.0, 2.0, 3.0):
        c.append(PCase(f"2d_pow{p}", (45, 37), 0.25, 4, pow_=p, seed=1))
        c.append(PCase(f"3d_pow{p}", (37, 23, 6), 0.25, 4, 2, pow_=p, seed=2))
        c.append(PCase(f"2d_pow{p}_unknown_ring", (41, 39), 0.125, 16, pow_=p, grid="one", seed=3))
    # shape and radius classes (gap 3): windows of three words, rows starting mid-word, nx < 2 rn + 1, thin maps
    for rn in (1, 4, 16, 17):
        c.append(PCase(f"2d_rn{rn}_70x61", (70, 61), 0.25, rn, seed=4))
        c.append(PCase(f"3d_rn{rn}_67x35x3", (67, 35, 3), 0.25, rn, 1, seed=5))
    c.append(PCase("2d_aligned_64x32_rn16", (64, 32), 0.25, 16, seed=6))
    c.append(PCase("2d_narrow_5x40_rn4", (5, 40), 0.25, 4, seed=7))
    c.append(PCase("2d_narrow_40x5_rn17", (40, 5), 0.25, 17, seed=7))
    for dims in ((1, 37), (37, 1), (2, 3), (3, 2), (1, 1)):
        c.append(PCase(f"2d_thin_{dims[0]}x{dims[1]}", dims, 0.5, 4, grid="full" if dims == (1, 1) else "sparse", seed=8))
    c.append(PCase("2d_thin_3x33_dense", (3, 33), 0.5, 1, grid="full", seed=8))
    c.append(PCase("3d_nz1_hn2", (33, 31, 1), 0.25, 4, 2, seed=9))
    c.append(PCase("3d_hn_ge_nz", (35, 13, 7), 0.25, 4, 8, seed=10))
    c.append(PCase("3d_hn1", (33, 31, 3), 0.25, 4, 1, seed=11))  # 3069 voxels: nvox not a multiple of 32
    for dims in ((1, 1, 9), (2, 2, 2), (3, 1, 2), (1, 40, 3)):
        c.append(PCase("3d_thin_" + "x".join(map(str, dims)), dims, 0.5, 4, 2, grid="full" if dims == (2, 2, 2) else "sparse", seed=12))
    # the largest radius the rank table accepts (gap 4)
    c.append(PCase("2d_rn_max", (2 * RN_MAX + 9, 2 * RN_MAX + 3), 0.25, RN_MAX, seed=13))
    c.append(PCase("3d_rn_max_pow2", (RN_MAX + 9, RN_MAX + 3, 3), 0.25, RN_MAX, 1, pow_=2.0, seed=14))
    # source classes and densities (gap 5)
    for kind in ("unknown", "one", "full", "int8"):
        c.append(PCase(f"2d_{kind}", (45, 37), 0.25, 4, grid=kind, seed=15))
        c.append(PCase(f"3d_{kind}_pow2", (21, 19, 5), 0.25, 4, 2, pow_=2.0, grid=kind, seed=16))
    c.append(PCase("2d_int8_pow3_rn16", (70, 61), 0.25, 16, pow_=3.0, grid="int8", seed=17))
    return c


def range_cases():
    """Source ranges (gap 6).  Maps of 40 x 30 (x 6) cells of 0.25 m at origin (-1, 0.5, 0.25), every cell a source."""
    c = []
    d2, d3 = (40, 30), (40, 30, 6)
    for name, rng, pos in (("inside", (2.0, 1.5), (4.0, 4.0)),
                           ("upper_clamp", (3.0, 2.0), (8.0, 7.0)),        # pos + range beyond the map: dim - 1, exclusive
                           ("lower_clamp", (3.0, 2.0), (-0.5, 1.0)),
                           ("zero_on_y", (2.0, 0.0), (4.0, 4.0)),           # lo == hi on one axis: empty
                           ("pos_outside_high", (1.0, 1.0), (30.0, 30.0)),  # both corners clamp to dim - 1: empty
                           ("pos_outside_low", (1.0, 1.0), (-30.0, -30.0)),
                           ("whole_map_and_more", (100.0, 100.0), (4.0, 4.0)),
                           ("on_cell_boundaries", (1.0, 0.75), (4.0, 4.25)),
                           ("zero_range", (0.0, 0.0), (4.0, 4.0))):         # norm 0: the whole map
        c.append(PCase("2d_range_" + name, d2, 0.25, 2, grid="full", range_=rng, pos=pos, seed=20))
    for name, rng, pos in (("inside", (2.0, 1.5, 0.5), (4.0, 4.0, 1.0)),
                           ("upper_clamp", (3.0, 2.0, 1.0), (8.0, 7.0, 1.5)),
                           ("zero_on_z", (2.0, 1.5, 0.0), (4.0, 4.0, 1.0)),
                           ("pos_outside", (1.0, 1.0, 1.0), (4.0, 4.0, 9.0)),
                           ("whole_map_and_more", (100.0, 100.0, 100.0), (4.0, 4.0, 1.0))):
        c.append(PCase("3d_range_" + name, d3, 0.25, 2, 1, grid="full", range_=rng, pos=pos, seed=21))
    return c


POTENTIAL = {c.name: c for c in potential_cases() + range_cases()}
assert len(POTENTIAL) == len(potential_cases() + range_cases())

# the one larger map: the layer-wise scipy statement (scenarios.potential_from_map) is its second witness
BIG = dict(dims=(256, 256, 64), origin=(-12.8, -12.8, -3.2), res=0.1, radius=(1.0, 1.0, 1.0), n_boxes=60, edge_m=(0.5, 3.0))


def big_grid():
    import scenarios as S

    return S.box_map(BIG["dims"], BIG["res"], BIG["origin"], BIG["n_boxes"], BIG["edge_m"], seed=5)


# ---- search-region cases ---------------------------------------------------------------------------------
class RCase:
    def __init__(self, name, dims, origin, res, path, radius, dense=False):
        self.name, self.dims, self.origin, self.res = name, tuple(dims), tuple(origin), res
        self.path, self.radius, self.dense = np.asarray(path, dtype=np.float64), tuple(radius), dense

    def ref_args(self):
        D = len(self.dims)
        return pb.make_args(D, ACC, np.zeros(int(np.prod(self.dims)), np.int8), self.dims, self.origin, self.res,
                            np.zeros((1, D)), start=dict(pos=(0,) * D), goal=dict(pos=(0,) * D))

    def restate(self):
        return restate_region(self.path, self.dims, self.origin, self.res, self.radius, self.dense)

    def reference(self):
        return pb.reference_search_region(self.ref_args(), self.path, self.radius, int(np.prod(self.dims)), self.dense)


def region_cases():
    c = []
    d2, o2, d3, o3, res = (45, 37), (-1.0, 0.5), (37, 23, 11), (-1.0, 0.5, 0.25), 0.25
    paths2 = dict(
        one_point=[[3.0, 4.0]],
        repeated=[[3.0, 4.0], [3.0, 4.0], [3.0, 4.0]],                        # max_diff = 0, s = inf
        short=[[3.0, 4.0], [3.1, 4.05], [3.15, 4.2], [3.3, 4.3]],              # segments under 0.8 cells
        starts_outside=[[-3.0, 4.0], [3.0, 4.0], [5.0, 6.0]],                  # the ray breaks at once, the end cell stays
        leaves=[[3.0, 4.0], [30.0, 4.5], [4.0, 8.0]],
        on_boundaries=[[0.0, 1.5], [2.25, 3.75], [5.0, 3.75], [5.0, 8.0]],     # origin + k res exactly
        long=[[-0.5, 1.0], [9.5, 9.0], [0.0, 9.2], [10.0, 0.7]])
    for name, p in paths2.items():
        for dense in (False, True):
            c.append(RCase(f"2d_{name}_{'dense' if dense else 'sparse'}", d2, o2, res, p, (0.5, 0.3), dense))
    c.append(RCase("2d_radius0", d2, o2, res, paths2["long"], (0.0, 0.0)))
    c.append(RCase("2d_radius_over_map", d2, o2, res, paths2["short"], (20.0, 20.0)))
    c.append(RCase("2d_radius_one_axis", d2, o2, res, paths2["long"], (0.0, 1.1)))
    paths3 = dict(
        one_point=[[3.0, 4.0, 1.0]],
        repeated=[[3.0, 4.0, 1.0], [3.0, 4.0, 1.0]],
        short=[[3.0, 4.0, 1.0], [3.1, 4.05, 1.1], [3.15, 4.2, 1.15]],
        starts_outside=[[3.0, 4.0, -2.0], [3.0, 4.0, 1.0], [5.0, 5.0, 2.5]],
        on_boundaries=[[0.0, 1.5, 0.5], [2.25, 3.75, 1.25], [5.0, 3.75, 2.75]],
        long=[[-0.5, 1.0, 0.5], [7.5, 6.0, 2.8], [0.0, 6.0, 0.3]])
    for name, p in paths3.items():
        for dense in (False, True):
            c.append(RCase(f"3d_{name}_{'dense' if dense else 'sparse'}", d3, o3, res, p, (0.5, 0.3, 0.25), dense))
    c.append(RCase("3d_radius0", d3, o3, res, paths3["long"], (0.0, 0.0, 0.0)))
    c.append(RCase("3d_radius_over_map", d3, o3, res, paths3["short"], (20.0, 20.0, 20.0)))
    return c


REGION = {c.name: c for c in region_cases()}


# ---- the pins ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(POTENTIAL))
def test_potential_restatement_matches_reference(name):
    case = POTENTIAL[name]
    same_array(case.restate(), case.reference(), name)


def test_potential_restatement_twice_matches_reference_twice():
    """A second updatePotentialMap on the same planner takes the field's positive cells as sources."""
    for name in ("2d_pow2.0", "3d_pow0.5", "2d_int8"):
        case = POTENTIAL[name]
        once = case.restate()
        same_array(case.restate(once), case.reference(once), name)


def test_range_cases_lose_a_row_to_the_clamp_and_can_be_empty():
    """The expected [lo, hi) from the rule: the clamped upper corner is exclusive, so a range that reaches past the
    map stops one row short of its edge; a range that is zero on an axis is empty."""
    boxes = {c.name: source_box(c.dims, c.origin, c.res, c.range_, c.pos) for c in range_cases()}
    assert boxes["2d_range_upper_clamp"][1] == [39, 29] and boxes["3d_range_upper_clamp"][1][:2] == [39, 29]
    assert boxes["2d_range_whole_map_and_more"] == ([0, 0], [39, 29])
    assert boxes["2d_range_zero_range"] == ([0, 0], [40, 30])
    for empty in ("2d_range_zero_on_y", "2d_range_pos_outside_high", "2d_range_pos_outside_low", "3d_range_zero_on_z",
                  "3d_range_pos_outside"):
        lo, hi = boxes[empty]
        assert any(h <= l for l, h in zip(lo, hi)), empty
        c = POTENTIAL[empty]
        np.testing.assert_array_equal(c.restate(), c.grid())  # no source: the grid comes back as it was
    c = POTENTIAL["2d_range_upper_clamp"]
    f = c.restate().reshape(30, 40)
    assert (f[:, 39] < 100).all() and (f[29, :] < 100).all() and f[28, 38] == 100  # the last row and column only get stamped


def test_source_classes_are_present():
    g = POTENTIAL["2d_int8"].grid()
    assert len(np.unique(g)) == 256
    c = POTENTIAL["2d_pow3.0_unknown_ring"]
    f, g = c.restate(), c.grid()
    assert ((g == -1) & (f == 0)).any(), "stencil values in (1e-3, 1) turn unknown cells into 0"
    assert ((g == -1) & (f == -1)).any() and (f == 100).sum() == 1
    assert any(v == 0 for _, v in create_mask(2, c.res, c.radius, c.pow_))


def test_rank_table_limit_is_computed():
    assert distinct_stencil_radii(RN_MAX) < 255 <= distinct_stencil_radii(RN_MAX + 1) and RN_MAX > 17


def test_stencil_extension_keeps_scenarios_results():
    """scenarios.potential_from_map_stencil (3-D, grids without unknown cells) is this restatement's special case."""
    import scenarios as S

    rng = np.random.default_rng(4)
    dims, res, rad = (21, 19, 9), 0.25, (1.0, 1.0, 0.5)
    g = (rng.random(int(np.prod(dims))) < 0.03).astype(np.int8) * 100
    for p in (1.0, 2.0):
        np.testing.assert_array_equal(restate_potential(g, dims, (0, 0, 0), res, rad, p),
                                      S.potential_from_map_stencil(g, dims, res, rad, p))


def test_big_map_layerwise_statement_matches_reference():
    import scenarios as S

    g = big_grid()
    args = pb.make_args(3, ACC, g, BIG["dims"], BIG["origin"], BIG["res"], np.zeros((1, 3)), start=dict(pos=(0, 0, 0)),
                        goal=dict(pos=(0, 0, 0)))
    same_array(S.potential_from_map(g, BIG["dims"], BIG["res"], BIG["radius"]),
               pb.reference_potential_map(args, BIG["radius"], g.size))


@pytest.mark.parametrize("name", sorted(REGION))
def test_region_restatement_matches_reference(name):
    case = REGION[name]
    same_array(case.restate(), case.reference(), name)


def test_region_cases_cover_their_classes():
    r = {n: c.restate() for n, c in REGION.items()}
    assert r["2d_one_point_sparse"].sum() == 0 and r["3d_one_point_sparse"].sum() == 0  # no segment: no cell
    assert r["2d_one_point_dense"].sum() == 5 * 5 and r["3d_one_point_dense"].sum() == 5 * 5 * 3
    assert r["2d_radius0"].sum() > 20 and r["2d_radius_over_map"].all() and r["3d_radius_over_map"].all()
    assert 0 < r["2d_starts_outside_sparse"].sum() < r["2d_long_sparse"].sum()
    assert ray_trace(*REGION["2d_repeated_sparse"].path[:2], (45, 37), (-1.0, 0.5), 0.25) == []
