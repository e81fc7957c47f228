"""mplx_update_cells (csrc/mplx_update.cu: scatter_last_kernel, repack_occ_kernel, repack_occ2_kernel) and the
read-back mplx_read_map (unbrick_occ2_kernel) on every shape class, constructed edit pattern, value class and
upload path.

After every call the device is checked against two witnesses: the numpy restatement of tests/update_restatement.py
(pinned to the header's word rules by tests/test_update_restatement_cpu.py, and sharing no code with the kernels),
and a fresh ctx given the final grid.  The read-back must be bit-equal to both, the grid must be stored verbatim
and the Python MapUtil must have been edited in place.  The patterns aim at the brick geometry the re-pack relies
on: single voxels at every brick and pair boundary class, sorted runs that end at a brick row's end or wrap into
the next row or plane, a set and a later clear that must turn summary bits back to 0, duplicates presented
sorted, unsorted and descending.  Also here: a map of more than 2^30 voxels, launch counts, refusals, the
consumers after edits at brick edges, and the BatchPlanner's choice between a sparse and a full upload."""
import ctypes as C
import zlib

import numpy as np
import pytest

import oracle_bindings as ob
import update_restatement as R
from parity import assert_expansion_equal
from update_restatement import SHAPES, shape_dims

pytestmark = pytest.mark.gpu
ACC = 0x03
UPDATE_LAUNCHES = 3  # scatter_last_kernel, repack_occ_kernel, repack_occ2_kernel (the radix sort is not counted)
READ_OCC2_LAUNCHES = 1  # unbrick_occ2_kernel
VALUES = np.array([100, 0, -1, 1, 99, 101, 127, -128], dtype=np.int8)
FREE = VALUES[1:]  # every value class that is not occupied
SMALL = 70_000  # maps up to this many voxels also get a call that edits every voxel


def make_env(grid, dims, origin=None, res=0.1):
    from motion_primitive_library_b200 import MapUtil, env_map

    mu = MapUtil()
    mu.setMap((0.0,) * len(dims) if origin is None else origin, dims, np.array(grid, dtype=np.int8), res)
    return env_map(mu)


def apply(ref, idx, vals):
    """grid[idx[k]] = vals[k] in array order: the later entry for a voxel wins"""
    idx = np.asarray(idx, dtype=np.int64).reshape(-1)
    vals = np.asarray(vals, dtype=np.int8).reshape(-1)
    u, first = np.unique(idx[::-1], return_index=True)
    ref[u] = vals[::-1][first]


def masks(dims):
    """(x, y, z) masks of a brick row, a brick's y extent and its z extent"""
    return (7, 7, 7) if len(dims) == 3 else (31, 15, 0)


def end_bit(nvox):
    """the bits the radix sort must compare: the fewest that hold nvox - 1"""
    return max(1, int(nvox - 1).bit_length())


class Session:
    """A ctx under edit and the grid it must hold."""

    def __init__(self, grid, dims, origin=None, res=0.1):
        self.dims = dims
        self.nvox = R.nvox_of(dims)
        self.ref = np.array(grid, dtype=np.int8).reshape(-1)
        self.env = make_env(self.ref, dims, origin, res)
        self.calls = 0

    def update(self, idx, vals, what=""):
        idx = np.asarray(idx, dtype=np.int64).reshape(-1)
        vals = np.broadcast_to(np.asarray(vals, dtype=np.int8), idx.shape)
        before = self.env.launch_count()
        self.env.update_cells(idx, vals)
        assert self.env.launch_count() - before == (UPDATE_LAUNCHES if idx.size else 0), what
        apply(self.ref, idx, vals)
        self.calls += 1
        self.check(what)

    def check(self, what=""):
        env, ref, dims = self.env, self.ref, self.dims
        got = env.read_map()
        _, occ_r, pairs_r = R.views(ref, dims)
        fresh = make_env(ref, dims)
        want = fresh.read_map()
        fresh.close()
        assert got[0].tobytes() == ref.tobytes(), (what, "grid")
        assert env.map_util_.map.tobytes() == ref.tobytes(), (what, "MapUtil")
        for name, g, r, f in (("occupancy words", got[1], occ_r, want[1]), ("pair words", got[2], pairs_r, want[2])):
            bad = np.flatnonzero((g.reshape(len(g), -1) != r.reshape(len(r), -1)).any(1))
            if bad.size:
                w = int(bad[0])
                diff = (g.reshape(len(g), -1)[w] ^ r.reshape(len(r), -1)[w])
                b = [i for i in range(32) if any((int(d) >> i) & 1 for d in diff)]
                raise AssertionError(f"{what}: {name} differ from the restatement in {bad.size} words; word {w} "
                                     f"bits {b}: voxels {[R.coords(32 * w + i, dims) for i in b[:3]]}")
            assert g.tobytes() == f.tobytes(), (what, name, "fresh ctx")

    def close(self):
        self.env.close()


# ---- the constructed edit patterns ------------------------------------------------------------------
def axis_classes(n, mask, rems):
    """coordinates c < n with c & mask in rems, in the first two bricks and the last one, and 0, n - 1"""
    out = {0, n - 1}
    for base in (0, mask + 1, (n - 1) & ~mask):
        out |= {base + r for r in rems if 0 <= base + r < n}
    return sorted(out)


def vid(dims, x, y, z=0):
    v = np.asarray(x, np.int64) + dims[0] * (np.asarray(y, np.int64) + dims[1] * np.asarray(z, np.int64))
    return int(v) if v.ndim == 0 else v


def position_voxels(dims):
    """single voxels at every position class: x & mask in {0, 1, mask-1, mask} and x in {0, nx-1}; y at pair and
    brick boundaries; z at brick boundaries; the corners; voxel 0, the last voxel and the last partial word"""
    mx, my, mz = masks(dims)
    nx, ny = dims[0], dims[1]
    nz = dims[2] if len(dims) == 3 else 1
    xs = axis_classes(nx, mx, (0, 1, mx - 1, mx))
    ys = axis_classes(ny, my, (0, 1, 3, 4, 6, 7) if len(dims) == 3 else (0, 1, 14, 15))
    zs = axis_classes(nz, mz, (0, 1, 6, 7)) if len(dims) == 3 else [0]
    x0, y0, z0 = xs[len(xs) // 2], ys[len(ys) // 2], zs[len(zs) // 2]
    v = [vid(dims, x, y0, z0) for x in xs] + [vid(dims, x0, y, z0) for y in ys] + [vid(dims, x0, y0, z) for z in zs]
    v += [vid(dims, x, y, z) for x in (0, nx - 1) for y in (0, ny - 1) for z in (0, nz - 1)]
    nvox = R.nvox_of(dims)
    last = (nvox // 32) * 32
    v += [0, nvox - 1] + ([last, (last + nvox - 1) // 2] if last < nvox else [])
    return list(dict.fromkeys(v))


def x_runs(dims):
    """sorted runs along x: every start class to every end class in one row; runs across the row end into the next
    row and across the plane end into the next plane; stride-2 runs, where the skip rule never fires"""
    mx, _, _ = masks(dims)
    nx, ny = dims[0], dims[1]
    nz = dims[2] if len(dims) == 3 else 1
    nvox = R.nvox_of(dims)
    xs = axis_classes(nx, mx, (0, 1, mx - 1, mx))
    y0, z0 = ny // 2, nz // 2
    runs = [np.arange(vid(dims, s, y0, z0), vid(dims, e, y0, z0) + 1) for s in xs if s < 2 * (mx + 1) for e in xs
            if e > s]
    row_end = vid(dims, nx - 1, y0, z0)
    plane_end = vid(dims, nx - 1, ny - 1, max(0, z0 - 1))
    for end in (row_end, plane_end):
        for a, b in ((0, 1), (1, 2), (mx, mx + 2), (nx + 1, 3)):
            runs.append(np.arange(max(0, end - a), min(nvox, end + b + 1)))
    runs.append(np.arange(vid(dims, 0, y0, z0), min(nvox, vid(dims, 0, y0, z0) + 2 * nx + 3), 2))
    runs.append(np.arange(vid(dims, 1, y0, z0) if nx > 1 else 1, min(nvox, vid(dims, 0, y0, z0) + 3 * nx), 2))
    runs.append(np.arange(max(0, nvox - 40), nvox))
    return [r for r in runs if r.size]


def case_singles(s, rng):
    for v in position_voxels(s.dims):
        s.update([v], [100], f"single {R.coords(v, s.dims)}")


def case_set_clear(s, rng):
    """on a map with nothing occupied: occupy one voxel (the only occupied voxel of its successors' boxes), then
    clear it in a later call; its successors' summary bits go 1 and back to 0"""
    for k, v in enumerate(position_voxels(s.dims)):
        succ = R.successors(v, s.dims)
        x, y, z = R.coords(np.asarray(succ), s.dims)
        inner = np.asarray(succ)[(x > 0) & (y > 0) & (z > 0 if len(s.dims) == 3 else True)]
        s.update([v], [100], f"set {R.coords(v, s.dims)}")
        assert summary_bits(s.env, inner).all()
        s.update([v], [FREE[k % FREE.size]], f"clear {R.coords(v, s.dims)}")
        assert not summary_bits(s.env, inner).any(), (v, inner)


def summary_bits(env, vs):
    pairs = env.read_map()[2]
    return np.array([(int(pairs[v >> 5, 1]) >> (v & 31)) & 1 for v in vs], dtype=bool)


def case_runs(s, rng):
    for k, r in enumerate(x_runs(s.dims)):
        s.update(r, [100], f"run {r[0]}..{r[-1]} step {r[1] - r[0] if r.size > 1 else 1}")
        s.update(r, [FREE[k % FREE.size]], f"clear run {r[0]}..{r[-1]}")


def case_duplicates(s, rng):
    """duplicates within one call with different values, presented sorted (the host's presorted path), unsorted
    (the radix sort) and descending; the later entry in array order wins"""
    nvox = s.nvox
    for order in ("sorted", "unsorted", "descending"):
        base = rng.integers(0, nvox, min(200, 2 * nvox))
        idx = np.repeat(base, rng.integers(1, 5, base.size))
        if order == "sorted":
            idx = np.sort(idx, kind="stable")
        elif order == "descending":
            idx = np.sort(idx, kind="stable")[::-1]
        else:
            idx = rng.permutation(idx)
        s.update(idx, VALUES[rng.integers(0, VALUES.size, idx.size)], f"duplicates {order}")
    # one window written in descending order, pass after pass: only the last pass may win
    w = np.arange(max(0, nvox // 2 - 32), min(nvox, nvox // 2 + 32))[::-1]
    passes = 48
    vals = np.concatenate([np.full(w.size, FREE[p % FREE.size] if p % 2 else 100, np.int8) for p in range(passes)])
    s.update(np.tile(w, passes), vals, "descending passes")
    # the radix sort must compare bit end_bit - 1: X and X - 2^(end_bit - 1) agree below it.  Each X is written
    # twice, 33 entries apart, with its alias in between; the second write must win.
    hi = 1 << (end_bit(nvox) - 1)
    xs = np.arange(hi, nvox)[:64]
    if xs.size and nvox > 1:
        groups = [np.concatenate([[x], np.full(33, x - hi), [x]]) for x in xs]
        gv = [np.concatenate([[0], np.full(33, 1), [100]]).astype(np.int8) for _ in xs]
        perm = rng.permutation(len(groups))
        s.update(np.concatenate([groups[p] for p in perm]), np.concatenate([gv[p] for p in perm]), "aliases")


def case_sizes(s, rng):
    s.update(np.zeros(0, np.int64), np.zeros(0, np.int8), "n = 0")
    for v in (0, s.nvox - 1, s.nvox // 2):
        s.update([v], [VALUES[v % VALUES.size]], f"n = 1 at {v}")
    if s.nvox <= SMALL:
        idx = rng.permutation(s.nvox)
        s.update(idx, VALUES[rng.integers(0, VALUES.size, idx.size)], "n = nvox, random order")
        s.update(np.arange(s.nvox), np.where(rng.random(s.nvox) < 0.2, 100, 0).astype(np.int8), "n = nvox, in order")


CASES = {"singles": case_singles, "set_clear": case_set_clear, "runs": case_runs, "duplicates": case_duplicates,
         "sizes": case_sizes}


def background(dims, case, rng):
    n = R.nvox_of(dims)
    free = FREE[rng.integers(0, FREE.size, n)]
    if case in ("set_clear", "runs"):
        return free  # nothing occupied: every summary bit an edit sets is visible, and so is a stale one
    return np.where(rng.random(n) < 0.1, 100, free).astype(np.int8)


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("shape", list(SHAPES))
def test_edit_pattern(shape, case):
    dims = shape_dims(shape)
    rng = np.random.default_rng(zlib.crc32(f"{shape}/{case}".encode()))
    s = Session(background(dims, case, rng), dims)
    s.check("initial")
    CASES[case](s, rng)
    assert s.calls > 0
    s.close()


# ---- duplicates that a wrong order splits apart ---------------------------------------------------------------
def test_split_duplicates_keep_the_last_entry():
    """A voxel's entries must end up adjacent after the host's order check and the radix sort, or several threads of
    scatter_last_kernel store to its byte and any of them may land.  Two calls make many voxels depend on that:
    each voxel is written several times, from different warps, and only its last entry is occupied.
    * radix path: X in the upper half of the id range is written 8 times, each time followed by 32 entries of its
      alias X - 2^(end_bit - 1), which agrees with X on every bit but the top one the sort must compare;
    * windows of 64 voxels written in descending order, 16 passes each: every adjacent pair ascends or descends by
      one, so a presorted check that accepted a descending pair would skip the sort.
    The counts of voxels holding an earlier entry's value are reported, so a wrong order shows how often it wins."""
    dims = (64, 64, 64)
    nvox = R.nvox_of(dims)
    hi = 1 << (end_bit(nvox) - 1)
    rng = np.random.default_rng(77)
    s = Session(np.zeros(nvox, np.int8), dims)
    xs = rng.choice(np.arange(hi, nvox), 2048, replace=False)
    writes, gap = 8, 32
    group = lambda x: np.concatenate([np.r_[x, np.full(gap, x - hi)]] * (writes - 1) + [[x]])
    gvals = np.concatenate([np.r_[0, np.full(gap, 1)]] * (writes - 1) + [[100]]).astype(np.int8)
    radix_idx = np.concatenate([group(x) for x in xs])
    radix_vals = np.tile(gvals, xs.size)
    starts = np.sort(rng.choice(np.arange(0, nvox // 64), 64, replace=False)) * 64
    passes = 16
    desc = np.concatenate([np.tile(np.arange(a + 63, a - 1, -1), passes) for a in starts])
    desc_vals = np.tile(np.repeat(np.r_[np.zeros(passes - 1), 100].astype(np.int8), 64), starts.size)
    for what, idx, vals, last in (("alias groups (radix path)", radix_idx, radix_vals, xs),
                                  ("descending passes", desc, desc_vals, np.unique(desc))):
        s.env.update_cells(idx, vals)
        apply(s.ref, idx, vals)
        wrong = int((s.env.read_map()[0][last] != 100).sum())
        assert wrong == 0, f"{what}: {wrong} of {last.size} voxels hold an earlier entry's value"
        s.check(what)
    s.close()


# ---- launches and NULL outputs --------------------------------------------------------------------------
def test_read_map_outputs_and_launches():
    """every subset of NULL outputs is accepted; the unbrick kernel runs exactly when occ2 is requested"""
    dims = (17, 15, 9)
    rng = np.random.default_rng(3)
    s = Session(np.where(rng.random(R.nvox_of(dims)) < 0.2, 100, -1).astype(np.int8), dims)
    s.update(rng.integers(0, s.nvox, 300), [100], "edits")
    grid_r, occ_r, pairs_r = R.views(s.ref, dims)
    lib, h = s.env._lib, s.env.handle
    nw = (s.nvox + 31) // 32
    for mask in range(8):
        g, o, p = np.full(s.nvox, 7, np.int8), np.full(nw, 7, np.uint32), np.full((nw, 2), 7, np.uint32)
        ptrs = [a.ctypes.data if mask >> k & 1 else None for k, a in enumerate((g, o, p))]
        before = s.env.launch_count()
        assert lib.mplx_read_map(h, *ptrs) == 0
        assert s.env.launch_count() - before == (READ_OCC2_LAUNCHES if mask & 4 else 0), mask
        for k, (a, r) in enumerate(((g, grid_r), (o, occ_r), (p, pairs_r))):
            if mask >> k & 1:
                assert a.tobytes() == r.tobytes(), (mask, k)
            else:
                assert (a == 7).all(), (mask, k)  # not written
    s.close()


def test_update_before_set_map_is_refused():
    from motion_primitive_library_b200 import abi

    lib = abi.load()
    for dim in (2, 3):
        h = C.c_void_p()
        abi.check(lib.mplx_create(dim, 0, C.byref(h)))
        try:
            idx, val = np.array([0], np.int32), np.array([100], np.int8)
            assert lib.mplx_update_cells(h, idx.ctypes.data, val.ctypes.data, 1) == abi.MPLX_ERR_ARG
            assert b"mplx_set_map" in lib.mplx_last_error()
            assert lib.mplx_read_map(h, None, None, None) == abi.MPLX_ERR_ARG  # still no map
            assert lib.mplx_launch_count(h) == 0
        finally:
            lib.mplx_destroy(h)


# ---- a map of more than 2^30 voxels ------------------------------------------------------------------------
BIG = (1024, 1024, 1025)  # 1 074 790 400 voxels: ids need 31 bits


def host_available():
    """MemAvailable of /proc/meminfo in bytes (unlimited where it cannot be read)"""
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) << 10
    except OSError:
        pass
    return 1 << 62


def device_free():
    import torch

    return torch.cuda.mem_get_info(0)[0]


def test_large_indices():
    """ids above 2^30 through the radix path (end_bit = 31) and the presorted path; the grid and the occupancy words
    in full, the pair words against a fresh ctx in full and against the restatement within reach of the edits."""
    from motion_primitive_library_b200 import abi

    dims = BIG
    nvox = R.nvox_of(dims)
    assert (1 << 30) < nvox < (1 << 31) and end_bit(nvox) == 31
    need_host, need_dev = 6 << 30, 4 << 30  # measured peaks: about 5 GB of host and 3.5 GB of device memory
    if host_available() < need_host or device_free() < need_dev:
        pytest.skip(f"needs {need_host >> 30} GB of free host and {need_dev >> 30} GB of free device memory")
    nx, sxy = dims[0], dims[0] * dims[1]
    rng = np.random.default_rng(30)
    ref = np.zeros(nvox, np.int8)
    ref[rng.integers(0, nvox, 200_000)] = 100
    env = make_env(ref, dims)
    hi = 1 << 30
    # radix path: unsorted, above and below 2^30, duplicates with different values, X next to its alias X - 2^30
    top = np.arange(hi, nvox, 4099)
    alias = rng.choice(top, 50, replace=False)
    groups = np.concatenate([np.concatenate([[x], np.full(33, x - hi), [x]]) for x in alias])
    gvals = np.tile(np.concatenate([[0], np.full(33, 100), [100]]).astype(np.int8), alias.size)
    rnd = np.concatenate([rng.integers(hi, nvox, 20_000), rng.integers(0, hi, 5_000)])
    rnd = np.concatenate([rnd, rnd[:3000]])
    idx1 = np.concatenate([groups, rng.permutation(rnd)])
    val1 = np.concatenate([gvals, VALUES[rng.integers(0, VALUES.size, rnd.size)]])
    # presorted path: runs across brick rows in the last plane, the 2^30 boundary, and the last voxel
    z = dims[2] - 1
    runs = [np.arange(hi - 40, hi + 40), np.arange(5 + nx * 9 + sxy * z, 40 + nx * 9 + sxy * z),
            np.arange(nvox - nx - 9, nvox)]
    idx2 = np.concatenate(runs)
    idx2 = np.sort(np.concatenate([idx2, idx2[::7]]), kind="stable")
    val2 = VALUES[rng.integers(0, VALUES.size, idx2.size)]
    lib, h = env._lib, env.handle
    for idx, val in ((idx1, val1), (idx2, val2)):
        before = env.launch_count()
        env.update_cells(idx, val)
        assert env.launch_count() - before == UPDATE_LAUNCHES
        apply(ref, idx, val)
    touched = np.concatenate([idx1, idx2])
    # refusal: an index equal to nvox; nothing applied, no launch
    before = env.launch_count()
    bad = np.array([5, nvox - 1, nvox], np.int32)
    vals = np.full(3, 100, np.int8)
    assert lib.mplx_update_cells(h, bad.ctypes.data, vals.ctypes.data, 3) == abi.MPLX_ERR_ARG
    assert b"outside" in lib.mplx_last_error() and env.launch_count() == before

    got = env.read_map()
    assert same(got[0], ref), "grid"
    assert same(env.map_util_.map, ref), "MapUtil"
    del got
    occ_full = np.packbits(ref == 100, bitorder="little")
    occ_full = np.concatenate([occ_full, np.zeros((-occ_full.size) % 4, np.uint8)]).view("<u4")
    g2, o2, p2 = env.read_map()
    del g2
    assert o2.tobytes() == occ_full.tobytes(), "occupancy words"
    del occ_full
    words = R.reach_words(touched, dims)
    occ_r, pairs_r = R.views_at(ref, dims, words)
    assert o2[words].tobytes() == occ_r.tobytes()
    bad_w = np.flatnonzero((p2[words] != pairs_r).any(1))
    assert bad_w.size == 0, ("pair words within reach of the edits", words[bad_w[:8]])
    env.close()
    del env
    fresh = make_env(ref, dims)
    del ref
    assert p2.tobytes() == fresh.read_map()[2].tobytes(), "pair words against a fresh ctx"
    fresh.close()


def same(a, b, chunk=1 << 26):
    """a == b without a temporary of the map's size"""
    return a.size == b.size and all(np.array_equal(a[k:k + chunk], b[k:k + chunk]) for k in range(0, a.size, chunk))


# ---- the consumers after edits at brick edges ----------------------------------------------------------------
def consumer_scene(dim):
    from scenarios import Scenario, control_set

    dims = (45, 37, 29) if dim == 3 else (77, 45)
    return Scenario(f"brick_edges_{dim}d", dims, 0.1, tuple(-d * 0.05 for d in dims), ACC, control_set(1.0, 3, dim),
                    v_max=3.0, n_boxes=4 if dim == 3 else 3, edge_m=(0.4, 1.0), seed=8)


def brick_edge_voxels(dims):
    """voxels at brick corners (every axis at c & mask in {0, mask}) and every voxel of the last, padded brick"""
    mx, my, mz = masks(dims)
    ax = [np.array([c for c in range(n) if c & m in (0, m)]) for n, m in zip(dims, (mx, my, mz))]
    last = [np.arange(n & ~m if n & m else n - m - 1, n) for n, m in zip(dims, (mx, my, mz))]
    out = []
    for sel in (ax, last):
        g = np.meshgrid(*sel, indexing="ij")
        out.append(vid(dims, *[a.reshape(-1) for a in g]))
    return np.unique(np.concatenate(out))


@pytest.mark.parametrize("dim", [3, 2])
def test_consumers_after_edits_at_brick_edges(dim):
    """Obstacles placed at brick corners and in the last padded brick, some removed again, single voxels toggled:
    kernels 0, 2 and 5 against the oracle on the final grid (counts, actions, successors and keys bit-exact, costs
    exact), mplx_edges_is_free the same way, and mplx_plan_batch against a fresh ctx."""
    from test_edges_oracle_vs_ref import edges_of

    sc = consumer_scene(dim)
    dims = sc.dim_cells
    rng = np.random.default_rng(40 + dim)
    nodes = sc.frontier(1500, seed=9)
    s = Session(sc.grid(), dims, sc.origin, sc.res)
    e = s.env
    e.set_control(sc.control)
    e.set_u(sc.U)
    e.set_v_max(sc.v_max)
    before = e.expand(nodes)
    edge = brick_edge_voxels(dims)
    edge = edge[(s.ref[edge] != 100)]
    s.update(edge, [100], "place at brick edges")  # ascending: the presorted path
    drop = rng.permutation(edge)[: edge.size // 2]
    s.update(drop, FREE[rng.integers(0, FREE.size, drop.size)], "remove half")  # the radix path
    for v in edge[:: max(1, edge.size // 12)]:
        s.update([v], [0 if s.ref[v] == 100 else 100], "toggle one")
    final = s.ref.copy()
    orc_env = ob.OracleEnv(dim, sc.control, sc.U, final, dims, sc.origin, sc.res, v_max=sc.v_max)
    orc = orc_env.expand(nodes, nthreads=8)
    for k in (0, 2, 5):
        e.set_kernel(k)
        st = assert_expansion_equal(e.expand(nodes, want=("succ", "cost", "action", "key")), orc, exact_cost=True)
        assert 0 < st["finite"] < st["successors"]
    e.set_kernel(0)
    assert e.expand(nodes).cost.tobytes() != before.cost.tobytes()  # the edits reached the primitives
    parents, actions, _ = edges_of(orc_env, nodes, rng, extra=400)
    fo, co = orc_env.edges_is_free(parents, actions)
    fg, cg = e.is_free_edges(parents, actions)
    np.testing.assert_array_equal(fg, fo)
    assert cg.tobytes() == co.tobytes()
    fresh = make_env(final, dims, sc.origin, sc.res)
    fresh.set_control(sc.control)
    fresh.set_u(sc.U)
    fresh.set_v_max(sc.v_max)
    q = sc.frontier(64, seed=10, max_steps=0)
    a = e.plan_batch(q[:32], q[32:], max_expand=300)
    b = fresh.plan_batch(q[:32], q[32:], max_expand=300)
    for f in ("valid", "cost", "expanded", "n_closed"):
        assert a[f].tobytes() == b[f].tobytes(), f
    for f in ("actions", "closed"):
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a[f], b[f])), f
    fresh.close()
    s.close()


# ---- the host upload path -----------------------------------------------------------------------------------
def _batch_paths(args, starts, goals):
    from motion_primitive_library_b200 import planner as P

    out = {}
    for path in ("lockstep", "device", "device_cost_terms", "device_grow", "auto"):
        bp = P.BatchPlanner(args, path=path)
        try:
            out[path] = bp.plan_detail(starts, goals)
        finally:
            bp.close()
    return out


def _same_detail(a, b, what):
    ra, _, aa, ca = a
    rb, _, ab, cb = b
    assert ra.tobytes() == rb.tobytes(), what
    assert all(x.tobytes() == y.tobytes() for x, y in zip(aa, ab)), (what, "actions")
    assert all(x.tobytes() == y.tobytes() for x, y in zip(ca, cb)), (what, "closed")


@pytest.mark.parametrize("with_potential", [False, True])
def test_batch_planner_upload_path(with_potential):
    """A BatchPlanner session edited through update_cells: a journal of exactly journalLimit() entries goes as a
    sparse update, one entry more as a full upload, two edit calls between plans as one sparse update, and an edit
    that restores the original values as a sparse update.  After every step every path answers as a fresh session
    on the final grid; with a potential map installed at open, the full upload re-sends it from the host copy."""
    from motion_primitive_library_b200 import planner as P

    sc = consumer_scene(3)
    dims = np.asarray(sc.dim_cells)
    grid = np.array(sc.grid(), dtype=np.int8).reshape(-1)
    nvox = grid.size
    limit = nvox // 64  # MapUtil::journalLimit()
    rng = np.random.default_rng(50)
    pot = np.where(grid == 100, 100, rng.integers(0, 50, nvox)).astype(np.int8) if with_potential else None
    nodes = sc.frontier(24, seed=11, max_steps=0)
    starts, goals = nodes[:12].copy(), nodes[12:].copy()
    base = dict(v_max=sc.v_max, max_num=400)
    if with_potential:
        base.update(potential=pot, potential_weight=0.5)

    def args_for(g):
        return P.make_args(3, ACC, g, sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=starts["pos"][0]),
                           goal=dict(pos=goals["pos"][0]), **base)

    def cells_of(idx):
        idx = np.asarray(idx, dtype=np.int64)
        return np.stack([idx % dims[0], idx // dims[0] % dims[1], idx // (dims[0] * dims[1])], 1).astype(np.int32)

    cur = grid.copy()
    sess = {p: P.BatchPlanner(args_for(grid), path=p) for p in ("lockstep", "device", "device_cost_terms",
                                                                 "device_grow", "auto")}
    try:
        for bp in sess.values():
            bp.plan(starts, goals)
        # the walls go through the queries' start-goal midpoints
        mids = np.floor(((starts["pos"] + goals["pos"]) / 2 - np.asarray(sc.origin)) / sc.res).astype(np.int64)
        wall = np.unique([vid(dims, m[0], np.clip(m[1] + dy, 0, dims[1] - 1), np.clip(m[2] + dz, 0, dims[2] - 1))
                          for m in mids for dy in range(-2, 3) for dz in range(-2, 3)])
        assert 2 * wall.size < limit
        journal = 0  # MapUtil's journal: entries since the open or the last truncation
        two = [(wall[::2], np.full(wall[::2].size, 100, np.int8)), (wall[1::3], np.full(wall[1::3].size, -1, np.int8))]
        steps = [  # (edit calls, expected (full, delta) increments)
            (two, (0, 1)),  # two calls between plans: one sparse update
            ("fill", (0, 1)),  # the journal at exactly journalLimit(): sparse
            ([(wall[:1], np.zeros(1, np.int8))], (1, 0)),  # one entry past it: truncated, a full upload
            ("restore", (0, 1)),  # every changed voxel back to its original value
        ]
        for k, (calls, inc) in enumerate(steps):
            if calls == "fill":
                n = limit - journal
                idx = np.concatenate([wall, rng.integers(0, nvox, n)])[:n]
                calls = [(idx, np.full(n, 100, np.int8))]
            elif calls == "restore":
                back = np.flatnonzero(cur != grid)
                assert 0 < back.size <= limit
                calls = [(back, grid[back])]
            for idx, val in calls:
                apply(cur, idx, val)
                journal += idx.size
                journal = 0 if journal > limit else journal
            assert (k != 1 or journal == limit) and (k != 2 or journal == 0)
            fresh = _batch_paths(args_for(cur), starts, goals)
            for path, bp in sess.items():
                f0, d0 = bp.map_uploads()
                for idx, val in calls:
                    bp.update_cells(cells_of(idx), val)
                _same_detail(bp.plan_detail(starts, goals), fresh[path], (k, path))
                assert tuple(np.subtract(bp.map_uploads(), (f0, d0))) == inc, (k, path)
        assert cur.tobytes() == grid.tobytes()
    finally:
        for bp in sess.values():
            bp.close()
