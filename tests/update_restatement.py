"""What mplx_read_map must return for a grid, restated in numpy from the rules of the map views, with no code
shared with csrc/mplx_pack.cuh:

* the grid bytes, verbatim;
* occupancy word w, bit b: voxel i = 32w + b is occupied, i.e. its byte is 100 (map_util.h:48); 0 for i >= nvox;
* pair word w = {occupancy word w, summary word w}; summary bit of voxel (x, y[, z]): the OR of the occupancy of
  the box {x-1, x} x {y-1, y} (x {z-1, z}), a cell outside the map counting as occupied; 1 for i >= nvox.

`views_at` evaluates the rules on a chosen set of words only, so maps of a billion voxels are checked without
temporaries of the map's size.  `brick_geometry` restates the brick layout of the device copy (occ2): 3-D bricks
of 8x8x8 voxels in which a pair holds 8 x by 4 y of one z, 2-D bricks of 32x16 in which a pair holds one row of
32 x; bricks counted x fastest, 16 pairs per brick."""
import numpy as np

import fixtures

OCCUPIED = 100

# the shape classes of tests/test_update_paths_gpu.py and tests/test_update_restatement_cpu.py: sizes of 1 and
# around the brick extents on every axis, nz = 1 / ny = 1, nx = 1, and voxel counts with and without a partial
# last word
SHAPES_3D = [(1, 1, 1), (1, 1, 40), (8, 8, 8), (7, 9, 1), (9, 7, 3), (16, 16, 16), (17, 15, 9), (33, 8, 17),
             (64, 64, 64)]
SHAPES_2D = [(1, 1), (1, 50), (31, 15), (32, 16), (33, 17), (64, 1), (65, 33), (100, 3), "corridor"]
SHAPES = {("x".join(map(str, s)) if s != "corridor" else s): s for s in SHAPES_3D + SHAPES_2D}


def shape_dims(name):
    s = SHAPES[name]
    return tuple(int(d) for d in fixtures.corridor()["dim"]) if s == "corridor" else s


def nvox_of(dims):
    return int(np.prod(np.asarray(dims, dtype=np.int64)))


def coords(i, dims):
    """(x, y, z) of voxel ids i (z = 0 in 2-D)"""
    i = np.asarray(i, dtype=np.int64)
    nx, ny = int(dims[0]), int(dims[1])
    return i % nx, (i // nx) % ny, i // (nx * ny)


def summary_bits(grid, dims, i):
    """summary bit of each voxel id in i (all < nvox)"""
    grid = np.asarray(grid).reshape(-1).view(np.int8)
    i = np.asarray(i, dtype=np.int64)
    nx, sxy = int(dims[0]), int(dims[0]) * int(dims[1])
    x, y, z = coords(i, dims)
    three = len(dims) == 3
    s = np.zeros(i.shape, dtype=bool)
    for dz in (0, 1) if three else (0,):
        for dy in (0, 1):
            for dx in (0, 1):
                outside = (x < dx) | (y < dy) | (z < dz)
                j = np.where(outside, 0, i - dx - dy * nx - dz * sxy)
                s |= outside | (grid[j] == OCCUPIED)
    return s


def _pack(bits):
    """bool[..., 32] -> uint32[...], bit b from bits[..., b]"""
    return (bits.astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32)


def views_at(grid, dims, words):
    """(occupancy words, pair words [len, 2]) of the given word indices"""
    grid = np.asarray(grid).reshape(-1).view(np.int8)
    nvox = nvox_of(dims)
    assert grid.size == nvox
    words = np.asarray(words, dtype=np.int64).reshape(-1)
    i = words[:, None] * 32 + np.arange(32, dtype=np.int64)[None, :]
    inside = i < nvox
    ic = np.where(inside, i, 0)
    occ = inside & (grid[ic] == OCCUPIED)
    summ = ~inside | summary_bits(grid, dims, ic)
    o = _pack(occ)
    return o, np.stack([o, _pack(summ)], axis=-1)


def views(grid, dims):
    """(grid int8[nvox], occupancy uint32[nw], pairs uint32[nw, 2]): mplx_read_map's three outputs"""
    grid = np.asarray(grid).reshape(-1).view(np.int8)
    nw = (nvox_of(dims) + 31) // 32
    occ, pairs = views_at(grid, dims, np.arange(nw))
    return grid.copy(), occ, pairs


def reach_words(idx, dims):
    """the words whose occupancy or summary bits an edit of voxels idx can change: those of v + {0,1}^dim"""
    idx = np.unique(np.asarray(idx, dtype=np.int64))
    nx, sxy, nvox = int(dims[0]), int(dims[0]) * int(dims[1]), nvox_of(dims)
    offs = [dx + dy * nx + dz * sxy for dz in ((0, 1) if len(dims) == 3 else (0,)) for dy in (0, 1) for dx in (0, 1)]
    v = (idx[:, None] + np.asarray(offs, dtype=np.int64)[None, :]).reshape(-1)
    return np.unique(np.minimum(v, nvox - 1) >> 5)


def successors(v, dims):
    """the voxels whose summary box holds voxel v: v + {0,1}^dim inside the map"""
    x, y, z = (int(c) for c in coords(v, dims))
    nx, ny = int(dims[0]), int(dims[1])
    nz = int(dims[2]) if len(dims) == 3 else 1
    out = []
    for dz in (0, 1) if len(dims) == 3 else (0,):
        for dy in (0, 1):
            for dx in (0, 1):
                if x + dx < nx and y + dy < ny and z + dz < nz:
                    out.append(int(v) + dx + dy * nx + dz * nx * ny)
    return out


def brick_geometry(dims):
    """(pair index, bit) of every voxel in the brick buffer, and its pair count"""
    three = len(dims) == 3
    bx, by, bz = (8, 8, 8) if three else (32, 16, 1)
    nx, ny = int(dims[0]), int(dims[1])
    nz = int(dims[2]) if three else 1
    nbx, nby, nbz = -(-nx // bx), -(-ny // by), -(-nz // bz)
    x, y, z = coords(np.arange(nvox_of(dims)), dims)
    brick = x // bx + nbx * (y // by + nby * (z // bz))
    if three:  # a pair: 8 x by 4 y of one z; inside it x fastest, then y
        pair, bit = brick * 16 + (z % 8) * 2 + (y % 8) // 4, (x % 8) + 8 * (y % 4)
    else:  # a pair: one row of 32 x
        pair, bit = brick * 16 + y % 16, x % 32
    return pair, bit, nbx * nby * nbz * 16
