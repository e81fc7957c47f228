"""The numpy restatement of mplx_read_map's three views (tests/update_restatement.py) pinned, without a GPU, to
the word rules and the brick layout of csrc/mplx_pack.cuh compiled with g++ (tests/update_views_host.cpp): on
every shape class of tests/test_update_paths_gpu.py, random grids at several densities and grids holding every
int8 value, the occupancy words, the voxel-order pair words read back from the brick buffer through occ2_pair /
occ2_bit, each voxel's (pair, bit) and the padding bits of the brick buffer must all agree with the rules."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

import update_restatement as R
from update_restatement import SHAPES, shape_dims

HERE = Path(__file__).resolve().parent


def test_shape_classes_cover_word_and_row_classes():
    dims = [shape_dims(n) for n in SHAPES]
    assert any(R.nvox_of(d) % 32 == 0 for d in dims) and any(R.nvox_of(d) % 32 != 0 for d in dims)
    assert any(d[0] == 1 for d in dims if len(d) == 3) and any(d[0] == 1 for d in dims if len(d) == 2)
    assert any(d[2] == 1 for d in dims if len(d) == 3) and any(d[1] == 1 for d in dims if len(d) == 2)


@pytest.fixture(scope="module")
def header(tmp_path_factory):
    so = tmp_path_factory.mktemp("update_views") / "update_views_host.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", str(so),
                           str(HERE / "update_views_host.cpp")])
    lib = C.CDLL(str(so))
    lib.uv_pair_count.argtypes = [C.c_int] * 4
    lib.uv_pair_count.restype = C.c_size_t
    lib.uv_views.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 5
    lib.uv_views.restype = None
    return lib


def header_views(lib, grid, dims):
    d3 = tuple(dims) + (1,) * (3 - len(dims))
    nvox = R.nvox_of(dims)
    nw = (nvox + 31) // 32
    g = np.ascontiguousarray(grid, dtype=np.int8)
    npairs = lib.uv_pair_count(len(dims), *d3)
    occ, bricks, pairs = np.zeros(nw, np.uint32), np.zeros((npairs, 2), np.uint32), np.zeros((nw, 2), np.uint32)
    pair_of, bit_of = np.zeros(nvox, np.uint32), np.zeros(nvox, np.uint8)
    lib.uv_views(g.ctypes.data, len(dims), *d3, occ.ctypes.data, bricks.ctypes.data, pairs.ctypes.data,
                 pair_of.ctypes.data, bit_of.ctypes.data)
    return occ, bricks, pairs, pair_of, bit_of


def grids(dims, seed):
    """random grids at several densities of 100 over non-occupied values, and grids holding every int8 value"""
    rng = np.random.default_rng(seed)
    n = R.nvox_of(dims)
    free = np.array([0, -1, 1, 99, 101, 127, -128], dtype=np.int8)
    for p in (0.0, 0.03, 0.3, 0.9, 1.0):
        yield f"p{p}", np.where(rng.random(n) < p, 100, free[rng.integers(0, free.size, n)]).astype(np.int8)
    every = np.arange(-128, 128, dtype=np.int64)
    yield "every_int8", np.resize(every, n).astype(np.int8)
    yield "every_int8_shuffled", rng.permutation(np.resize(every, max(n, 256)))[:n].astype(np.int8)


@pytest.mark.parametrize("name", list(SHAPES))
def test_restatement_matches_header_rules(header, name):
    dims = shape_dims(name)
    pair_r, bit_r, npairs_r = R.brick_geometry(dims)
    checked = 0
    for label, g in grids(dims, seed=len(name) * 31 + sum(dims)):
        grid, occ_r, pairs_r = R.views(g, dims)
        assert grid.tobytes() == g.tobytes()
        occ, bricks, pairs, pair_of, bit_of = header_views(header, g, dims)
        assert bricks.shape[0] == npairs_r
        np.testing.assert_array_equal(pair_of, pair_r, err_msg=f"{name} {label}: pair of a voxel")
        np.testing.assert_array_equal(bit_of, bit_r, err_msg=f"{name} {label}: bit of a voxel")
        assert occ.tobytes() == occ_r.tobytes(), (name, label, "occupancy words")
        bad = np.flatnonzero((pairs != pairs_r).any(1))
        assert bad.size == 0, (name, label, "pair words", bad[:8], pairs[bad[:2]], pairs_r[bad[:2]])
        # every brick-buffer bit no voxel owns (padding) reads 1 in both words
        owned = np.zeros(npairs_r, dtype=np.uint64)
        np.bitwise_or.at(owned, pair_r, np.uint64(1) << bit_r.astype(np.uint64))
        pad = (~owned) & np.uint64(0xFFFFFFFF)
        for k in (0, 1):
            assert ((bricks[:, k].astype(np.uint64) & pad) == pad).all(), (name, label, "padding", k)
        checked += 1
    assert checked == 7
    # the rules themselves, on a few voxels stated by hand
    g = np.zeros(R.nvox_of(dims), np.int8)
    occ, pairs = R.views_at(g, dims, [0])
    assert occ[0] == 0 and pairs[0, 1] & 1 == 1  # voxel 0: its box reaches outside the map


def test_value_classes():
    """only 100 is occupied: 101, 127, -1 and -128 are not"""
    dims = (8, 4)
    g = np.zeros(32, np.int8)
    g[:8] = [100, 101, 127, -1, -128, 99, 1, 0]
    occ, pairs = R.views_at(g, dims, [0])
    assert occ[0] == 1 and pairs[0, 0] == 1
    # summary: row 0 and column 0 read outside; (1, 1) holds (0, 0) in its box; every other voxel is free
    s = int(pairs[0, 1])
    want = 0xFF | (1 << 8) | (1 << 16) | (1 << 24) | (1 << 9)
    assert s == want, hex(s)


def test_summary_past_nvox_and_partial_last_word():
    dims = (5, 3, 3)  # 45 voxels: the second word holds 13 voxels and 19 bits past nvox
    g = np.zeros(45, np.int8)
    occ, pairs = R.views_at(g, dims, [1])
    assert occ[0] == 0
    assert (int(pairs[0, 1]) >> 13) == (1 << 19) - 1


def test_reach_words_and_successors():
    dims = (33, 8, 17)
    nx, sxy = 33, 33 * 8
    v = 5 + 3 * nx + 2 * sxy
    assert R.successors(v, dims) == [v, v + 1, v + nx, v + nx + 1, v + sxy, v + sxy + 1, v + sxy + nx, v + sxy + nx + 1]
    assert R.successors(R.nvox_of(dims) - 1, dims) == [R.nvox_of(dims) - 1]
    w = R.reach_words([v], dims)
    assert set(w) == {(v + o) >> 5 for o in (0, 1, nx, nx + 1, sxy, sxy + 1, sxy + nx, sxy + nx + 1)}
