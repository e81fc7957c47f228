"""The ray trace of MapPlanner::setSearchRegion on the CPU: search::segment_cells (csrc/mplx_search.cuh), the one walk
that mplx_set_search_region_path runs on the host and the batch tunnel build runs on the device, compiled by g++,
gives cell for cell what region_path_cells' own per-segment loop gave (restated in tests/segment_cells_host.cpp), on
random 2-D and 3-D paths that leave the map part-way through a segment, repeat points and have segments of 0 and 1
steps."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent


@pytest.fixture(scope="module")
def sc(tmp_path_factory):
    so = tmp_path_factory.mktemp("sc") / "libsc.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(so),
                           str(HERE / "segment_cells_host.cpp")])
    L = C.CDLL(str(so))
    for fn in (L.sc_walk, L.sc_loop):
        fn.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                       C.c_int]
        fn.restype = C.c_int
    return L


def trace(fn, dim, mdim, origin, res, path, dense):
    md = np.array(list(mdim) + [1] * (3 - len(mdim)), np.int32)
    org = np.array(list(origin) + [0.0] * (3 - len(origin)))
    p = np.ascontiguousarray(path, dtype=np.float64)
    cap = 1 << 16
    out = np.zeros(cap * 3, np.int32)
    n = fn(dim, md.ctypes.data, org.ctypes.data, float(res), p.ctypes.data, len(p), 1 if dense else 0,
           out.ctypes.data, cap)
    assert n >= 0
    return out[:3 * n].reshape(-1, 3)


def random_path(rng, dim, lo, hi, res):
    """Points inside and around the map; some segments are shorter than one step (0 samples) or a little longer
    (1 sample), some points repeat."""
    n = int(rng.integers(1, 12))
    pts = [rng.uniform(lo - 1.0, hi + 1.0)]
    for _ in range(n - 1):
        kind = rng.integers(4)
        if kind == 0:
            step = rng.uniform(-0.5, 0.5, dim) * res * 0.8  # max_diff 0
        elif kind == 1:
            step = np.full(dim, 0.8 * res * 1.5) * rng.choice([-1, 1], dim)  # max_diff 1
        elif kind == 2:
            step = np.zeros(dim)  # a repeated point
        else:
            step = rng.uniform(-(hi - lo), hi - lo)  # long, often leaving the map
        pts.append(pts[-1] + step)
    return np.array(pts)


@pytest.mark.parametrize("dim,mdim,res", [(2, (45, 38), 0.25), (2, (17, 64), 0.1), (3, (20, 19, 13), 0.25),
                                          (3, (9, 31, 7), 0.5)])
@pytest.mark.parametrize("dense", [False, True])
def test_walk_equals_the_segment_loop(sc, dim, mdim, res, dense):
    rng = np.random.default_rng(dim * 100 + sum(mdim) + int(dense))
    origin = np.array([-m * res / 2 for m in mdim]) + rng.uniform(-0.1, 0.1, dim)
    lo = origin
    hi = origin + np.array(mdim) * res
    total = left = 0
    for _ in range(300):
        path = random_path(rng, dim, lo, hi, res)
        a = trace(sc.sc_walk, dim, mdim, origin, res, path, dense)
        b = trace(sc.sc_loop, dim, mdim, origin, res, path, dense)
        assert np.array_equal(a, b), path
        total += len(a)
        left += int(((a[:, :dim] < 0) | (a[:, :dim] >= np.array(mdim))).any())
    assert total > 1000 and (dense or left > 0)


def test_walk_stops_at_the_first_cell_outside(sc):
    dim, mdim, res = 2, (10, 10), 1.0
    origin = (0.0, 0.0)
    path = np.array([[0.5, 5.5], [14.5, 5.5]])  # leaves the map at x = 10
    cells = trace(sc.sc_walk, dim, mdim, origin, res, path, False)
    xs = cells[:-1, 0]
    assert xs.max() == 9 and cells[-1, 0] == 14  # the samples stop inside; the end point's cell is pushed as is
    assert np.array_equal(cells, trace(sc.sc_loop, dim, mdim, origin, res, path, False))
