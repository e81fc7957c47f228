"""The per-query tunnels of the batched searches (mplx_set_batch_regions) on the CPU:
  - the brick build (csrc/mplx_tunnel.cuh geometry, restated in tests/tunnel_bricks_host.cpp and compiled by g++)
    gives, voxel for voxel, the region a dense stamp of the same path cells gives, as mplx_set_search_region_path's
    region_stamp_kernel stamps it, on random 2-D and 3-D paths;
  - the new entry points are declared in include/mplx.h with the signatures abi.py binds."""
import ctypes as C
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest

from motion_primitive_library_b200 import abi

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent


@pytest.fixture(scope="module")
def tb(tmp_path_factory):
    so = tmp_path_factory.mktemp("tb") / "libtb.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", str(so),
                           str(HERE / "tunnel_bricks_host.cpp")])
    L = C.CDLL(str(so))
    vp = C.c_void_p
    L.tb_build.argtypes = [C.c_int, vp, C.c_int, vp, vp, vp, C.POINTER(C.c_int64), vp]
    L.tb_build.restype = C.c_int
    return L


def dense_stamp(dim, mdim, cells, r):
    """region_stamp_kernel (csrc/mplx_maps.cu): every (path cell, box offset) inside the map sets its voxel."""
    nz = mdim[2] if dim == 3 else 1
    out = np.zeros((nz, mdim[1], mdim[0]), np.uint8)
    for c in cells:
        lo = [max(c[k] - r[k], 0) for k in range(dim)]
        hi = [min(c[k] + r[k], mdim[k] - 1) for k in range(dim)]
        if any(lo[k] > hi[k] for k in range(dim)):
            continue
        if dim == 3:
            out[lo[2]:hi[2] + 1, lo[1]:hi[1] + 1, lo[0]:hi[0] + 1] = 1
        else:
            out[0, lo[1]:hi[1] + 1, lo[0]:hi[0] + 1] = 1
    return out.reshape(-1)


def random_paths(rng, dim, mdim, n_q):
    """Per query: a random walk of cells that wanders off the map, runs along its edges and repeats cells, or a
    single cell."""
    paths = []
    for q in range(n_q):
        n = 1 if q % 5 == 0 else int(rng.integers(2, 40))
        c = np.array([rng.integers(-3, m + 3) for m in mdim[:dim]])
        pts = []
        for _ in range(n):
            pts.append(c.copy())
            c = c + rng.integers(-2, 3, size=dim)
            if q % 7 == 3:
                c[0] = 0  # along the edge
        cells = np.zeros((n, 3), np.int32)
        cells[:, :dim] = np.array(pts)
        if q % 4 == 1:
            cells = np.vstack([cells, cells[:3]])  # repeated cells
        paths.append(cells)
    return paths


@pytest.mark.parametrize("dim,mdim,r", [
    (2, (37, 29, 1), (0, 0, 0)), (2, (37, 29, 1), (3, 1, 0)), (2, (64, 16, 1), (9, 4, 0)),
    (3, (21, 18, 13), (0, 0, 0)), (3, (21, 18, 13), (2, 3, 1)), (3, (33, 17, 9), (5, 0, 8)),
])
def test_brick_build_equals_dense_stamp(tb, dim, mdim, r):
    rng = np.random.default_rng(sum(mdim) * 7 + sum(r) + dim)
    n_q = 23
    paths = random_paths(rng, dim, mdim, n_q)
    off = np.zeros(n_q + 1, np.int64)
    off[1:] = np.cumsum([len(p) for p in paths])
    cells = np.ascontiguousarray(np.vstack(paths), dtype=np.int32)
    md = np.array(mdim, np.int32)
    rr = np.array(r, np.int32)
    nvox = int(np.prod(mdim[:dim]))
    out = np.zeros(n_q * nvox, np.uint8)
    nb = C.c_int64()
    assert tb.tb_build(dim, md.ctypes.data, n_q, off.ctypes.data, cells.ctypes.data, rr.ctypes.data, C.byref(nb),
                       out.ctypes.data) == 0
    touched = 0
    for q in range(n_q):
        want = dense_stamp(dim, mdim, paths[q][:, :dim], r)
        assert np.array_equal(out[q * nvox:(q + 1) * nvox], want), q
        touched += int(want.sum() > 0)
    assert touched > n_q // 2
    # storage follows the tunnels: never more bricks than the queries' boxes can touch
    per = 1
    for k in range(dim):
        per *= (2 * r[k] + 1 + 6) // 8 + 1
    assert 0 < nb.value <= len(cells) * per


def test_new_entry_points_are_declared_and_bound():
    header = (ROOT / "include" / "mplx.h").read_text()
    sigs = {
        "mplx_set_batch_regions": r"int mplx_set_batch_regions\(mplx_ctx \*ctx, int n_q, const int64_t \*pt_offset, "
                                  r"const double \*pts, const double \*radius,\s+int dense\);",
        "mplx_batch_regions_info": r"int mplx_batch_regions_info\(mplx_ctx \*ctx, int32_t \*n_q, int64_t \*n_bricks, "
                                   r"int64_t \*bytes\);",
        "mplx_read_batch_region": r"int mplx_read_batch_region\(mplx_ctx \*ctx, int q, uint8_t \*out\);",
    }
    for name, pat in sigs.items():
        assert re.search(pat, header), name
        assert name in abi.EXPORTED_SYMBOLS
    assert "mplx_tunnel.cu" in (ROOT / "motion_primitive_library_b200" / "csrc" / "Makefile").read_text()
