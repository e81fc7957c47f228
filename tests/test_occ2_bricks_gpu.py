"""The fixed-point kernels on maps where the brick layout of occ2 (csrc/mplx_pack.cuh) has padding and where
decisions sit on brick edges.

occ2 stores each voxel's occupancy and candidate-summary bit in bricks of 8x8x8 voxels (2-D: 32x16), so a
map whose dims are not multiples of the brick has padded bricks, and a cell on a brick face has neighbours
whose bits live in another brick's line.  Every case runs kernels 5 (expand_fx_kernel), 0 (auto:
expand_fxn_kernel + fx_resolve_kernel, shown by the launch count) and 2 (register kernel, no occ2) against
the CPU oracle with exact costs, and against the reference where oracle/_ref is built:

  faces       obstacles on brick faces and corners of a map with odd dims
  boundary    starts on cell boundaries that are brick boundaries, with the voxel the reference puts sample
              0 in (blocked) or the one across the boundary (free, but a candidate) occupied: the uncertain
              samples read summary bits of cells on both sides of a brick edge
  padding     starts next to the map's edges, moving out of it: samples cross into the padded bricks
"""
from __future__ import annotations

import numpy as np
import pytest

from oracle_bindings import WAYPOINT_DTYPE
from test_fx_paths_gpu import ACC, Case, boundary, emitted_mask, product_set, ref_cell, run_kernels, same_mask, u_values

pytestmark = pytest.mark.gpu

KERNELS = (5, 0, 2)
BRICK = {3: (8, 8, 8), 2: (32, 16)}
MAPS = {3: dict(mdim=(43, 29, 21), origin=(-2.1373, -1.5519, -1.1017)),
        2: dict(mdim=(203, 77), origin=(-9.8713, -4.0291))}


def brick_face_grid(mdim, dim, rng, frac):
    """Occupied voxels drawn from the cells on brick faces (a coordinate at either end of its brick), and
    every brick corner inside the map."""
    cells = np.stack(np.meshgrid(*[np.arange(m) for m in mdim], indexing="ij"), -1).reshape(-1, dim)
    b = np.asarray(BRICK[dim])
    r = cells % b
    end = (r == 0) | (r == b - 1)
    face = end.any(1)
    corner = end.all(1)
    occ = (face & (rng.random(len(cells)) < frac)) | corner
    grid = np.zeros(int(np.prod(mdim)), np.int8)
    idx = cells[occ, 0] + mdim[0] * cells[occ, 1]
    if dim == 3:
        idx = idx + mdim[0] * mdim[1] * cells[occ, 2]
    grid[idx] = 100
    return grid, int(face.sum()), int(corner.sum())


def acc_case(dim, grid=None, res=0.15):
    m = MAPS[dim]
    return Case(dim, ACC, product_set(*[u_values(ACC)] * dim), m["mdim"], m["origin"], res, grid=grid, v_max=2.5)


def n_nodes(dim):
    return 1201 if dim == 3 else 2003  # >= 64*256 primitive slots: kernel 0 is the fxn pair


@pytest.mark.parametrize("dim", [3, 2])
def test_obstacles_on_brick_faces(dim):
    rng = np.random.default_rng(40 + dim)
    m = MAPS[dim]
    grid, n_face, n_corner = brick_face_grid(m["mdim"], dim, rng, 0.08)
    case = acc_case(dim, grid)
    n = n_nodes(dim)
    nodes = np.zeros(n, dtype=WAYPOINT_DTYPE)
    cells = rng.integers(1, np.asarray(m["mdim"]) - 1, (n, dim))
    nodes["pos"][:, :dim] = np.asarray(m["origin"]) + np.round((cells + rng.random((n, dim))) * case.res / 0.05) * 0.05
    nodes["vel"][:, :dim] = rng.integers(-3, 4, (n, dim)) * 0.5
    orc, _ = run_kernels(case, nodes, kernels=KERNELS)
    st = emitted_mask(orc)
    assert n_corner > 8 and np.isinf(orc["cost"][st]).sum() > 1000 and np.isfinite(orc["cost"][st]).sum() > 1000


@pytest.mark.parametrize("dim", [3, 2])
def test_uncertain_samples_on_brick_edges(dim):
    """As test_fx_paths_gpu's boundary starts: every start on a cell boundary on every axis, and on the axis
    that separates the two candidate cells of the test, a brick boundary."""
    rng = np.random.default_rng(50 + dim)
    m = MAPS[dim]
    case = acc_case(dim)
    n = n_nodes(dim)
    b = np.asarray(BRICK[dim])
    mdim = np.asarray(m["mdim"])
    o = np.asarray(m["origin"])
    k = rng.integers(2, mdim - 2, (n, dim))
    axis = rng.integers(0, dim, n)
    rows = np.arange(n)
    # on `axis` a brick boundary j*b[axis], 1 <= j, inside [2, mdim - 2)
    k[rows, axis] = rng.integers(1, (mdim[axis] - 3) // b[axis] + 1) * b[axis]
    nodes = np.zeros(n, dtype=WAYPOINT_DTYPE)
    nodes["pos"][:, :dim] = boundary(o, case.res, k)
    still = rng.random((n, dim)) < 0.5
    nodes["vel"][:, :dim] = np.where(still, 0.0, rng.integers(-2, 3, (n, dim)) * 0.5)
    y = (nodes["pos"][:, :dim] - o) * (1.0 / case.res)
    assert (np.abs(y - k) < 1e-9).all()
    c0 = ref_cell(nodes["pos"][:, :dim], o, case.res)
    other = c0.copy()
    other[rows, axis] = np.where(c0[rows, axis] == k[rows, axis], k[rows, axis] - 1, k[rows, axis])
    # c0 and `other` lie in different bricks along `axis`
    assert ((c0[rows, axis] // b[axis]) != (other[rows, axis] // b[axis])).all()
    blocked = rng.random(n) < 0.3
    case.grid[case.index(np.where(blocked[:, None], c0, other))] = 100
    orc, _ = run_kernels(case, nodes, kernels=KERNELS)
    live = emitted_mask(orc) & ~same_mask(orc, nodes, dim)
    assert int((live & np.isfinite(orc["cost"])).sum()) > 1000
    assert int((live & np.isinf(orc["cost"])).sum()) > 1000


@pytest.mark.parametrize("dim", [3, 2])
def test_primitives_leaving_through_padded_bricks(dim):
    """Starts within two cells of a map edge with velocity pointing out of the map on that axis; the map's
    dims are not multiples of the brick, so the last brick on each axis is padded and samples past the edge
    have addresses in it (or past it)."""
    rng = np.random.default_rng(60 + dim)
    m = MAPS[dim]
    mdim = np.asarray(m["mdim"])
    assert (mdim % np.asarray(BRICK[dim]) != 0).all()
    grid, _, _ = brick_face_grid(m["mdim"], dim, rng, 0.02)
    case = acc_case(dim, grid)
    n = n_nodes(dim)
    o = np.asarray(m["origin"])
    cells = rng.integers(2, mdim - 2, (n, dim))
    axis = rng.integers(0, dim, n)
    high = rng.random(n) < 0.7  # the high edges border the padding
    rows = np.arange(n)
    cells[rows, axis] = np.where(high, mdim[axis] - 1 - rng.integers(0, 2, n), rng.integers(0, 2, n))
    nodes = np.zeros(n, dtype=WAYPOINT_DTYPE)
    nodes["pos"][:, :dim] = o + (cells + rng.choice([0.0, 0.5, 0.25], (n, dim))) * case.res
    nodes["vel"][:, :dim] = rng.integers(-2, 3, (n, dim)) * 0.5
    nodes["vel"][rows, axis] = np.where(high, 1.0, -1.0) * rng.choice([0.5, 1.0], n)
    orc, _ = run_kernels(case, nodes, kernels=KERNELS)
    em = emitted_mask(orc)
    # most primitives of these nodes leave the map: blocked; some turn back in time and stay free
    assert np.isinf(orc["cost"][em]).sum() > 3000 and np.isfinite(orc["cost"][em]).sum() > 100
