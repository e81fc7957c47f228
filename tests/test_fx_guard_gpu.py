"""The fixed-point kernels on the guard-banded occ2 buffer (csrc/mplx_pack.cuh) and their two sample loops.

The device copy of the map is stored padded by a guard band of G = 32 cells on every side, every bit of it
set.  Where every sample of a primitive provably stays within G cells of the map (fx_band: the start cell in
the map, the displacement bound + 2 <= G), the sample loop addresses its cells without testing them against
the map; any other primitive takes the literal loop.  A plan whose samples may reach past the band
(maxn + 2 > G) runs the checked loop, which tests every sample.  Every case runs kernels 5 (expand_fx_kernel),
0 (auto: expand_fxn_kernel + fx_resolve_kernel, shown by the launch count) and 2 (register kernel, no occ2)
against the CPU oracle with exact costs, and against the reference where oracle/_ref is built:

  faces       starts next to every face, edge and corner of odd-sized 3-D and 2-D maps, moving out of it or
              along it: samples land in the guard band (unchecked loop)
  checked     the same starts in a plan with maxn + 2 > G, speeds that carry samples far past the band
  outside     starts outside the map (rows that fail fx_band): the literal loop in the unchecked plan
  update      the same after sparse edits of cells on the map's faces (mplx_update_cells)
  read_map    mplx_read_map after a set and after updates: the voxel-order views, restated in numpy
"""
from __future__ import annotations

import numpy as np
import pytest

import update_restatement as ur
from oracle_bindings import WAYPOINT_DTYPE
from test_fx_paths_gpu import ACC, Case, emitted_mask, product_set, run_kernels, u_values

pytestmark = pytest.mark.gpu

KERNELS = (5, 0, 2)
GUARD = 32  # kOcc2Guard
MAPS = {3: dict(mdim=(43, 29, 21), origin=(-2.1373, -1.5519, -1.1017)),
        2: dict(mdim=(203, 77), origin=(-9.8713, -4.0291))}
RES = 0.15


def maxn(v_max, res=RES, T=1.0):
    return max(5, int(np.ceil(v_max * T / res)))


def n_nodes(dim):
    return 1201 if dim == 3 else 2003  # >= 64*256 primitive slots: kernel 0 is the fxn pair


def face_grid(mdim, dim, rng, frac):
    """Occupied voxels drawn from the cells within two cells of a face of the map."""
    cells = np.stack(np.meshgrid(*[np.arange(m) for m in mdim], indexing="ij"), -1).reshape(-1, dim)
    m = np.asarray(mdim)
    near = ((cells < 2) | (cells >= m - 2)).any(1)
    occ = near & (rng.random(len(cells)) < frac)
    grid = np.zeros(int(np.prod(mdim)), np.int8)
    idx = cells[occ, 0] + mdim[0] * cells[occ, 1]
    if dim == 3:
        idx = idx + mdim[0] * mdim[1] * cells[occ, 2]
    grid[idx] = 100
    return grid


def edge_nodes(rng, n, dim, speed, outside=0):
    """On each axis independently: next to the low face, next to the high face or anywhere inside, so every
    face, edge and corner of the map is met.  On a face axis the velocity points out of the map (mostly) or
    into it; `outside` > 0 puts that many cells between the start and the face, outside the map."""
    m = MAPS[dim]
    mdim, o = np.asarray(m["mdim"]), np.asarray(m["origin"])
    side = rng.integers(0, 3, (n, dim))  # 0 low face, 1 high face, 2 inside
    depth = rng.integers(0, 3, (n, dim))
    cells = np.where(side == 0, depth, np.where(side == 1, mdim - 1 - depth, rng.integers(0, mdim, (n, dim))))
    if outside:
        cells = np.where(side == 0, -1 - rng.integers(0, outside, (n, dim)), cells)
        cells = np.where(side == 1, mdim + rng.integers(0, outside, (n, dim)), cells)
    nodes = np.zeros(n, dtype=WAYPOINT_DTYPE)
    nodes["pos"][:, :dim] = o + (cells + rng.choice([0.0, 0.5, 0.25], (n, dim))) * RES
    mag = rng.choice(speed, (n, dim))
    out = rng.random((n, dim)) < 0.75
    sign = np.where(side == 0, -1.0, 1.0) * np.where(out, 1.0, -1.0)
    nodes["vel"][:, :dim] = np.where(side == 2, rng.choice(np.concatenate([-np.asarray(speed), speed]), (n, dim)),
                                     sign * mag)
    return nodes


def case_for(dim, v_max, grid=None):
    m = MAPS[dim]
    return Case(dim, ACC, product_set(*[u_values(ACC)] * dim), m["mdim"], m["origin"], RES, grid=grid, v_max=v_max)


@pytest.mark.parametrize("dim", [3, 2])
def test_starts_on_every_face_edge_and_corner(dim):
    v_max = 4.5  # maxn 30: the unchecked loop
    assert maxn(v_max) + 2 <= GUARD
    rng = np.random.default_rng(70 + dim)
    case = case_for(dim, v_max, face_grid(MAPS[dim]["mdim"], dim, rng, 0.02))
    nodes = edge_nodes(rng, n_nodes(dim), dim, (0.5, 1.5, 3.0, 4.5))
    orc, _ = run_kernels(case, nodes, kernels=KERNELS)
    em = emitted_mask(orc)
    assert np.isinf(orc["cost"][em]).sum() > 3000 and np.isfinite(orc["cost"][em]).sum() > 300


@pytest.mark.parametrize("dim", [3, 2])
def test_plan_past_the_guard_band_runs_the_checked_loop(dim):
    v_max = 7.5  # maxn 50: samples may travel 50 cells, past the 32 of the band
    assert maxn(v_max) + 2 > GUARD
    rng = np.random.default_rng(80 + dim)
    case = case_for(dim, v_max, face_grid(MAPS[dim]["mdim"], dim, rng, 0.02))
    nodes = edge_nodes(rng, n_nodes(dim), dim, (1.5, 4.5, 6.5, 7.0))
    orc, _ = run_kernels(case, nodes, kernels=KERNELS)
    em = emitted_mask(orc)
    assert np.isinf(orc["cost"][em]).sum() > 3000 and np.isfinite(orc["cost"][em]).sum() > 50


@pytest.mark.parametrize("dim", [3, 2])
def test_rows_outside_the_band_take_the_literal_loop(dim):
    """Starts up to 40 cells outside the map: their rows fail fx_band and the unchecked plan decides those
    primitives with the literal loop; some turn back into the map in time, and all of them are blocked by
    their first sample, which the reference puts outside the map."""
    v_max = 4.5
    rng = np.random.default_rng(90 + dim)
    case = case_for(dim, v_max, face_grid(MAPS[dim]["mdim"], dim, rng, 0.02))
    nodes = edge_nodes(rng, n_nodes(dim), dim, (0.5, 3.0, 4.5), outside=40)
    orc, _ = run_kernels(case, nodes, kernels=KERNELS)
    em = emitted_mask(orc)
    assert np.isinf(orc["cost"][em]).sum() > 3000


@pytest.mark.parametrize("dim", [3, 2])
def test_expansion_and_read_map_after_updates(dim):
    """mplx_read_map after the set and after sparse edits of cells on and next to the faces equals the
    voxel-order views restated from the grid, and the expansions near the faces match the oracle on the
    edited grid."""
    rng = np.random.default_rng(100 + dim)
    m = MAPS[dim]
    mdim = tuple(m["mdim"])
    grid = face_grid(mdim, dim, rng, 0.02)
    case = case_for(dim, 4.5, grid.copy())
    env = case.gpu()
    try:
        for got, want in zip(env.read_map(), ur.views(grid, mdim)):
            assert got.tobytes() == want.tobytes()
        cells = np.stack(np.meshgrid(*[np.arange(d) for d in mdim], indexing="ij"), -1).reshape(-1, dim)
        near = ((cells < 3) | (cells >= np.asarray(mdim) - 3)).any(1)
        idx = case.index(cells[near])
        pick = idx[rng.random(idx.size) < 0.1]
        vals = rng.choice(np.array([100, 0, 100, -1], dtype=np.int8), pick.size)
        env.update_cells(pick, vals)
        grid[pick] = vals
        for got, want in zip(env.read_map(), ur.views(grid, mdim)):
            assert got.tobytes() == want.tobytes()
        case.grid = grid
        nodes = edge_nodes(rng, n_nodes(dim), dim, (0.5, 1.5, 3.0, 4.5))
        orc, _ = run_kernels(case, nodes, kernels=KERNELS, env=env)
        em = emitted_mask(orc)
        assert np.isinf(orc["cost"][em]).sum() > 1000 and np.isfinite(orc["cost"][em]).sum() > 300
    finally:
        env.close()
