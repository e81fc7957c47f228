"""Constructed stored edges, one per branch of mplx_edges_is_free / mplx_edges_cells, shared with
tests/test_edges_paths_gpu.py, and their witnesses on the CPU:

  is_free, intrinsic cost   the oracle against the REFERENCE's env_map::is_free(pr) / calculate_intrinsic_cost(pr)
                            (oracle/_ref or its recordings), bit for bit;
  cells                     the oracle's walk against `walk_acc`, a plain-numpy restatement of
                            Primitive::sample(n) + floatToInt + getIndex for ACC edges (map_planner.cpp:135-151).

Each case asserts, from the restatement, that its branch is taken.  Edges with more than 2^20 samples and NaN
velocities have no CPU witness (the reference would allocate n + 1 waypoints; a NaN max_vel is compared
differently by every implementation): for them the bar is the contract of include/mplx.h and csrc/mplx_edges.cu —
not free, no cells, finite work — and only the GPU file runs them."""
import math

import numpy as np
import pytest

import oracle_bindings as ob
from reference_record import same_array

ACC = 0x03
INT_MIN = -2 ** 31
EDGE_N_MAX = 1 << 20  # kEdgeNMax, csrc/mplx_edges.cu
RES, T = 0.25, 1.0
DIMS = {2: (37, 29), 3: (37, 29, 11)}       # nx not a multiple of 32
ORIGIN = {2: (-1.0, 0.5), 3: (-1.0, 0.5, 0.25)}


def controls(dim):
    from scenarios import control_set

    return control_set(1.0, 3, dim)


def action_of(dim, u):
    U = controls(dim)
    return int(np.flatnonzero((U == np.asarray(u, dtype=np.float64)).all(1))[0])


def grid_of(dim):
    g = np.zeros(DIMS[dim][::-1], dtype=np.int8)
    g[..., 20:23, 12:15] = 100  # one block (through every z-layer)
    g[..., 3, 30] = -1
    return g.reshape(-1)


def oracle_env(dim, region=None, v_max=-1.0):
    return ob.OracleEnv(dim, ACC, controls(dim), grid_of(dim), DIMS[dim], ORIGIN[dim], RES, T=T, w=10.0, v_max=v_max,
                        region=region)


def centre(dim, cell):
    return [ORIGIN[dim][k] + (cell[k] + 0.5) * RES for k in range(dim)]


# ---- the plain-numpy walk ----------------------------------------------------------------------------------
def to_cell(p, origin):
    x = (p - origin) / RES - 0.5
    if not abs(x) < 2147483648.0:  # NaN / beyond int: what the reference's cvttsd2si yields
        return INT_MIN
    return int(math.copysign(math.floor(abs(x) + 0.5), x))


def wrap32(v):
    return (v + 2 ** 31) % 2 ** 32 - 2 ** 31


def sample_count(dim, parent, u):
    """n = ceil(max_v T / res) of an ACC edge: v is linear, max_v = max(|v(0)|, |v(T)|) over the axes."""
    max_v = 0.0
    for k in range(dim):
        v0 = float(parent["vel"][k])
        max_v = max(max_v, max(abs(v0), abs(u[k] * T + v0)))
    return math.ceil(max_v * T / RES)


def walk_acc(dim, parent, u):
    """(cells, ids) of getLinkedNodes' walk: n + 1 samples at t = i (T / n), p(t) = u/2 t t + v t + p, an entry
    whenever getIndex (int arithmetic, no bounds test) differs from the previous one, prev_id starting at -1."""
    n = sample_count(dim, parent, u)
    dt = T / n if n else math.inf
    cells, ids, prev = [], [], -1
    for i in range(n + 1):
        t = i * dt if n else math.nan  # 0 * inf
        pn = []
        for k in range(dim):
            p = float(u[k]) / 2 * t * t + float(parent["vel"][k]) * t + float(parent["pos"][k])
            pn.append(to_cell(p, ORIGIN[dim][k]))
        idx = pn[0] + DIMS[dim][0] * pn[1] + (DIMS[dim][0] * DIMS[dim][1] * pn[2] if dim == 3 else 0)
        idx = wrap32(idx)
        if idx != prev:
            cells.append(pn)
            ids.append(idx)
            prev = idx
    return cells, ids


def inside(dim, cell):
    return all(0 <= cell[k] < DIMS[dim][k] for k in range(dim))


# ---- the cases ------------------------------------------------------------------------------------------
def constructed(dim):
    """[(name, parent, action)] with the branch of each case asserted from the restatement."""
    out = []
    zero, last = (0,) * dim, tuple(d - 1 for d in DIMS[dim])

    def add(name, pos, vel, u):
        w = np.zeros((), dtype=ob.WAYPOINT_DTYPE)
        w["pos"][:dim], w["vel"][:dim] = pos, vel
        out.append((name, w, action_of(dim, u)))
        return w

    u0 = (0.0,) * dim
    # n = 0: at rest under u = 0; dt = T / 0, the one sample at 0 * inf = NaN
    w = add("rest_n0", centre(dim, (5,) * dim), u0, u0)
    assert sample_count(dim, w, u0) == 0 and walk_acc(dim, w, u0)[0] == [[INT_MIN] * dim]
    # a NaN position with a finite velocity: every sample converts to INT_MIN, one entry
    w = add("nan_pos", [math.nan] + centre(dim, (5,) * dim)[1:], (1.0,) + (0.0,) * (dim - 1), u0)
    assert walk_acc(dim, w, u0)[0] == [[INT_MIN] + [5] * (dim - 1)]
    # leaving the map through every face: only the t = T sample is outside
    for k in range(dim):
        for side, cell in ((-1, 1), (1, DIMS[dim][k] - 2)):
            c = [6] * dim
            c[k] = cell
            vel = [0.0] * dim
            vel[k] = side * 0.5  # two cells per T: n = 2, the samples lie in cell, cell + side, cell + 2 side
            w = add(f"leaves_axis{k}_{'low' if side < 0 else 'high'}", centre(dim, c), vel, u0)
            cells, _ = walk_acc(dim, w, u0)
            assert all(inside(dim, x) for x in cells[:-1]) and not inside(dim, cells[-1]) and len(cells) == 3
    # entering from outside; far outside on both sides
    c = [6] * dim
    c[0] = -3
    add("enters_from_low_x", centre(dim, c), [1.0] + [0.0] * (dim - 1), u0)
    add("far_outside", [1e12] * dim, [-1.0] * dim, u0)
    add("beyond_int", [1e300] * dim, [1.0] * dim, u0)
    # the prev_id = -1 quirk: the walk starts in cell (-1, 0[, 0]) whose index is -1, so that cell is dropped
    c = [0] * dim
    c[0] = -1
    w = add("first_index_minus_one", centre(dim, c), [0.5] + [0.0] * (dim - 1), u0)
    cells, ids = walk_acc(dim, w, u0)
    assert to_cell(float(w["pos"][0]), ORIGIN[dim][0]) == -1 and ids[0] == 0 and cells[0] == [0] * dim and len(cells) == 2
    # getIndex wraps for negative cells: (-1, 1) aliases (nx - 1, 0); rows below the map have negative indices
    c = [0] * dim
    c[0], c[1] = -1, 1
    w = add("aliases_last_cell_of_row0", centre(dim, c), [0.0, -0.25] + [0.0] * (dim - 2), u0)
    assert walk_acc(dim, w, u0)[1][0] == DIMS[dim][0] - 1
    c = [4, 1] + [0] * (dim - 2)
    w = add("negative_indices", centre(dim, c), [0.25, -1.0] + [0.0] * (dim - 2), u0)
    assert min(walk_acc(dim, w, u0)[1]) < -1
    # through the obstacle block, along its face, through the unknown cell, and a plain free edge
    c = [11, 21] + [5] * (dim - 2)
    add("hits_block", centre(dim, c), [1.0, 0.0] + [0.0] * (dim - 2), (1.0,) + (0.0,) * (dim - 1))
    c = [10, 19] + [5] * (dim - 2)
    add("along_block", centre(dim, c), [1.0, 0.0] + [0.0] * (dim - 2), u0)
    c = [28, 3] + [0] * (dim - 2)
    add("through_unknown", centre(dim, c), [1.0, 0.0] + [0.0] * (dim - 2), u0)
    add("free_diagonal", centre(dim, (2,) * dim), [1.0] * dim, (-1.0,) * dim)
    add("decelerates_to_rest", centre(dim, (8,) * dim), [1.0] * dim, (-1.0,) * dim)
    # samples exactly on cell boundaries
    add("on_boundaries", [ORIGIN[dim][k] + 6 * RES for k in range(dim)], [0.5] * dim, u0)
    add("corner_cell_low", centre(dim, zero), [0.25] * dim, u0)
    add("corner_cell_high", centre(dim, last), [-0.25] * dim, u0)
    return out


def batch(dim):
    cases = constructed(dim)
    parents = np.array([w for _, w, _ in cases], dtype=ob.WAYPOINT_DTYPE)
    actions = np.array([a for _, _, a in cases], dtype=np.int32)
    return [n for n, _, _ in cases], parents, actions


def region_of(dim):
    """Everything but a slab of rows, so that some otherwise free edges end outside the region."""
    r = np.ones(DIMS[dim][::-1], dtype=np.uint8)
    r[..., 8:10, :] = 0
    return r.reshape(-1)


def contract_only(dim):
    """Edges without a CPU witness: n beyond kEdgeNMax, NaN / infinite velocities."""
    rows = []
    for vel in ([1e6] + [0.0] * (dim - 1), [math.nan] + [0.0] * (dim - 1), [0.0] * (dim - 1) + [math.inf],
                [(EDGE_N_MAX + 1) * RES] + [0.0] * (dim - 1)):
        w = np.zeros((), dtype=ob.WAYPOINT_DTYPE)
        w["pos"][:dim], w["vel"][:dim] = centre(dim, (5,) * dim), vel
        rows.append(w)
    assert sample_count(dim, rows[0], (0.0,) * dim) > EDGE_N_MAX and sample_count(dim, rows[3], (0.0,) * dim) == EDGE_N_MAX + 1
    return np.array(rows, dtype=ob.WAYPOINT_DTYPE), np.full(len(rows), action_of(dim, (0.0,) * dim), dtype=np.int32)


def largest_served(dim):
    """n == kEdgeNMax exactly: the largest edge that is still walked (oracle witness only)."""
    w = np.zeros(1, dtype=ob.WAYPOINT_DTYPE)
    w["pos"][0, :dim], w["vel"][0, 0] = centre(dim, (5,) * dim), EDGE_N_MAX * RES
    assert sample_count(dim, w[0], (0.0,) * dim) == EDGE_N_MAX
    return w, np.array([action_of(dim, (0.0,) * dim)], dtype=np.int32)


# ---- the pins ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("with_region", [False, True])
def test_constructed_edges_oracle_matches_reference(dim, with_region):
    names, parents, actions = batch(dim)
    env = oracle_env(dim, region_of(dim) if with_region else None)
    fo, co = env.edges_is_free(parents, actions)
    fr, cr = ob.ref_edges_is_free(env, parents, actions)
    same_array(fo, fr, "free")
    same_array(co, cr, "cost", bits=True)
    free = dict(zip(names, fo))
    assert not free["rest_n0"] and not free["nan_pos"] and not free["hits_block"] and not free["first_index_minus_one"]
    assert not any(free[n] for n in names if n.startswith("leaves_"))
    assert free["along_block"] and free["through_unknown"] and free["corner_cell_low"] and free["corner_cell_high"]
    assert bool(free["decelerates_to_rest"]) != with_region  # it crosses the slab the region leaves out


@pytest.mark.parametrize("dim", [2, 3])
def test_constructed_edges_oracle_walk_matches_numpy_walk(dim):
    names, parents, actions = batch(dim)
    off, cells = oracle_env(dim).edges_cells(parents, actions)
    U = controls(dim)
    for i, name in enumerate(names):
        want, _ = walk_acc(dim, parents[i], U[actions[i]])
        got = cells[off[i]:off[i + 1]]
        assert got.tolist() == want, name
    lengths = dict(zip(names, np.diff(off)))
    assert lengths["rest_n0"] == 1 and lengths["first_index_minus_one"] == 2 and lengths["negative_indices"] > 3
