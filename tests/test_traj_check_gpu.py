"""mplx_traj_check (env_map.traverse_trajectories): trajectories checked against the map and the dynamic limits on
the device, against the host restatement (env_map_host::traverse_trajectory, is_free, validate_primitive in
mpl_host.hpp, pinned to the reference by tests/test_traj_check_vs_ref.py) on the same inputs.

Accuracy contract (DESIGN.md §8): without time scaling, status and cost are bit for bit, for every control; so are
seg_free and seg_valid for VEL and ACC paths.  On JRK paths max_vel goes through CUDA's cbrt / acos / cos, so a
segment's seg_free may differ only where the host's max_v * T / res is within 1e-9 relative of an integer, and its
seg_valid only where a maximum is within 1e-9 relative of its limit (or, for the yaw test, d within 1e-12 of
cos(yaw_max)).  A scaled path's samples go through Lambda::getTau's closed-form quartic, so its cost may differ
only where a host sample lies within 1e-9 (1 + |x|) of a cell boundary, or, with a gradient weight, by 1e-9
relative: |vel| = v / lambda carries getTau's rounding into the sum.  As in mplx_traj_scale, the final sample's time
can land an ulp past the last lambda segment, where getTau finds no root and the sample is the start state; the
two sides may disagree about that one sample (start state against a root near the end).  The exceptions are
counted and reported."""
import ctypes as C
import warnings

import numpy as np
import pytest

import traj_check_bindings as CB
from motion_primitive_library_b200 import MapUtil, TrajSolverBatch, abi, env_map
from motion_primitive_library_b200 import planner as P

pytestmark = pytest.mark.gpu

VEL, ACC, JRK, YAW = CB.VEL, CB.ACC, CB.JRK, CB.YAW
SCALE, SCALE_DOWN = 1, 2
EXCEPTIONS = {"seg_free": 0, "seg_valid": 0, "cost": 0, "cost_gradient": 0, "cost_final_row": 0}
COMPARED = {"segments": 0, "scaled_paths": 0, "scaled_gradient_paths": 0}
MDIM3, RES3, ORIGIN3 = (48, 40, 16), 0.25, (-6.0, -5.0, -2.0)
MDIM2, RES2, ORIGIN2 = (64, 48), 0.2, (-6.4, -4.8)


def test_struct_layout():
    assert C.sizeof(abi.TrajCheckOut) == 4 * C.sizeof(C.c_void_p) + 8
    assert abi.TrajCheckOut.seconds.offset == 4 * C.sizeof(C.c_void_p)
    assert [f[0] for f in abi.TrajCheckOut._fields_] == ["status", "cost", "seg_free", "seg_valid", "seconds"]


@pytest.fixture(scope="module")
def solvers():
    s = {2: TrajSolverBatch(2), 3: TrajSolverBatch(3)}
    yield s
    for x in s.values():
        x.close()


def world(dim, seed):
    if dim == 3:
        return CB.random_grid(MDIM3, seed), MDIM3, ORIGIN3, RES3
    return CB.random_grid(MDIM2, seed, p_occ=0.02), MDIM2, ORIGIN2, RES2


def make_env(dim, grid, mdim, origin, res, limits):
    mu = MapUtil()
    mu.setMap(np.asarray(origin, dtype=np.float64), np.asarray(mdim), grid.copy(), res)
    e = env_map(mu, device=0)
    e.set_control(ACC)
    e.set_u(np.zeros((1, dim)))
    for k, v in limits.items():
        getattr(e, "set_" + k)(v)
    return e


def device_paths(s, dim, control, yaw, n_paths, seed, lo, hi, n_wp=(2, 14)):
    """mplx_traj_solve outputs (TrajSolverBatch.solve) through random waypoints in [lo, hi)"""
    rng = np.random.default_rng(seed)
    ws, wc, dts = [], [], []
    for _ in range(n_paths):
        n = int(rng.integers(n_wp[0], n_wp[1] + 1))
        w = np.zeros(n, dtype=P.WAYPOINT_DTYPE)
        w["pos"][:, :dim] = lo + (hi - lo) * rng.random((n, dim))
        w["yaw"] = rng.uniform(-3, 3, n)
        ws.append(w)
        wc.append(np.full(n, control | (YAW if yaw else 0), dtype=np.uint8))
        dts.append(rng.uniform(0.5, 3, n - 1))
    res, _ = s[dim].solve(ws, control | (YAW if yaw else 0), wp_control=wc, dts=dts)
    assert all(r["status"] == 1 for r in res)
    return [dict(seg_t=r["seg_t"], coeff=r["coeff"]) for r in res], np.full(n_paths, control | (YAW if yaw else 0),
                                                                             dtype=np.uint8)


def box(mdim, origin, res, margin=0.1):
    lo = np.asarray(origin, dtype=np.float64)
    ext = np.asarray(mdim) * res
    return lo + margin * ext, lo + (1 - margin) * ext


def host_of(dim, grid, mdim, origin, res, paths, ctl, limits, **kw):
    return CB.traj_check(dim, grid, mdim, origin, res, paths, ctl, nthreads=8, **limits, **kw)


def flat(dev, key):
    """the per-segment flags in their waypoint slots: a path's last slot holds 0, a path without segments has none"""
    return np.concatenate([np.append(r[key], 0).astype(np.uint8) for r in dev if len(r[key])] + [np.zeros(0, np.uint8)])


def near_integer(x):
    return abs(x - round(x)) <= 1e-9 * max(abs(x), 1.0)


def yaw_d(c, t, dim):
    """validate_yaw's d = v.normalized() . (cos yaw, sin yaw) at both ends of a segment (numpy's arithmetic)"""
    out = []
    for te in (0.0, t):
        v = np.array([np.polyval(np.polyder(np.array([c[a][0] / 120, c[a][1] / 24, c[a][2] / 6, c[a][3] / 2, c[a][4],
                                                      c[a][5]])), te) for a in range(2)])
        yaw = np.polyval(np.array([c[dim][0] / 120, c[dim][1] / 24, c[dim][2] / 6, c[dim][3] / 2, c[dim][4], c[dim][5]]), te)
        if np.linalg.norm(v) > 0:
            out.append(v[0] / np.linalg.norm(v) * np.cos(yaw) + v[1] / np.linalg.norm(v) * np.sin(yaw))
    return out


def segment_exception_ok(key, c, t, ctl, dim, res, limits):
    """whether a segment's disagreement is one the contract allows: on JRK paths max_v * T / res within 1e-9 of an
    integer (seg_free) or a maximum within 1e-9 of its limit (seg_valid); on yaw paths d within 1e-12 of
    cos(yaw_max) (seg_valid)"""
    jrk = ctl & 15 == JRK
    if key == "seg_free":
        return jrk and near_integer(max(CB.max_abs(c[a], t, 1) for a in range(dim)) * t / res)
    near = []
    if jrk:
        for order, lim in ((1, limits.get("v_max", -1)), (2, limits.get("a_max", -1))):
            if lim > 0:
                near += [abs(CB.max_abs(c[a], t, order) - lim) <= 1e-9 * lim for a in range(dim)]
    ym = limits.get("yaw_max", -1)
    if ctl & YAW and ym > 0:
        near += [abs(d - np.cos(ym)) <= 1e-12 for d in yaw_d(c, t, dim)]
    return any(near)


def compare(dev, host, paths, ctl, dim, res, limits, host_samples=None, origin=None, gradient=0.0, final_row=None):
    """device against host under the contract; host_samples(p, N): the host's sample rows of scaled path p;
    final_row(p, cost): whether the device's cost is the host's with the final sample at the other end"""
    st = np.array([r["status"] for r in dev], dtype=np.int32)
    cost = np.array([r["cost"] for r in dev])
    assert st.tobytes() == host["status"].tobytes()
    bad = np.nonzero(cost.view(np.uint64) != host["cost"].view(np.uint64))[0]
    if host_samples is not None:
        COMPARED["scaled_paths"] += len(cost)
        COMPARED["scaled_gradient_paths"] += len(cost) if gradient > 0 else 0
    for p in bad:
        assert host_samples is not None, (p, cost[p], host["cost"][p])
        h = host["cost"][p]
        if gradient > 0 and np.isfinite(h) and abs(cost[p] - h) <= 1e-9 * (1 + abs(h)):
            EXCEPTIONS["cost_gradient"] += 1
            continue
        if near_boundary(host_samples, int(p), dim, origin, res, limits["v_max"]):
            EXCEPTIONS["cost"] += 1
            continue
        assert final_row(int(p), cost[p]), (p, cost[p], h)
        EXCEPTIONS["cost_final_row"] += 1
    offs = host["offset"]
    COMPARED["segments"] += int(offs[-1])
    for key in ("seg_free", "seg_valid"):
        got, want = flat(dev, key), host[key]
        assert got.size == want.size
        for k in np.nonzero(got != want)[0]:
            p = int(np.searchsorted(offs, k, side="right") - 1)
            j = int(k - offs[p])
            assert segment_exception_ok(key, np.asarray(paths[p]["coeff"][j]), float(paths[p]["seg_t"][j]), int(ctl[p]),
                                        dim, res, limits), (key, p, j)
            EXCEPTIONS[key] += 1


def py_cost(rows, dim, grid, mdim, origin, res, pot=None, pw=0.0, gw=0.0):
    """traverse_trajectory over sample rows, in numpy (not bit for bit): to explain a final-row disagreement"""
    prev, c = 0xFFFFFFFF, 0.0
    mdim = np.asarray(mdim)
    for r in rows:
        x = (r[:dim] - np.asarray(origin)) / res - 0.5
        pn = np.where(x >= 0, np.floor(x + 0.5), np.ceil(x - 0.5)).astype(np.int64)
        idx = int(pn[0] + mdim[0] * pn[1] + (mdim[0] * mdim[1] * pn[2] if dim == 3 else 0)) & 0xFFFFFFFF
        if idx == prev:
            continue
        prev = idx
        if (pn < 0).any() or (pn >= mdim).any():
            return np.inf
        if pot is not None:
            if pot[idx] >= 100:
                return np.inf
            if pot[idx] > 0:
                c += pw * pot[idx] + gw * np.linalg.norm(r[dim:2 * dim])
        elif grid[idx] == 100:
            return np.inf
    return c


def final_row_explainer(dim, grid, mdim, origin, res, sc, host_samples, device_samples, limits, pot=None, pw=0.0,
                        gw=0.0):
    """final_row for compare: the two sides disagree about the final sample only, one taking the start state
    (getTau found no root) and the other a root near the end.  The device's own sample rows (mplx_traj_scale's
    sampling, the same traj_row under the same lambda) must agree with the host's on every earlier row, and the
    host's rows with the final one replaced by the device's must give the device's cost."""
    def explain(p, dev_cost):
        N = int(np.ceil(limits["v_max"] * sc[p]["total_t"] / res))
        rows, drows = host_samples(p, N)[0], device_samples(p, N)
        if not np.allclose(drows[:-1, :2 * dim], rows[:-1, :2 * dim], rtol=1e-7, atol=1e-7):
            return False
        start = rows[0, :dim].tobytes()
        if (rows[-1, :dim].tobytes() == start) == (drows[-1, :dim].tobytes() == start):
            return False  # not a start-against-root disagreement
        alt = rows.copy()
        alt[-1] = drows[-1]
        want = py_cost(alt, dim, grid, mdim, origin, res, pot, pw, gw)
        return bool((np.isinf(want) and np.isinf(dev_cost)) or abs(want - dev_cost) <= 1e-6 * (1 + abs(dev_cost)))

    return explain


def near_boundary(host_samples, p, dim, origin, res, v_max):
    """a host sample of path p within 1e-9 (1 + |x|) of a cell boundary (origin + k res)"""
    rows, total = host_samples(p)
    N = int(np.ceil(v_max * total / res))
    pos = host_samples(p, N)[0][:, :dim]
    x = (pos - np.asarray(origin)) / res
    return bool((np.abs(x - np.round(x)) * res <= 1e-9 * (1 + np.abs(pos))).any())


CASES = [(dim, control, yaw) for dim in (2, 3) for control in (VEL, ACC, JRK) for yaw in (False, True)]


@pytest.mark.parametrize("dim,control,yaw", CASES)
@pytest.mark.parametrize("with_region", [False, True])
def test_solved_paths(solvers, dim, control, yaw, with_region):
    grid, mdim, origin, res = world(dim, 5 * dim + control + yaw)
    limits = dict(v_max=1.5, a_max=1.0, j_max=2.0, yaw_max=0.9)
    e = make_env(dim, grid, mdim, origin, res, limits)
    region = None
    if with_region:
        region = (np.random.default_rng(dim + control).random(grid.size) < 0.95).astype(np.uint8)
        e.set_search_region(region)
    lo, hi = box(mdim, origin, res, margin=-0.05)
    paths, ctl = device_paths(solvers, dim, control, yaw, 300, 11 * dim + control + yaw, lo, hi)
    dev, sec = e.traverse_trajectories(paths, ctl)
    host = host_of(dim, grid, mdim, origin, res, paths, ctl, limits, region=region)
    compare(dev, host, paths, ctl, dim, res, limits)
    assert sec > 0 and host["status"].all()
    assert np.isinf(host["cost"]).any() and (host["cost"] == 0).any()
    real = np.ones(host["seg_free"].size, dtype=bool)
    real[host["offset"][1:] - 1] = False
    assert host["seg_free"][real].any() and not host["seg_free"][real].all()
    assert (control == VEL and not yaw) or not host["seg_valid"][real].all()
    e.close()


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("route", ["set_potential", "update_potential_map"])
@pytest.mark.parametrize("gradient", [0.0, 0.6])
def test_potential(solvers, dim, route, gradient):
    grid, mdim, origin, res = world(dim, 70 + dim)
    grid[grid < 0] = 0
    limits = dict(v_max=1.2, a_max=2.0)
    e = make_env(dim, grid, mdim, origin, res, limits)
    e.set_potential_weight(0.25)
    e.set_gradient_weight(gradient)
    if route == "set_potential":
        rng = np.random.default_rng(dim)
        pot = np.where(grid == 100, 100, rng.integers(-3, 60, grid.size))
        pot[rng.random(grid.size) < 0.003] = 120
        pot = pot.astype(np.int8)
        e.set_potential_map(pot)
        host_grid = grid
    else:
        pot = e.update_potential_map([0.8] * dim)
        host_grid = pot
    assert (pot > 0).any() and (pot >= 100).any()
    lo, hi = box(mdim, origin, res)
    paths, ctl = device_paths(solvers, dim, JRK, dim == 2, 300, 90 + dim, lo, hi)
    dev, _ = e.traverse_trajectories(paths, ctl)
    host = host_of(dim, host_grid, mdim, origin, res, paths, ctl, limits, potential=pot, potential_weight=0.25,
                   gradient_weight=gradient)
    compare(dev, host, paths, ctl, dim, res, limits)
    fin = host["cost"][np.isfinite(host["cost"])]
    assert (fin > 0).any() and np.isinf(host["cost"]).any()
    e.close()


@pytest.mark.parametrize("dim,control", [(2, ACC), (3, ACC), (3, JRK), (2, JRK)])
@pytest.mark.parametrize("mode", [SCALE, SCALE_DOWN])
def test_scaled(solvers, dim, control, mode):
    """mplx_traj_scale's outputs fed in directly: the device's lambda on both sides"""
    grid, mdim, origin, res = world(dim, 30 + dim)
    limits = dict(v_max=1.3, a_max=1.0)
    e = make_env(dim, grid, mdim, origin, res, limits)
    lo, hi = box(mdim, origin, res)
    paths, ctl = device_paths(solvers, dim, control, False, 200, 130 + dim + mode, lo, hi)
    kw = dict(ri=0.8, rf=1.4) if mode == SCALE else dict(mv=0.7, ri=1.0, rf=1.0)
    sc, _ = solvers[dim].scale(paths, mode, with_lambda=True, **kw)
    assert sum(r["status"] == 1 for r in sc) > 10
    dev, _ = e.traverse_trajectories(paths, ctl, scaled=sc)
    host = host_of(dim, grid, mdim, origin, res, paths, ctl, limits, scaled=sc)

    def host_samples(p, N=1):
        r = P.traj_scale(dim, paths[p]["seg_t"], paths[p]["coeff"], mode, control=control, n_samples=N, **kw)
        assert sc[p]["status"] == 1 and r["status"] == 1
        return r["samples"], r["total_t"]

    def device_samples(p, N):
        return solvers[dim].scale([paths[p]], mode, n_samples=N, **kw)[0][0]["samples"]

    compare(dev, host, paths, ctl, dim, res, limits, host_samples=host_samples, origin=origin,
            final_row=final_row_explainer(dim, grid, mdim, origin, res, sc, host_samples, device_samples, limits))
    unscaled, _ = e.traverse_trajectories(paths, ctl)
    assert any(a["status"] != b["status"] or a["cost"] != b["cost"] for a, b in zip(dev, unscaled))
    # the same paths on a potential field with a gradient weight
    e.set_potential_weight(0.2)
    e.set_gradient_weight(0.5)
    pot = np.where(grid == 100, 100, np.random.default_rng(mode).integers(0, 50, grid.size)).astype(np.int8)
    e.set_potential_map(pot)
    dev, _ = e.traverse_trajectories(paths, ctl, scaled=sc)
    host = host_of(dim, grid, mdim, origin, res, paths, ctl, limits, scaled=sc, potential=pot, potential_weight=0.2,
                   gradient_weight=0.5)
    compare(dev, host, paths, ctl, dim, res, limits, host_samples=host_samples, origin=origin, gradient=0.5,
            final_row=final_row_explainer(dim, grid, mdim, origin, res, sc, host_samples, device_samples, limits, pot,
                                          0.2, 0.5))
    e.close()


def test_update_cells_without_reupload(solvers):
    dim = 3
    grid, mdim, origin, res = world(dim, 3)
    grid[:] = 0
    limits = dict(v_max=1.0, a_max=1.0)
    e = make_env(dim, grid, mdim, origin, res, limits)
    lo, hi = box(mdim, origin, res)
    paths, ctl = device_paths(solvers, dim, ACC, False, 100, 17, lo, hi)
    before, _ = e.traverse_trajectories(paths, ctl)
    assert all(r["cost"] == 0 for r in before)
    rng = np.random.default_rng(1)
    idx = rng.choice(grid.size, grid.size // 50, replace=False)
    e.update_cells(idx, np.full(idx.size, 100, dtype=np.int8))
    grid2 = grid.copy()
    grid2[idx] = 100
    after, _ = e.traverse_trajectories(paths, ctl)
    host = host_of(dim, grid2, mdim, origin, res, paths, ctl, limits)
    compare(after, host, paths, ctl, dim, res, limits)
    assert np.isinf(host["cost"]).any()
    e.close()


def test_sample_counts_across_warps(solvers):
    """N from 1 to above 10^5 samples per path, across warp (32) and CTA (128) boundaries, on a potential field with a
    gradient weight: every counted sample adds a term, so the previous-index rule at chunk edges and the in-order sum
    show in the cost bit for bit"""
    dim = 2
    grid, mdim, origin, res = world(dim, 9)
    grid[:] = 0
    pot = np.random.default_rng(9).integers(-3, 60, grid.size).astype(np.int8)
    p = P.traj_solve(dim, ACC, pos=np.array([[-5.5, -4.0], [-1.0, 3.5], [1.0, -3.0], [5.5, 4.0]]), v=1.0, n_samples=1)
    path = dict(seg_t=p["seg_t"], coeff=p["coeff"])
    total = float(np.sum(p["seg_t"]))
    e = make_env(dim, grid, mdim, origin, res, {})
    e.set_potential_weight(0.3)
    e.set_gradient_weight(0.7)
    e.set_potential_map(pot)
    seen, costs = set(), []
    for n in (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1000, 4097, 150_000):
        v = n * res / total * (1 - 1e-12)
        limits = dict(v_max=v)
        e.set_v_max(v)
        dev, _ = e.traverse_trajectories([path], ACC)
        host = host_of(dim, grid, mdim, origin, res, [path], [ACC], limits, potential=pot, potential_weight=0.3,
                       gradient_weight=0.7)
        compare(dev, host, [path], [ACC], dim, res, limits)
        assert host["status"][0] == 1
        seen.add(int(np.ceil(v * total / res)))
        costs.append(host["cost"][0])
    e.close()
    assert max(seen) > 100_000 and 1 in seen and 33 in seen and 129 in seen
    assert np.isfinite(costs).all() and costs[-1] > costs[3] > 0


def test_wrapped_index_rule(solvers):
    """defined behaviour 4 on the device: the end sample's index 2^32 wraps to the start's 0, so with N = 1 it is not
    counted (cost 0); with N = 2 the middle sample is counted and lies outside (+inf).  The env never gets set_u or
    set_control: the checks read only the limits."""
    grid, mdim, origin, res, paths = CB.wrapped_index_case()
    mu = MapUtil()
    mu.setMap(np.asarray(origin), np.asarray(mdim), grid.copy(), res)
    e = env_map(mu, device=0)
    for k, want in ((1, 0.0), (2, np.inf)):
        limits = dict(v_max=k / 65536)
        e.set_v_max(limits["v_max"])
        dev, _ = e.traverse_trajectories(paths, VEL)
        host = host_of(3, grid, mdim, origin, res, paths, [VEL], limits)
        compare(dev, host, paths, [VEL], 3, res, limits)
        assert host["status"][0] == 1 and host["cost"][0] == want
    e.close()


def test_batch_independence_and_launches(solvers):
    dim = 3
    grid, mdim, origin, res = world(dim, 21)
    limits = dict(v_max=1.5, a_max=1.0)
    e = make_env(dim, grid, mdim, origin, res, limits)
    lo, hi = box(mdim, origin, res, margin=-0.05)
    paths, ctl = device_paths(solvers, dim, JRK, False, 2000, 23, lo, hi)
    base, _ = e.traverse_trajectories(paths, ctl)
    perm = np.random.default_rng(2).permutation(len(paths))
    shuf, _ = e.traverse_trajectories([paths[i] for i in perm], ctl[perm])
    for k, i in enumerate(perm):
        assert shuf[k]["cost"] == base[i]["cost"] or (np.isnan(shuf[k]["cost"]) and np.isnan(base[i]["cost"]))
        assert shuf[k]["status"] == base[i]["status"]
        assert (shuf[k]["seg_free"] == base[i]["seg_free"]).all() and (shuf[k]["seg_valid"] == base[i]["seg_valid"]).all()
    halves = e.traverse_trajectories(paths[:700], ctl[:700])[0] + e.traverse_trajectories(paths[700:], ctl[700:])[0]
    for a, b in zip(halves, base):
        assert a["cost"] == b["cost"] and a["status"] == b["status"] and (a["seg_free"] == b["seg_free"]).all()
    launches = []
    for n in (1, 10, 2000):
        l0 = e.launch_count()
        e.traverse_trajectories(paths[:n], ctl[:n])
        launches.append(e.launch_count() - l0)
    # a batch in which no path has a segment has no waypoint slot: the segment kernel runs on one block
    empty = dict(seg_t=np.zeros(0), coeff=np.zeros((0, dim + 1, 6)))
    l0 = e.launch_count()
    out, _ = e.traverse_trajectories([empty, empty], ctl[:2])
    launches.append(e.launch_count() - l0)
    assert [(o["status"], o["cost"]) for o in out] == [(0, 0.0), (0, 0.0)]
    assert launches == [3, 3, 3, 3]
    e.close()


def test_defined_behaviours(solvers):
    dim = 3
    grid, mdim, origin, res = world(dim, 4)
    lo, hi = box(mdim, origin, res)
    paths, ctl = device_paths(solvers, dim, ACC, False, 6, 5, lo, hi)
    bad = [dict(p) for p in paths]
    bad[0]["seg_t"] = np.array(bad[0]["seg_t"]); bad[0]["seg_t"][0] = -1.0
    bad[1]["seg_t"] = np.array(bad[1]["seg_t"]); bad[1]["seg_t"][-1] = np.nan
    bad[2]["coeff"] = np.array(bad[2]["coeff"]); bad[2]["coeff"][-1, 0, 0] = np.inf
    bad.append(dict(seg_t=np.zeros(0), coeff=np.zeros((0, 4, 6))))
    c = np.append(ctl, ACC)
    for vm in (-1.0, 0.0, 1.0, 1e9):
        limits = dict(v_max=vm, a_max=0.8)
        e = make_env(dim, grid, mdim, origin, res, limits)
        dev, _ = e.traverse_trajectories(bad, c)
        host = host_of(dim, grid, mdim, origin, res, bad, c, limits)
        compare(dev, host, bad, c, dim, res, limits)
        want = [0, 0, 0, 1, 1, 1, 0] if vm == 1.0 else [0] * 7
        assert host["status"].tolist() == want
        e.close()


def test_refusals():
    dim = 2
    grid, mdim, origin, res = world(dim, 1)
    lib = abi.load()
    h = C.c_void_p()
    abi.check(lib.mplx_create(dim, 0, C.byref(h)))
    offset = np.array([0, 3], dtype=np.int64)
    seg_t = np.ones(3)
    coeff = np.zeros((3, 3, 6))
    ctl = np.array([ACC], dtype=np.uint8)
    st = np.full(1, 7, dtype=np.int32)
    cost = np.full(1, 7.0)
    fr = np.full(3, 7, dtype=np.uint8)
    out = abi.TrajCheckOut(st.ctypes.data, cost.ctypes.data, fr.ctypes.data, fr.ctypes.data, 0.0)

    def call(n=1, off=offset, s=seg_t, cf=coeff, c=ctl, tt=None, nl=None, lam=None, o=out):
        return lib.mplx_traj_check(h, n, abi.ptr(off), abi.ptr(s), abi.ptr(cf), abi.ptr(c), abi.ptr(tt), abi.ptr(nl),
                                   abi.ptr(lam), None if o is None else C.byref(o))

    assert call() == abi.MPLX_ERR_ARG  # no map
    mu = np.ascontiguousarray(grid)
    abi.check(lib.mplx_set_map(h, mu.ctypes.data, np.asarray(mdim, dtype=np.int32).ctypes.data,
                               np.asarray(origin, dtype=np.float64).ctypes.data, res))
    assert call() == abi.MPLX_ERR_ARG  # no params
    U = np.zeros((1, dim))
    abi.check(lib.mplx_set_params(h, ACC, 1.0, 10.0, 1.0, 1.0, -1.0, -1.0, -1.0, U.ctypes.data, 1, dim))
    l0 = lib.mplx_launch_count(h)
    nl = np.array([1], dtype=np.int32)
    tt = np.ones(1)
    lam = np.zeros((3 * 5 * dim, 7))
    refusals = [
        dict(n=-1), dict(off=None), dict(off=np.array([1, 3], dtype=np.int64)), dict(off=np.array([0, 3, 2], dtype=np.int64), n=2),
        dict(o=None), dict(o=abi.TrajCheckOut(None, cost.ctypes.data, None, None, 0.0)),
        dict(o=abi.TrajCheckOut(st.ctypes.data, None, None, None, 0.0)), dict(s=None), dict(cf=None), dict(c=None),
        dict(lam=lam), dict(lam=lam, nl=nl), dict(lam=lam, tt=tt), dict(nl=nl, tt=tt),
        dict(lam=lam, nl=np.array([-1], dtype=np.int32), tt=tt), dict(lam=lam, nl=np.array([31], dtype=np.int32), tt=tt),
    ]
    for kw in refusals:
        assert call(**kw) == abi.MPLX_ERR_ARG, kw
        assert st[0] == 7 and cost[0] == 7.0 and (fr == 7).all() and out.seconds == 0.0, kw
    assert lib.mplx_launch_count(h) == l0
    assert call(lam=lam, nl=np.array([30], dtype=np.int32), tt=tt) == abi.MPLX_OK  # 3 slots * 5 * dim
    assert call(n=0) == abi.MPLX_OK
    lib.mplx_destroy(h)


def test_report_exceptions():
    """the contract's allowed disagreements seen by the tests above (run last in this module): each kind stays rare.
    Bounds: a cell-boundary cost difference or a segment flag difference in at most 1 % of what was compared, a
    final-row difference in at most 5 % of the scaled paths, a gradient-rounding difference in at most 25 % of the
    scaled paths on a field with a gradient weight."""
    warnings.warn(f"traj_check exceptions allowed by the accuracy contract: {EXCEPTIONS} of {COMPARED}")
    seg = EXCEPTIONS["seg_free"] + EXCEPTIONS["seg_valid"]
    assert seg <= 0.01 * COMPARED["segments"], (EXCEPTIONS, COMPARED)
    assert EXCEPTIONS["cost"] <= 0.01 * COMPARED["scaled_paths"], (EXCEPTIONS, COMPARED)
    assert EXCEPTIONS["cost_final_row"] <= 0.05 * COMPARED["scaled_paths"], (EXCEPTIONS, COMPARED)
    assert EXCEPTIONS["cost_gradient"] <= 0.25 * COMPARED["scaled_gradient_paths"], (EXCEPTIONS, COMPARED)
