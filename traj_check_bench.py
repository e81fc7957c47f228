"""Throughput of mplx_traj_check (env_map.traverse_trajectories) against the host restatement (mplh_traj_check).

The 3-D 512^3, 0.1 m map of scenarios.cfg3 (its boxes, v_max 3, a_max 2), occupancy only and with a potential
field (mplx_update_potential_map, radius 0.5 m, weights 0.1 / 0.2).  The trajectories are mplx_traj_solve's JRK
output through random walks (steps of up to 1 m per axis, segment times from the L-inf allocation with v = 1)
at 1 024 / 4 096 / 16 384 paths of 16 / 64 / 256 waypoints, checked as solved and after mplx_traj_scale's
scale_down(mv = 1.5, 1, 1).  Per size: the device time of the kernels (CUDA events, median of --reps), the host
clock around the synchronous call (copies included), the host restatement on --host-threads threads where its
estimate from 64 paths is under --host-budget seconds, the samples the call evaluates at most (sum of N + 1 over
the paths; a path stops at its first collision) and the bytes the call moves (computed from the shapes).  Prints
one JSON line per size and the card's name and power limit, read in the same run."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

import scenarios as S  # noqa: E402
from motion_primitive_library_b200 import MapUtil, TrajSolverBatch, env_map  # noqa: E402
from motion_primitive_library_b200 import planner as P  # noqa: E402

JRK, SCALE_DOWN = 0x07, 2


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def walks(rng, n_paths, n_wp, lo, hi):
    start = lo + (hi - lo) * rng.random((n_paths, 1, 3))
    return list(start + np.cumsum(rng.uniform(-1, 1, (n_paths, n_wp, 3)), axis=1))


def call_bytes(n_paths, n_wp, scaled):
    """host-to-device and device-to-host bytes of one call: offsets, segment times, coefficients, control, the
    lambda slots when scaled, status, cost and the two segment flags"""
    b = 8 * (n_paths + 1) + 8 * n_wp + 8 * 4 * 6 * n_wp + n_paths
    if scaled:
        b += 8 * n_paths + 4 * n_paths + 8 * 7 * 15 * n_wp
    return b + 4 * n_paths + 8 * n_paths + 2 * n_wp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", default="1024,4096,16384")
    ap.add_argument("--waypoints", default="16,64,256")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-threads", type=int, default=8)
    ap.add_argument("--host-budget", type=float, default=20.0, help="seconds the host restatement may take per size")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    sc = S.cfg3()
    grid = sc.grid()
    mu = MapUtil()
    mu.setMap(sc.origin, sc.dim_cells, grid.copy(), sc.res)
    env = env_map(mu, device=0)
    env.set_control(sc.control)
    env.set_u(sc.U)
    env.set_v_max(sc.v_max)
    env.set_a_max(sc.a_max)
    solver = TrajSolverBatch(3)
    lo = np.asarray(sc.origin) + 0.2 * np.asarray(sc.dim_cells) * sc.res
    hi = np.asarray(sc.origin) + 0.8 * np.asarray(sc.dim_cells) * sc.res
    rng = np.random.default_rng(0)
    limits = dict(v_max=sc.v_max, a_max=sc.a_max)
    for field in ("occupancy", "potential"):
        host_grid, pot = grid, None
        if field == "potential":
            env.set_potential_weight(0.1)
            env.set_gradient_weight(0.2)
            pot = env.update_potential_map([0.5] * 3)
            host_grid = pot
        for n_wp in [int(x) for x in a.waypoints.split(",")]:
            for n_paths in [int(x) for x in a.paths.split(",")]:
                res, _ = solver.solve(walks(rng, n_paths, n_wp, lo, hi), JRK)
                paths = [dict(seg_t=r["seg_t"], coeff=r["coeff"]) for r in res]
                scaled_res, _ = solver.scale(paths, SCALE_DOWN, mv=1.5, with_lambda=True)
                for scaled in (None, scaled_res):
                    env.traverse_trajectories(paths[: min(64, n_paths)], JRK,
                                              scaled=None if scaled is None else scaled[: min(64, n_paths)])
                    dev, wall = [], []
                    for _ in range(a.reps):
                        t0 = time.perf_counter()
                        out, sec = env.traverse_trajectories(paths, JRK, scaled=scaled)
                        wall.append(time.perf_counter() - t0)
                        dev.append(sec)
                    totals = [s["total_t"] if s["status"] == 1 else float(np.sum(p["seg_t"]))
                              for s, p in zip(scaled_res, paths)] if scaled is not None else \
                        [float(np.sum(p["seg_t"])) for p in paths]
                    samples = int(sum(np.ceil(sc.v_max * t / sc.res) + 1 for t in totals))
                    costs = np.array([o["cost"] for o in out])
                    row = dict(field=field, scaled=scaled is not None, paths=n_paths, waypoints=n_wp,
                               samples_max=samples, collided=int(np.isinf(costs).sum()),
                               bytes=call_bytes(n_paths, n_paths * n_wp, scaled is not None),
                               device_ms=round(1e3 * float(np.median(dev)), 3),
                               call_ms=round(1e3 * float(np.median(wall)), 3))
                    kw = dict(potential=pot, potential_weight=0.1, gradient_weight=0.2, scaled=scaled, **limits)
                    # the estimate: a call of 1 path (the map copies) and the time per path of a call of 64
                    t_of = {}
                    for m in (1, min(64, n_paths)):
                        t0 = time.perf_counter()
                        P.traj_check(3, host_grid, sc.dim_cells, sc.origin, sc.res, paths[:m], JRK,
                                     nthreads=a.host_threads, **dict(kw, scaled=None if scaled is None else scaled[:m]))
                        t_of[m] = time.perf_counter() - t0
                    m = max(t_of)
                    est = t_of[1] + (t_of[m] - t_of[1]) * n_paths / max(m - 1, 1)
                    if est <= a.host_budget:
                        t0 = time.perf_counter()
                        h = P.traj_check(3, host_grid, sc.dim_cells, sc.origin, sc.res, paths, JRK,
                                         nthreads=a.host_threads, **kw)
                        row.update(host_s=round(time.perf_counter() - t0, 3), host_threads=a.host_threads,
                                   host_same_cost=int((h["cost"].view(np.uint64) == costs.view(np.uint64)).sum()))
                    else:
                        row.update(host_s=None, host_skipped=f"estimated {est:.0f} s on {a.host_threads} threads")
                    print(json.dumps(row), flush=True)
    solver.close()
    env.close()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
