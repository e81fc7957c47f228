"""Throughput of mplx_traj_solve (TrajSolverBatch) against the host's dense TrajSolver restatement.

setPath JRK and ACC paths with yaw VEL, 3-D, at 1 024 / 4 096 / 16 384 paths of 16 / 64 / 256 waypoints (random
walks, segment times from the L-inf allocation with v = 1).  Per size: the device time of the kernels (CUDA
events), the host clock around the synchronous call (copies included), and the host restatement (mpl_host.hpp,
dense, cubic in the path length) on all host cores where its estimate from one path is under a minute; the rest
are named as skipped.  Prints one JSON line per size and the card's name and power limit, read in the same run.

--scale times mplx_traj_scale (TrajSolverBatch.scale) instead: scale_down(mv = 0.5, 1, 1) of the device's solved
trajectories with sample(--scale-samples), against the host Trajectory's scale_down + sample on all host cores."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

from motion_primitive_library_b200 import TrajSolverBatch  # noqa: E402
from motion_primitive_library_b200 import planner as P  # noqa: E402

NAMES = {0x07: "JRK", 0x03: "ACC"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def _host_one(args):
    control, path = args
    return P.traj_solve(3, control, pos=path, v=1.0, n_samples=1)["segments"]


def _host_scale(args):
    seg_t, coeff, control, n_samples = args
    return P.traj_scale(3, seg_t, coeff, 2, mv=0.5, control=control, n_samples=n_samples)["status"]


def scale_main(a):
    cores = os.cpu_count() or 1
    s = TrajSolverBatch(3)
    rng = np.random.default_rng(0)
    ns = a.scale_samples
    for control in (0x07, 0x03):
        for n_wp in [int(x) for x in a.waypoints.split(",")]:
            for n_paths in [int(x) for x in a.paths.split(",")]:
                paths = [np.cumsum(rng.uniform(-1, 1, (n_wp, 3)), axis=0) for _ in range(n_paths)]
                res, _ = s.solve(paths, control)
                s.scale(res[: min(64, n_paths)], 2, mv=0.5, n_samples=ns)  # warm-up: module load, scratch
                s.scale(res, 2, mv=0.5, n_samples=ns)
                dev, wall = [], []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    out, sec = s.scale(res, 2, mv=0.5, n_samples=ns)
                    wall.append(time.perf_counter() - t0)
                    dev.append(sec)
                row = dict(leg="scale_down", control=NAMES[control], dim=3, paths=n_paths, waypoints=n_wp, samples=ns,
                           scaled=sum(o["status"] == 1 for o in out), device_ms=round(1e3 * float(np.median(dev)), 3),
                           call_ms=round(1e3 * float(np.median(wall)), 3))
                t0 = time.perf_counter()
                _host_scale((res[0]["seg_t"], res[0]["coeff"], control, ns))
                est = (time.perf_counter() - t0) * n_paths / cores
                if est <= a.host_budget:
                    t0 = time.perf_counter()
                    with ProcessPoolExecutor(cores) as ex:
                        list(ex.map(_host_scale, [(r["seg_t"], r["coeff"], control, ns) for r in res],
                                    chunksize=max(1, n_paths // (4 * cores))))
                    row.update(host_s=round(time.perf_counter() - t0, 3), host_cores=cores)
                else:
                    row.update(host_s=None, host_skipped=f"estimated {est:.0f} s on {cores} cores")
                print(json.dumps(row), flush=True)
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paths", default="1024,4096,16384")
    ap.add_argument("--waypoints", default="16,64,256")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-budget", type=float, default=60.0, help="seconds the host restatement may take per size")
    ap.add_argument("--scale", action="store_true", help="time mplx_traj_scale (scale_down) instead of the solve")
    ap.add_argument("--scale-samples", type=int, default=100, help="sample(N) of each scaled trajectory")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    if a.scale:
        scale_main(a)
        print(json.dumps({"card": card()}), flush=True)
        return
    cores = os.cpu_count() or 1
    s = TrajSolverBatch(3)
    rng = np.random.default_rng(0)
    for control in (0x07, 0x03):
        for n_wp in [int(x) for x in a.waypoints.split(",")]:
            for n_paths in [int(x) for x in a.paths.split(",")]:
                paths = [np.cumsum(rng.uniform(-1, 1, (n_wp, 3)), axis=0) for _ in range(n_paths)]
                s.solve(paths[: min(64, n_paths)], control)  # warm-up: module load, scratch
                s.solve(paths, control)
                dev, wall = [], []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    res, sec = s.solve(paths, control)
                    wall.append(time.perf_counter() - t0)
                    dev.append(sec)
                assert all(r["status"] == 1 for r in res)
                row = dict(control=NAMES[control], yaw="VEL", dim=3, paths=n_paths, waypoints=n_wp,
                           device_ms=round(1e3 * float(np.median(dev)), 3), call_ms=round(1e3 * float(np.median(wall)), 3))
                t0 = time.perf_counter()
                _host_one((control, paths[0]))
                est = (time.perf_counter() - t0) * n_paths / cores
                if est <= a.host_budget:
                    t0 = time.perf_counter()
                    with ProcessPoolExecutor(cores) as ex:
                        list(ex.map(_host_one, [(control, p) for p in paths], chunksize=max(1, n_paths // (4 * cores))))
                    row.update(host_s=round(time.perf_counter() - t0, 3), host_cores=cores)
                else:
                    row.update(host_s=None, host_skipped=f"estimated {est:.0f} s on {cores} cores")
                print(json.dumps(row), flush=True)
    s.close()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
