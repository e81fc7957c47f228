"""Device search (mplx_plan_batch) against the lock-step loop of MPL::MultiQueryPlanner on the cfg5 workload
(512^3 cfg3 map, JRK-125, setEpsilon(2), <= 1000 expansions per query): the full 4096-query set and batches of
16, 64, 256 and 1024 of its queries.  The two paths alternate within every size, each in its own session that
plans the set twice (the second pass, which recycles the search memory, is reported).  Prints one JSON line with
expansions/s, seconds, the arena slots and bytes, whether both paths gave identical results (validity, cost
bits, expansions, closed sets, trajectories), and the card name and power limit read in the same run.

With --workload cfg4 the same comparison runs the cost-term device search (mplx_plan_batch_cost_terms) against
the lock-step loop on the distance-map planner's plan: the 512^3 map replaced by its potential field
(MapPlanner::updatePotentialMap on the device, as bench.py's cfg4), ACC x YAW-81, yaw_max 0.7, wyaw 1, potential
weight 0.5, the cfg5 queries, eps 2, <= 1000 expansions per query.

    python search_bench.py [--workload cfg5|cfg4] [--sizes 16,64,256,1024,4096] [--repeat 2]
"""
from __future__ import annotations

import argparse
import json
import subprocess

import numpy as np


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim = [x.strip() for x in out.split(",")]
        return dict(name=name, power_limit=plim)
    except Exception as e:  # noqa: BLE001
        import torch

        return dict(name=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,64,256,1024,4096")
    ap.add_argument("--repeat", type=int, default=2, help="alternations of the two paths per size")
    ap.add_argument("--workload", choices=("cfg5", "cfg4"), default="cfg5")
    a = ap.parse_args()
    import cfg5_bench
    import scenarios as S
    from motion_primitive_library_b200 import planner as P

    if a.workload == "cfg5":
        sc = S.cfg3()
        grid = sc.grid()
        q = cfg5_bench.make_queries(sc, 4096, 20.0)
        args = P.make_args(3, sc.control, grid, sc.dim_cells, sc.origin, sc.res, sc.U,
                           start=dict(pos=q["start"]["pos"][0]), goal=dict(pos=q["goal"]["pos"][0]), v_max=sc.v_max,
                           a_max=sc.a_max, T=sc.T, w=sc.w, max_num=1000, eps=2.0)
        device_path = "device"
        workload = "cfg5 queries (512^3 cfg3, JRK-125, eps 2, <= 1000 expansions/query)"
    else:
        from motion_primitive_library_b200 import MapUtil, env_map

        sc = S.cfg4()
        mu = MapUtil()
        mu.setMap(sc.origin, sc.dim_cells, sc.grid(), sc.res)
        e = env_map(mu, device=0)
        e.set_potential_weight(sc.potential_weight)
        e.set_gradient_weight(sc.gradient_weight)
        field = e.update_potential_map(sc.potential_radius).copy()  # the grid becomes the field (map_planner.cpp:387)
        e.close()
        q = cfg5_bench.make_queries(sc, 4096, 20.0)
        args = P.make_args(3, sc.control, field, sc.dim_cells, sc.origin, sc.res, sc.U,
                           start=dict(pos=q["start"]["pos"][0]), goal=dict(pos=q["goal"]["pos"][0]), v_max=sc.v_max,
                           yaw_max=sc.yaw_max, wyaw=sc.wyaw, T=sc.T, w=sc.w, max_num=1000, eps=2.0, potential=field,
                           potential_weight=sc.potential_weight, gradient_weight=sc.gradient_weight)
        device_path = "device_cost_terms"
        workload = ("cfg4 queries (512^3 cfg3-style map replaced by its potential field, ACCxYAW-81, yaw_max 0.7, "
                    "wyaw 1, potential weight 0.5, eps 2, <= 1000 expansions/query)")
    runs = []
    for n in [int(x) for x in a.sizes.split(",")]:
        st, go = q["start"][:n], q["goal"][:n]
        outs = {}
        for rep in range(a.repeat):
            for path in (device_path, "lockstep"):
                s = P.BatchPlanner(args, path=path)
                try:
                    s.plan_detail(st, go)  # pass 1 allocates the search memory
                    res, tot, acts, closed = s.plan_detail(st, go)
                finally:
                    s.close()
                outs.setdefault(path, []).append((res, tot, acts, closed))
                runs.append(dict(queries=n, path=path, rep=rep, seconds=tot["seconds"],
                                 expansions=tot["nodes"], expansions_per_s=tot["nodes"] / tot["seconds"],
                                 slots=tot["slots"], arena_bytes=tot["arena_bytes"]))
        d, l = outs[device_path][-1], outs["lockstep"][-1]
        same = (np.array_equal(d[0], l[0]) and all(np.array_equal(x, y) for x, y in zip(d[2], l[2]))
                and all(np.array_equal(x, y) for x, y in zip(d[3], l[3])))
        for r in runs:
            if r["queries"] == n:
                r["identical"] = bool(same)
    summary = {}
    for n in sorted({r["queries"] for r in runs}):
        best = {p: min((r for r in runs if r["queries"] == n and r["path"] == p), key=lambda r: r["seconds"])
                for p in (device_path, "lockstep")}
        summary[str(n)] = dict(device_s=best[device_path]["seconds"], lockstep_s=best["lockstep"]["seconds"],
                               speedup=best["lockstep"]["seconds"] / best[device_path]["seconds"],
                               identical=best[device_path]["identical"])
    print(json.dumps(dict(workload=workload, card=card(), summary=summary, runs=runs)))


if __name__ == "__main__":
    main()
