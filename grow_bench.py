"""The growing device search (mplx_plan_batch_grow, BatchPlanner path "device_grow"; AUTO for unbounded plans)
against the bounded device search and the lock-step loop.  Three workloads:

  cap1000    the cfg5 queries (512^3 cfg3, JRK-125, eps 2) at the cap they run with today, 1 000 expansions:
             "device" (worst-case arenas) against "device_grow" (arenas sized for the batch);
  cap20000   the same queries at cap 20 000 (SURVEY.md §8d): "device", "device_grow" and, at the sizes in
             --lockstep-sizes, "lockstep";
  unbounded  config 1's plan (the corridor, ACC, v_max = a_max = 1, eps 1, max_num -1) on the corridor map with a
             wall across it at x cell 400, so that the goals of every fourth query (beyond the wall) cannot be
             reached and their searches exhaust the reachable lattice: "auto" (the growing search) against
             "lockstep".

The paths alternate within every size, each in its own session that plans the set twice (the second pass, which
recycles the search memory, is reported), --repeat times; the faster run is reported.  Prints one JSON line with
seconds, slots, first-round arena bytes, rounds, reruns, whether all paths gave identical results (validity, cost
bits, expansions, closed sets, trajectories), and the card name and power limit read in the same run.

    python grow_bench.py --workload cap1000|cap20000|unbounded [--sizes ...] [--repeat 2]
"""
from __future__ import annotations

import argparse
import json

import numpy as np

from search_bench import card

DEFAULT_SIZES = dict(cap1000="16,64,256,1024,4096", cap20000="16,64,256", unbounded="16,64,256")


def cfg5_args(max_num):
    import cfg5_bench
    import scenarios as S
    from motion_primitive_library_b200 import planner as P

    sc = S.cfg3()
    q = cfg5_bench.make_queries(sc, 4096, 20.0)
    args = P.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U,
                       start=dict(pos=q["start"]["pos"][0]), goal=dict(pos=q["goal"]["pos"][0]), v_max=sc.v_max,
                       a_max=sc.a_max, T=sc.T, w=sc.w, max_num=max_num, eps=2.0)
    return args, q["start"], q["goal"]


def corridor_args(n_max, seed=1):
    import sys
    from pathlib import Path

    sys.path.insert(0, str(Path(__file__).resolve().parent / "tests"))
    import fixtures
    from motion_primitive_library_b200 import planner as P

    c = fixtures.corridor()
    g = c["grid"].reshape(199, 799).copy()
    g[:, 400] = 100
    args = P.make_args(2, 0x03, g.reshape(-1), c["dim"], c["origin"], c["res"], fixtures.U_2d(),
                       start=dict(pos=c["start"]), goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0)
    rng = np.random.default_rng(seed)
    free = np.argwhere(g == 0)
    left, right = free[free[:, 1] < 390], free[free[:, 1] > 410]
    pos = lambda ij: ((ij[1] + 0.5) * c["res"] + c["origin"][0], (ij[0] + 0.5) * c["res"] + c["origin"][1])
    S = np.zeros(n_max, dtype=P.WAYPOINT_DTYPE)
    G = np.zeros(n_max, dtype=P.WAYPOINT_DTYPE)
    for k in range(n_max):
        S["pos"][k, :2] = pos(left[rng.integers(len(left))])
        G["pos"][k, :2] = pos((right if k % 4 == 3 else left)[rng.integers(len(right if k % 4 == 3 else left))])
    return args, S, G


def identical(a, b):
    return bool(np.array_equal(a[0], b[0]) and a[0]["cost"].tobytes() == b[0]["cost"].tobytes()
                and all(np.array_equal(x, y) for x, y in zip(a[2], b[2]))
                and all(np.array_equal(x, y) for x, y in zip(a[3], b[3])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=tuple(DEFAULT_SIZES), default="cap1000")
    ap.add_argument("--sizes", default=None)
    ap.add_argument("--lockstep-sizes", default="16,64", help="cap20000: sizes the lock-step loop also runs")
    ap.add_argument("--repeat", type=int, default=2, help="alternations of the paths per size")
    a = ap.parse_args()
    from motion_primitive_library_b200 import planner as P

    sizes = [int(x) for x in (a.sizes or DEFAULT_SIZES[a.workload]).split(",")]
    if a.workload == "cap1000":
        args, S, G = cfg5_args(1000)
        paths = lambda n: ("device", "device_grow")
        workload = "cfg5 queries (512^3 cfg3, JRK-125, eps 2, <= 1000 expansions/query)"
    elif a.workload == "cap20000":
        args, S, G = cfg5_args(20000)
        ls = {int(x) for x in a.lockstep_sizes.split(",") if x}
        paths = lambda n: ("device", "device_grow") + (("lockstep",) if n in ls else ())
        workload = "cfg5 queries (512^3 cfg3, JRK-125, eps 2, <= 20000 expansions/query)"
    else:
        args, S, G = corridor_args(max(sizes))
        paths = lambda n: ("auto", "lockstep")
        workload = ("config 1 (corridor with a wall at x cell 400, ACC, v_max = a_max = 1, eps 1, unbounded); "
                    "every fourth goal beyond the wall")
    runs, summary = [], {}
    for n in sizes:
        st, go = S[:n], G[:n]
        outs = {}
        for rep in range(a.repeat):
            for path in paths(n):
                s = P.BatchPlanner(args, path=path)
                try:
                    s.plan_detail(st, go)  # pass 1 allocates the search memory
                    d = s.plan_detail(st, go)
                finally:
                    s.close()
                outs[path] = d
                tot = d[1]
                runs.append(dict(queries=n, path=path, ran=tot["path"], rep=rep, seconds=tot["seconds"],
                                 expansions=tot["nodes"], slots=tot["slots"], arena_bytes=tot["arena_bytes"],
                                 rounds=tot["grow_rounds"], reruns=tot["grow_reruns"],
                                 first_cap=tot["grow_first_cap"], last_cap=tot["grow_last_cap"],
                                 to_lockstep=tot["grow_lockstep"]))
        ps = paths(n)
        same = all(identical(outs[ps[0]], outs[p]) for p in ps[1:])
        best = {p: min((r for r in runs if r["queries"] == n and r["path"] == p), key=lambda r: r["seconds"]) for p in ps}
        summary[str(n)] = dict(identical=same, unreachable=int((outs[ps[0]][0]["valid"] == 0).sum()),
                               **{p: {k: best[p][k] for k in ("seconds", "ran", "slots", "arena_bytes", "rounds",
                                                              "reruns", "first_cap", "last_cap", "to_lockstep")}
                                  for p in ps})
    print(json.dumps(dict(workload=workload, card=card(), summary=summary, runs=runs)))


if __name__ == "__main__":
    main()
