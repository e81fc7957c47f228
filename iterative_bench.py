"""MapPlanner::iterativePlan for cfg5's 4 096 queries as one batch, round by round (tunnel radius 0.5 m, eps 2,
<= 1000 expansions per plan, max_iter 3 and 10).  Two routes for each round's tunnels, run one after the other in
the same process and alternated over --repeat passes:
  recorded   mplx_set_batch_regions_recorded: the paths the last search recorded, traced on the device;
  host       mplx_plan_batch_trajectories to the host, then mplx_set_batch_regions from those points.
Per round: queries still running, tunnel build (wall time of the synchronous call; for the host route also the
trajectory read-back), search (CUDA events) and kernel launches.  Then MultiQueryPlanner::iterativePlan
(BatchPlanner.iterative_plan, whole batch) and the single-query MapPlanner::iterativePlan (mplh_iterative_plan) on the
first --single queries; every route must give identical per-query results.  Prints the card and its power limit and
one JSON line.

    python iterative_bench.py [--queries 4096] [--repeat 2] [--single 256]"""
import argparse
import json
import subprocess
import time

import numpy as np


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def loop(e, S, G, radius, max_iter, route):
    """iterativePlan from the first plan's trajectories, each round one plan_batch over the running queries."""
    n = len(S)
    e.set_batch_regions([], radius)  # the first plan is untunnelled
    r0 = e.plan_batch(S, G, eps=2.0, max_expand=1000, trajectories=True)
    its, ok = np.zeros(n, np.int32), np.zeros(n, bool)
    cost, expd, valid = r0["cost"].copy(), r0["expanded"].copy(), r0["valid"].copy()
    prev = np.zeros(n)
    running = np.flatnonzero(r0["valid"] != 0)
    ok[running] = True
    from_ = running.astype(np.int32)  # each running query's place in the last search
    rounds = []
    while running.size:
        t0 = time.perf_counter()
        if route == "recorded":
            e.set_batch_regions_recorded(from_, radius)
        else:
            trajs, _ = e.batch_trajectories(capacity=1 << 20)
            e.set_batch_regions([trajs[i]["nodes"]["pos"][:, :3] if len(trajs[i]["nodes"]) else S["pos"][q:q + 1, :3]
                                 for i, q in zip(from_, running)], radius)
        build = time.perf_counter() - t0
        l0 = e.launch_count()
        r = e.plan_batch(S[running], G[running], eps=2.0, max_expand=1000, trajectories=True)
        rounds.append(dict(running=int(running.size), build_s=build, search_s=float(r["seconds"]),
                           launches=int(e.launch_count() - l0)))
        nxt, pos = [], []
        for i, q in enumerate(running):
            its[q] += 1
            valid[q], cost[q], expd[q] = r["valid"][i], r["cost"][i], r["expanded"][i]
            if not r["valid"][i]:
                ok[q] = False
                continue
            if prev[q] == r["cost"][i]:
                continue
            prev[q] = r["cost"][i]
            if its[q] < max_iter:
                nxt.append(q)
                pos.append(i)
        running = np.array(nxt, np.int64)
        from_ = np.array(pos, np.int32)
    return dict(its=its, ok=ok, cost=cost, expanded=expd, valid=valid), rounds


def same(a, b, qs):
    return all(int(a["its"][q]) == int(b["its"][q]) and bool(a["ok"][q]) == bool(b["ok"][q])
               and int(a["valid"][q]) == int(b["valid"][q]) and int(a["expanded"][q]) == int(b["expanded"][q])
               and np.float64(a["cost"][q]).tobytes() == np.float64(b["cost"][q]).tobytes() for q in qs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=4096)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--single", type=int, default=256)
    ap.add_argument("--max-iter", default="3,10")
    a = ap.parse_args()
    import cfg5_bench
    import scenarios as SC
    from motion_primitive_library_b200 import MapUtil, env_map
    from motion_primitive_library_b200 import planner as P

    print("card:", card(), flush=True)
    sc = SC.cfg3()
    grid = sc.grid()
    q = cfg5_bench.make_queries(sc, a.queries, 20.0)
    S, G = q["start"], q["goal"]
    radius = [0.5, 0.5, 0.5]
    mu = MapUtil()
    mu.setMap(sc.origin, sc.dim_cells, grid, sc.res)
    e = env_map(mu, device=0)
    e.set_control(sc.control)
    e.set_u(sc.U)
    e.set_dt(sc.T)
    e.set_w(sc.w)
    e.set_v_max(sc.v_max)
    e.set_a_max(sc.a_max)
    args = P.make_args(3, sc.control, grid, sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=S["pos"][0]),
                       goal=dict(pos=G["pos"][0]), v_max=sc.v_max, a_max=sc.a_max, T=sc.T, w=sc.w, max_num=1000, eps=2.0)
    out = dict(card=card(), queries=a.queries, radius=radius, runs=[])
    e.plan_batch(S, G, eps=2.0, max_expand=1000, trajectories=True)  # warm-up: modules, arenas
    for max_iter in [int(x) for x in a.max_iter.split(",")]:
        res = {}
        for rep in range(a.repeat):
            for route in ("recorded", "host"):
                t0 = time.perf_counter()
                r, rounds = loop(e, S, G, radius, max_iter, route)
                wall = time.perf_counter() - t0
                res.setdefault(route, r)
                out["runs"].append(dict(max_iter=max_iter, route=route, rep=rep, wall_s=wall, rounds=rounds))
                print(json.dumps(out["runs"][-1]), flush=True)
        s = P.BatchPlanner(args, path="device")
        try:
            t0 = time.perf_counter()
            bres, bits, bok = s.iterative_plan(S, G, radius, max_iter)
            bwall = time.perf_counter() - t0
        finally:
            s.close()
        batch = dict(its=bits, ok=bok, cost=bres["cost"], expanded=bres["expanded"], valid=bres["valid"])
        n1 = min(a.single, a.queries)
        single = dict(its=np.zeros(n1, np.int32), ok=np.zeros(n1, bool), cost=np.zeros(n1),
                      expanded=np.zeros(n1, np.int32), valid=np.zeros(n1, np.int32))
        t0 = time.perf_counter()
        for k in range(n1):
            aq = P.make_args(3, sc.control, grid, sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=S["pos"][k]),
                             goal=dict(pos=G["pos"][k]), v_max=sc.v_max, a_max=sc.a_max, T=sc.T, w=sc.w, max_num=1000,
                             eps=2.0)
            _, last = P.iterative_plan(aq, radius, max_iter)
            single["its"][k], single["ok"][k] = last["iterations"], bool(last["ok"])
            single["cost"][k], single["expanded"][k], single["valid"][k] = last["cost"], last["expanded"], last["valid"]
        swall = time.perf_counter() - t0
        allq = range(a.queries)
        summary = dict(max_iter=max_iter, batch_wall_s=bwall, single_wall_s=swall, single_queries=n1,
                       recorded_equals_host=same(res["recorded"], res["host"], allq),
                       batch_equals_recorded=same(batch, res["recorded"], allq),
                       single_equals_batch=same(single, batch, range(n1)),
                       iterations_hist=np.bincount(bits).tolist(), ok=int(bok.sum()))
        out.setdefault("summary", []).append(summary)
        print(json.dumps(summary), flush=True)
    e.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
