"""What per-query tunnels cost on the cfg5 workload (512^3 cfg3 map, JRK-125, setEpsilon(2), <= 1000 expansions per
query, 4096 queries by default).  Each query's tunnel surrounds its own route: the waypoints of its untunnelled plan
(start and goal where that plan found none), --radius metres on every axis, ray-traced.  Three runs:
  tunnels     mplx_set_batch_regions, then one mplx_plan_batch over the whole batch, query q in tunnel q;
  sequential  one query at a time, its tunnel installed ctx-wide (mplx_set_search_region_path), the way a caller
              without per-query tunnels has to plan such a batch; on the first --sequential queries only, as it is
              slow, with its time per query;
  untunnelled the same batch without tunnels.
For each: slots, tunnel bytes, tunnel build time (wall, synchronous call) and search time (CUDA events, best of
--repeat after one warm-up).  The sequential run's results must equal the tunnelled batch's for its queries.  Prints
one JSON line with the card name and power limit read in the same run.

    python tunnel_bench.py [--queries 4096] [--radius 0.5] [--sequential 256] [--repeat 3]
"""
from __future__ import annotations

import argparse
import json
import time

import numpy as np

from search_bench import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=4096)
    ap.add_argument("--radius", type=float, default=0.5)
    ap.add_argument("--sequential", type=int, default=256)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    import cfg5_bench
    import scenarios as S
    from motion_primitive_library_b200 import MapUtil, abi, env_map

    sc = S.cfg3()
    q = cfg5_bench.make_queries(sc, a.queries, 20.0)
    st, go = q["start"], q["goal"]
    mu = MapUtil()
    mu.setMap(sc.origin, sc.dim_cells, sc.grid(), sc.res)
    e = env_map(mu, device=0)
    e.set_control(sc.control)
    e.set_u(sc.U)
    e.set_dt(sc.T)
    e.set_w(sc.w)
    e.set_v_max(sc.v_max)
    e.set_a_max(sc.a_max)
    kw = dict(eps=2.0, max_expand=1000, closed=False)
    n = len(st)
    rad = np.full(3, a.radius)

    def best(f):
        f()  # warm-up
        return min((f() for _ in range(a.repeat)), key=lambda r: r[0])

    # the untunnelled batch, and the routes from its trajectories
    plain_s, plain = best(lambda: (lambda r: (r["seconds"], r))(e.plan_batch(st, go, **kw)))
    routed = e.plan_batch(st, go, trajectories=True, **kw)
    routes = []
    for i in range(n):
        nodes = routed["trajectories"][i]["nodes"]
        routes.append(nodes["pos"] if len(nodes) else np.stack([st["pos"][i], go["pos"][i]]))
    route_pts = int(sum(len(r) for r in routes))

    def build():
        t0 = time.perf_counter()
        e.set_batch_regions(routes, rad)
        return time.perf_counter() - t0, e.batch_regions_info()

    build_s, info = best(build)
    tun_s, tun = best(lambda: (lambda r: (r["seconds"], r))(e.plan_batch(st, go, **kw)))
    e.set_batch_regions([], rad)

    # one query at a time with a ctx-wide tunnel (no region read-back, as a planner would call it)
    lib, h = abi.load(), e.handle
    m = min(a.sequential, n)
    seq = []
    t0 = time.perf_counter()
    region_s = search_s = 0.0
    for i in range(m):
        p = np.ascontiguousarray(routes[i], dtype=np.float64)
        t1 = time.perf_counter()
        abi.check(lib.mplx_set_search_region_path(h, p.ctypes.data, len(p), rad.ctypes.data, 0, None))
        t2 = time.perf_counter()
        r = e.plan_batch(st[i:i + 1], go[i:i + 1], **kw)
        region_s += t2 - t1
        search_s += r["seconds"]
        seq.append(r)
    seq_wall = time.perf_counter() - t0
    abi.check(lib.mplx_set_search_region(h, None))
    same = all(int(r["valid"][0]) == int(tun["valid"][i]) and int(r["expanded"][0]) == int(tun["expanded"][i])
               and np.float64(r["cost"][0]).tobytes() == np.float64(tun["cost"][i]).tobytes()
               and np.array_equal(r["actions"][0], tun["actions"][i]) for i, r in enumerate(seq))
    e.close()
    print(json.dumps(dict(
        workload=f"cfg5 queries (512^3 cfg3, JRK-125, eps 2, <= 1000 expansions/query), {n} queries, tunnels of "
                 f"{a.radius} m around each query's untunnelled route ({route_pts} route points)",
        card=card(),
        tunnels=dict(search_s=tun_s, build_wall_s=build_s, slots=int(tun["slots"]), tunnel_bytes=info["bytes"],
                     bricks=info["n_bricks"], bytes_per_query=info["bytes"] / n, valid=int(tun["valid"].sum()),
                     expanded=int(tun["expanded"].sum())),
        sequential=dict(queries=m, wall_s=seq_wall, wall_s_per_query=seq_wall / max(m, 1), region_wall_s=region_s,
                        search_s=search_s, slots=1, tunnel_bytes=int((mu.map.size + 31) // 32 * 4),
                        identical_to_tunnels=bool(same)),
        untunnelled=dict(search_s=plain_s, slots=int(plain["slots"]), tunnel_bytes=0, build_wall_s=0.0,
                         valid=int(plain["valid"].sum()), expanded=int(plain["expanded"].sum())))))


if __name__ == "__main__":
    main()
