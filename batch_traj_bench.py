"""What recording the planned trajectories costs on the cfg5 workload (512^3 cfg3 map, JRK-125, setEpsilon(2),
<= 1000 expansions per query, 4096 queries by default): the device search (mplx_plan_batch) without and with
trajectory recording, mplx_plan_batch_trajectories without and with samples, and the whole pipeline plan ->
trajectories -> mplx_traj_check (traverse_trajectories), against the same pipeline on MultiQueryPlanner's lock-step
loop with host-built trajectories (BatchPlanner.plan_detail(trajectories=True), then the host's traverse_trajectory).
The recording search runs twice: with the automatic room (an eighth of the search budget) and with a room of
--small-room-mib, which displaces no arena at cfg5, so that the cost of the recording kernel and that of the room
show apart.  Each measurement is the best of --repeat runs, after one warm-up run that allocates the search memory.
Prints one JSON line with the device seconds of the kernels (CUDA events), the wall seconds of the pipelines, whether
recording changed any search result, whether the two pipelines gave bitwise the same trajectories and checks, and the
card name and power limit read in the same run.

    python batch_traj_bench.py [--queries 4096] [--repeat 3] [--n-samples 64] [--small-room-mib 64]
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
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--n-samples", type=int, default=64)
    ap.add_argument("--small-room-mib", type=int, default=64)
    a = ap.parse_args()
    import cfg5_bench
    import scenarios as S
    from motion_primitive_library_b200 import MapUtil, env_map
    from motion_primitive_library_b200 import planner as P

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

    def best(f):
        f()  # warm-up: allocates the search memory and the trajectory room
        return min((f() for _ in range(a.repeat)), key=lambda r: r[0])

    off = best(lambda: (e.plan_batch(st, go, **kw)["seconds"], None))

    def on(room=0):
        r = e.plan_batch(st, go, trajectories=True, traj_room_bytes=room, **kw)
        return r["seconds"], r

    small_s, r_small = best(lambda: on(a.small_room_mib << 20))
    r_off = e.plan_batch(st, go, **kw)
    on_s, r_on = best(on)  # the last search call recorded: mplx_plan_batch_trajectories reads it
    identical = (np.array_equal(r_on["valid"], r_off["valid"]) and r_on["cost"].tobytes() == r_off["cost"].tobytes()
                 and all(np.array_equal(x, y) for x, y in zip(r_on["actions"], r_off["actions"])))
    cap = sum(len(x) + 1 for x in r_on["actions"] if len(x))
    traj_s = best(lambda: (e.batch_trajectories(0, cap)[1], None))[0]
    traj_samples_s = best(lambda: (e.batch_trajectories(a.n_samples, cap)[1], None))[0]

    def pipeline():
        t0 = time.perf_counter()
        r = e.plan_batch(st, go, trajectories=True, **kw)
        chk, check_s = e.traverse_trajectories(r["trajectories"], sc.control)
        return time.perf_counter() - t0, (r, chk, check_s)

    e2e_s, (r_p, chk, check_s) = best(pipeline)
    e.close()
    n_traj = sum(1 for x in r_p["actions"] if len(x))

    # the lock-step loop with host-built trajectories, checked on the host
    args = P.make_args(3, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U,
                       start=dict(pos=st["pos"][0]), goal=dict(pos=go["pos"][0]), v_max=sc.v_max, a_max=sc.a_max,
                       T=sc.T, w=sc.w, max_num=1000, eps=2.0)
    bp = P.BatchPlanner(args, path="lockstep")
    try:
        bp.plan_detail(st, go, closed=False)  # allocates the search states

        def lockstep():
            t0 = time.perf_counter()
            _, tot, _, _, trajs = bp.plan_detail(st, go, closed=False, trajectories=True)
            t1 = time.perf_counter()
            hchk = P.traj_check(3, sc.grid(), sc.dim_cells, sc.origin, sc.res, trajs, sc.control, v_max=sc.v_max,
                                nthreads=8)
            return time.perf_counter() - t0, (tot, trajs, hchk, t1 - t0)

        lock_s, (tot_l, trajs_l, hchk, lock_plan_s) = best(lockstep)
    finally:
        bp.close()
    same_traj = all(x[k].tobytes() == y[k].tobytes() for x, y in zip(trajs_l, r_p["trajectories"])
                    for k in ("nodes", "seg_t", "coeff"))
    same_check = all(int(h) == c["status"] and np.float64(hc).tobytes() == np.float64(c["cost"]).tobytes()
                     for h, hc, c in zip(hchk["status"], hchk["cost"], chk))
    print(json.dumps(dict(
        workload=f"cfg5 queries (512^3 cfg3, JRK-125, eps 2, <= 1000 expansions/query), {a.queries} queries",
        card=card(),
        search_s=off[0], search_recording_s=on_s, recording_overhead=on_s / off[0] - 1.0,
        search_recording_small_room_s=small_s, small_room_mib=a.small_room_mib,
        small_room_overhead=small_s / off[0] - 1.0, small_room_rounds_identical=bool(
            all(np.array_equal(x, y) for x, y in zip(r_small["actions"], r_on["actions"]))),
        trajectories_s=traj_s, trajectories_samples_s=traj_samples_s, n_samples=a.n_samples,
        pipeline_wall_s=e2e_s, pipeline_check_s=check_s, trajectories=n_traj, waypoint_slots=cap,
        checked_finite=int(sum(1 for c in chk if c["status"] and np.isfinite(c["cost"]))),
        identical_with_recording=bool(identical),
        lockstep_pipeline_wall_s=lock_s, lockstep_plan_wall_s=lock_plan_s, lockstep_path=tot_l["path"],
        lockstep_trajectories_identical=bool(same_traj), lockstep_checks_identical=bool(same_check))))


if __name__ == "__main__":
    main()
