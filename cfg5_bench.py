"""BASELINE.json config 5 — the path's multi-GPU workload: many (start, goal) queries on one 512^3
voxel map, JRK control, planned in lock-step by MPL::MultiQueryPlanner (one device launch per
iteration expands the current node of every live query of the rank; host A* bookkeeping spread over
the rank's host cores) and SHARDED over ranks by query (strong scaling: the query set is fixed).
The only collectives are the set-up broadcast of the map and the final all-gather of the per-query
results and counters (SURVEY.md §8e); there is no exchange during the search.

Used by `bench.py` (the `multi_query` object of the default line, and `--workload cfg5`) and by
`tools/batch_queries.py`.
"""
from __future__ import annotations

import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np


def make_queries(sc, n_queries: int, min_dist: float, seed: int = 5):
    """Start/goal pairs: free cell centres at rest, at least min_dist apart (SURVEY.md §8d cfg5)."""
    from motion_primitive_library_b200 import planner

    pts = sc.frontier(4 * n_queries, seed=11, max_steps=0)["pos"]
    rng = np.random.default_rng(seed)
    ext = min(sc.dim_cells) * sc.res
    q = np.zeros(n_queries, dtype=[("start", planner.WAYPOINT_DTYPE), ("goal", planner.WAYPOINT_DTYPE)])
    k = 0
    while k < n_queries:
        i, j = rng.integers(0, len(pts), 2)
        if np.abs(pts[i] - pts[j]).max() >= min(min_dist, 0.4 * ext):
            q["start"]["pos"][k], q["goal"]["pos"][k] = pts[i], pts[j]
            k += 1
    return q


def run(sc, grid, local: int, n_queries: int = 4096, max_expand: int = 1000, min_dist: float = 20.0,
        ref_queries: int = 32, repeat: int = 2, eps: float = 2.0):
    """Plan the query set sharded over the ranks of the default process group (or alone).
    Returns the result dict on every rank (counters are reduced).  `repeat` passes over the same set in one
    planner session: the first allocates the search states, the others recycle them (the fastest is reported)."""
    import torch.distributed as dist

    from motion_primitive_library_b200 import planner, sharding
    import scenarios as S

    on = dist.is_available() and dist.is_initialized()
    rank = dist.get_rank() if on else 0
    world = dist.get_world_size() if on else 1
    q = make_queries(sc, n_queries, min_dist)

    def make(start, goal):
        a = planner.make_args(3, sc.control, grid, sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=start),
                              goal=dict(pos=goal), v_max=sc.v_max, a_max=sc.a_max, T=sc.T, w=sc.w, max_num=max_expand, eps=eps)
        a.device = local
        return a

    res_dtype = [("valid", "i4"), ("cost", "f8"), ("expanded", "i4"), ("n_closed", "i4"), ("n_actions", "i4")]
    # host threads of this rank's planner: its share of the CPUs the job may use (the ranks of one box share the
    # cgroup quota; every rank spawning a thread per CPU oversubscribed an 8-rank run 8x), within its affinity mask
    import os

    local_world = int(os.environ.get("LOCAL_WORLD_SIZE", str(world))) if on else 1
    n_threads = max(1, min(len(os.sched_getaffinity(0)), S.effective_cpus() // max(1, local_world)))
    os.environ["MPLH_THREADS"] = str(n_threads)
    sl = sharding.shard_slice(len(q), rank, world)
    session = planner.BatchPlanner(make(q["start"]["pos"][0], q["goal"]["pos"][0])) if sl.stop > sl.start else None

    def run_slice(mine):
        if len(mine) == 0:
            return np.zeros(0, dtype=res_dtype), dict(expansions=0, iterations=0, seconds_max=0.0, t_pop_max=0.0,
                                                      t_device_max=0.0, t_relax_max=0.0, device_path=0)
        res, tot = session.plan(mine["start"], mine["goal"])
        return res, dict(expansions=tot["nodes"], iterations=tot["iterations"], seconds_max=tot["seconds"],
                         t_pop_max=tot["t_pop"], t_device_max=tot["t_device"], t_relax_max=tot["t_relax"],
                         device_path=1 if tot["path"] == "device" else 0)

    # pass 0 allocates (and page-faults) the search-state memory of every query; later passes recycle it
    passes = []
    for _ in range(max(1, repeat)):
        if on:
            dist.barrier()
        passes.append(sharding.run_sharded(q, run_slice))
    res, cnt = passes[-1] if len(passes) == 1 else min(passes[1:], key=lambda rc: rc[1]["seconds_max"])
    first_seconds = passes[0][1]["seconds_max"]
    t_rel = session.close() if session is not None else 0.0
    if on:
        import torch

        tr = torch.tensor([t_rel], dtype=torch.float64, device="cuda")
        dist.all_reduce(tr, op=dist.ReduceOp.MAX)
        t_rel = float(tr.item())
    cnt["t_release_max"] = t_rel
    secs = cnt["seconds_max"]
    # the device search (mplx_plan_batch) runs each query's whole A* on the GPU: no pop / relax phases on the host
    path = "device" if cnt.get("device_path", 0) else "lockstep"
    phases = ({"device_search": cnt["t_device_max"]} if path == "device" else
              {"pop": cnt["t_pop_max"], "device+pcie": cnt["t_device_max"], "relax": cnt["t_relax_max"]})
    out = {
        "workload": f"cfg5: {n_queries} start/goal pairs >= {min_dist} m apart, {sc.name}, setEpsilon({eps:g}), <= {max_expand} expansions/query, "
                    f"queries sharded over {world} rank(s)",
        "n_gpus": world, "scaling": "strong", "value": cnt["expansions"] / secs, "unit": "expansions/s",
        "expansions": int(cnt["expansions"]), "seconds": secs, "passes": len(passes),
        "first_pass_seconds": first_seconds, "session_close_seconds": cnt["t_release_max"], "lockstep_iterations_sum": int(cnt["iterations"]) if path == "lockstep" else 0,
        "queries": n_queries, "queries_solved": int(res["valid"].sum()), "epsilon": eps, "max_expand": max_expand, "host_threads_per_rank": n_threads,
        "path": path, "phase_seconds_max": phases,
        "what": "sum of node expansions / max over ranks of MultiQueryPlanner::plan wall time (path device: every query's "
                "whole A* on the GPU, mplx_plan_batch; path lockstep: device expansion + PCIe + host A* bookkeeping) for one pass over the query set in a session whose search states are recycled from "
                "the previous pass (first_pass_seconds = the pass that allocates them; session_close_seconds = freeing "
                "them at the end, once per session)",
    }
    if rank == 0 and ref_queries > 0:
        import sys
        from pathlib import Path

        sys.path.insert(0, str(Path(__file__).resolve().parent / "tests"))
        import planner_bindings as pb

        if pb.ref_planner_available():
            n = min(ref_queries, n_queries)
            nt = S.effective_cpus()
            t0 = time.perf_counter()
            with ThreadPoolExecutor(nt) as ex:  # ctypes releases the GIL: one reference planner per thread
                outs = list(ex.map(lambda k: pb.plan_reference(make(q["start"]["pos"][k], q["goal"]["pos"][k])), range(n)))
            dt = time.perf_counter() - t0
            exp = sum(o["n_closed"] for o in outs)
            same = all(o["n_closed"] == res["n_closed"][k] and o["valid"] == res["valid"][k]
                       and (not o["valid"] or o["cost"] == res["cost"][k]) for k, o in enumerate(outs))
            plan_s = sum(o["seconds"] for o in outs)  # inside MapPlanner::plan only (no map set-up, no teardown)
            out["reference"] = {"value": exp / (plan_s / min(nt, n)), "unit": "expansions/s", "queries": n, "threads": min(nt, n),
                                "wall_seconds": dt, "plan_seconds_sum": plan_s, "same_results_as_gpu": bool(same),
                                "what": "the reference's MapPlanner::plan (oracle/_ref), one query per host thread, time "
                                        "inside plan() only"}
    return out
