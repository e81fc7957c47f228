#!/usr/bin/env python
"""bench.py — node-expansions/sec of the H100 expansion engine (and of the reference CPU path).

A "step" is one pass of the hot path (batched env_map::get_succ) over one batch of
synthetic frontier nodes.  Default workload: the north_star target — 512^3 voxel map @0.1 m,
3-D ACC control, 27 primitives per node (BASELINE.json metric "on 512^3 voxel map").

  python bench.py --gpus 1 --steps K --warmup W [--workload 512c_acc27|cfg2|cfg3|cfg4]
  python bench.py --impl reference ...      # the reference's CPU path (oracle) on the host cores
  python bench.py ... --dump-outputs DIR    # also write the last timed step's results as DIR/*.npy

Prints ONE JSON line (rank 0).  See DESIGN.md §Measurement for the definition of every key.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

METRIC = "node-expansions/sec (frontier x |U| primitives validated+costed) on 512^3 voxel map"
UNIT = "expansions/s"
S_IN = 112  # bytes of one frontier node (3-D Waypoint payload)
S_OUT = 132  # bytes of one successor record: 112 Waypoint + 8 cost + 4 action + 8 key


def emit(line: dict) -> None:
    """Print the JSON line as the LAST line of stdout: the reference planner (oracle/_ref) printf()s its own
    messages through C stdio, whose buffer would otherwise be flushed after Python's at exit."""
    try:
        C.CDLL(None).fflush(None)
    except Exception:
        pass
    sys.stdout.flush()
    # the reference's messages end with an ANSI reset and no newline: start a fresh line for the JSON
    print("\n" + json.dumps(line), flush=True)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="512c_acc27")
    ap.add_argument("--nodes", type=int, default=1 << 18, help="frontier nodes per step per GPU")
    ap.add_argument("--cpu-seconds", type=float, default=12.0, help="budget of the cpu_baseline leg")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-multi-query", action="store_true", help="skip the cfg5 leg (sharded many-query planning)")
    ap.add_argument("--no-replay", action="store_true", help="skip the replay-frontier batch sweep")
    ap.add_argument("--mq-queries", type=int, default=4096)
    ap.add_argument("--mq-max-expand", type=int, default=1000)
    ap.add_argument("--mq-eps", type=float, default=2.0, help="cfg5: the planner's setEpsilon (weighted A*)")
    ap.add_argument("--kernel", type=int, default=0,
                    help="0 = auto, 1 = literal loop, 2 = register, 3 = flat, 4 = dealing, 5 = fixed-point")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step returned (a fixed sample of its nodes) as DIR/<name>.npy")
    return ap.parse_args()


def make_env(sc, device):
    from motion_primitive_library_b200 import MapUtil, env_map

    mu = MapUtil()
    mu.setMap(sc.origin, sc.dim_cells, sc.grid(), sc.res)
    e = env_map(mu, device=device)
    e.set_control(sc.control)
    e.set_u(sc.U)
    e.set_dt(sc.T)
    e.set_w(sc.w)
    e.set_wyaw(sc.wyaw)
    e.set_v_max(sc.v_max)
    e.set_a_max(sc.a_max)
    e.set_j_max(sc.j_max)
    e.set_yaw_max(sc.yaw_max)
    if sc.potential_radius is not None:
        e.set_potential_weight(sc.potential_weight)
        e.set_gradient_weight(sc.gradient_weight)
        if sc._pot is None:
            # MapPlanner::updatePotentialMap on the device (mplx_update_potential_map; bit-exact against the
            # reference's own function, tests/test_maps_gpu.py) — the scipy generator of scenarios.py needs
            # minutes at 512^3.  The CPU arms receive this very field as their potential_map_.
            sc._pot = e.update_potential_map(sc.potential_radius).copy()
        else:
            e.set_potential_map(sc.potential())
    e._sync_params()
    return e


class ClockSampler:
    """SM clock and throttle reasons sampled DURING the timed region.

    Polls NVML from a background thread (a timed region of a few ms is far shorter than
    nvidia-smi's minimum loop period); falls back to `nvidia-smi -lms` when pynvml is missing."""

    REASONS = {0x8: "hw_slowdown", 0x40: "hw_thermal_slowdown", 0x20: "sw_thermal_slowdown", 0x4: "sw_power_cap"}

    def __init__(self, gpu_index=0):
        self.idx = gpu_index
        self.samples = []
        self._stop = False
        self._thr = None
        self._h = None
        try:
            import pynvml

            pynvml.nvmlInit()
            self.nv = pynvml
            # CUDA_VISIBLE_DEVICES may remap ordinals: resolve through the PCI bus id of the torch device
            import torch

            bus = torch.cuda.get_device_properties(gpu_index).pci_bus_id if hasattr(
                torch.cuda.get_device_properties(gpu_index), "pci_bus_id") else None
            self._h = pynvml.nvmlDeviceGetHandleByIndex(gpu_index)
            if bus is not None:
                for i in range(pynvml.nvmlDeviceGetCount()):
                    h = pynvml.nvmlDeviceGetHandleByIndex(i)
                    if pynvml.nvmlDeviceGetPciInfo(h).bus == bus:
                        self._h = h
            self.sm_max = float(pynvml.nvmlDeviceGetMaxClockInfo(self._h, pynvml.NVML_CLOCK_SM))
        except Exception:
            self.nv = None

    def _poll(self):
        nv = self.nv
        while not self._stop:
            try:
                sm = nv.nvmlDeviceGetClockInfo(self._h, nv.NVML_CLOCK_SM)
                rs = nv.nvmlDeviceGetCurrentClocksEventReasons(self._h) if hasattr(
                    nv, "nvmlDeviceGetCurrentClocksEventReasons") else nv.nvmlDeviceGetCurrentClocksThrottleReasons(self._h)
                pw = nv.nvmlDeviceGetPowerUsage(self._h) / 1000.0
                self.samples.append((float(sm), int(rs), pw))
            except Exception:
                break
            time.sleep(0.0005)

    def start(self):
        if self.nv is None:
            return
        import threading

        self._thr = threading.Thread(target=self._poll, daemon=True)
        self._thr.start()

    def stop(self):
        if self.nv is None or self._thr is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvml unavailable"]}
        self._stop = True
        self._thr.join(timeout=2)
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": self.sm_max, "reasons": ["no samples"]}
        sm = sorted(s[0] for s in self.samples)
        reasons = set()
        for _, rs, _ in self.samples:
            for bit, nm in self.REASONS.items():
                if rs & bit:
                    reasons.add(nm)
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": self.sm_max, "samples": len(self.samples),
                "power_w_max": max(s[2] for s in self.samples), "reasons": sorted(reasons), "source": "nvml"}


def algorithmic_bytes(nU, mean_samples_per_node, mean_succ_per_node, has_region):
    """SURVEY.md §8d: B = S_in + sum_samples*b_vox + N_succ*S_out per expansion."""
    b_vox = 1.0 + (0.125 if has_region else 0.0)
    return S_IN + mean_samples_per_node * b_vox + mean_succ_per_node * S_OUT


class CpuArm:
    """The reference's CPU implementation of the path, timed on the host cores.

    kind "reference": oracle/_ref/libmplref.so — the UNMODIFIED reference headers
    (env_map<Dim>::get_succ and everything under it) compiled against the Eigen/Boost stand-ins of
    oracle/shim; one env_map per std::thread (get_succ is not re-entrant), map shared read-only.
    kind "port": the oracle restatement (bit-identical results, fewer allocations) when _ref is absent."""

    def __init__(self, sc):
        sys.path.insert(0, str(ROOT / "tests"))
        import oracle_bindings as ob

        self.ob = ob
        self.env = ob.OracleEnv.from_scenario(sc)
        self.kind = "reference" if ob.ref_available() else "port"

    def timed(self, nodes, threads):
        if self.kind == "reference":
            return self.ob.ref_timed(self.env, nodes, nthreads=threads)
        return self.env.timed(nodes, nthreads=threads)

    def describe(self, threads):
        if self.kind == "reference":
            return (f"unmodified reference env_map::get_succ (oracle/_ref: the reference's include/ + Eigen/Boost "
                    f"stand-ins, g++ -O2), {threads} std::threads")
        return f"oracle restatement of env_map::get_succ (g++ -O2, no FMA), {threads} std::threads"


def cpu_reference(sc, nodes, threads, budget_s):
    """Time the CPU arm on a bounded sample of the same frontier (~budget_s seconds of all-core work)."""
    arm = CpuArm(sc)
    probe = nodes[: min(len(nodes), 64 * threads)]
    t = arm.timed(probe, threads)
    rate = len(probe) / max(t["seconds"], 1e-9)
    n = int(min(len(nodes), max(len(probe), rate * budget_s / 2)))
    done, secs = 0, 0.0
    while secs < budget_s * 0.8:
        t = arm.timed(nodes[:n], threads)
        done += n
        secs += t["seconds"]
    return dict(rate=done / secs, n=done, seconds=secs, kind=arm.kind, desc=arm.describe(threads))


def host_threads():
    """Threads for the CPU arm: every CPU the process may use (cgroup quota respected — running 128
    threads inside a 16-CPU quota only adds throttling and would flatter the GPU)."""
    from scenarios import effective_cpus

    return effective_cpus()


def config_dict(sc, n, world):
    """The `config` object of the JSON line — identical for both arms (same workload, same step)."""
    nU = sc.nU
    slots = n * nU
    return {"workload": sc.name, "map": "x".join(str(d) for d in sc.dim_cells) + f" @{sc.res} m int8",
            "control": f"0x{sc.control:02x}", "primitives_per_node": nU, "nodes_per_step_per_gpu": n,
            "frontier": "reachable lattice states (random free cell centres + <=6 random valid controls), seed 7+rank",
            "parallelism": f"replicas x{world}, frontier sharded",
            "l2": f"per-step working set {(n * 112 + slots * 132 + int(np.prod(sc.dim_cells))) / 1e6:.0f} MB "
                  f"(frontier + successor records + map) exceeds the H100's 50 MB L2"}


def run_reference(args, sc, rank, world):
    if rank != 0:
        return
    threads = host_threads()
    arm = CpuArm(sc)
    # the same step as the GPU arm: args.nodes frontier nodes of the same generator and seed (rank 0's slice)
    per_step = args.nodes
    batch = sc.frontier(per_step, seed=7)
    for _ in range(args.warmup):
        arm.timed(batch, threads)
    dt = 0.0
    for _ in range(args.steps):
        dt += arm.timed(batch, threads)["seconds"]
    v = per_step * args.steps / dt
    line = {
        "impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": config_dict(sc, per_step, max(1, args.gpus)),
        "cpu_baseline": {"value": v, "unit": UNIT, "cores": threads, "kind": arm.kind,
                         "sample": f"{per_step} frontier nodes/step x {args.steps} steps; {arm.describe(threads)}"},
        "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    emit(line)


def parity_spot_check(env, sc, nodes):
    """Expand `nodes` through the C ABI (the kernel the timed region uses) and compare with the CPU
    checker: the reference itself (oracle/_ref) when present, else the restatement.  Counts, actions,
    successor waypoints and keys bit-exact; costs exact for occupancy planning, 1e-6 relative otherwise.
    Returns {"nodes": n, "successors": s, "against": ...}; raises on any mismatch."""
    sys.path.insert(0, str(ROOT / "tests"))
    import oracle_bindings as ob
    from parity import assert_expansion_equal

    orc_env = ob.OracleEnv.from_scenario(sc)
    threads = host_threads()
    against = "reference" if ob.ref_available() else "port"
    o = ob.ref_expand(orc_env, nodes, nthreads=threads) if against == "reference" else orc_env.expand(nodes, nthreads=threads, lattice=False)
    g = env.expand(nodes, want=("succ", "cost", "action", "key"))
    st = assert_expansion_equal(g, o, exact_cost=sc.potential_radius is None and not (sc.control & 16))
    return {"nodes": int(len(nodes)), "successors": st["successors"], "against": against}


def run_cfg5_workload(args, rank, local, world):
    """`--workload cfg5`: the whole line is the sharded many-query planning run (BASELINE.json configs[4]).
    A step = planning the full query set once; value = expansions/s of the whole job, end to end (device
    expansion + PCIe + host A* bookkeeping + release of the search states)."""
    import scenarios as S

    sc5 = S.cfg3()
    if args.impl == "reference":
        if rank != 0:
            return
        sys.path.insert(0, str(ROOT / "tests"))
        import cfg5_bench
        import planner_bindings as pb
        from concurrent.futures import ThreadPoolExecutor

        from motion_primitive_library_b200 import planner

        q = cfg5_bench.make_queries(sc5, args.mq_queries, 20.0)
        nt = host_threads()
        n = min(len(q), 8 * nt)  # bounded sample of the same query set
        grid = sc5.grid()

        def one(k):
            a = planner.make_args(3, sc5.control, grid, sc5.dim_cells, sc5.origin, sc5.res, sc5.U,
                                  start=dict(pos=q["start"]["pos"][k]), goal=dict(pos=q["goal"]["pos"][k]), v_max=sc5.v_max,
                                  a_max=sc5.a_max, T=sc5.T, w=sc5.w, max_num=args.mq_max_expand, eps=args.mq_eps)
            return pb.plan_reference(a)

        vals = []
        for it in range(args.warmup + args.steps):
            with ThreadPoolExecutor(nt) as ex:
                outs = list(ex.map(one, range(n)))
            if it >= args.warmup:
                vals.append(sum(o["n_closed"] for o in outs) / (sum(o["seconds"] for o in outs) / min(nt, n)))
        v = float(np.mean(vals))
        emit({"impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": args.gpus,
                          "steps": args.steps, "warmup": args.warmup, "ms_per_step": None, "higher_is_better": True,
                          "scaling": "strong", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
                          "config": {"workload": "cfg5", "queries": args.mq_queries, "max_expand": args.mq_max_expand, "epsilon": args.mq_eps,
                                     "map": "512x512x512 @0.1 m int8", "control": "0x07", "primitives_per_node": 125},
                          "cpu_baseline": {"value": v, "unit": UNIT, "cores": nt, "kind": "reference",
                                           "sample": f"{n} of the {args.mq_queries} queries per step, one reference MapPlanner::plan per "
                                                     f"host thread, time inside plan() only"},
                          "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}})
        return
    import torch
    import torch.distributed as dist

    import cfg5_bench
    from motion_primitive_library_b200 import sharding

    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; the expansion engine has no CPU fallback")
    torch.cuda.set_device(local)
    if world > 1:
        sharding.bind_to_gpu_numa(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    grid = sharding.broadcast_array(sc5.grid() if rank == 0 else None, src=0)
    sampler = ClockSampler(local)
    runs = []
    for it in range(args.warmup + args.steps):
        if it == args.warmup and rank == 0:
            sampler.start()
        r = cfg5_bench.run(sc5, grid, local, n_queries=args.mq_queries, max_expand=args.mq_max_expand, eps=args.mq_eps,
                           ref_queries=32 if (world == 1 and it == 0) else 0)
        if it >= args.warmup:
            runs.append(r)
        elif it == 0:
            first = r
    if rank == 0:
        clocks = sampler.stop()
        secs = float(np.mean([r["seconds"] for r in runs]))
        v = runs[0]["expansions"] / secs
        line = {"metric": METRIC, "value": v, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                "ms_per_step": 1e3 * secs, "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f64",
                "data": "synthetic",
                "config": {"workload": "cfg5", "queries": args.mq_queries, "max_expand": args.mq_max_expand, "epsilon": args.mq_eps,
                           "map": "512x512x512 @0.1 m int8", "control": "0x07", "primitives_per_node": 125,
                           "parallelism": f"queries sharded over {world} rank(s), map broadcast once, results all-gathered"},
                "clocks": clocks, "multi_query": runs[-1], "reference_check": (first if args.warmup else runs[0]).get("reference"),
                "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": None, "d2h_bytes_per_step": None,
                        "note": "the value IS end to end: every iteration copies the popped nodes to the device and the "
                                "{key, action} records of their successors back"},
                "roofline": None, "cpu_baseline": None}
        emit(line)
    if world > 1:
        dist.destroy_process_group()


def replay_sweep(env, sc, lib, stream, local, max_nodes=65536):
    """Record the pop order of one long A* query on the workload's map (MPL::MapPlanner::plan with the GPU env,
    speculative batches of 64), then re-expand that sequence through mplx_expand_device in batches of
    B = 1, 256, 4096, 65536 nodes (inputs resident in HBM, CUDA events on the launching stream): the pure
    expansion rate on the frontier a search really produces, and how it depends on the batch size."""
    import torch

    from motion_primitive_library_b200 import abi, planner
    from motion_primitive_library_b200.abi import SuccOut

    pts = sc.frontier(64, seed=3, max_steps=0)["pos"]
    d = np.abs(pts[:, None, :] - pts[None, :, :]).max(-1)
    i, j = np.unravel_index(np.argmax(d), d.shape)  # the farthest pair of the sample: a long search
    a = planner.make_args(sc.Dim, sc.control, sc.grid(), sc.dim_cells, sc.origin, sc.res, sc.U, start=dict(pos=pts[i]),
                          goal=dict(pos=pts[j]), v_max=sc.v_max, a_max=sc.a_max, T=sc.T, w=sc.w, max_num=max_nodes, speculate=64)
    a.device = local
    t0 = time.perf_counter()
    tr = planner.plan_trace(a, cap=max_nodes)
    plan_s = time.perf_counter() - t0
    trace = tr["trace"]
    n, nU = len(trace), sc.nU
    if n < 256:
        return {"nodes": int(n), "note": "query solved too quickly for a sweep"}
    d_nodes = torch.from_numpy(np.ascontiguousarray(trace).view(np.uint8).reshape(n, 112)).cuda()
    bmax = min(n, 65536)
    slots = bmax * nU
    d_count = torch.empty(bmax, dtype=torch.int32, device="cuda")
    d_succ = torch.empty((slots, 112), dtype=torch.uint8, device="cuda")
    d_cost = torch.empty(slots, dtype=torch.float64, device="cuda")
    d_action = torch.empty(slots, dtype=torch.int32, device="cuda")
    d_key = torch.empty(slots, dtype=torch.int64, device="cuda")
    out_d = SuccOut(d_count.data_ptr(), d_succ.data_ptr(), d_cost.data_ptr(), d_action.data_ptr(), d_key.data_ptr(), None)
    stream.wait_stream(torch.cuda.current_stream())
    res = {}
    for B in (1, 256, 4096, 65536):
        if B > n:
            continue
        total = min(n, 2048 if B == 1 else n) // B * B  # bound the single-node case
        def run_once():
            for off in range(0, total, B):
                abi.check(lib.mplx_expand_device(env.handle, d_nodes.data_ptr() + off * 112, B, C.byref(out_d), stream.cuda_stream))
        run_once()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 3
        e0.record(stream)
        for _ in range(reps):
            run_once()
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        res[str(B)] = {"expansions_per_s": total / (ms * 1e-3), "us_per_batch": 1e3 * ms / (total // B), "nodes": int(total)}
    return {"nodes": int(n), "query": {"expanded": int(tr["expanded"]), "valid": int(tr["valid"]), "plan_seconds": plan_s,
                                        "speculate": 64},
            "batch_sweep": res,
            "what": "A* pop order of one long query (MPL::MapPlanner::plan, GPU env) replayed through mplx_expand_device"}


def dump_outputs(out_dir, n, nU, d_count, d_succ, d_cost, d_action, d_key, budget_bytes=48 << 20):
    """What mplx_expand_device returned in the last timed step, for a fixed seeded sample of the frontier nodes
    (all of them when they fit `budget_bytes`), as float64 .npy files: count [k], succ [k, nU, 14] (the
    Waypoint's pos, vel, acc, jrk, yaw, t), cost [k, nU], blocked [k, nU], action [k, nU], key [k, nU, 2] (high
    and low 32 bits).  A successor whose primitive collides has cost +inf in the API; here it has blocked = 1 and
    cost 0, so that every value written is finite.  Slots past a node's count hold no successor and are 0."""
    import torch

    per_node = nU * (14 + 1 + 1 + 1 + 2) * 8 + 8
    k = min(n, budget_bytes // per_node)
    idx = np.sort(np.random.default_rng(0).choice(n, size=k, replace=False)) if k < n else np.arange(n)
    it = torch.from_numpy(idx).to(d_count.device)
    count = d_count[it].cpu().numpy()
    valid = np.arange(nU)[None, :] < count[:, None]
    key = d_key.view(n, nU)[it].cpu().numpy().view(np.uint64)
    cost = d_cost.view(n, nU)[it].cpu().numpy()
    blocked = np.isposinf(cost)
    arrays = {
        "sample_index": idx,
        "count": count,
        "succ": d_succ.view(n, nU, 112)[it].view(torch.float64).cpu().numpy(),
        "cost": np.where(blocked, 0.0, cost),
        "blocked": blocked,
        "action": d_action.view(n, nU)[it].cpu().numpy(),
        "key": np.stack([key >> np.uint64(32), key & np.uint64(0xFFFFFFFF)], axis=-1),
    }
    out_dir.mkdir(parents=True, exist_ok=True)
    for name, a in arrays.items():
        a = a.astype(np.float64)
        if a.ndim >= 2:
            a[~valid] = 0.0
        if not np.isfinite(a).all():
            raise RuntimeError(f"bench.py: non-finite values in the {name} output of the timed step")
        np.save(out_dir / f"{name}.npy", a)


def kernel_name(which, sc, n_nodes, sms):
    """The kernel mplx_set_kernel(which) launches for this workload on a device with `sms` SMs (auto rule:
    mplx_kernels.cu launch_expand)."""
    names = {1: "mplx::expand_seq_kernel", 2: "mplx::expand_reg_kernel", 3: "mplx::expand_flat_kernel", 4: "mplx::expand_deal_kernel"}
    if which in names:
        return names[which]
    if (sc.control & 16) == 0 and sc.potential_radius is None and sc.nU <= 256:
        # occupancy planning: fixed-point sample loop; node-cooperative rows + flat items for large batches
        return "mplx::expand_fxn_kernel" if n_nodes * sc.nU >= 64 * 256 and sc.v_max > 0 else "mplx::expand_fx_kernel"
    heavy = (sc.control & 15) >= 7 or (sc.control & 16) != 0 or sc.potential_radius is not None
    big = n_nodes * sc.nU >= 2 * 256 * sms * 4 * 8
    return "mplx::expand_deal_kernel" if heavy and big else "mplx::expand_reg_kernel"


def main():
    args = parse()
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    import scenarios as S

    if args.workload == "cfg5":
        run_cfg5_workload(args, rank, local, world)
        return
    sc = S.WORKLOADS[args.workload]()
    if args.impl == "reference":
        run_reference(args, sc, rank, world)
        return

    import torch
    import torch.distributed as dist

    from motion_primitive_library_b200 import abi
    from motion_primitive_library_b200.abi import SuccOut, WAYPOINT_DTYPE

    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; the expansion engine has no CPU fallback "
                         "(use --impl reference for the CPU path)")
    torch.cuda.set_device(local)
    numa = None
    if world > 1:
        from motion_primitive_library_b200 import sharding

        numa = sharding.bind_to_gpu_numa(local)  # before any pinned allocation
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lib = abi.load()

    # ---- inputs: every rank holds the full map (replica) and its own slice of the frontier ----
    env = make_env(sc, local)
    env.set_kernel(args.kernel)
    n, nU = args.nodes, sc.nU
    nodes_np = sc.frontier(n, seed=7 + rank)
    slots = n * nU

    # measured algorithmic bytes (untimed stats pass)
    d_nodes = torch.from_numpy(nodes_np.view(np.uint8).reshape(n, 112)).cuda()
    d_count = torch.empty(n, dtype=torch.int32, device="cuda")
    d_succ = torch.empty((slots, 112), dtype=torch.uint8, device="cuda")
    d_cost = torch.empty(slots, dtype=torch.float64, device="cuda")
    d_action = torch.empty(slots, dtype=torch.int32, device="cuda")
    d_key = torch.empty(slots, dtype=torch.int64, device="cuda")
    out_d = SuccOut(d_count.data_ptr(), d_succ.data_ptr(), d_cost.data_ptr(), d_action.data_ptr(), d_key.data_ptr(), None)
    # a dedicated non-default stream: the kernel, and the CUDA events that time it, are both
    # issued on this stream (mplx_expand_device treats a NULL stream as "the ctx's own stream",
    # so torch's legacy default stream, whose handle is 0, must not be used here)
    stream = torch.cuda.Stream()
    assert stream.cuda_stream != 0
    stream.wait_stream(torch.cuda.current_stream())

    def step_device():
        abi.check(lib.mplx_expand_device(env.handle, d_nodes.data_ptr(), n, C.byref(out_d), stream.cuda_stream))

    env.enable_stats(True)
    step_device()
    torch.cuda.synchronize()
    samples, succ_total = env.last_stats()
    env.enable_stats(False)
    mean_samples, mean_succ = samples / n, succ_total / n
    bytes_per_exp = algorithmic_bytes(nU, mean_samples, mean_succ, False)

    # ---- untimed spot check: a slice of the very frontier that is timed, against the CPU checker ----
    parity_checked = parity_spot_check(env, sc, nodes_np[: min(n, 4096)])

    for _ in range(args.warmup):
        step_device()
    torch.cuda.synchronize()
    launches0 = env.launch_count()
    if world > 1:
        dist.barrier()
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
    ev[0].record(stream)
    for k in range(args.steps):
        step_device()
        ev[k + 1].record(stream)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    clocks = sampler.stop() if rank == 0 else None
    elapsed_ms = ev[0].elapsed_time(ev[-1])
    kernel_ms = [ev[k].elapsed_time(ev[k + 1]) for k in range(args.steps)]
    if args.dump_outputs and rank == 0:
        dump_outputs(Path(args.dump_outputs), n, nU, d_count, d_succ, d_cost, d_action, d_key)
    gpu_launches = env.launch_count() - launches0  # kernels of this library launched inside the timed region
    t_el = torch.tensor([elapsed_ms], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(t_el, op=dist.ReduceOp.MAX)
    elapsed_ms = float(t_el.item())
    value = world * n * args.steps / (elapsed_ms * 1e-3)

    # ---- e2e: the reference-facing C-ABI calls with HOST (pinned) buffers, copies inside the timed region.
    #   e2e        mplx_expand_packed, flags=DROP_INF: what the A* host consumes per successor — state fields
    #              marked by the control flag + cost + action + key, +inf successors dropped on the device
    #              (graph_search.h:81), double-buffered over two streams.  This is the call the planner makes.
    #   e2e_full   mplx_expand: the literal get_succ contract (112 B Waypoint + cost + action + key, inf kept).
    e2e = None
    e2e_full = None
    e2e_state = None
    if not args.no_e2e:
        from motion_primitive_library_b200.abi import PackedOut

        def timed_host(step, steps):
            for _ in range(2):
                step()
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            l0 = env.launch_count()
            t0 = time.perf_counter()
            for _ in range(steps):
                step()
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            t_e = torch.tensor([t1 - t0], dtype=torch.float64, device="cuda")
            if world > 1:
                dist.all_reduce(t_e, op=dist.ReduceOp.MAX)
            return float(t_e.item()), env.launch_count() - l0

        e2e_steps = max(3, min(args.steps, 10))
        h_nodes = env._pinned_empty(n, WAYPOINT_DTYPE)
        h_nodes[:] = nodes_np
        nstate = sc.Dim * bin(sc.control & 15).count("1") + (1 if sc.control & 16 else 0)
        # occupancy planning: the finite edge cost is a function of the action alone and the coordinates of a
        # successor are needed only when its key is new to the search, where the host planner evaluates them
        # itself (MPL::MultiQueryPlanner, env_map_gpu::forward_from_pod): the stream is {key, u16 action}.
        # Potential-field / yaw planning streams the cost too.
        keys_only = sc.potential_radius is None and not (sc.control & 16)
        pb = dict(count=env._pinned_empty(n, np.int32), offset=env._pinned_empty(n, np.int64),
                  action=env._pinned_empty(slots, np.uint16), key=env._pinned_empty(slots, np.uint64))
        if not keys_only:
            pb["cost"] = env._pinned_empty(slots, np.float64)

        def packed_out(b):
            return PackedOut(b["count"].ctypes.data, b["offset"].ctypes.data, abi.ptr(b.get("state")),
                             abi.ptr(b.get("cost")), b["action"].ctypes.data, b["key"].ctypes.data, slots, 0, 0)

        out_p = packed_out(pb)

        def step_packed():
            abi.check(lib.mplx_expand_packed(env.handle, h_nodes.ctypes.data, n, abi.PACK_DROP_INF, C.byref(out_p)))

        secs, launches = timed_host(step_packed, e2e_steps)
        kept = int(out_p.total)
        assert int(pb["count"].sum()) == kept and 0 < kept <= succ_total  # the result is read on the host
        rec_bytes = 8 + 2 + (0 if keys_only else 8)
        e2e = {"value": world * n * e2e_steps / secs, "unit": UNIT, "h2d_bytes_per_step": int(n * 112),
               "d2h_bytes_per_step": int(n * 12 + kept * rec_bytes), "steps": e2e_steps,
               "ms_per_step": 1e3 * secs / e2e_steps, "launches": int(launches), "records_per_step": kept,
               "d2h_gbs": (n * 12 + kept * rec_bytes) * e2e_steps / secs / 1e9,
               "call": "mplx_expand_packed(flags=MPLX_PACK_DROP_INF), pinned host buffers: per finite successor "
                       + ("key + u16 action (cost = f(action), coordinates rebuilt by the host for new states only)"
                          if keys_only else "cost + key + u16 action") + "; per node count + offset"}
        # the same call with the state fields and the cost in the stream (round-1 protocol)
        pb["state"] = env._pinned_empty(slots * nstate, np.float64)
        if "cost" not in pb:
            pb["cost"] = env._pinned_empty(slots, np.float64)
        out_p = packed_out(pb)
        secs, launches = timed_host(step_packed, max(3, e2e_steps // 2))
        e2e_state = {"value": world * n * max(3, e2e_steps // 2) / secs, "unit": UNIT, "h2d_bytes_per_step": int(n * 112),
                     "d2h_bytes_per_step": int(n * 12 + kept * (8 * nstate + 8 + 2 + 8)),
                     "ms_per_step": 1e3 * secs / max(3, e2e_steps // 2), "launches": int(launches),
                     "call": f"mplx_expand_packed with {nstate} state doubles + cost + key + u16 action per finite successor"}
        del pb

        h_count = env._pinned_empty(n, np.int32)
        h_succ = env._pinned_empty(slots, WAYPOINT_DTYPE)
        h_cost = env._pinned_empty(slots, np.float64)
        h_action = env._pinned_empty(slots, np.int32)
        h_key = env._pinned_empty(slots, np.uint64)
        out_h = SuccOut(h_count.ctypes.data, h_succ.ctypes.data, h_cost.ctypes.data, h_action.ctypes.data,
                        h_key.ctypes.data, None)

        def step_host():
            abi.check(lib.mplx_expand(env.handle, h_nodes.ctypes.data, n, C.byref(out_h)))

        secs, launches = timed_host(step_host, max(3, e2e_steps // 2))
        assert int(h_count.sum()) == succ_total
        e2e_full = {"value": world * n * max(3, e2e_steps // 2) / secs, "unit": UNIT,
                    "h2d_bytes_per_step": int(n * 112), "d2h_bytes_per_step": int(n * 4 + slots * (112 + 8 + 4 + 8)),
                    "ms_per_step": 1e3 * secs / max(3, e2e_steps // 2), "launches": int(launches),
                    "call": "mplx_expand: full get_succ contract, 132 B per successor slot, +inf kept"}

    # ---- replay frontier (SURVEY.md §8d i): the nodes a real A* pops, re-expanded in batches of B ----
    replay = None
    if not args.no_replay and rank == 0 and args.workload in ("512c_acc27", "cfg2"):
        replay = replay_sweep(env, sc, lib, stream, local)

    # ---- cfg5 leg: the path's actual multi-GPU split — 4096 start/goal queries sharded over the ranks ----
    multi_query = None
    if not args.no_multi_query and args.workload == "512c_acc27":
        import cfg5_bench
        from motion_primitive_library_b200 import sharding

        sc5 = S.cfg3()  # same map generator and seed as the headline workload, JRK-125 controls
        grid5 = sharding.broadcast_array(sc.grid() if rank == 0 else None, src=0)  # the one set-up collective
        env.close()
        torch.cuda.empty_cache()
        multi_query = cfg5_bench.run(sc5, grid5, local, n_queries=args.mq_queries, max_expand=args.mq_max_expand, eps=args.mq_eps,
                                     ref_queries=32 if world == 1 else 0)

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    peaks = {}
    pk = ROOT / "MEASURED_PEAKS.json"
    if pk.exists():
        peaks = json.loads(pk.read_text())
    peak_gbs = float(peaks.get("hbm_gbs", 3350.0))  # fallback: H100 SXM data sheet
    k_ms = float(np.mean(kernel_ms))
    achieved = bytes_per_exp * n / (k_ms * 1e-3) / 1e9
    roofline = {"bound": "hbm", "achieved": achieved, "peak": peak_gbs, "unit": "GB/s", "frac": achieved / peak_gbs,
                "traffic": None, "peak_source": "measured" if pk.exists() else "fallback",
                "kernel": kernel_name(args.kernel, sc, n, torch.cuda.get_device_properties(local).multi_processor_count),
                "kernel_ms": k_ms,
                "algorithmic_bytes_per_expansion": bytes_per_exp,
                "mean_samples_per_expansion": mean_samples, "mean_successors_per_expansion": mean_succ}

    cpu_baseline = None
    if world == 1 and not args.no_cpu_baseline:
        threads = host_threads()
        r = cpu_reference(sc, nodes_np, threads, args.cpu_seconds)
        cpu_baseline = {"value": r["rate"], "unit": UNIT, "cores": threads, "kind": r["kind"],
                        "sample": f"{r['n']} expansions drawn from the same frontier, {r['seconds']:.1f} s; {r['desc']}"}

    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": elapsed_ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f64", "data": "synthetic",
        "config": config_dict(sc, n, world), "primitives_per_sec": value * nU, "parity_checked": parity_checked,
        "clocks": clocks, "numa": numa, "e2e": e2e, "e2e_state_records": e2e_state, "e2e_full_contract": e2e_full, "gpu_launches": int(gpu_launches),
        "roofline": roofline, "replay": replay, "multi_query": multi_query,
        "cpu_baseline": cpu_baseline,
    }
    emit(line)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
