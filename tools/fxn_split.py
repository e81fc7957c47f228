#!/usr/bin/env python
"""Where the headline step's time goes: mplx_expand_device on the 512^3 ACC-27 frontier (bench.py's
default workload, 2^18 nodes, seed 7), timed with CUDA events over --steps steps after --warmup.

Output sets, in one process:
  default      every output of bench.py (count, successor records, cost, action, key);
  succ=NULL    the same without the 112-byte successor records;
  count only   succ, key, action and cost NULL;
  succ only    count and the successor records.
Library switches, one child process each (they are read once per process), every output:
  no L2 window   MPLX_NO_L2_WINDOW=1: the voxel bitmap pairs get no persisting access-policy window;
  per-lane       MPLX_FXN_SPAN=0: every output written by per-lane stores;
  span succ      MPLX_FXN_SPAN=1: the records through the CTA-span staging, the rest per lane;
  span succ+ka   MPLX_FXN_SPAN=3: records, keys and actions staged;
  span all       MPLX_FXN_SPAN=7: records, keys, actions and costs staged (the default).
SM clock, power and throttle reasons are sampled during every timed window (bench.ClockSampler, else nvidia-smi): a card with a
low power limit may cap its clocks under the write stream.  Prints the card, its power limit and the L2 sizes
next to the numbers.  MPLX_LIB selects the library as everywhere.
Usage: python tools/fxn_split.py [--steps 1000] [--warmup 10] [--reps 3]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

CHILDREN = {
    "no L2 window": {"MPLX_NO_L2_WINDOW": "1"},
    "per-lane": {"MPLX_FXN_SPAN": "0"},
    "span succ": {"MPLX_FXN_SPAN": "1"},
    "span succ+ka": {"MPLX_FXN_SPAN": "3"},
    "span all": {"MPLX_FXN_SPAN": "7"},
}


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    props = torch.cuda.get_device_properties(0)
    persist = C.c_int(0)
    try:
        rt = C.CDLL("libcudart.so.12")
        rt.cudaDeviceGetAttribute(C.byref(persist), 108, 0)  # cudaDevAttrMaxPersistingL2CacheSize
    except OSError:
        persist.value = -1
    return {"nvidia_smi": q, "l2_bytes": props.L2_cache_size, "max_persisting_l2_bytes": persist.value}


class SmiSampler:
    """Clock, power and throttle reasons from `nvidia-smi -lms` while a window runs: the fallback where
    bench.ClockSampler has no NVML bindings."""

    QUERY = "clocks.sm,power.draw,clocks_throttle_reasons.sw_power_cap,clocks_throttle_reasons.hw_slowdown,"\
            "clocks_throttle_reasons.sw_thermal_slowdown"

    def start(self):
        self.p = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.QUERY}", "--format=csv,noheader,nounits", "-i", "0",
                                   "-lms", "20"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)

    def stop(self):
        self.p.terminate()
        out, _ = self.p.communicate(timeout=10)
        rows = [[x.strip() for x in line.split(",")] for line in out.splitlines() if line.count(",") == 4]
        if not rows:
            return {"sm_mhz": None, "reasons": ["no samples"]}
        sm = sorted(float(r[0]) for r in rows)
        names = ("sw_power_cap", "hw_slowdown", "sw_thermal_slowdown")
        reasons = sorted({nm for r in rows for nm, v in zip(names, r[2:]) if v.lower() == "active"})
        return {"sm_mhz": sm[len(sm) // 2], "power_w_max": max(float(r[1]) for r in rows), "reasons": reasons,
                "samples": len(rows), "source": "nvidia-smi"}


def sampler():
    import bench

    s = bench.ClockSampler(0)
    return s if s.nv is not None else SmiSampler()


def measure(steps, warmup, reps, setups):
    import numpy as np
    import torch

    import bench
    import scenarios as S
    from motion_primitive_library_b200 import abi
    from motion_primitive_library_b200.abi import SuccOut

    sc = S.cfg_headline()
    n, nU = 1 << 18, sc.nU
    slots = n * nU
    torch.cuda.set_device(0)
    lib = abi.load()
    env = bench.make_env(sc, 0)
    nodes = sc.frontier(n, seed=7)
    d_nodes = torch.from_numpy(nodes.view(np.uint8).reshape(n, 112)).cuda()
    d_count = torch.empty(n, dtype=torch.int32, device="cuda")
    d_succ = torch.empty((slots, 112), dtype=torch.uint8, device="cuda")
    d_cost = torch.empty(slots, dtype=torch.float64, device="cuda")
    d_action = torch.empty(slots, dtype=torch.int32, device="cuda")
    d_key = torch.empty(slots, dtype=torch.int64, device="cuda")
    cnt, succ, cost, act, key = (d_count.data_ptr(), d_succ.data_ptr(), d_cost.data_ptr(), d_action.data_ptr(),
                                 d_key.data_ptr())
    outs = {"default": SuccOut(cnt, succ, cost, act, key, None),
            "succ=NULL": SuccOut(cnt, None, cost, act, key, None),
            "count only": SuccOut(cnt, None, None, None, None, None),
            "succ only": SuccOut(cnt, succ, None, None, None, None)}
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    res, clocks = {}, {}
    for rep in range(reps):
        for name in setups:
            out = outs[name]

            def step():
                abi.check(lib.mplx_expand_device(env.handle, d_nodes.data_ptr(), n, C.byref(out), stream.cuda_stream))

            for _ in range(warmup):
                step()
            torch.cuda.synchronize()
            smp = sampler()
            smp.start()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record(stream)
            for _ in range(steps):
                step()
            ev[1].record(stream)
            torch.cuda.synchronize()
            c = smp.stop()
            res.setdefault(name, []).append(ev[0].elapsed_time(ev[1]) / steps)
            clocks.setdefault(name, []).append(c)
    env.close()
    return {"ms": res, "clocks": clocks}


def fmt_clocks(cs):
    sm = [c.get("sm_mhz") for c in cs if c.get("sm_mhz")]
    pw = [c.get("power_w_max") for c in cs if c.get("power_w_max")]
    rs = sorted({r for c in cs for r in c.get("reasons", [])})
    return (f"sm {min(sm):.0f}-{max(sm):.0f} MHz" if sm else "sm n/a") + (f", power max {max(pw):.0f} W" if pw else "") + \
        f", throttle {','.join(rs) or 'none'}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", default=None, help="comma-separated set-up names (default: all)")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        print(json.dumps(measure(a.steps, a.warmup, a.reps, ["default"])))
        return
    only = set(a.only.split(",")) if a.only else None
    inproc = [s for s in ("default", "succ=NULL", "count only", "succ only") if only is None or s in only]
    r = measure(a.steps, a.warmup, a.reps, inproc) if inproc else {"ms": {}, "clocks": {}}
    res, clocks = r["ms"], r["clocks"]
    for name, env in CHILDREN.items():
        if only is not None and name not in only:
            continue
        child = subprocess.run([sys.executable, __file__, "--child", "--steps", str(a.steps), "--warmup", str(a.warmup),
                                "--reps", str(a.reps)], env=dict(os.environ, **env), capture_output=True, text=True,
                               check=True)
        cr = json.loads(child.stdout.strip().splitlines()[-1])
        res[name], clocks[name] = cr["ms"]["default"], cr["clocks"]["default"]
    info = card()
    print(f"card: {info['nvidia_smi']}  L2 {info['l2_bytes'] >> 20} MiB, max persisting "
          f"{info['max_persisting_l2_bytes'] / 2**20:.1f} MiB  lib: {os.environ.get('MPLX_LIB', 'default')}")
    for name, ms in res.items():
        print(f"  {name:14s} ms/step " + " ".join(f"{x:.4f}" for x in ms) + f"   min {min(ms):.4f}   "
              + fmt_clocks(clocks[name]))


if __name__ == "__main__":
    main()
