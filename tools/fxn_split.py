#!/usr/bin/env python
"""Where the headline step's time goes: mplx_expand_device on the 512^3 ACC-27 frontier (bench.py's
default workload, 2^18 nodes, seed 7), timed with CUDA events over --steps steps after --warmup, in
three set-ups:
  default      every output of bench.py (count, successor records, cost, action, key);
  succ=NULL    the same without the 112-byte successor records (the record stream leaves the L2);
  no L2 window MPLX_NO_L2_WINDOW=1: the voxel bitmap pairs get no persisting access-policy window.
The L2 switch is read once per process, so that set-up runs in a child process.  Prints the card,
its power limit and the L2 sizes next to the numbers.  MPLX_LIB selects the library as everywhere.
Usage: python tools/fxn_split.py [--steps 20] [--warmup 3] [--reps 3]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


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
    outs = {"default": SuccOut(d_count.data_ptr(), d_succ.data_ptr(), d_cost.data_ptr(), d_action.data_ptr(),
                               d_key.data_ptr(), None),
            "succ=NULL": SuccOut(d_count.data_ptr(), None, d_cost.data_ptr(), d_action.data_ptr(), d_key.data_ptr(), None)}
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    res = {}
    for rep in range(reps):
        for name in setups:
            out = outs[name]

            def step():
                abi.check(lib.mplx_expand_device(env.handle, d_nodes.data_ptr(), n, C.byref(out), stream.cuda_stream))

            for _ in range(warmup):
                step()
            torch.cuda.synchronize()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record(stream)
            for _ in range(steps):
                step()
            ev[1].record(stream)
            torch.cuda.synchronize()
            res.setdefault(name, []).append(ev[0].elapsed_time(ev[1]) / steps)
    env.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        print(json.dumps(measure(a.steps, a.warmup, a.reps, ["default"])))
        return
    res = measure(a.steps, a.warmup, a.reps, ["default", "succ=NULL"])
    child = subprocess.run([sys.executable, __file__, "--child", "--steps", str(a.steps), "--warmup", str(a.warmup),
                            "--reps", str(a.reps)], env=dict(os.environ, MPLX_NO_L2_WINDOW="1"),
                           capture_output=True, text=True, check=True)
    res["no L2 window"] = json.loads(child.stdout.strip().splitlines()[-1])["default"]
    info = card()
    print(f"card: {info['nvidia_smi']}  L2 {info['l2_bytes'] >> 20} MiB, max persisting "
          f"{info['max_persisting_l2_bytes'] / 2**20:.1f} MiB  lib: {os.environ.get('MPLX_LIB', 'default')}")
    for name, ms in res.items():
        print(f"  {name:13s} ms/step " + " ".join(f"{x:.4f}" for x in ms) + f"   min {min(ms):.4f}")


if __name__ == "__main__":
    main()
