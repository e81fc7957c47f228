#!/usr/bin/env python
"""What a map change costs the device, sparse against full.

  python map_update_bench.py [--warmup W]     # prints ONE JSON line

For the headline 512^3 map and the cfg2 256^3 map it times
  * the full path a changed grid takes without sparse updates: mplx_set_map (grid copy + both packs),
    and the potential-map and search-region re-sends that follow it when those are set;
  * mplx_update_cells for k changed voxels, k from 1 up past the point where it costs as much as the
    full path, for two patterns: k uniformly random voxels (unsorted: the radix-sort path), and one solid
    box of k voxels in index order (the already-sorted path).
Each time is a host clock around one synchronous call (both entry points return after a stream
synchronise), after warm-up calls of the same shape; the median and the minimum of the repeats are
reported.  `crossover_k` is the smallest k whose median update time reaches the median set_map time;
the journal limit of MapUtil (host/mpl_host.hpp, kJournalFraction) is set from it."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))


def card_info(device=0):
    """Name and power limit of the card, read now (the numbers are only meaningful with them)."""
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(device)
        name = pynvml.nvmlDeviceGetName(h)
        return {"name": name.decode() if isinstance(name, bytes) else name,
                "power_limit_w": pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0}
    except Exception:
        out = subprocess.run(["nvidia-smi", "-i", str(device), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1])} if len(out) == 2 else {"name": None, "power_limit_w": None}


def _time(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return {"median_ms": 1e3 * float(np.median(ts)), "min_ms": 1e3 * float(np.min(ts)), "reps": reps}


def _box(dims, k, rng):
    """Indices of one solid box of about k voxels (a cube of side round(k^(1/3))), in index order."""
    s = max(1, int(round(k ** (1.0 / 3.0))))
    s = min(s, *dims)
    lo = [int(rng.integers(0, d - s + 1)) for d in dims]
    z, y, x = np.meshgrid(*(np.arange(lo[a], lo[a] + s) for a in (2, 1, 0)), indexing="ij")
    return (x + dims[0] * y + dims[0] * dims[1] * z).reshape(-1).astype(np.int32)


def measure_map(sc, ks, warmup, device=0):
    from motion_primitive_library_b200 import MapUtil, abi, env_map

    lib = abi.load()
    grid = np.ascontiguousarray(sc.grid(), dtype=np.int8)
    dims = tuple(int(d) for d in sc.dim_cells)
    nvox = grid.size
    mu = MapUtil()
    mu.setMap(sc.origin, dims, grid, sc.res)
    env = env_map(mu, device=device)
    h = env.handle
    dim32 = np.ascontiguousarray(dims, dtype=np.int32)
    org = np.ascontiguousarray(sc.origin, dtype=np.float64)
    pot = np.ascontiguousarray(np.where(grid == 100, 100, 0).astype(np.int8))  # any int8 field: only the copy is timed
    region = np.ones(nvox, dtype=np.uint8)

    def set_map():
        abi.check(lib.mplx_set_map(h, grid.ctypes.data, dim32.ctypes.data, org.ctypes.data, sc.res))

    full = {"set_map": _time(set_map, warmup, 10),
            "set_potential": _time(lambda: abi.check(lib.mplx_set_potential(h, pot.ctypes.data, 0.1, 0.0)), warmup, 10),
            "set_search_region": _time(lambda: abi.check(lib.mplx_set_search_region(h, region.ctypes.data)), warmup, 10)}
    full["set_map_potential_region_ms"] = sum(full[k]["median_ms"] for k in ("set_map", "set_potential", "set_search_region"))
    set_map()
    rng = np.random.default_rng(11)
    out = {"map": "x".join(str(d) for d in dims), "nvox": nvox, "full_path": full, "update_cells": {}}
    for pattern in ("random", "box"):
        rows = []
        for k in ks:
            if k > nvox:
                continue
            idx = rng.integers(0, nvox, k, dtype=np.int64).astype(np.int32) if pattern == "random" else _box(dims, k, rng)
            vals = np.where(rng.random(idx.size) < 0.5, 100, 0).astype(np.int8)

            def upd():
                abi.check(lib.mplx_update_cells(h, idx.ctypes.data, vals.ctypes.data, idx.size))

            reps = 20 if idx.size <= (1 << 18) else 5
            rows.append({"k": int(idx.size), **_time(upd, warmup, reps)})
        t_full = full["set_map"]["median_ms"]
        cross = next((r["k"] for r in rows if r["median_ms"] >= t_full), None)
        out["update_cells"][pattern] = {"rows": rows, "crossover_k": cross,
                                        "crossover_fraction": None if cross is None else cross / nvox}
    env.close()
    return out


def run(warmup):
    import torch

    import scenarios as S

    if not torch.cuda.is_available():
        raise SystemExit("map_update_bench.py: no CUDA device; the map-update path has no CPU fallback")
    ks = [1, 64, 4096, 1 << 15, 1 << 18, 1 << 20, 1 << 21, 1 << 22, 1 << 23, 1 << 24, 1 << 25]
    warmup = max(1, warmup)
    card = card_info(0)
    maps = [measure_map(S.cfg_headline(), ks, warmup), measure_map(S.cfg2(), ks, warmup)]
    card_after = card_info(0)
    return {"workload": "map_update", "metric": "ms per map change (host clock around the synchronous call)",
            "unit": "ms", "higher_is_better": False, "gpu": card, "gpu_after": card_after, "maps": maps,
            "note": "full path = what a changed grid costs when it is re-uploaded: mplx_set_map, then the potential "
                    "map and the search region re-sent when set"}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    print(json.dumps(run(ap.parse_args().warmup)), flush=True)
