"""The CTA-span copy-out of expand_fxn_kernel (csrc/mplx_fxn.cu, csrc/mplx_span.cuh) through mplx_expand_device.

A CTA stages its successor records, keys, actions and costs in shared memory, one contiguous span of slots per
array with the holes past each node's count filled, and copies each span out with plain stores at its unaligned
edges and bulk copies for the rest.  Every case runs every selectable kernel into device arrays that sit between
guard bytes, at offsets from 16-byte alignment, and checks the results bit for bit against the CPU oracle, that
no byte outside the arrays changed and that the auto kernel launched expand_fxn_kernel + fx_resolve_kernel.
Which outputs are staged follows the launcher's rule (span_mask); the forced legs run every staging mask in a
child process, where MPLX_FXN_SPAN is read afresh."""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle_bindings as ob
from parity import assert_expansion_equal
from test_fx_paths_gpu import (ACC, JRK, KERNELS, NTHREADS, ORDER, THREADS, VEL, WANT, Case, boundary_case, emitted_mask,
                               matrix_case, overflow_case, product_set, queue_capacity, random_nodes, same_mask)

pytestmark = pytest.mark.gpu

GUARD = 384  # bytes of pattern before and after every array; a multiple of 128
PATTERN = 0xA5
SPAN_MIN_LOOP = 20  # kSpanMinLoop (csrc/mplx_fxn.cu)
SIZES = dict(succ=ob.WAYPOINT_DTYPE.itemsize, cost=8, action=4, key=8, lattice=4 * ob.LATTICE_MAX)


def span_mask(case):
    """The outputs the launcher stages by default (bits 1 succ, 2 key + action, 4 cost) when all are requested:
    none on the sorted path (JRK/SNP), keys, actions and costs only where the plan bounds the sample loops at
    maxn = ceil(v_max T / res) >= 20 samples (the whole table where v_max <= 0 or for VEL)."""
    if ORDER[case.control] >= 3:
        return 0
    maxn = 128 if case.v_max <= 0 or case.control == VEL else math.ceil(case.v_max * case.T / case.res)
    return 7 if maxn >= SPAN_MIN_LOOP else 1


def expand_guarded(env, nodes, want, offsets=None, kernel=0):
    """mplx_expand_device into arrays that start offsets[name] bytes past a 128-byte line, each with GUARD pattern
    bytes before and after; returns the Expansion after checking that the guards are intact."""
    import torch

    from motion_primitive_library_b200 import abi
    from motion_primitive_library_b200.env import Expansion

    offsets = offsets or {}
    env._sync_params()
    n, nU = nodes.size, env.U_.shape[0]
    dev = torch.device("cuda", 0)
    d_nodes = torch.from_numpy(nodes.view(np.uint8).copy()).to(dev)
    raw, arr = {}, {}
    for name in ("count",) + tuple(want):
        size = 4 * n if name == "count" else n * nU * SIZES[name]
        off = offsets.get(name, 0)
        raw[name] = torch.full((2 * GUARD + off + size,), PATTERN, dtype=torch.uint8, device=dev)
        assert raw[name].data_ptr() % 128 == 0
        arr[name] = raw[name][GUARD + off:GUARD + off + size]
        assert arr[name].data_ptr() % 128 == off % 128
    out = abi.SuccOut(*[arr[k].data_ptr() if k in arr else None for k in ("count", "succ", "cost", "action", "key", "lattice")])
    before = env.launch_count()
    abi.check(env._lib.mplx_expand_device(env.handle, d_nodes.data_ptr(), n, C.byref(out), None))
    abi.check(env._lib.mplx_sync(env.handle))
    assert env.launch_count() - before == (2 if kernel == 0 else 1), kernel  # kernel 0: fxn + resolve
    for name, r in raw.items():
        h = r.cpu().numpy()
        lo, hi = GUARD + offsets.get(name, 0), h.size - GUARD
        assert (h[:lo] == PATTERN).all() and (h[hi:] == PATTERN).all(), f"{name}: bytes outside the array written"
    host = {k: v.cpu().numpy() for k, v in arr.items()}
    return Expansion(nU, host["count"].view(np.int32),
                     host["succ"].view(ob.WAYPOINT_DTYPE) if "succ" in host else None,
                     host["cost"].view(np.float64) if "cost" in host else None,
                     host["action"].view(np.int32) if "action" in host else None,
                     host["key"].view(np.uint64) if "key" in host else None,
                     host["lattice"].view(np.int32).reshape(-1, ob.LATTICE_MAX) if "lattice" in host else None)


OUTPUTS = ("succ", "cost", "action", "key")
WANTS = [OUTPUTS, ("cost", "action", "key")] + [tuple(x for x in OUTPUTS if x != drop) for drop in OUTPUTS]
# key and action 8 / 4 bytes past 16-byte alignment, succ 16-byte but not 128-byte aligned
OFFSETS = [dict(), dict(succ=48, key=8, action=4, cost=8, count=4), dict(succ=16, key=24, action=12, cost=120)]


def check_all(case, nodes, wants=WANTS, offsets=OFFSETS, kernels=KERNELS):
    orc = case.oracle().expand(nodes, nthreads=NTHREADS)
    env = case.gpu()
    for k in kernels:
        env.set_kernel(k)
        for want in wants:
            for off in offsets:
                assert_expansion_equal(expand_guarded(env, nodes, want, off, k), orc, exact_cost=True)
    return orc


def test_headline_plan_with_ambiguous_primitives():
    """ACC-27 starts on cell boundaries next to obstacles: many primitives are queued and resolved; 1201 nodes
    is not a multiple of the 9 nodes of a CTA."""
    case, nodes = boundary_case(0.15, seed=31)
    assert nodes.size % (THREADS // case.nU) != 0 and span_mask(case) == 7
    orc = check_all(case, nodes)
    em = emitted_mask(orc)
    assert np.isinf(orc["cost"][em]).sum() > 2000 and np.isfinite(orc["cost"][em]).sum() > 2000


@pytest.mark.parametrize("per_axis", [(4, 8), (8, 8), (8, 16), (16, 16)], ids=["32", "64", "128", "256"])
def test_full_cta_spans_2d(per_axis):
    """2-D VEL sets of 32 / 64 / 128 / 256 controls: npb * nU = 256, the largest span."""
    m = dict(mdim=(211, 97), origin=(-31.1337, -14.2791), res=0.3)
    from scenarios import box_map

    grid = box_map(m["mdim"], m["res"], m["origin"], n_boxes=12, edge_m=(0.9, 3.0), seed=per_axis[0] + per_axis[1])
    U = product_set(np.linspace(-2.0, 2.0, per_axis[0]), np.linspace(-2.0, 2.0, per_axis[1]))
    case = Case(2, VEL, U, m["mdim"], m["origin"], m["res"], grid=grid, v_max=2.5)
    assert (THREADS // case.nU) * case.nU == 256 and span_mask(case) == 7
    n = max(64 * THREADS // case.nU + 37, 301)
    nodes = random_nodes(np.random.default_rng(per_axis[1]), n, case, 2, np.asarray(case.mdim) - 2)
    check_all(case, nodes, wants=WANTS[:2], offsets=OFFSETS[:2], kernels=(0,))


def test_sorted_path_jrk125():
    """JRK-125 (the CTA sort of the sample loop, SORT = true): the per-lane stores, the sorted path never stages."""
    case = matrix_case(3, JRK, False, 23)
    case.U = product_set(*[(-2.0, -1.0, 0.0, 1.0, 2.0)] * 3)
    assert span_mask(case) == 0
    nodes = random_nodes(np.random.default_rng(24), 301, case, 2, np.asarray(case.mdim) - 2)
    assert nodes.size * case.nU >= 64 * THREADS
    check_all(case, nodes, wants=WANTS[:3], offsets=OFFSETS[:2])


@pytest.mark.parametrize("with_region", [False, True], ids=["map", "region"])
def test_lattice_and_region(with_region):
    """LAT on (lattice ids requested), with and without a search region, every output staged."""
    case = lattice_case(with_region)
    assert span_mask(case) == 7
    nodes = random_nodes(np.random.default_rng(42), 703, case, 2, np.asarray(case.mdim) - 2)
    check_all(case, nodes, wants=[WANT, ("cost", "lattice")], offsets=OFFSETS[:2], kernels=(0,))


def lattice_case(with_region):
    case = matrix_case(3, ACC, with_region, 41)
    case.v_max = 3.5  # maxn = ceil(3.5 / 0.15) = 24: keys, actions and costs staged too
    return case


def forced_leg():
    """Run in a child process with MPLX_FXN_SPAN set: the headline and the lattice + region cases."""
    case, nodes = boundary_case(0.15, seed=31)
    check_all(case, nodes, wants=WANTS, offsets=OFFSETS[:2], kernels=(0,))
    case = lattice_case(True)
    nodes = random_nodes(np.random.default_rng(42), 703, case, 2, np.asarray(case.mdim) - 2)
    check_all(case, nodes, wants=[WANT, ("cost", "lattice")], offsets=OFFSETS[1:2], kernels=(0,))
    print("forced leg ok")


@pytest.mark.parametrize("mask", [0, 1, 3, 7])
def test_forced_span_modes(mask):
    """Every staging mask of the unsorted path (MPLX_FXN_SPAN, read once per process) in a child process."""
    here = Path(__file__).resolve().parent
    env = dict(os.environ, MPLX_FXN_SPAN=str(mask),
               PYTHONPATH=os.pathsep.join([str(here), str(here.parent), os.environ.get("PYTHONPATH", "")]))
    out = subprocess.run([sys.executable, "-s", "-c", "import test_fxn_span_out_gpu as t; t.forced_leg()"], cwd=here,
                         env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "forced leg ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


def test_full_ambiguity_queue():
    """More queued primitives than a queue segment holds: the in-kernel literal loop (verdict 3) decides."""
    case, nodes, site, holed, away = overflow_case(False)
    orc = check_all(case, nodes, wants=[OUTPUTS, ("cost",)], offsets=OFFSETS[1:2], kernels=(0,))
    # the primitives overflow_case queues (test_fx_paths_gpu.py): more than a segment holds
    n, nU = nodes.size, case.nU
    em = emitted_mask(orc).reshape(n, nU)
    ux = case.U[orc["action"].reshape(n, nU), 0]
    queued = em & ~same_mask(orc, nodes, 3).reshape(n, nU) & ((ux == 0.0) | (ux == away[site][:, None]))
    queued &= holed[site][:, None]
    seg = (np.arange(n) // (THREADS // nU)) & 63
    assert (np.bincount(seg, weights=queued.sum(1), minlength=64) > queue_capacity(n * nU)).any()
