"""The per-query round bookkeeping of MultiQueryPlanner::iterativePlan (host/iterative_rounds.hpp), compiled by g++
and driven by scripted round results, against MapPlanner::iterativePlan's loop (map_planner.cpp:413-430) restated
here: the previous cost starts at 0 and is compared with ==, a failed plan returns false, max_num caps the plans."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent


@pytest.fixture(scope="module")
def ir(tmp_path_factory):
    so = tmp_path_factory.mktemp("ir") / "libir.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", str(so),
                           str(HERE / "iterative_rounds_host.cpp")])
    L = C.CDLL(str(so))
    L.ir_run.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.POINTER(C.c_int)] * 3
    L.ir_run.restype = None
    return L


def run(L, rounds, max_num):
    planned = np.array([1 if c is not None else 0 for c in rounds] or [0], np.int32)
    cost = np.array([c if c is not None else 0.0 for c in rounds] or [0.0])
    its, ok, used = C.c_int(), C.c_int(), C.c_int()
    L.ir_run(planned.ctypes.data, cost.ctypes.data, len(rounds), max_num, C.byref(its), C.byref(ok), C.byref(used))
    return its.value, ok.value, used.value


def loop(rounds, max_num):
    """map_planner.cpp:413-430 with round r's plan() giving rounds[r] (None = failed)."""
    prev, cnt = 0.0, 0
    while cnt < max_num:
        cnt += 1
        c = rounds[cnt - 1]
        if c is None:
            return cnt, 0
        if prev == c:
            break
        prev = c
    return cnt, 1


@pytest.mark.parametrize("rounds,max_num,want", [
    ([0.0, 5.0], 3, (1, 1, 1)),                 # a first cost of 0.0 equals the initial previous cost
    ([5.0, 4.0, 4.0, 3.0], 10, (3, 1, 3)),      # equal costs end the loop
    ([5.0, 4.0, None, 3.0], 10, (3, 0, 3)),     # a failure mid-loop returns false
    ([None], 3, (1, 0, 1)),                     # a failure in round 1
    ([5.0, 4.0, 3.0, 2.0, 1.0], 3, (3, 1, 3)),  # the cap
    ([5.0], 1, (1, 1, 1)),                      # max_num 1
    ([5.0], 0, (0, 1, 0)),                      # max_num 0: no plan
    ([5.0, 5.0 + 1e-12, 5.0 + 1e-12], 10, (3, 1, 3)),  # == on doubles, no tolerance
])
def test_scripted_rounds(ir, rounds, max_num, want):
    assert run(ir, rounds, max_num) == want
    its, ok = loop(rounds, max_num) if max_num > 0 else (0, 1)
    assert (its, ok) == want[:2]


def test_random_scripts_follow_the_loop(ir):
    rng = np.random.default_rng(3)
    for _ in range(2000):
        n = int(rng.integers(1, 8))
        rounds = [None if rng.random() < 0.1 else float(rng.choice([0.0, 1.0, 2.0, 3.0])) for _ in range(n)]
        max_num = int(rng.integers(1, n + 1))
        its, ok, used = run(ir, rounds, max_num)
        assert (its, ok) == loop(rounds, max_num) and used == its
