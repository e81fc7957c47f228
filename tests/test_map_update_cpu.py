"""Sparse map updates without a GPU: MapUtil::setCells and its change journal, the word rules shared by
the full and the sparse packs (tests/map_update_host.cpp), and the new entry points' refusal to run
without a device."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

HERE = Path(__file__).resolve().parent


def test_journal_and_pack_rules(tmp_path):
    exe = tmp_path / "map_update_host"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-pthread", "-o", str(exe), str(HERE / "map_update_host.cpp")])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    print(out.stdout[-2000:])
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    assert "map_update_host fails 0" in out.stdout


def test_update_entry_points_refuse_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the refusal path is only reachable on a CPU-only host")
    import fixtures
    from motion_primitive_library_b200 import abi
    from motion_primitive_library_b200 import planner as P

    lib = abi.load()
    idx = np.zeros(1, dtype=np.int32)
    val = np.zeros(1, dtype=np.int8)
    assert lib.mplx_update_cells(None, idx.ctypes.data, val.ctypes.data, 1) == abi.MPLX_ERR_ARG
    assert lib.mplx_read_map(None, None, None, None) == abi.MPLX_ERR_ARG
    hl, _ = P._host()
    assert hl.mplh_batch_update_cells(None, idx.ctypes.data, val.ctypes.data, 1) != 0
    assert hl.mplh_batch_map_uploads(None, C.byref(C.c_int64()), C.byref(C.c_int64())) != 0
    c = fixtures.corridor()
    a = P.make_args(2, 0x03, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                    goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0)
    with pytest.raises(RuntimeError, match="no CUDA device|CPU fallback"):
        P.BatchPlanner(a)
