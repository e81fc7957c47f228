"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol
include/mplx.h declares, and refuses to compute without a CUDA device (no CPU fallback)."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def test_header_symbols_all_exported():
    from motion_primitive_library_b200 import abi

    lib = abi.load()
    header = (ROOT / "include" / "mplx.h").read_text()
    declared = set(re.findall(r"\b(mplx_[a-z_]+)\s*\(", header))
    declared -= {"mplx_ctx"}
    assert declared == set(abi.EXPORTED_SYMBOLS), declared ^ set(abi.EXPORTED_SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), f"libmplx.so does not export {name}"


def test_struct_layouts():
    from motion_primitive_library_b200 import abi

    assert abi.WAYPOINT_DTYPE.itemsize == 112
    assert C.sizeof(abi.SuccOut) == 6 * C.sizeof(C.c_void_p)
    assert b"sm_90a" in abi.load().mplx_build_info()


def test_no_cpu_fallback_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the refusal path is only reachable on a CPU-only host")
    from motion_primitive_library_b200 import MapUtil, abi, env_map

    h = C.c_void_p()
    rc = abi.load().mplx_create(3, 0, C.byref(h))
    assert rc == abi.MPLX_ERR_CUDA
    assert b"no CPU fallback" in abi.load().mplx_last_error()
    mu = MapUtil()
    mu.setMap((0, 0), (4, 4), np.zeros(16, dtype=np.int8), 1.0)
    with pytest.raises(abi.MplxError):
        env_map(mu)


def test_host_planner_entry_points_refuse_without_gpu():
    """libmpl_host.so (C++ host planner with the GPU env): every entry point loads, resolves libmplx and
    fails loudly — never plans on the CPU — when no device is present."""
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present; the refusal path is only reachable on a CPU-only host")
    import fixtures
    from motion_primitive_library_b200 import planner as P

    c = fixtures.corridor()
    a = P.make_args(2, 0x03, c["grid"], c["dim"], c["origin"], c["res"], fixtures.U_2d(), start=dict(pos=c["start"]),
                    goal=dict(pos=c["goal"]), v_max=1.0, a_max=1.0)
    q = np.zeros(2, dtype=P.WAYPOINT_DTYPE)
    for call in (lambda: P.plan(a), lambda: P.lpa_session(a, [("plan",)]), lambda: P.iterative_plan(a, (0.5, 0.5), 2),
                 lambda: P.plan_trajectory(a, 5), lambda: P.plan_batch(a, q, q)):
        with pytest.raises(RuntimeError, match="no CUDA device|CPU fallback"):
            call()


def test_bad_arguments_rejected_before_cuda():
    from motion_primitive_library_b200 import abi

    h = C.c_void_p()
    assert abi.load().mplx_create(4, 0, C.byref(h)) == abi.MPLX_ERR_ARG
    assert abi.load().mplx_create(3, 0, None) == abi.MPLX_ERR_ARG


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under the package or include/ may reference it."""
    pkg = ROOT / "motion_primitive_library_b200"
    offenders = []
    for p in list(pkg.rglob("*")) + list((ROOT / "include").rglob("*")):
        if p.is_file() and p.suffix in {".py", ".cu", ".cuh", ".h", ".cpp", ".hpp"} or p.name == "Makefile":
            if p.is_file() and re.search(r"oracle|liboracle|orc_", p.read_text(errors="ignore")):
                offenders.append(str(p.relative_to(ROOT)))
    assert not offenders, offenders
