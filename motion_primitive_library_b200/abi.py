"""ctypes binding of libmplx.so (include/mplx.h) — plumbing only.

The product is the C-ABI library; this module loads it and exposes thin, typed wrappers.
It raises loudly when the library (the CUDA extension) is missing: there is no CPU or
PyTorch fallback for the node-expansion path.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import numpy as np

PKG_DIR = Path(__file__).resolve().parent
LIB_PATH = PKG_DIR / "lib" / "libmplx.so"

MPLX_OK, MPLX_ERR_ARG, MPLX_ERR_CUDA, MPLX_ERR_ALLOC = 0, 1, 2, 3
VEL, ACC, JRK, SNP = 0x01, 0x03, 0x07, 0x0F
VELxYAW, ACCxYAW, JRKxYAW, SNPxYAW = 0x11, 0x13, 0x17, 0x1F
LATTICE_MAX = 13

# Waypoint<Dim> payload (include/mplx.h mplx_waypoint; reference include/mpl_basis/waypoint.h:33-38)
WAYPOINT_DTYPE = np.dtype(
    [("pos", "<f8", 3), ("vel", "<f8", 3), ("acc", "<f8", 3), ("jrk", "<f8", 3), ("yaw", "<f8"), ("t", "<f8")]
)
assert WAYPOINT_DTYPE.itemsize == 112

# Every symbol include/mplx.h declares (the CPU test-suite checks the .so exports all of them).
EXPORTED_SYMBOLS = (
    "mplx_create",
    "mplx_destroy",
    "mplx_last_error",
    "mplx_set_map",
    "mplx_set_potential",
    "mplx_set_potential_weights",
    "mplx_set_search_region",
    "mplx_update_potential_map",
    "mplx_set_search_region_path",
    "mplx_set_params",
    "mplx_expand",
    "mplx_expand_device",
    "mplx_expand_packed",
    "mplx_edges_is_free",
    "mplx_edges_cells",
    "mplx_set_kernel",
    "mplx_sync",
    "mplx_launch_count",
    "mplx_enable_stats",
    "mplx_last_stats",
    "mplx_stream",
    "mplx_host_alloc",
    "mplx_host_free",
    "mplx_build_info",
)


class SuccOut(C.Structure):
    """mplx_succ_out"""

    _fields_ = [
        ("count", C.c_void_p),
        ("succ", C.c_void_p),
        ("cost", C.c_void_p),
        ("action", C.c_void_p),
        ("key", C.c_void_p),
        ("lattice", C.c_void_p),
    ]


class PackedOut(C.Structure):
    """mplx_packed_out"""

    _fields_ = [
        ("count", C.c_void_p),
        ("offset", C.c_void_p),
        ("state", C.c_void_p),
        ("cost", C.c_void_p),
        ("action", C.c_void_p),
        ("key", C.c_void_p),
        ("capacity", C.c_int64),
        ("total", C.c_int64),
        ("nstate", C.c_int32),
    ]


PACK_DROP_INF = 1


class MplxError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libmplx error {code}: {msg}")
        self.code = code


_lib = None


def load() -> C.CDLL:
    """Load libmplx.so; fail loudly if it has not been built (python __graft_entry__.py build)."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("MPLX_LIB", LIB_PATH))
    if not path.exists():
        raise ImportError(
            f"{path} not found: the sm_90a CUDA engine is not built. Run "
            f"`python -c 'import __graft_entry__ as g; g.build()'` (or make -C "
            f"motion_primitive_library_b200/csrc). There is no CPU fallback for this path."
        )
    lib = C.CDLL(str(path))
    vp, i32, f64 = C.c_void_p, C.c_int, C.c_double
    lib.mplx_create.argtypes = [i32, i32, C.POINTER(vp)]
    lib.mplx_create.restype = i32
    lib.mplx_destroy.argtypes = [vp]
    lib.mplx_destroy.restype = i32
    lib.mplx_last_error.argtypes = []
    lib.mplx_last_error.restype = C.c_char_p
    lib.mplx_set_map.argtypes = [vp, vp, vp, vp, f64]
    lib.mplx_set_map.restype = i32
    lib.mplx_set_potential.argtypes = [vp, vp, f64, f64]
    lib.mplx_set_potential.restype = i32
    lib.mplx_set_potential_weights.argtypes = [vp, f64, f64]
    lib.mplx_set_potential_weights.restype = i32
    lib.mplx_set_search_region.argtypes = [vp, vp]
    lib.mplx_set_search_region.restype = i32
    lib.mplx_update_potential_map.argtypes = [vp, vp, f64, vp, vp, f64, f64, vp]
    lib.mplx_update_potential_map.restype = i32
    lib.mplx_set_search_region_path.argtypes = [vp, vp, i32, vp, i32, vp]
    lib.mplx_set_search_region_path.restype = i32
    lib.mplx_set_params.argtypes = [vp, i32, f64, f64, f64, f64, f64, f64, f64, vp, i32, i32]
    lib.mplx_set_params.restype = i32
    lib.mplx_expand.argtypes = [vp, vp, i32, C.POINTER(SuccOut)]
    lib.mplx_expand.restype = i32
    lib.mplx_expand_device.argtypes = [vp, vp, i32, C.POINTER(SuccOut), vp]
    lib.mplx_expand_device.restype = i32
    lib.mplx_expand_packed.argtypes = [vp, vp, i32, i32, C.POINTER(PackedOut)]
    lib.mplx_expand_packed.restype = i32
    lib.mplx_edges_is_free.argtypes = [vp, vp, vp, i32, vp, vp]
    lib.mplx_edges_is_free.restype = i32
    lib.mplx_edges_cells.argtypes = [vp, vp, vp, i32, vp, vp, C.c_int64, C.POINTER(C.c_int64), vp, vp]
    lib.mplx_edges_cells.restype = i32
    lib.mplx_set_kernel.argtypes = [vp, i32]
    lib.mplx_set_kernel.restype = i32
    lib.mplx_sync.argtypes = [vp]
    lib.mplx_sync.restype = i32
    lib.mplx_launch_count.argtypes = [vp]
    lib.mplx_launch_count.restype = C.c_int64
    lib.mplx_enable_stats.argtypes = [vp, i32]
    lib.mplx_enable_stats.restype = i32
    lib.mplx_last_stats.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    lib.mplx_last_stats.restype = i32
    lib.mplx_stream.argtypes = [vp]
    lib.mplx_stream.restype = vp
    lib.mplx_host_alloc.argtypes = [C.c_size_t]
    lib.mplx_host_alloc.restype = vp
    lib.mplx_host_free.argtypes = [vp]
    lib.mplx_host_free.restype = None
    lib.mplx_build_info.argtypes = []
    lib.mplx_build_info.restype = C.c_char_p
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != MPLX_OK:
        raise MplxError(rc, load().mplx_last_error().decode())


def ptr(a) -> int | None:
    """Address of a numpy array / torch tensor / None."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()  # torch.Tensor
