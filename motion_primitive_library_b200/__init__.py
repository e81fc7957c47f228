"""motion_primitive_library_b200 — B200-native node expansion for search-based motion-primitive planning.

The product is libmplx.so (hand-written sm_90a CUDA behind the C ABI of include/mplx.h).
This package holds the host-side mirror of the reference's operator interface for that one
path (benchmark input generators live in scenarios.py at the repository root).
"""
from . import abi  # noqa: F401
from .env import Expansion, MapUtil, env_map  # noqa: F401

__all__ = ["abi", "env_map", "MapUtil", "Expansion"]
