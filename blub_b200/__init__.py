"""blub_b200 -- H100-native APIC/FLIP fluid-step core (drop-in for Wumpf/blub's HybridFluid path).

The product is ``libblubcore.so`` (hand-written sm_90a CUDA behind the C ABI of ``include/blub_fluid.h``); this
package is only the ctypes mirror of the reference's ``HybridFluid`` interface used by tests and ``bench.py``.
There is no CPU fallback: importing works anywhere (so that symbols can be checked), but creating a fluid without
the built library or without an H100 raises.
"""
from .fluid import (  # noqa: F401
    DT_120HZ,
    BlubError,
    HybridFluid,
    SolverConfig,
    kernel_launch_count,
    lib,
    lib_path,
    scene_info,
)

__all__ = ["HybridFluid", "SolverConfig", "BlubError", "DT_120HZ", "lib", "lib_path", "scene_info", "kernel_launch_count"]
