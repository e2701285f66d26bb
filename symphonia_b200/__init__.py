"""symphonia_b200 -- H100 (sm_90a) batched audio-synthesis engine behind Symphonia's decoder seam.

The product is `libsymgpu.so` (CUDA kernels + C ABI, see include/symgpu.h).  This package is the
thin host-side harness: a ctypes binding (`_native`), an `Engine` wrapper that moves numpy / torch
buffers through the ABI, and seeded synthetic workload generators used by tests and bench.py.
There is no CPU implementation of the synthesis path here: importing works without a GPU (so the
CPU test tier can check symbols and host logic) but creating an Engine without one raises.
"""
from ._native import NativeLibraryMissing, lib, lib_path  # noqa: F401
from .engine import Engine, SymgpuError  # noqa: F401

__all__ = ["Engine", "SymgpuError", "NativeLibraryMissing", "lib", "lib_path"]
