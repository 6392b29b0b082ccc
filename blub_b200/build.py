"""Builds libblubcore.so in-tree with nvcc for sm_90a (no torch, no JIT cache).

    python -m blub_b200.build [--force] [--verbose]
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libblubcore.so")
SOURCES = ["pcg.cu", "fluid_kernels.cu", "transfer_kernels.cu", "flow_kernels.cu", "load_kernels.cu", "body_kernels.cu", "viscosity_kernels.cu", "mesh_body.cpp", "hybrid_fluid.cu", "slab.cu", "solids.cu", "mesh_voxelizer.cu", "scene.cpp", "state_file.cpp",
           "c_api.cpp"]
# the mesh voxelizer shares its arithmetic with a host twin and a NumPy restatement: no FMA contraction, so that all three agree bit for bit
EXTRA_FLAGS = {"mesh_voxelizer.cu": ["-fmad=false"]}
HEADERS = ["common.cuh", "blub_core.hpp", "fluid_kernels.hpp", "voxelize_core.hpp", "xoshiro.hpp", "grid_words.cuh", "grid_reduce.cuh", os.path.join("..", "..", "include", "blub_fluid.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function", "--expt-relaxed-constexpr",
]


def _stale(obj, deps):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    objs, rebuilt = [], False
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        obj = os.path.join(objdir, src + ".o")
        objs.append(obj)
        if force or _stale(obj, [sp] + hdrs):
            cmd = [NVCC] + FLAGS + EXTRA_FLAGS.get(src, []) + (["-Xptxas", "-v"] if verbose else []) + ["-x", "cu", "-c", sp, "-o", obj]
            if verbose:
                print(" ".join(cmd), flush=True)
            subprocess.check_call(cmd)
            rebuilt = True
    if rebuilt or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart", "-lz"]  # zlib: CRC-32 of the state file
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    # headless runner over the C ABI only (SURVEY section 8 f2): a plain C++ program linked against libblubcore.so
    runner, rsrc = os.path.join(HERE, "blub_run"), os.path.join(CSRC, "blub_run.cpp")
    if force or _stale(runner, [rsrc, LIB, os.path.join(HERE, "..", "include", "blub_fluid.h")]):
        cmd = [NVCC, "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets", "-o", runner, rsrc, "-L" + HERE, "-lblubcore", "-Xlinker", "-rpath,$ORIGIN"]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
