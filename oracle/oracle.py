"""ctypes front-end of the CPU oracle (oracle/blub_oracle.c).

TEST INFRASTRUCTURE ONLY -- see the header of blub_oracle.c.  Imported by tests/,
``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` legs, never by
the product package ``blub_b200``.  PARITY UNPINNED (no runnable reference, no golden vectors).
"""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libbluboracle.so")

# f32 of Duration::from_nanos(1e9 / 120).as_secs_f32() (simulation_controller.rs:33-39, SURVEY B14)
DT_120HZ = float(np.float32(8333333e-9))

SOLID, FLUID, AIR = 0, 1, -1

ARR_POS, ARR_ROWX, ARR_ROWY, ARR_ROWZ = 0, 1, 2, 3
ARR_UX, ARR_UY, ARR_UZ, ARR_MARKER = 4, 5, 6, 7
ARR_P_VEL, ARR_P_DEN, ARR_RESIDUAL, ARR_LL, ARR_VOXEL, ARR_SEARCH, ARR_AUX = 8, 9, 10, 11, 12, 13, 14

STAGES = [
    "p2g", "divergence_compute", "solve_velocity", "binning", "divergence_remove", "extrapolate",
    "transfer_clear", "advect", "set_boundary_marker", "density_gather_error", "solve_density",
    "position_change", "extrapolate2", "correct_particles",
]


def build(force: bool = False) -> str:
    """Compile the oracle with the Makefile next to this file (gcc only)."""
    src = os.path.join(_HERE, "blub_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        # OpenMP: never more threads than CPUs this process may run on, and sleep (not spin) at barriers -- the oracle's
        # loops are short, and a spinning 128-thread team on a CPU-limited box is slower than one thread
        try:
            ncpu = len(os.sched_getaffinity(0))
        except AttributeError:
            ncpu = os.cpu_count() or 1
        os.environ.setdefault("OMP_NUM_THREADS", str(max(1, min(ncpu, 64))))
        os.environ.setdefault("OMP_WAIT_POLICY", "passive")
        build()
        L = C.CDLL(_LIB_PATH)
        L.orc_create.restype = C.c_void_p
        L.orc_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint32]
        L.orc_destroy.argtypes = [C.c_void_p]
        L.orc_add_fluid_cube.restype = C.c_uint32
        L.orc_add_fluid_cube.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int)]
        L.orc_set_particles.argtypes = [C.c_void_p, C.c_uint32] + [C.c_void_p] * 4
        L.orc_set_gravity.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
        L.orc_set_solver_config.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_int, C.c_int]
        L.orc_set_rebin_frequency.argtypes = [C.c_void_p, C.c_uint32]
        L.orc_set_quirks.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        L.orc_set_voxels.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_set_reduce_mode.argtypes = [C.c_void_p, C.c_int]
        L.orc_num_particles.restype = C.c_uint32
        L.orc_num_particles.argtypes = [C.c_void_p]
        L.orc_step_counter.restype = C.c_uint32
        L.orc_step_counter.argtypes = [C.c_void_p]
        L.orc_last_solve.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int)]
        L.orc_last_scalars.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float)]
        L.orc_array.restype = C.c_void_p
        L.orc_array.argtypes = [C.c_void_p, C.c_int]
        L.orc_step.argtypes = [C.c_void_p, C.c_float]
        L.orc_step_stages.argtypes = [C.c_void_p, C.c_float, C.c_int, C.c_int]
        L.orc_solve.argtypes = [C.c_void_p, C.c_int, C.c_float]
        for name in ("orc_stage_p2g",):
            getattr(L, name).argtypes = [C.c_void_p, C.c_float]
        _lib = L
    return _lib


def _f3(v):
    return (C.c_float * 3)(*[float(x) for x in v])


class OracleFluid:
    """Mirror of HybridFluid (src/simulation/hybrid_fluid.rs) on the CPU restatement."""

    PARTICLES_PER_GRID_CELL = 8  # hybrid_fluid.rs:90

    def __init__(self, nx, ny, nz, max_num_particles):
        self.L = lib()
        self.nx, self.ny, self.nz = int(nx), int(ny), int(nz)
        self.n = self.nx * self.ny * self.nz
        self.max_num_particles = int(max_num_particles)
        self.h = C.c_void_p(self.L.orc_create(self.nx, self.ny, self.nz, self.max_num_particles))

    def close(self):
        if self.h:
            self.L.orc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- setup ------------------------------------------------------------------------------
    def add_fluid_cube(self, min_grid, max_grid):
        trunc = C.c_int(0)
        return int(self.L.orc_add_fluid_cube(self.h, _f3(min_grid), _f3(max_grid), C.byref(trunc))), bool(trunc.value)

    def set_gravity_grid(self, g):
        self.L.orc_set_gravity(self.h, _f3(g))

    def set_particles(self, pos4, rowx=None, rowy=None, rowz=None):
        pos4 = np.ascontiguousarray(pos4, dtype=np.float32).reshape(-1, 4)
        rows = [None if r is None else np.ascontiguousarray(r, dtype=np.float32).reshape(-1, 4) for r in (rowx, rowy, rowz)]
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        self.L.orc_set_particles(self.h, pos4.shape[0], ptr(pos4), ptr(rows[0]), ptr(rows[1]), ptr(rows[2]))

    def set_solver_config(self, which, error_tolerance=0.1, max_num_iterations=32, error_check_frequency=4):
        self.L.orc_set_solver_config(self.h, which, error_tolerance, max_num_iterations, error_check_frequency)

    def set_rebin_frequency(self, f):
        self.L.orc_set_rebin_frequency(self.h, int(f))

    def set_quirks(self, precond_mode=0, cap_p2g=0, cap_density=0, binning_mode=0):
        self.L.orc_set_quirks(self.h, precond_mode, cap_p2g, cap_density, binning_mode)

    def set_reduce_mode(self, as_written):
        """B16: True = drop the last first-level partial when N % 16384 != 0, as the reference's host code does."""
        self.L.orc_set_reduce_mode(self.h, 1 if as_written else 0)

    def set_voxels(self, rgba):
        rgba = np.ascontiguousarray(rgba, dtype=np.float32).reshape(self.n, 4)
        self.L.orc_set_voxels(self.h, rgba.ctypes.data_as(C.c_void_p))

    # -- state ------------------------------------------------------------------------------
    @property
    def num_particles(self):
        return int(self.L.orc_num_particles(self.h))

    def _arr(self, which, shape, dtype):
        ptr = self.L.orc_array(self.h, which)
        n = int(np.prod(shape))
        buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr)
        return np.frombuffer(buf, dtype=dtype).reshape(shape)

    def grid(self, which):
        dt = np.int8 if which == ARR_MARKER else (np.uint32 if which == ARR_LL else np.float32)
        return self._arr(which, (self.nz, self.ny, self.nx), dt)

    def voxels(self):
        return self._arr(ARR_VOXEL, (self.nz, self.ny, self.nx, 4), np.float32)

    def particles(self, which=ARR_POS):
        return self._arr(which, (self.max_num_particles, 4), np.float32)[: self.num_particles]

    def last_solve(self, which):
        e, it = C.c_float(0), C.c_int(0)
        self.L.orc_last_solve(self.h, which, C.byref(e), C.byref(it))
        return float(e.value), int(it.value)

    def last_scalars(self, which):
        """(alpha_K, beta_{K-1}, sigma_K) of the last iteration K of the last solve, as float32 values."""
        out = (C.c_float * 3)()
        self.L.orc_last_scalars(self.h, which, out)
        return tuple(np.float32(out[k]) for k in range(3))

    # -- stepping ---------------------------------------------------------------------------
    def step(self, dt=DT_120HZ):
        self.L.orc_step(self.h, dt)

    def step_stages(self, dt, frm, to):
        self.L.orc_step_stages(self.h, dt, frm, to)

    def solve(self, which, dt=DT_120HZ):
        """PCG on the rhs currently in grid(ARR_RESIDUAL) with the markers in grid(ARR_MARKER)."""
        self.L.orc_solve(self.h, which, dt)


# -- scene JSON (src/scene/mod.rs:19-43, 109-144) ---------------------------------------------
def load_scene(path):
    with open(path) as fh:
        return json.load(fh)


def fluid_from_scene(cfg, cls=OracleFluid):
    """Scene::create_fluid_from_config (src/scene/mod.rs:109-144): world -> grid units."""
    fl = cfg["fluid"]
    d = fl["grid_dimension"]
    f32 = np.float32
    scale = f32(fl["grid_to_world_scale"])
    fluid = cls(d["x"], d["y"], d["z"], fl["max_num_particles"])
    for cube in fl["fluid_cubes"]:
        mn = [f32(cube["min"][k]) / scale for k in "xyz"]
        mx = [f32(cube["max"][k]) / scale for k in "xyz"]
        fluid.add_fluid_cube(mn, mx)
    g = cfg["gravity"]
    fluid.set_gravity_grid([f32(g[k]) / scale for k in "xyz"])
    return fluid
