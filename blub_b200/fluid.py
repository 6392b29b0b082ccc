"""ctypes mirror of the reference's ``HybridFluid`` (src/simulation/hybrid_fluid.rs) over libblubcore.so.

Method names, argument meaning and defaults follow the Rust interface so that parity tests read like the reference's
call sites (src/scene/mod.rs:109-144,166-214).  All compute happens in the CUDA library; nothing here falls back to
NumPy or to the oracle.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

# Duration::from_nanos(1e9 / 120).as_secs_f32() (simulation_controller.rs:33-39)
DT_120HZ = float(np.float32(8333333e-9))

# the 14 stages of one step, in the order of HybridFluid::step (hybrid_fluid.rs:770-977); indices for step_stages / step_timed
STAGES = [
    "p2g", "divergence_compute", "solve_velocity", "binning", "divergence_remove", "extrapolate",
    "transfer_clear", "advect", "set_boundary_marker", "density_gather_error", "solve_density",
    "position_change", "extrapolate2", "correct_particles",
]
TAP_POS, TAP_VX, TAP_VY, TAP_VZ, TAP_UX, TAP_UY, TAP_UZ, TAP_MARKER, TAP_P_VEL, TAP_P_DEN, TAP_RESIDUAL, TAP_SOLID_VOXELS = range(12)

BLUB_OK = 0
BLUB_WARN_TRUNCATED = 100
TAG_CENSUS_FRAC_BITS = 16  # BLUB_TAG_CENSUS_FRAC_BITS: census sums are sums of rint(value * 2^16)
TAG_CENSUS_MAX = 256       # tags per census
LOAD_PROBES_MAX = 16            # BLUB_LOAD_PROBES_MAX
LOAD_HISTORY_LENGTH = 1024      # BLUB_LOAD_HISTORY_LENGTH: records per probe in the device ring
LOAD_FORCE_FRAC_BITS = 16       # BLUB_LOAD_FORCE_FRAC_BITS: force sums are sums of rint(q * 2^16)
LOAD_TORQUE_FRAC_BITS = 8       # BLUB_LOAD_TORQUE_FRAC_BITS: torque sums are sums of rint(r_b * q * 2^8)
BODIES_MAX = 16                 # BLUB_BODIES_MAX
BODY_HISTORY_LENGTH = 1024      # BLUB_BODY_HISTORY_LENGTH: records per body in the device ring


class BlubError(RuntimeError):
    pass


class SolverConfig(C.Structure):
    """pressure_solver.rs:57-62"""

    _fields_ = [("error_tolerance", C.c_float), ("max_num_iterations", C.c_int32), ("error_check_frequency", C.c_int32)]


class SolverSample(C.Structure):
    _fields_ = [("error", C.c_float), ("iteration_count", C.c_int32)]


class Quirks(C.Structure):
    _fields_ = [("precond_mode", C.c_int32), ("reserved", C.c_int32 * 7)]


class FluidView(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "particles_position_ll", "particles_velocity_x", "particles_velocity_y", "particles_velocity_z",
        "grid_velocity_x", "grid_velocity_y", "grid_velocity_z", "marker", "pressure_from_velocity", "pressure_from_density")]


class RigidObject(C.Structure):
    """BlubRigidObject: StaticObjectConfig + RigidAnimation (src/scene/models.rs:11-46) for an analytic box / sphere."""

    _fields_ = [("world_position", C.c_float * 3), ("scale", C.c_float), ("rotation_angles_deg", C.c_float * 3), ("shape", C.c_int32),
                ("half_extent", C.c_float * 3), ("has_translation", C.c_int32), ("translation_target", C.c_float * 3),
                ("translation_curve", C.c_int32), ("translation_duration", C.c_float), ("has_rotation", C.c_int32),
                ("rotation_axis", C.c_float * 3), ("rotation_deg_per_sec", C.c_float)]

    @classmethod
    def from_dict(cls, obj):
        o = cls()
        o.world_position[:] = [float(v) for v in obj["world_position"]]
        o.scale = float(obj.get("scale", 1.0))
        o.rotation_angles_deg[:] = [float(v) for v in obj.get("rotation_angles", (0, 0, 0))]
        o.shape = {"box": 0, "sphere": 1, "mesh": 2}[obj.get("shape", "box")]
        o.half_extent[:] = [float(v) for v in obj.get("half_extent", (0, 0, 0))]
        tr, rot = obj.get("translation"), obj.get("rotation")
        if tr:
            o.has_translation = 1
            o.translation_target[:] = [float(v) for v in tr["target"]]
            o.translation_curve = 1 if tr.get("curve", "Linear") == "SmoothStep" else 0
            o.translation_duration = float(tr["duration"])
        if rot:
            o.has_rotation = 1
            o.rotation_axis[:] = [float(v) for v in rot["axis"]]
            o.rotation_deg_per_sec = float(rot["deg_per_sec"])
        return o


class RigidState(C.Structure):
    _fields_ = [("centre_voxel", C.c_float * 3), ("velocity_voxel", C.c_float * 3), ("axis_scaled", C.c_float * 3), ("rotation", C.c_float * 9)]


class SceneInfo(C.Structure):
    _fields_ = [("grid_dimension", C.c_uint32 * 3), ("max_num_particles", C.c_uint32), ("grid_to_world_scale", C.c_float),
                ("world_position", C.c_float * 3), ("gravity", C.c_float * 3), ("num_fluid_cubes", C.c_uint32),
                ("num_static_objects", C.c_uint32)]


class StateInfo(C.Structure):
    _fields_ = [("grid_dimension", C.c_uint32 * 3), ("max_num_particles", C.c_uint32), ("num_particles", C.c_uint32), ("step_count", C.c_uint32),
                ("format_version", C.c_uint32)]


class FluidSource(C.Structure):
    """BlubFluidSource: a source box in grid cells and its velocity in cells/s."""

    _fields_ = [("min_grid", C.c_float * 3), ("max_grid", C.c_float * 3), ("velocity_grid", C.c_float * 3)]


class FluidDrain(C.Structure):
    _fields_ = [("min_grid", C.c_float * 3), ("max_grid", C.c_float * 3)]


class TagCensus(C.Structure):
    """BlubTagCensus: what the particles of one tag add up to (sums in 2^16 fixed point)."""

    _fields_ = [("count", C.c_uint64), ("position_sum_fx", C.c_int64 * 3), ("velocity_sum_fx", C.c_int64 * 3), ("cell_min", C.c_int32 * 3),
                ("cell_max", C.c_int32 * 3)]


class Viscosity(C.Structure):
    """BlubViscosity: kinematic viscosity in cells^2/s, the solve's absolute tolerance (cells/s) and iteration cap."""

    _fields_ = [("kinematic_viscosity", C.c_float), ("error_tolerance", C.c_float), ("max_num_iterations", C.c_int32), ("reserved", C.c_uint32)]


class LoadProbe(C.Structure):
    """BlubLoadProbe: a box of cells and a pivot, in grid cells."""

    _fields_ = [("min_grid", C.c_float * 3), ("max_grid", C.c_float * 3), ("pivot_grid", C.c_float * 3)]


class SolidLoad(C.Structure):
    """BlubSolidLoad: one step's pressure force (2^16 fixed point) and torque (2^8) on the solids of a probe box."""

    _fields_ = [("step", C.c_uint32), ("wetted_faces", C.c_uint32), ("force_fx", C.c_int64 * 3), ("torque_fx", C.c_int64 * 3)]


class Body(C.Structure):
    """BlubBody: a floating box (shape 0, half extents) or sphere (shape 1, radius half_extent[0]) in grid cells, cells/s and rad/s."""

    _fields_ = [("shape", C.c_int32), ("half_extent", C.c_float * 3), ("relative_density", C.c_float), ("centre", C.c_float * 3),
                ("rotation", C.c_float * 4), ("velocity", C.c_float * 3), ("angular_velocity", C.c_float * 3)]

    @classmethod
    def from_dict(cls, d):
        b = cls()
        shape = d.get("shape", "box")
        if isinstance(shape, str) and shape not in ("box", "sphere", "mesh"):
            raise BlubError(f"body shape {shape!r}: must be \"box\", \"sphere\" or \"mesh\"")
        b.shape = {"box": 0, "sphere": 1, "mesh": 2}[shape] if isinstance(shape, str) else int(shape)
        ext = d["half_extent"]
        b.half_extent[:] = [float(ext)] * 3 if np.ndim(ext) == 0 else [float(v) for v in ext]
        b.relative_density = float(d["relative_density"])
        b.centre[:] = [float(v) for v in d["centre"]]
        b.rotation[:] = [float(v) for v in d.get("rotation", (1.0, 0.0, 0.0, 0.0))]
        b.velocity[:] = [float(v) for v in d.get("velocity", (0.0, 0.0, 0.0))]
        b.angular_velocity[:] = [float(v) for v in d.get("angular_velocity", (0.0, 0.0, 0.0))]
        return b

    def to_dict(self):
        return {"shape": {1: "sphere", 2: "mesh"}.get(self.shape, "box"), "half_extent": tuple(self.half_extent), "relative_density": self.relative_density,
                "centre": tuple(self.centre), "rotation": tuple(self.rotation), "velocity": tuple(self.velocity),
                "angular_velocity": tuple(self.angular_velocity)}


class MeshBodyProperties(C.Structure):
    """BlubMeshBodyProperties: a mesh body's volume, centre of mass, inertia, principal frame and body-frame bounds (DESIGN.md §8)."""

    _fields_ = [("volume", C.c_double), ("centroid", C.c_double * 3), ("inertia", C.c_double * 9), ("principal_moments", C.c_double * 3),
                ("principal_rotation", C.c_double * 4), ("bounds_lo", C.c_float * 3), ("bounds_hi", C.c_float * 3), ("mass", C.c_float),
                ("moments", C.c_float * 3), ("scale", C.c_float), ("num_vertices", C.c_uint32), ("num_triangles", C.c_uint32)]

    def to_dict(self):
        out = {name: getattr(self, name) for name in ("volume", "mass", "scale", "num_vertices", "num_triangles")}
        for name in ("centroid", "principal_moments", "principal_rotation", "bounds_lo", "bounds_hi", "moments"):
            out[name] = tuple(getattr(self, name))
        out["inertia"] = np.array(list(self.inertia)).reshape(3, 3)
        return out


class MeshBodyShape(C.Structure):
    _fields_ = [("mesh", C.c_void_p), ("scale", C.c_float)]


def quat_matrix(q):
    """The float64 rotation matrix of the quaternion q = (w, x, y, z)."""
    w, x, y, z = [float(v) for v in q]
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def mesh_body_properties(positions, triangles, scale):
    """blub_mesh_body_properties (host only): checks a closed mesh and returns its mass properties and principal frame as a dict (mass and
    moments for relative density 1).  Raises BlubError on a mesh a mesh body cannot take."""
    pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
    idx = np.ascontiguousarray(triangles, dtype=np.uint32).reshape(-1)
    p = MeshBodyProperties()
    _check(lib().blub_mesh_body_properties(pos.ctypes.data_as(C.c_void_p), pos.shape[0], idx.ctypes.data_as(C.c_void_p), idx.shape[0], float(scale),
                                           C.byref(p)))
    return p.to_dict()


def mesh_body_vertices(positions, triangles, scale):
    """blub_mesh_body_vertices (host only): the float32 body-frame vertices [n, 3] a mesh body of this mesh and scale stores."""
    pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
    idx = np.ascontiguousarray(triangles, dtype=np.uint32).reshape(-1)
    out = np.zeros_like(pos)
    _check(lib().blub_mesh_body_vertices(pos.ctypes.data_as(C.c_void_p), pos.shape[0], idx.ctypes.data_as(C.c_void_p), idx.shape[0], float(scale),
                                         out.ctypes.data_as(C.c_void_p)))
    return out


class BodyRecord(C.Structure):
    """BlubBodyRecord: one step's load on a body (BlubSolidLoad's fixed point) and its pose after the step."""

    _fields_ = [("step", C.c_uint32), ("wetted_faces", C.c_uint32), ("force_fx", C.c_int64 * 3), ("torque_fx", C.c_int64 * 3),
                ("centre", C.c_float * 3), ("rotation", C.c_float * 4), ("velocity", C.c_float * 3), ("angular_velocity", C.c_float * 3),
                ("reserved", C.c_uint32)]


def lib_path() -> str:
    return os.path.join(_HERE, "libblubcore.so")


_lib = None


def lib():
    """Load libblubcore.so; fails loudly when it has not been built (``python -m blub_b200.build``)."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise BlubError(f"{path} is missing: build it with `python -m blub_b200.build` (there is no CPU fallback)")
    L = C.CDLL(path)
    vp, u32, f3 = C.c_void_p, C.c_uint32, C.POINTER(C.c_float)
    sig = {
        "blub_fluid_create": (C.c_int, [C.POINTER(vp), u32, u32, u32, u32, C.c_int, vp]),
        "blub_fluid_destroy": (None, [vp]),
        "blub_fluid_create_slab": (C.c_int, [C.POINTER(vp), u32, u32, u32, u32, C.c_int, vp, C.c_int, C.c_int]),
        "blub_fluid_slab_window": (C.c_int, [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]),
        "blub_fluid_attach_slab_peers": (C.c_int, [vp, C.POINTER(vp), C.c_int]),
        "blub_fluid_slab_error": (C.c_int, [vp]),
        "blub_solid_voxelize": (C.c_int, [vp, C.POINTER(u32), C.POINTER(RigidObject), C.c_float, f3, C.c_double, C.c_double, C.c_int, vp,
                                          C.POINTER(RigidState)]),
        "blub_simulation_delta_ns": (C.c_uint64, [C.c_uint64]),
        "blub_duration_as_secs_f32": (C.c_float, [C.c_uint64]),
        "blub_timer_steps_in_frame": (u32, [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.c_uint64, C.c_uint64]),
        "blub_fluid_stream": (vp, [vp]),
        "blub_device_malloc": (C.c_int, [C.POINTER(vp), C.c_size_t, C.c_int]),
        "blub_device_free": (C.c_int, [vp]),
        "blub_mesh_create": (C.c_int, [C.POINTER(vp), vp, u32, vp, u32, C.c_int]),
        "blub_mesh_load_obj": (C.c_int, [C.POINTER(vp), C.c_char_p, C.c_int]),
        "blub_mesh_destroy": (None, [vp]),
        "blub_mesh_info": (C.c_int, [vp, C.POINTER(u32), C.POINTER(u32)]),
        "blub_obj_read": (C.c_int, [C.c_char_p, vp, u32, vp, u32, C.POINTER(u32)]),
        "blub_solid_voxelize_mesh": (C.c_int, [vp, C.POINTER(u32), vp, C.POINTER(RigidObject), C.c_float, f3, C.c_double, C.c_double, C.c_int, vp,
                                               C.POINTER(RigidState)]),
        "blub_scene_static_object": (C.c_int, [C.c_char_p, u32, C.POINTER(RigidObject), C.c_char_p, C.c_size_t]),
        "blub_ipc_export": (C.c_int, [vp, C.c_char_p]),
        "blub_ipc_open": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(vp)]),
        "blub_ipc_close": (C.c_int, [vp]),
        "blub_enable_peer_access": (C.c_int, [C.c_int, C.c_int]),
        "blub_fluid_add_cube": (C.c_int, [vp, f3, f3]),
        "blub_fluid_add_cube_tagged": (C.c_int, [vp, f3, f3, u32]),
        "blub_fluid_set_gravity_grid": (C.c_int, [vp, f3]),
        "blub_fluid_num_particles": (u32, [vp]),
        "blub_fluid_grid_dimension": (None, [vp, C.POINTER(u32)]),
        "blub_fluid_solver_config": (C.POINTER(SolverConfig), [vp, C.c_int]),
        "blub_fluid_rebinning_frequency": (C.POINTER(u32), [vp]),
        "blub_fluid_solver_stats": (C.c_size_t, [vp, C.c_int, C.POINTER(SolverSample), C.c_size_t]),
        "blub_fluid_update_statistics": (None, [vp]),
        "blub_fluid_set_solid_voxels": (C.c_int, [vp, vp]),
        "blub_fluid_step": (C.c_int, [vp, C.c_double]),
        "blub_fluid_view": (C.c_int, [vp, C.POINTER(FluidView)]),
        "blub_fluid_set_quirks": (C.c_int, [vp, C.POINTER(Quirks)]),
        "blub_fluid_synchronize": (C.c_int, [vp]),
        "blub_fluid_save_state": (C.c_int, [vp, C.c_char_p]),
        "blub_fluid_load_state": (C.c_int, [C.POINTER(vp), C.c_char_p, C.c_int, vp]),
        "blub_state_info": (C.c_int, [C.c_char_p, C.POINTER(StateInfo)]),
        "blub_fluid_step_count": (u32, [vp]),
        "blub_fluid_set_flow": (C.c_int, [vp, C.POINTER(FluidSource), u32, C.POINTER(FluidDrain), u32]),
        "blub_fluid_flow_counters": (C.c_int, [vp, C.POINTER(C.c_uint64)]),
        "blub_fluid_has_flow": (C.c_int, [vp]),
        "blub_fluid_set_flow_tagged": (C.c_int, [vp, C.POINTER(FluidSource), C.POINTER(u32), u32, C.POINTER(FluidDrain), u32]),
        "blub_fluid_paint_tags": (C.c_int, [vp, f3, f3, u32]),
        "blub_fluid_tag_census": (C.c_int, [vp, u32, u32, C.POINTER(TagCensus)]),
        "blub_fluid_set_load_probes": (C.c_int, [vp, C.POINTER(LoadProbe), u32]),
        "blub_fluid_load_history": (C.c_int, [vp, u32, C.POINTER(SolidLoad), u32, C.POINTER(u32)]),
        "blub_load_probe_cells": (C.c_int, [C.POINTER(u32), C.POINTER(LoadProbe), C.POINTER(u32), C.POINTER(u32)]),
        "blub_scene_load_probes": (C.c_int, [C.c_char_p, C.POINTER(LoadProbe), u32, C.POINTER(u32)]),
        "blub_fluid_set_viscosity": (C.c_int, [vp, C.POINTER(Viscosity)]),
        "blub_fluid_viscosity": (C.c_int, [vp, C.POINTER(Viscosity)]),
        "blub_fluid_last_viscosity_solve": (C.c_int, [vp, C.POINTER(C.c_int32), C.POINTER(C.c_float)]),
        "blub_fluid_viscosity_only": (C.c_int, [vp, C.c_double]),
        "blub_scene_viscosity": (C.c_int, [C.c_char_p, C.POINTER(C.c_float)]),
        "blub_fluid_set_bodies": (C.c_int, [vp, C.POINTER(Body), u32]),
        "blub_fluid_body_history": (C.c_int, [vp, u32, C.POINTER(BodyRecord), u32, C.POINTER(u32)]),
        "blub_fluid_bodies": (C.c_int, [vp, C.POINTER(Body), u32, C.POINTER(u32)]),
        "blub_scene_bodies": (C.c_int, [C.c_char_p, C.POINTER(Body), u32, C.POINTER(u32)]),
        "blub_mesh_body_properties": (C.c_int, [vp, u32, vp, u32, C.c_float, C.POINTER(MeshBodyProperties)]),
        "blub_mesh_body_vertices": (C.c_int, [vp, u32, vp, u32, C.c_float, vp]),
        "blub_fluid_set_bodies_meshes":(C.c_int, [vp, C.POINTER(Body), C.POINTER(MeshBodyShape), u32]),
        "blub_fluid_body_mass_properties": (C.c_int, [vp, u32, C.POINTER(MeshBodyProperties)]),
        "blub_scene_body_model": (C.c_int, [C.c_char_p, u32, C.c_char_p, C.c_size_t, C.POINTER(C.c_float)]),
        "blub_last_error": (C.c_char_p, []),
        "blub_version": (C.c_char_p, []),
        "blub_scene_load": (C.c_int, [C.POINTER(vp), C.c_char_p, C.c_int, vp]),
        "blub_scene_info": (C.c_int, [C.c_char_p, C.POINTER(SceneInfo)]),
        "blub_fluid_download": (C.c_int, [vp, C.c_int, vp, C.c_size_t]),
        "blub_fluid_upload": (C.c_int, [vp, C.c_int, vp, C.c_size_t]),
        "blub_fluid_set_particles": (C.c_int, [vp, u32, vp, vp, vp, vp]),
        "blub_fluid_step_stages": (C.c_int, [vp, C.c_double, C.c_int, C.c_int]),
        "blub_fluid_solve_only": (C.c_int, [vp, C.c_int, C.c_double]),
        "blub_fluid_last_solve": (C.c_int, [vp, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int32)]),
        "blub_fluid_solver_work": (C.c_int, [vp, C.POINTER(u32)]),
        "blub_fluid_last_solve_scalars": (C.c_int, [vp, C.c_int, C.POINTER(C.c_float)]),
        "blub_fluid_time_solve": (C.c_int, [vp, C.c_int, C.c_double, C.c_int, C.POINTER(C.c_float)]),
        "blub_fluid_time_steps": (C.c_int, [vp, C.c_double, C.c_int, C.POINTER(C.c_float)]),
        "blub_fluid_step_timed": (C.c_int, [vp, C.c_double, C.POINTER(C.c_float)]),
        "blub_fluid_set_graph_replay": (C.c_int, [vp, C.c_int]),
        "blub_fluid_set_solver_path": (C.c_int, [vp, C.c_int]),
        "blub_fluid_set_transfer_path": (C.c_int, [vp, C.c_int]),
        "blub_kernel_launch_count": (C.c_uint64, [C.c_int]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    _lib = L
    return L


def _check(rc, allow=(BLUB_OK,)):
    if rc not in allow:
        raise BlubError(f"libblubcore error {rc}: {lib().blub_last_error().decode()}")
    return rc


def _f3(v):
    return (C.c_float * 3)(*[float(x) for x in v])


def ipc_open(handle: bytes, device: int) -> int:
    out = C.c_void_p()
    _check(lib().blub_ipc_open(handle, device, C.byref(out)))
    return int(out.value)


def enable_peer_access(device: int, peer: int):
    _check(lib().blub_enable_peer_access(device, peer))


def solid_voxelize(rgba16f_device_ptr, dims, obj, scale, fluid_world_position, t, dt, clear_first=True, cuda_stream=None):
    """Write one analytic rigid solid (dict, see RigidObject.from_dict) into an RGBA16F device volume; returns its RigidState."""
    d = (C.c_uint32 * 3)(*[int(v) for v in dims])
    st = RigidState()
    _check(lib().blub_solid_voxelize(rgba16f_device_ptr, d, C.byref(RigidObject.from_dict(obj)), float(scale), _f3(fluid_world_position), float(t),
                                     float(dt), 1 if clear_first else 0, cuda_stream, C.byref(st)))
    return st


def obj_read(path):
    """Positions [nv, 3] float32 and triangles [nt, 3] uint32 of a Wavefront OBJ, read by the library's host-side loader."""
    import numpy as np
    counts = (C.c_uint32 * 2)()
    _check(lib().blub_obj_read(os.fsencode(path), None, 0, None, 0, counts))
    pos = np.zeros((counts[0], 3), dtype=np.float32)
    idx = np.zeros(counts[1], dtype=np.uint32)
    _check(lib().blub_obj_read(os.fsencode(path), pos.ctypes.data_as(C.c_void_p), counts[0], idx.ctypes.data_as(C.c_void_p), counts[1], counts))
    return pos, idx.reshape(-1, 3)


class Mesh:
    """Device-resident triangle mesh for the hull voxelizer (MeshVertices / MeshIndices of the reference's voxelization pass)."""

    def __init__(self, positions=None, triangles=None, obj_path=None, device=0):
        import numpy as np
        self.h = C.c_void_p()
        if obj_path is not None:
            _check(lib().blub_mesh_load_obj(C.byref(self.h), os.fsencode(obj_path), device))
        else:
            pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
            idx = np.ascontiguousarray(triangles, dtype=np.uint32).reshape(-1)
            _check(lib().blub_mesh_create(C.byref(self.h), pos.ctypes.data_as(C.c_void_p), pos.shape[0], idx.ctypes.data_as(C.c_void_p), idx.shape[0], device))

    def info(self):
        nv, nt = C.c_uint32(), C.c_uint32()
        _check(lib().blub_mesh_info(self.h, C.byref(nv), C.byref(nt)))
        return int(nv.value), int(nt.value)

    def voxelize(self, rgba16f_device_ptr, dims, placement, scale, fluid_world_position, t, dt, clear_first=True, cuda_stream=None):
        """One draw of the reference's voxelization pass for this mesh (placement: dict as for RigidObject.from_dict, shape ignored)."""
        d = (C.c_uint32 * 3)(*[int(v) for v in dims])
        st = RigidState()
        obj = placement if isinstance(placement, RigidObject) else RigidObject.from_dict(dict(placement, shape="mesh"))
        _check(lib().blub_solid_voxelize_mesh(rgba16f_device_ptr, d, self.h, C.byref(obj), float(scale), _f3(fluid_world_position), float(t), float(dt),
                                              1 if clear_first else 0, cuda_stream, C.byref(st)))
        return st

    def close(self):
        if self.h:
            lib().blub_mesh_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def scene_static_object(path, index):
    """(model path, RigidObject placement) of static_objects[index] of a scene file."""
    obj = RigidObject()
    buf = C.create_string_buffer(1024)
    _check(lib().blub_scene_static_object(os.fsencode(path), index, C.byref(obj), buf, len(buf)))
    return buf.value.decode(), obj


def kernel_launch_count(reset=False) -> int:
    return int(lib().blub_kernel_launch_count(1 if reset else 0))


def scene_info(path):
    info = SceneInfo()
    _check(lib().blub_scene_info(os.fsencode(path), C.byref(info)))
    return info


def _load_probes(probes):
    """[(min, max[, pivot])] in grid cells -> a BlubLoadProbe array; the pivot defaults to the box centre (min + max) / 2 in float32."""
    arr = (LoadProbe * max(len(probes), 1))()
    for k, (mn, mx, *pivot) in enumerate(probes):
        mn, mx = np.asarray(mn, dtype=np.float32), np.asarray(mx, dtype=np.float32)
        pv = np.asarray(pivot[0], dtype=np.float32) if pivot and pivot[0] is not None else (mn + mx) * np.float32(0.5)
        arr[k].min_grid[:], arr[k].max_grid[:], arr[k].pivot_grid[:] = [float(v) for v in mn], [float(v) for v in mx], [float(v) for v in pv]
    return arr


def load_probe_cells(dims, probe):
    """The cells [lo, hi) a load probe (min, max[, pivot]) holds on a grid of `dims` cells (host only)."""
    lo, hi = (C.c_uint32 * 3)(), (C.c_uint32 * 3)()
    _check(lib().blub_load_probe_cells((C.c_uint32 * 3)(*[int(d) for d in dims]), _load_probes([probe]), lo, hi))
    return tuple(lo), tuple(hi)


def scene_load_probes(path):
    """The scene's fluid.load_probes in grid cells: [(min, max, pivot)] (host only)."""
    count = C.c_uint32(0)
    arr = (LoadProbe * LOAD_PROBES_MAX)()
    _check(lib().blub_scene_load_probes(os.fsencode(path), arr, LOAD_PROBES_MAX, C.byref(count)))
    return [(tuple(p.min_grid), tuple(p.max_grid), tuple(p.pivot_grid)) for p in arr[:count.value]]


def scene_viscosity(path):
    """The scene's fluid.viscosity (m^2/s) in cells^2/s: value / grid_to_world_scale^2, 0.0 without the key (host only)."""
    out = C.c_float(0)
    _check(lib().blub_scene_viscosity(os.fsencode(path), C.byref(out)))
    return float(out.value)


def scene_bodies(path):
    """The scene's fluid.bodies in grid cells, cells/s and rad/s, as dicts (see Body.to_dict; host only)."""
    count = C.c_uint32(0)
    arr = (Body * BODIES_MAX)()
    _check(lib().blub_scene_bodies(os.fsencode(path), arr, BODIES_MAX, C.byref(count)))
    return [b.to_dict() for b in arr[:min(count.value, BODIES_MAX)]]


def scene_body_model(path, body):
    """(resolved OBJ path, scale in cells per model unit) of the scene's mesh body `body` (host only)."""
    buf = C.create_string_buffer(4096)
    scale = C.c_float(0.0)
    _check(lib().blub_scene_body_model(os.fsencode(path), int(body), buf, len(buf), C.byref(scale)))
    return buf.value.decode(), scale.value


def state_info(path):
    """Validates a state file written by HybridFluid.save_state (host only) and returns its StateInfo."""
    info = StateInfo()
    _check(lib().blub_state_info(os.fsencode(path), C.byref(info)))
    return info


class HybridFluid:
    """HybridFluid::new (hybrid_fluid.rs:92-100)."""

    PARTICLES_PER_GRID_CELL = 8  # hybrid_fluid.rs:90

    def __init__(self, nx, ny, nz, max_num_particles, device=0, cuda_stream=None, _handle=None):
        self.L = lib()
        self.device = device
        if _handle is None:
            h = C.c_void_p()
            _check(self.L.blub_fluid_create(C.byref(h), nx, ny, nz, max_num_particles, device, cuda_stream))
            self.h = h
        else:
            self.h = _handle
        d = (C.c_uint32 * 3)()
        self.L.blub_fluid_grid_dimension(self.h, d)
        self.nx, self.ny, self.nz = int(d[0]), int(d[1]), int(d[2])
        self.n = self.nx * self.ny * self.nz

    @classmethod
    def create_slab(cls, nx, ny, nz_owned, max_num_particles, rank, world, device=0, cuda_stream=None):
        """Rank `rank` of a z-slab decomposition (4 ghost planes on both sides of the nz_owned owned planes)."""
        L = lib()
        h = C.c_void_p()
        _check(L.blub_fluid_create_slab(C.byref(h), nx, ny, nz_owned, max_num_particles, device, cuda_stream, rank, world))
        return cls(0, 0, 0, 0, _handle=h)

    def slab_window(self):
        w, n = C.c_void_p(), C.c_size_t()
        _check(self.L.blub_fluid_slab_window(self.h, C.byref(w), C.byref(n)))
        return int(w.value), int(n.value)

    def attach_slab_peers(self, windows):
        arr = (C.c_void_p * len(windows))(*windows)
        _check(self.L.blub_fluid_attach_slab_peers(self.h, arr, len(windows)))

    def slab_error(self):
        return int(self.L.blub_fluid_slab_error(self.h))

    def ipc_export_window(self):
        buf = C.create_string_buffer(64)
        _check(self.L.blub_ipc_export(self.slab_window()[0], buf))
        return bytes(buf.raw)

    @classmethod
    def from_scene(cls, path, device=0, cuda_stream=None):
        """Scene::new + create_fluid_from_config (src/scene/mod.rs:56-144) on an unchanged scene JSON."""
        L = lib()
        h = C.c_void_p()
        _check(L.blub_scene_load(C.byref(h), os.fsencode(path), device, cuda_stream))
        return cls(0, 0, 0, 0, device=device, _handle=h)

    @classmethod
    def from_state(cls, path, device=0, cuda_stream=None):
        """A fluid restored from a file of save_state: its next step is bit for bit the one the saved fluid would have taken.
        The solid-voxel volume is not part of the state; attach it again with set_solid_voxels."""
        L = lib()
        h = C.c_void_p()
        _check(L.blub_fluid_load_state(C.byref(h), os.fsencode(path), device, cuda_stream))
        return cls(0, 0, 0, 0, device=device, _handle=h)

    def save_state(self, path):
        """Waits for the enqueued steps, then writes everything a later step depends on to `path` (atomically)."""
        _check(self.L.blub_fluid_save_state(self.h, os.fsencode(path)))

    @property
    def step_count(self):
        return int(self.L.blub_fluid_step_count(self.h))

    def close(self):
        if getattr(self, "h", None):
            self.L.blub_fluid_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- reference surface --------------------------------------------------------------------
    def add_fluid_cube(self, min_grid, max_grid, tag=0):
        """hybrid_fluid.rs:620-678; every new particle carries the particle tag `tag` (uint32).  True when truncated to max_num_particles."""
        rc = _check(self.L.blub_fluid_add_cube_tagged(self.h, _f3(min_grid), _f3(max_grid), int(tag)), allow=(BLUB_OK, BLUB_WARN_TRUNCATED))
        return rc == BLUB_WARN_TRUNCATED

    def set_gravity_grid(self, g):
        _check(self.L.blub_fluid_set_gravity_grid(self.h, _f3(g)))

    @property
    def num_particles(self):
        return int(self.L.blub_fluid_num_particles(self.h))

    def grid_dimension(self):
        return self.nx, self.ny, self.nz

    def pressure_solver_config_velocity(self):
        return self.L.blub_fluid_solver_config(self.h, 0).contents

    def pressure_solver_config_density(self):
        return self.L.blub_fluid_solver_config(self.h, 1).contents

    def set_solver_config(self, which, error_tolerance=0.1, max_num_iterations=32, error_check_frequency=4):
        c = self.L.blub_fluid_solver_config(self.h, which).contents
        c.error_tolerance, c.max_num_iterations, c.error_check_frequency = error_tolerance, max_num_iterations, error_check_frequency

    def set_rebin_frequency(self, f):
        self.L.blub_fluid_rebinning_frequency(self.h)[0] = int(f)

    def pressure_solver_stats(self, which):
        buf = (SolverSample * 100)()
        n = self.L.blub_fluid_solver_stats(self.h, which, buf, 100)
        return [(buf[k].error, buf[k].iteration_count) for k in range(n)]

    def update_statistics(self):
        self.L.blub_fluid_update_statistics(self.h)

    def set_solid_voxels(self, device_ptr):
        _check(self.L.blub_fluid_set_solid_voxels(self.h, device_ptr))

    def step(self, dt=DT_120HZ):
        _check(self.L.blub_fluid_step(self.h, dt))

    def view(self):
        v = FluidView()
        _check(self.L.blub_fluid_view(self.h, C.byref(v)))
        return v

    def set_quirks(self, precond_mode=0):
        q = Quirks()
        q.precond_mode = precond_mode
        _check(self.L.blub_fluid_set_quirks(self.h, C.byref(q)))

    def synchronize(self):
        _check(self.L.blub_fluid_synchronize(self.h))

    # -- taps ---------------------------------------------------------------------------------
    def download_grid(self, tap):
        dt = np.int8 if tap == TAP_MARKER else np.float32
        out = np.empty((self.nz, self.ny, self.nx), dtype=dt)
        _check(self.L.blub_fluid_download(self.h, tap, out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    def upload_grid(self, tap, arr):
        dt = np.int8 if tap == TAP_MARKER else np.float32
        arr = np.ascontiguousarray(arr, dtype=dt).reshape(self.nz, self.ny, self.nx)
        _check(self.L.blub_fluid_upload(self.h, tap, arr.ctypes.data_as(C.c_void_p), arr.nbytes))

    def download_particles(self, tap=TAP_POS):
        out = np.empty((self.num_particles, 4), dtype=np.float32)
        if out.size:
            _check(self.L.blub_fluid_download(self.h, tap, out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    def set_particles(self, pos4, rowx=None, rowy=None, rowz=None):
        pos4 = np.ascontiguousarray(pos4, dtype=np.float32).reshape(-1, 4)
        rows = [None if r is None else np.ascontiguousarray(r, dtype=np.float32).reshape(-1, 4) for r in (rowx, rowy, rowz)]
        ptr = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        _check(self.L.blub_fluid_set_particles(self.h, pos4.shape[0], ptr(pos4), ptr(rows[0]), ptr(rows[1]), ptr(rows[2])))

    def step_stages(self, dt, frm, to):
        _check(self.L.blub_fluid_step_stages(self.h, dt, frm, to))

    def solve_only(self, which, dt=DT_120HZ):
        _check(self.L.blub_fluid_solve_only(self.h, which, dt))

    def last_solve(self, which):
        e, it = C.c_float(0), C.c_int32(0)
        _check(self.L.blub_fluid_last_solve(self.h, which, C.byref(e), C.byref(it)))
        return float(e.value), int(it.value)

    def last_solve_scalars(self, which):
        """(alpha, beta, sigma) the last solve of a field left, as float32 values (conventions per solver path: blub_fluid.h)."""
        out = (C.c_float * 3)()
        _check(self.L.blub_fluid_last_solve_scalars(self.h, which, out))
        return tuple(np.float32(out[k]) for k in range(3))

    def solver_work(self):
        """{tiles, columns, cells_per_tile, cells_per_column} of the most recent solve's work lists."""
        out = (C.c_uint32 * 4)()
        _check(self.L.blub_fluid_solver_work(self.h, out))
        return {"tiles": int(out[0]), "columns": int(out[1]), "cells_per_tile": int(out[2]), "cells_per_column": int(out[3])}

    def time_solve(self, which, dt, repetitions):
        ms = (C.c_float * repetitions)()
        _check(self.L.blub_fluid_time_solve(self.h, which, dt, repetitions, ms))
        return [float(x) for x in ms]

    def step_timed(self, dt=DT_120HZ):
        ms = (C.c_float * 14)()
        _check(self.L.blub_fluid_step_timed(self.h, dt, ms))
        return [float(x) for x in ms]

    def set_solver_path(self, persistent):
        """True / 1: persistent cooperative PCG, dense tiles + column list (default); False / 0: three kernels per iteration;
        2 / "tma": TMA-staged tiles; 4 / "dense": tile kernel without the sparsity skip; 6 / "tiles": tile kernel with the sparse tile bodies."""
        names = {"tma": 2, "dense": 4, "tiles": 6}
        mode = names[persistent] if persistent in names else (int(persistent) if persistent not in (True, False) else (1 if persistent else 0))
        _check(self.L.blub_fluid_set_solver_path(self.h, mode))

    def set_flow(self, sources=(), drains=()):
        """Replaces the flow set: sources = [(min, max, velocity[, tag])], drains = [(min, max)], boxes in grid cells, velocities in cells/s;
        the particles a source emits carry its tag (default 0).  Empty lists clear it.  Raises BlubError (and changes nothing) on overlaps, more
        than 16 boxes of a kind, non-finite values, boxes empty after clamping, z-slab ranks and a fluid inside a step."""
        src = (FluidSource * max(len(sources), 1))()
        tags = (C.c_uint32 * max(len(sources), 1))()
        for k, (mn, mx, vel, *tag) in enumerate(sources):
            src[k].min_grid[:], src[k].max_grid[:], src[k].velocity_grid[:] = [float(v) for v in mn], [float(v) for v in mx], [float(v) for v in vel]
            tags[k] = int(tag[0]) if tag else 0
        drn = (FluidDrain * max(len(drains), 1))()
        for k, (mn, mx) in enumerate(drains):
            drn[k].min_grid[:], drn[k].max_grid[:] = [float(v) for v in mn], [float(v) for v in mx]
        _check(self.L.blub_fluid_set_flow_tagged(self.h, src, tags, len(sources), drn, len(drains)))

    # -- particle tags ------------------------------------------------------------------------
    def paint_tags(self, min_grid, max_grid, tag):
        """Tags every particle whose cell lies in the box (corners clamped as add_fluid_cube clamps them, max exclusive).  Enqueued on the
        fluid's stream, no synchronisation."""
        _check(self.L.blub_fluid_paint_tags(self.h, _f3(min_grid), _f3(max_grid), int(tag)))

    def particle_tags(self):
        """The tag of every particle in array order: a uint32 view of the fourth column of the positions."""
        return self.download_particles(TAP_POS)[:, 3].view(np.uint32)

    def tag_census(self, first=0, count=TAG_CENSUS_MAX):
        """Census of tags first .. first + count - 1 (count <= 256): the raw fields of BlubTagCensus as arrays ("count", "position_sum_fx",
        "velocity_sum_fx", "cell_min", "cell_max"), plus "centroid" and "mean_velocity" (float64, NaN for an empty tag).  Synchronises."""
        count = int(count)
        out = (TagCensus * max(count, 1))()
        _check(self.L.blub_fluid_tag_census(self.h, int(first), count, out))
        recs = out[:count]
        res = {"count": np.array([r.count for r in recs], dtype=np.uint64)}
        for name, dt in (("position_sum_fx", np.int64), ("velocity_sum_fx", np.int64), ("cell_min", np.int32), ("cell_max", np.int32)):
            res[name] = np.array([list(getattr(r, name)) for r in recs], dtype=dt).reshape(-1, 3)
        scale = float(1 << TAG_CENSUS_FRAC_BITS)
        with np.errstate(invalid="ignore", divide="ignore"):
            n = res["count"].astype(np.float64)[:, None]
            res["centroid"] = res["position_sum_fx"].astype(np.float64) / scale / n
            res["mean_velocity"] = res["velocity_sum_fx"].astype(np.float64) / scale / n
        return res

    # -- solid load probes --------------------------------------------------------------------
    def set_viscosity(self, nu, error_tolerance=1e-4, max_num_iterations=200):
        """Kinematic viscosity in cells^2/s (m^2/s / grid_to_world_scale^2); 0 turns the stage off.  Every step then ends its stage 0 with
        the implicit diffusion of the grid velocity, solved to max |residual| <= error_tolerance (cells/s) or max_num_iterations.  Raises
        BlubError (and changes nothing) on a negative or non-finite nu, a tolerance that is not finite and above 0, a cap outside
        [1, 10000], z-slab ranks and a fluid inside a step."""
        v = Viscosity(float(nu), float(error_tolerance), int(max_num_iterations), 0)
        _check(self.L.blub_fluid_set_viscosity(self.h, C.byref(v)))

    def viscosity(self):
        """(kinematic viscosity in cells^2/s, error_tolerance, max_num_iterations); a viscosity of 0.0 means off."""
        v = Viscosity()
        _check(self.L.blub_fluid_viscosity(self.h, C.byref(v)))
        return float(v.kinematic_viscosity), float(v.error_tolerance), int(v.max_num_iterations)

    def last_viscosity_solve(self):
        """(iterations, [max |residual| per component]) of the last viscosity solve.  Synchronises."""
        it, e = C.c_int32(0), (C.c_float * 3)()
        _check(self.L.blub_fluid_last_viscosity_solve(self.h, C.byref(it), e))
        return int(it.value), [float(x) for x in e]

    def viscosity_only(self, dt=DT_120HZ):
        """Test hook: the viscosity stage on the grid velocity and marker as they are (tap uploads), nothing else."""
        _check(self.L.blub_fluid_viscosity_only(self.h, dt))

    def set_load_probes(self, probes=()):
        """Replaces the load probe set: probes = [(min, max[, pivot])] in grid cells (at most 16; pivot default: the box centre).  Resets the
        history.  An empty list clears the set.  Raises BlubError (and changes nothing) on too many probes, non-finite values, boxes empty
        after clamping to [0, dim], z-slab ranks and a fluid inside a step."""
        _check(self.L.blub_fluid_set_load_probes(self.h, _load_probes(probes), len(probes)))

    def load_history(self, probe, capacity=LOAD_HISTORY_LENGTH):
        """The newest records of one probe, oldest first: the raw fields of BlubSolidLoad as arrays ("step", "wetted_faces", "force_fx",
        "torque_fx") plus float64 "force" (cells^4/s^2 per unit density) and "torque" (cells^5/s^2).  Synchronises."""
        capacity = int(capacity)
        out = (SolidLoad * max(capacity, 1))()
        count = C.c_uint32(0)
        _check(self.L.blub_fluid_load_history(self.h, int(probe), out, capacity, C.byref(count)))
        recs = out[:count.value]
        res = {"step": np.array([r.step for r in recs], dtype=np.uint32), "wetted_faces": np.array([r.wetted_faces for r in recs], dtype=np.uint32),
               "force_fx": np.array([list(r.force_fx) for r in recs], dtype=np.int64).reshape(-1, 3),
               "torque_fx": np.array([list(r.torque_fx) for r in recs], dtype=np.int64).reshape(-1, 3)}
        res["force"] = res["force_fx"].astype(np.float64) / float(1 << LOAD_FORCE_FRAC_BITS)
        res["torque"] = res["torque_fx"].astype(np.float64) / float(1 << LOAD_TORQUE_FRAC_BITS)
        return res

    # -- floating bodies ----------------------------------------------------------------------
    def set_bodies(self, bodies=()):
        """Replaces the floating bodies: dicts {"shape": "box" | "sphere", "half_extent": (hx, hy, hz) or a radius, "relative_density",
        "centre", "rotation" (w, x, y, z; default identity), "velocity", "angular_velocity"} in grid cells, cells/s and rad/s (at most 16).
        Resets the history; an empty list clears the set.  Raises BlubError (and changes nothing) on a body that breaks a rule of
        blub_fluid_set_bodies, z-slab ranks and a fluid inside a step.
        A mesh body is {"shape": "mesh", "mesh": Mesh or (positions [n, 3], triangles [m, 3]), "scale": cells per model unit, "relative_density",
        "centre", "rotation", ...}: centre and rotation place the mesh's model origin and axes (DESIGN.md §8 "Mesh bodies"); it goes through
        blub_fluid_set_bodies_meshes, which also refuses what blub_mesh_body_properties refuses."""
        arr = (Body * max(len(bodies), 1))()
        shapes = (MeshBodyShape * max(len(bodies), 1))()
        keep = []  # meshes made here live until the set has copied them
        for k, b in enumerate(bodies):
            if not isinstance(b, Body) and b.get("mesh") is not None:
                m = b["mesh"]
                if not isinstance(m, Mesh):
                    m = Mesh(m[0], m[1], device=self.device)
                keep.append(m)
                arr[k] = Body.from_dict(dict(b, shape=2, half_extent=(1.0, 1.0, 1.0)))
                shapes[k].mesh, shapes[k].scale = m.h, float(b["scale"])
            else:
                arr[k] = b if isinstance(b, Body) else Body.from_dict(b)
        if keep:
            _check(self.L.blub_fluid_set_bodies_meshes(self.h, arr, shapes, len(bodies)))
        else:
            _check(self.L.blub_fluid_set_bodies(self.h, arr, len(bodies)))

    def body_mass_properties(self, body):
        """The mass properties of mesh body `body` as stored (see mesh_body_properties; mass and moments with its relative density)."""
        p = MeshBodyProperties()
        _check(self.L.blub_fluid_body_mass_properties(self.h, int(body), C.byref(p)))
        return p.to_dict()

    def mesh_body_model_pose(self, body):
        """(origin, R_model): where the current pose of mesh body `body` puts the mesh's model origin and model axes (R_model maps model
        to grid coordinates): R_model = R_body R_p^T, origin = c - R_model (scale * centroid), in float64."""
        b, p = self.bodies()[int(body)], self.body_mass_properties(body)
        R = quat_matrix(b["rotation"]) @ quat_matrix(p["principal_rotation"]).T
        return np.asarray(b["centre"], dtype=np.float64) - R @ (float(p["scale"]) * np.asarray(p["centroid"])), R

    def bodies(self):
        """The current bodies as dicts (the pose the next step writes).  Synchronises."""
        arr = (Body * BODIES_MAX)()
        count = C.c_uint32(0)
        _check(self.L.blub_fluid_bodies(self.h, arr, BODIES_MAX, C.byref(count)))
        return [b.to_dict() for b in arr[:count.value]]

    def body_history(self, body, capacity=BODY_HISTORY_LENGTH):
        """The newest records of one body, oldest first: "step", "wetted_faces", "force_fx", "torque_fx" as recorded, float64 "force"
        (cells^4/s^2 per unit density) and "torque" (cells^5/s^2), and float32 "centre", "rotation", "velocity", "angular_velocity" after
        the step.  Synchronises."""
        capacity = int(capacity)
        out = (BodyRecord * max(capacity, 1))()
        count = C.c_uint32(0)
        _check(self.L.blub_fluid_body_history(self.h, int(body), out, capacity, C.byref(count)))
        recs = out[:count.value]
        res = {"step": np.array([r.step for r in recs], dtype=np.uint32), "wetted_faces": np.array([r.wetted_faces for r in recs], dtype=np.uint32)}
        for name in ("force_fx", "torque_fx"):
            res[name] = np.array([list(getattr(r, name)) for r in recs], dtype=np.int64).reshape(-1, 3)
        for name, width in (("centre", 3), ("rotation", 4), ("velocity", 3), ("angular_velocity", 3)):
            res[name] = np.array([list(getattr(r, name)) for r in recs], dtype=np.float32).reshape(-1, width)
        res["force"] = res["force_fx"].astype(np.float64) / float(1 << LOAD_FORCE_FRAC_BITS)
        res["torque"] = res["torque_fx"].astype(np.float64) / float(1 << LOAD_TORQUE_FRAC_BITS)
        return res

    def download_solid_voxels(self):
        """The solid volume the step reads (BLUB_TAP_SOLID_VOXELS) as float16 [nz, ny, nx, 4]."""
        out = np.empty((self.nz, self.ny, self.nx, 4), dtype=np.float16)
        _check(self.L.blub_fluid_download(self.h, TAP_SOLID_VOXELS, out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    @property
    def has_flow(self):
        """True while the flow set is not empty (the particle count then lives on the device)."""
        return self.L.blub_fluid_has_flow(self.h) == 1

    @property
    def flow_counters(self):
        """Cumulative {"emitted", "drained", "refused"} particle counts of the sources and drains (synchronises)."""
        out = (C.c_uint64 * 3)()
        _check(self.L.blub_fluid_flow_counters(self.h, out))
        return {"emitted": int(out[0]), "drained": int(out[1]), "refused": int(out[2])}

    def set_transfer_path(self, scatter):
        """True / "scatter" (default): warp-aggregated atomic scatter; False / "gather": deterministic gather P2G over per-step cell lists."""
        _check(self.L.blub_fluid_set_transfer_path(self.h, 1 if scatter in (True, 1, "scatter") else 0))

    def stream(self):
        """The CUDA stream (as an integer handle) the fluid's work is enqueued on."""
        return self.L.blub_fluid_stream(self.h)

    def set_graph_replay(self, enabled):
        _check(self.L.blub_fluid_set_graph_replay(self.h, 1 if enabled else 0))

    def time_steps(self, dt, steps):
        ms = C.c_float(0)
        _check(self.L.blub_fluid_time_steps(self.h, dt, steps, C.byref(ms)))
        return float(ms.value)
