"""CPU-side tests: the C ABI library loads and exports every declared symbol, the scene loader reads blub scenes,
fixtures match the reference's shipped scenes (stored verbatim under tests/golden/reference_scenes).  No compute calls: no GPU here."""
import json
import os
import re

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SCENES = os.path.join(util.HERE, "golden", "reference_scenes")  # the reference's scenes/*.json, unchanged


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "blub_fluid.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(blub_[a-z_0-9]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    L = blub_b200.lib()
    syms = declared_symbols()
    assert len(syms) >= 25
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/blub_fluid.h but not exported"
    assert b"sm_90a" in L.blub_version()


def test_ctypes_mirror_binds_every_declared_symbol():
    L = blub_b200.lib()
    for s in declared_symbols():
        assert getattr(L, s).argtypes is not None, f"{s} has no ctypes signature in blub_b200/fluid.py"


def test_struct_layouts():
    import ctypes as C
    assert C.sizeof(F.SolverConfig) == 12 and C.sizeof(F.SolverSample) == 8
    assert C.sizeof(F.Quirks) == 32 and C.sizeof(F.FluidView) == 80


def test_no_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(blub_b200.BlubError):
        blub_b200.HybridFluid(64, 64, 64, 1000)


def test_invalid_arguments_are_reported_not_thrown():
    L = blub_b200.lib()
    assert L.blub_fluid_step(None, 0.01) == 1
    assert b"NULL" in L.blub_last_error()
    assert L.blub_fluid_num_particles(None) == 0
    assert L.blub_fluid_solver_stats(None, 0, None, 0) == 0


@pytest.mark.parametrize("name,dims,maxp,cubes", [
    ("dam_halfhalf", (128, 64, 64), 1238328, 1),
    ("dam_halfhalf_highres", (256, 128, 128), 10193528, 1),
    ("single_cell_debug", (64, 64, 128), 1238328, 1),
    ("dam_256", (256, 256, 256), 16500000, 1),
])
def test_scene_info(name, dims, maxp, cubes):
    info = blub_b200.scene_info(util.scene_path(name))
    assert tuple(info.grid_dimension) == dims and info.max_num_particles == maxp
    assert info.num_fluid_cubes == cubes and info.num_static_objects == 0
    assert abs(info.gravity[1] + 9.81) < 1e-6


def test_scene_loader_key_order_and_static_objects(tmp_path):
    sc = {
        "static_objects": [{"model": "models/x.obj", "scale": 1.0, "world_position": {"z": 0, "y": 0, "x": 0},
                            "rotation_angles": {"x": 0, "y": 90.0, "z": 0},
                            "animation": {"rotation": {"axis": {"x": 0, "y": 1, "z": 0}, "deg_per_sec": 20.0}}}],
        "fluid": {"fluid_cubes": [], "grid_dimension": {"z": 32, "x": 64, "y": 48}, "grid_to_world_scale": 2.5e-2,
                  "max_num_particles": 7, "world_position": {"x": -1.5, "y": 0.0, "z": 1e1}},
        "gravity": {"y": -9.81, "x": 0.0, "z": 0.0},
    }
    p = tmp_path / "s.json"
    p.write_text(json.dumps(sc))
    info = blub_b200.scene_info(str(p))
    assert tuple(info.grid_dimension) == (64, 48, 32) and info.num_static_objects == 1 and info.num_fluid_cubes == 0
    assert info.world_position[0] == -1.5 and info.world_position[2] == 10.0
    assert abs(info.grid_to_world_scale - 0.025) < 1e-9


@pytest.mark.parametrize("text", ["", "{", '{"gravity": 1}', '{"gravity":{"x":0,"y":0,"z":0}}', "[1,2"])
def test_scene_loader_errors(tmp_path, text):
    p = tmp_path / "bad.json"
    p.write_text(text)
    with pytest.raises(blub_b200.BlubError):
        blub_b200.scene_info(str(p))
    with pytest.raises(blub_b200.BlubError):
        blub_b200.scene_info(str(tmp_path / "missing.json"))


def test_fixtures_match_reference_scenes():
    for name in ["single_cell_debug", "dam_halfhalf", "dam_halfhalf_highres", "filled_basin"]:
        ref = json.load(open(os.path.join(REF_SCENES, name + ".json")))
        mine = json.load(open(util.scene_path(name)))
        assert ref["fluid"] == mine["fluid"] and ref["gravity"] == mine["gravity"], name
    ref = json.load(open(os.path.join(REF_SCENES, "double_dam_wgpulogo.json")))  # config C5's fluid, without the LFS-stub mesh
    mine = json.load(open(util.scene_path("double_dam")))
    assert ref["fluid"] == mine["fluid"] and ref["gravity"] == mine["gravity"]


def test_loader_reads_every_reference_scene_unchanged():
    names = sorted(os.listdir(REF_SCENES))
    assert len(names) == 14, names
    for fn in names:
        info = blub_b200.scene_info(os.path.join(REF_SCENES, fn))
        ref = json.load(open(os.path.join(REF_SCENES, fn)))
        d = ref["fluid"]["grid_dimension"]
        assert tuple(info.grid_dimension) == (d["x"], d["y"], d["z"]), fn
        assert info.num_fluid_cubes == len(ref["fluid"]["fluid_cubes"]), fn
        assert info.num_static_objects == len(ref.get("static_objects", [])), fn


def test_oracle_scene_seeding_counts():
    # SURVEY 0.1: real particle counts of the shipped scenes
    f = util.oracle_from_scene("dam_halfhalf")
    assert f.num_particles == 1218672
    f = util.oracle_from_scene("single_cell_debug")
    assert f.num_particles == 8
    assert (np.floor(f.particles()[:, :3]) == [31, 31, 63]).all()


def test_simulation_clock_matches_the_timer_arithmetic():
    """src/timer.rs:94-126 + simulation_controller.rs:33-35 in integer nanoseconds (host-only helpers of the C ABI)."""
    import ctypes as C
    from blub_b200 import fluid as F

    L = F.lib()
    dt_ns = L.blub_simulation_delta_ns(120)
    assert dt_ns == 8333333
    assert L.blub_duration_as_secs_f32(dt_ns) == np.float32(F.DT_120HZ)  # the dt every step is given (SURVEY B14)
    assert L.blub_duration_as_secs_f32(3 * 10 ** 9 + 500_000_000) == np.float32(3.5)
    rendered, simulated = C.c_uint64(0), C.c_uint64(0)
    frame = int(1e9 / 60)  # Duration::from_secs_f64(1 / 60)
    per_frame = [L.blub_timer_steps_in_frame(C.byref(rendered), C.byref(simulated), frame, dt_ns) for _ in range(60)]
    assert per_frame == [2] * 60 and simulated.value == 120 * dt_ns <= rendered.value
    rendered, simulated = C.c_uint64(0), C.c_uint64(0)
    per_frame = [L.blub_timer_steps_in_frame(C.byref(rendered), C.byref(simulated), 20_000_000, dt_ns) for _ in range(50)]  # 50 fps
    assert set(per_frame) == {2, 3} and sum(per_frame) == 120 and per_frame[:5] == [2, 2, 3, 2, 3]
    assert rendered.value - simulated.value < dt_ns  # never ahead of the render clock, never a full step behind
