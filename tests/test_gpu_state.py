"""GPU: checkpoint / restart.  A fluid saved after step k and loaded in a new fluid continues bit for bit as the fluid that never stopped:
all ten arrays of blub_fluid_view, the last solve of both fields and the statistics history are compared exactly.  Every resumed run
crosses a re-sort or rebinning step after the load.  The cheapest checks come first."""
import json
import os
import subprocess

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import util
from tests.util import DT

pytestmark = pytest.mark.gpu

BLUB_ERR_INVALID_ARGUMENT = 1
RUNNER = os.path.join(os.path.dirname(F.lib_path()), "blub_run")
PARTICLE_TAPS = {"particles_position": F.TAP_POS, "particles_velocity_x": F.TAP_VX, "particles_velocity_y": F.TAP_VY, "particles_velocity_z": F.TAP_VZ}
GRID_TAPS = {"grid_velocity_x": F.TAP_UX, "grid_velocity_y": F.TAP_UY, "grid_velocity_z": F.TAP_UZ, "marker": F.TAP_MARKER,
             "pressure_from_velocity": F.TAP_P_VEL, "pressure_from_density": F.TAP_P_DEN}


def snapshot(f):
    f.synchronize()
    f.update_statistics()
    out = {name: f.download_particles(tap) for name, tap in PARTICLE_TAPS.items()}
    out.update({name: f.download_grid(tap) for name, tap in GRID_TAPS.items()})
    out["last_solve"] = [f.last_solve(0), f.last_solve(1)]
    out["stats"] = [f.pressure_solver_stats(0), f.pressure_solver_stats(1)]
    out["step_count"] = f.step_count
    return out


def assert_identical(a, b):
    for name in list(PARTICLE_TAPS) + list(GRID_TAPS):
        assert a[name].shape == b[name].shape and np.array_equal(a[name], b[name]), name
    for name in ("last_solve", "stats", "step_count"):
        assert a[name] == b[name], name


def resumed_equals_uninterrupted(tmp_path, scene, before, after, setup=lambda f: None, step=None):
    """`before` steps, save, close, load, `after` steps -- against before + after steps of one fluid."""
    step = step or (lambda f, k: f.step(DT))
    ref = blub_b200.HybridFluid.from_scene(util.scene_path(scene))
    setup(ref)
    for k in range(before + after):
        step(ref, k)
    want = snapshot(ref)
    ref.close()

    f = blub_b200.HybridFluid.from_scene(util.scene_path(scene))
    setup(f)
    for k in range(before):
        step(f, k)
    path = str(tmp_path / "state.blub")
    f.save_state(path)
    f.close()
    info = blub_b200.state_info(path)
    assert info.step_count == before and info.format_version == 1
    g = blub_b200.HybridFluid.from_state(path)
    assert g.step_count == before
    for k in range(before, before + after):
        step(g, k)
    got = snapshot(g)
    g.close()
    assert want["step_count"] == before + after
    assert_identical(want, got)
    return want


def test_saves_are_refused_inside_a_step_and_on_slab_ranks(tmp_path):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    f.step(DT)
    f.step_stages(DT, 0, 5)
    L = F.lib()
    path = str(tmp_path / "mid.blub")
    assert L.blub_fluid_save_state(f.h, os.fsencode(path)) == BLUB_ERR_INVALID_ARGUMENT
    assert b"inside a step" in L.blub_last_error() and not os.path.exists(path)
    f.step_stages(DT, 5, 14)  # the step is complete again
    f.save_state(path)
    assert blub_b200.state_info(path).step_count == 2
    f.close()
    s = blub_b200.HybridFluid.create_slab(64, 64, 32, 1000, rank=0, world=2)
    assert L.blub_fluid_save_state(s.h, os.fsencode(path)) == BLUB_ERR_INVALID_ARGUMENT
    assert b"z-slab" in L.blub_last_error()
    s.close()
    assert blub_b200.state_info(path).step_count == 2  # the refused save left the earlier file alone


def test_round_trip_files_are_byte_identical_and_loads_step_identically(tmp_path):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    for _ in range(10):
        f.step(DT)
    a, b = str(tmp_path / "a.blub"), str(tmp_path / "b.blub")
    f.save_state(a)
    g = blub_b200.HybridFluid.from_state(a)
    g.save_state(b)
    assert open(a, "rb").read() == open(b, "rb").read()
    assert not os.path.exists(a + ".tmp") and not os.path.exists(b + ".tmp")
    h = blub_b200.HybridFluid.from_state(a)
    for fl in (f, g, h):
        for _ in range(9):  # crosses the re-sort at step 16
            fl.step(DT)
    s = [snapshot(fl) for fl in (f, g, h)]
    assert_identical(s[0], s[1])
    assert_identical(s[0], s[2])


def test_save_waits_for_the_steps_in_flight(tmp_path):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_halfhalf"))
    for _ in range(12):
        f.step(DT)
    path = str(tmp_path / "inflight.blub")
    f.save_state(path)  # no synchronize before: the file holds the state after the last enqueued step
    want = snapshot(f)
    g = blub_b200.HybridFluid.from_state(path)
    assert_identical(want, snapshot(g))


def test_seeding_after_a_load_continues_the_particle_stream(tmp_path):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_halfhalf"))  # 1,218,672 particles, room for 1,238,328
    n0 = f.num_particles
    for _ in range(3):
        f.step(DT)
    path = str(tmp_path / "seed.blub")
    f.save_state(path)
    g = blub_b200.HybridFluid.from_state(path)
    for fl in (f, g):
        assert not fl.add_fluid_cube([100.0, 40.0, 20.0], [104.0, 44.0, 24.0])  # the RNG seed depends on num_particles
    assert f.num_particles == g.num_particles == n0 + 4 * 4 * 4 * 8
    assert np.array_equal(f.download_particles(), g.download_particles())


def test_default_paths_resume_bit_for_bit(tmp_path):
    """Scatter P2G, graph replay, column PCG on dam_halfhalf (1.2 M particles); steps 13..24 cross the re-sorts at 16 and 24 and the
    rebinning at 20."""
    want = resumed_equals_uninterrupted(tmp_path, "dam_halfhalf", 13, 12, setup=lambda f: f.set_rebin_frequency(20))
    assert len(want["stats"][0]) == len(want["stats"][1]) == 25


def test_non_default_settings_survive_the_round_trip(tmp_path):
    """Gather P2G, eager launches, precond_mode 1, solver 1e-4 / 128 / 4, rebinning every 5th step: all set before the save only."""

    def setup(f):
        f.set_transfer_path("gather")
        f.set_graph_replay(False)
        f.set_quirks(precond_mode=1)
        util.tight_solver(f)
        f.set_rebin_frequency(5)

    resumed_equals_uninterrupted(tmp_path, "dam_halfhalf", 13, 12, setup=setup)


def test_moving_solid_resumes_with_its_voxels_attached_again(tmp_path):
    import torch

    sc = json.load(open(util.scene_path("double_dam")))
    d = sc["fluid"]["grid_dimension"]
    dims, scale, origin = (d["x"], d["y"], d["z"]), sc["fluid"]["grid_to_world_scale"], [sc["fluid"]["world_position"][c] for c in "xyz"]
    # the box of tests/test_gpu_configs.py: it starts inside the left dam and moves through the fluid from the first step
    solid = {"world_position": [0.22, 0.20, 0.32], "scale": 1.0, "rotation_angles": [0.0, 0.0, 0.0], "shape": "box", "half_extent": [0.12, 0.20, 0.12],
             "translation": {"target": [0.84, 0.20, 0.32], "curve": "SmoothStep", "duration": 2.0}}
    vol = torch.zeros((dims[2], dims[1], dims[0], 4), dtype=torch.float16, device="cuda")
    torch.cuda.synchronize()
    attached = set()

    def step(f, k):  # Scene::step: time from the step index (not a running sum), voxelize, step the fluid
        if id(f) not in attached:
            f.set_solid_voxels(vol.data_ptr())
            attached.add(id(f))
        t = 0.5 + (k + 1) * DT
        F.solid_voxelize(vol.data_ptr(), dims, solid, scale, origin, t, DT, cuda_stream=f.stream())
        f.step(DT)

    resumed_equals_uninterrupted(tmp_path, "double_dam", 13, 12, setup=lambda f: f.set_rebin_frequency(20), step=step)
    assert (vol[..., 3] > 0).sum().item() > 20000


def test_runner_resumes_a_saved_run(tmp_path):
    a, x, y, s, t = (str(tmp_path / n) for n in ("a.blub", "x.f32", "y.f32", "s.json", "t.json"))
    scene = util.scene_path("dam_small")

    def run(*args):
        res = subprocess.run([RUNNER, scene, *args], capture_output=True, text=True, timeout=300)
        assert res.returncode == 0, res.stdout + res.stderr
        return res.stdout

    out = run("--steps", "20", "--rebin", "10", "--save-state", a, "--checkpoint-every", "16")
    assert out.count("saved the state") == 2 and "after step 20" in out
    assert blub_b200.state_info(a).step_count == 20
    out = run("--load-state", a, "--steps", "20", "--dump", x, "--stats", s)  # the rebinning frequency comes from the file
    assert "resumed" in out and "after step 20" in out
    run("--steps", "40", "--rebin", "10", "--dump", y, "--stats", t)
    assert open(x, "rb").read() == open(y, "rb").read()
    hs, ht = json.load(open(s)), json.load(open(t))
    assert len(hs["velocity"]) == 40 and hs["velocity"] == ht["velocity"] and hs["density"] == ht["density"]
    bad = subprocess.run([RUNNER, util.scene_path("dam_halfhalf"), "--load-state", a, "--steps", "1"], capture_output=True, text=True, timeout=300)
    assert bad.returncode == 1 and "not the scene's" in bad.stderr
