"""GPU: stage 7 with the density scatter fused in and stage 9 as a sparse finish (transfer_kernels.cu: advect_density_kernel,
density_finish_sparse_kernel; DESIGN.md §3.2) change no bit.  Every case runs a fluid created with BLUB_DENSITY_FUSE=on next to one created with BLUB_DENSITY_FUSE=off
(read when a fluid is created: the separate advection, the memset, the density scatter and the dense rhs pass), and the particles (tags
included), the three velocity rows, the grid velocities, the marker, the residual after stage 9 and both pressures must be equal bit for bit.
20 steps span the re-sorts of steps 0, 8 and 16."""
import json

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import util

pytestmark = pytest.mark.gpu

DT = F.DT_120HZ
STEPS = 20
GRID_TAPS = (F.TAP_UX, F.TAP_UY, F.TAP_UZ, F.TAP_MARKER, F.TAP_P_VEL, F.TAP_P_DEN, F.TAP_RESIDUAL)
PARTICLE_TAPS = (F.TAP_POS, F.TAP_VX, F.TAP_VY, F.TAP_VZ)
BODIES = [{"shape": "box", "half_extent": (2.0, 1.5, 2.5), "relative_density": 0.5, "centre": (9.0, 9.0, 10.0)},
          {"shape": "sphere", "half_extent": 2.5, "relative_density": 0.75, "centre": (22.0, 10.0, 21.0)}]
ROLL = {"pivot": (16.0, 8.0, 16.0), "translations": [{"direction": (1.0, 0.0, 0.0), "amplitude": 2.0, "frequency": 1.2, "phase": 0.4}],
        "rotation": {"axis": (0.0, 0.0, 1.0), "amplitude": 0.15, "frequency": 0.9, "phase": 0.0, "rate": 0.0}}
# the moving box of the double_dam_box workload
SOLID = {"world_position": [0.44, 0.20, 0.32], "scale": 1.0, "rotation_angles": [0.0, 0.0, 0.0], "shape": "box", "half_extent": [0.12, 0.20, 0.12],
         "translation": {"target": [0.84, 0.20, 0.32], "curve": "SmoothStep", "duration": 2.0}}


def make(monkeypatch, fuse, build):
    monkeypatch.setenv("BLUB_DENSITY_FUSE", "on" if fuse else "off")  # "on": the test grids are below the size the fused path starts at
    f = build()
    monkeypatch.delenv("BLUB_DENSITY_FUSE", raising=False)
    return f


def taps(f):
    f.synchronize()
    return [f.download_grid(t).tobytes() for t in GRID_TAPS] + [f.download_particles(t).tobytes() for t in PARTICLE_TAPS]


def assert_same(a, b, what):
    names = [str(t) for t in GRID_TAPS] + ["p" + str(t) for t in PARTICLE_TAPS]
    bad = [n for n, x, y in zip(names, a, b) if x != y]
    assert not bad, f"{what}: taps {bad} differ"


def scene(name):
    return lambda: blub_b200.HybridFluid.from_scene(util.scene_path(name))


def odd_x():
    """A 40 x 24 x 24 grid (x not a multiple of 32) with a block of water against the high x wall."""
    rng = np.random.default_rng(11)
    n = 30000
    pos = np.zeros((n, 4), np.float32)
    pos[:, 0] = rng.uniform(20.0, 38.9, n)
    pos[:, 1] = rng.uniform(1.1, 14.0, n)
    pos[:, 2] = rng.uniform(1.1, 22.9, n)
    pos[:, 3] = np.arange(n, dtype=np.uint32).view(np.float32)
    f = blub_b200.HybridFluid(40, 24, 24, n)
    f.set_particles(pos)
    return f


class Stepper:
    """Steps one fluid of a case: the odd steps stage by stage (the residual of stage 9 recorded), the others as one step."""

    def __init__(self, case, f):
        self.case, self.f, self.k = case, f, 0
        if case == "bodies":
            f.set_bodies(BODIES)
        elif case == "surface_tension":
            f.set_surface_tension(5.0)
        elif case == "solid":
            import torch

            sc = json.load(open(util.scene_path("double_dam")))
            d = sc["fluid"]["grid_dimension"]
            self.dims, self.scale = (d["x"], d["y"], d["z"]), sc["fluid"]["grid_to_world_scale"]
            self.origin = [sc["fluid"]["world_position"][c] for c in "xyz"]
            self.vol = torch.zeros((d["z"], d["y"], d["x"], 4), dtype=torch.float16, device="cuda:0")
            torch.cuda.synchronize()
            f.set_solid_voxels(self.vol.data_ptr())

    def step(self):
        f, k = self.f, self.k
        if self.case == "tank":
            f.set_tank_frame(F.tank_frame_at(ROLL, k * DT))
        if self.case == "solid":
            F.solid_voxelize(self.vol.data_ptr(), self.dims, SOLID, self.scale, self.origin, (k + 1) * DT, DT, cuda_stream=f.stream())
        residual = None
        if k % 2:
            f.step_stages(DT, 0, 10)
            f.synchronize()
            residual = f.download_grid(F.TAP_RESIDUAL).tobytes()
            f.step_stages(DT, 10, 14)
        else:
            f.step(DT)
        self.k += 1
        return taps(f) + [residual]


def run_pair(monkeypatch, case, build):
    fused, plain = Stepper(case, make(monkeypatch, True, build)), Stepper(case, make(monkeypatch, False, build))
    for k in range(STEPS):
        a, b = fused.step(), plain.step()
        assert_same(a[:-1], b[:-1], f"{case} step {k}")
        assert a[-1] == b[-1], f"{case} step {k}: the residual after stage 9 differs"
    return fused.f


@pytest.mark.parametrize("case", ["dam_small", "dam_halfhalf", "odd_x", "solid", "bodies", "tap", "tank", "surface_tension"])
def test_fused_density_changes_no_bit(monkeypatch, case):
    build = {"dam_small": scene("dam_small"), "dam_halfhalf": scene("dam_halfhalf"), "odd_x": odd_x, "solid": scene("double_dam"),
             "bodies": scene("dam_small"), "tap": scene("tap_small"), "tank": scene("dam_small"), "surface_tension": scene("dam_small")}[case]
    f = run_pair(monkeypatch, case, build)
    if case == "tap":
        assert f.flow_counters["emitted"] > 0 and f.flow_counters["drained"] > 0


def test_resumed_fluid(monkeypatch, tmp_path):
    """A fluid loaded from a state file has no schedule until its next re-sort: the fused kernel walks the chunks only."""
    src = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    for _ in range(11):
        src.step(DT)
    path = str(tmp_path / "mid.blub")
    src.save_state(path)
    run_pair(monkeypatch, "resume", lambda: blub_b200.HybridFluid.from_state(path))


@pytest.mark.parametrize("case", ["dam_small", "surface_tension"])
def test_density_volume_is_zero_after_a_fused_step(monkeypatch, case):
    """The sparse finish puts every word the fused scatter added to back to zero (with surface tension after stage 1 dirtied it too)."""
    s = Stepper(case, make(monkeypatch, True, scene("dam_small")))
    for _ in range(STEPS):
        s.step()
        assert not s.f.download_grid(F.TAP_DENSITY).any()
    # a stage 9 alone scatters the positions afresh and leaves the splat in the volume
    s.f.step_stages(DT, 9, 10)
    assert s.f.download_grid(F.TAP_DENSITY).sum() > 0
    s.f.step_stages(DT, 10, 14)


def test_fallback_after_an_upload_between_the_stages(monkeypatch):
    """Stages 0-7, new particle positions from the host, stages 8-13: stage 9 must scatter the uploaded positions, and the steps after it
    (whose fused stage 7 finds the volume not zero) must go on as the comparator's."""
    fluids = [make(monkeypatch, fuse, scene("dam_small")) for fuse in (True, False)]
    for k in range(STEPS):
        res = []
        for f in fluids:
            if k in (3, 12):
                f.step_stages(DT, 0, 8)
                f.synchronize()
                pos = f.download_particles(F.TAP_POS)
                rows = [f.download_particles(t) for t in (F.TAP_VX, F.TAP_VY, F.TAP_VZ)]
                pos[:, :3] = np.clip(pos[:, :3] + np.float32(0.03), 1.01, 30.99)
                f.set_particles(pos, *rows)
                f.step_stages(DT, 8, 14)
            else:
                f.step(DT)
            res.append(taps(f))
        assert_same(res[0], res[1], f"step {k}")


def test_fused_runs_are_deterministic(monkeypatch):
    a, b = (Stepper("dam_halfhalf", make(monkeypatch, True, scene("dam_halfhalf"))) for _ in range(2))
    for k in range(STEPS):
        x, y = a.step(), b.step()
        assert_same(x[:-1], y[:-1], f"step {k}")
        assert x[-1] == y[-1]
