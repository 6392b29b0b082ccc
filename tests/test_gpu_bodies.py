"""GPU: floating bodies (DESIGN.md §8, "Floating bodies").  A fluid whose bodies were cleared computes what a fluid that never had any
computes; the composite solid volume, the marker, the load sums and every integration step agree bit for bit with the NumPy restatement
(tests/body_ref.py); a box falls freely and comes to rest on the floor, a heavy one sinks to a film above it; a floating box finds the draft discrete hydrostatics
predicts; runs are reproducible, graph against eager; a saved fluid resumes bit for bit; refusals change nothing; and the runner's --bodies
trajectories equal a ctypes-driven run's."""
import json
import os
import subprocess

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import body_ref, util
from tests.test_gpu_loads import BOX, RUNNER, Solid, seed_around
from tests.test_gpu_state import snapshot
from tests.test_gpu_tags import assert_same_physics, bits
from tests.util import DT

pytestmark = pytest.mark.gpu

INV_DT = np.float32(1.0) / np.float32(DT)
SCENE_G = (0.0, float(np.float32(-9.81) / np.float32(0.01)), 0.0)  # the scenes' gravity in grid units, as blub_scene_load sets it
S30 = (float(np.float32(np.cos(np.radians(15)))), 0.0, float(np.float32(np.sin(np.radians(15)))), 0.0)  # 30 degrees about y
# two bodies clear of the double dam's moving box and walls
DOUBLE_DAM_BODIES = [body_ref.body("box", (5, 4, 6), 0.6, (108, 20, 40), S30, (0, 0, 0), (0, 0.5, 0)),
                     body_ref.body("sphere", 5, 0.8, (20, 30, 52), velocity=(2, 0, 0))]


def record(h, k=-1):
    return {"wetted_faces": int(h["wetted_faces"][k]), "force_fx": [int(v) for v in h["force_fx"][k]], "torque_fx": [int(v) for v in h["torque_fx"][k]]}


def pose(h, k=-1):
    return {name: tuple(float(v) for v in h[name][k]) for name in ("centre", "rotation", "velocity", "angular_velocity")}


def assert_integrated(before, h, gravity, dims, k=-1):
    want = body_ref.integrate(before, h["force_fx"][k], h["torque_fx"][k], DT, gravity, dims)
    got = pose(h, k)
    for name in got:
        assert np.array_equal(np.float32(got[name]), np.float32(want[name])), (name, got[name], want[name])


# ---- 1. nothing changes without bodies --------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("path", ["scatter", "gather"])
def test_cleared_bodies_change_nothing(tmp_path, path, graph):
    runs = []
    for had in (False, True):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
        f.set_transfer_path(path)
        f.set_graph_replay(graph)
        if had:
            f.set_bodies([body_ref.body(centre=(16, 20, 16), half_extent=(3, 3, 3)), body_ref.body("sphere", 4, 2.0, (10, 10, 10))])
            f.set_bodies([])
        for _ in range(70):
            f.step(DT)
            f.synchronize()
        save = str(tmp_path / f"{int(had)}.blub")
        f.save_state(save)
        runs.append((snapshot(f), open(save, "rb").read()))
    assert_same_physics(runs[0][0], runs[1][0])
    assert np.array_equal(bits(runs[0][0]["particles_position"]), bits(runs[1][0]["particles_position"]))
    assert runs[0][1] == runs[1][1]


# ---- 2. / 3. composite volume, marker and loads bit for bit --------------------------------------------------------------------
def test_composite_marker_loads_and_integration_match_the_restatement(tmp_path):
    import torch
    f = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
    solid = Solid(f, BOX)
    f.set_bodies(DOUBLE_DAM_BODIES)
    dims = f.grid_dimension()
    for _ in range(12):
        solid.step()
    state = str(tmp_path / "s.blub")
    f.save_state(state)
    before = f.bodies()
    # a probe around body 0 alone (two cells beyond its bounding box), pivot at its centre
    e, c = body_ref.bounding_extents(before[0]), np.float32(before[0]["centre"])
    f.set_load_probes([(np.floor(c - e) - 2, np.ceil(c + e) + 2, c)])
    solid.voxelize()
    f.step_stages(DT, 0, 1)
    borrowed = solid.vol.cpu().numpy()
    want = body_ref.composite(dims, borrowed, before)
    got = f.download_solid_voxels()
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))
    assert np.array_equal(borrowed, solid.vol.cpu().numpy())  # the borrowed volume is never written
    # the marker: a twin without bodies whose borrowed volume is the restated composite volume
    twin = blub_b200.HybridFluid.from_state(state)
    twin.set_bodies([])
    vol = torch.from_numpy(want).cuda()
    torch.cuda.synchronize()
    twin.set_solid_voxels(vol.data_ptr())
    twin.step_stages(DT, 0, 1)
    assert np.array_equal(f.download_grid(F.TAP_MARKER), twin.download_grid(F.TAP_MARKER))
    # stage 2: the sums on the marker and pressure of the velocity solve, the probe holding body 0 alone, the integration
    f.step_stages(DT, 1, 3)
    marker, p_vel = f.download_grid(F.TAP_MARKER), f.download_grid(F.TAP_P_VEL)
    for i, b in enumerate(before):
        h = f.body_history(i, 1)
        assert h["step"].tolist() == [12]
        assert record(h) == body_ref.loads(marker, p_vel, INV_DT, b), i
        assert record(h)["wetted_faces"] > 0
        assert_integrated(b, h, SCENE_G, dims)
    assert record(f.load_history(0, 1)) == record(f.body_history(0, 1))
    f.step_stages(DT, 3, 14)


# ---- 4. the integrator over a floating run ---------------------------------------------------------------------------------
def test_every_recorded_pose_is_the_restated_integration_of_the_previous_one():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
    f.set_bodies(DOUBLE_DAM_BODIES)
    dims = f.grid_dimension()
    prev = f.bodies()
    for step in range(200):
        f.step(DT)
        for i in range(len(prev)):
            h = f.body_history(i, 1)
            assert h["step"].tolist() == [step]
            assert_integrated(prev[i], h, SCENE_G, dims)
        prev = f.bodies()
    assert max(abs(b["velocity"][1]) for b in prev) > 0.0


# ---- 5. free fall, rest, sinking ---------------------------------------------------------------------------------------------
def test_a_box_falls_freely_and_rests_on_the_floor():
    f = blub_b200.HybridFluid(64, 64, 64, 1000)
    g = (0.0, -981.0, 0.0)
    f.set_gravity_grid(g)
    b = body_ref.body("box", (4, 3, 5), 0.7, (30, 50, 30), velocity=(5, 0, 0))
    f.set_bodies([b])
    for step in range(60):
        f.step(DT)
        h = f.body_history(0, 1)
        assert record(h) == {"wetted_faces": 0, "force_fx": [0, 0, 0], "torque_fx": [0, 0, 0]}
        b = body_ref.integrate(b, (0, 0, 0), (0, 0, 0), DT, g, (64, 64, 64))
        assert pose(h) == {k: b[k] for k in ("centre", "rotation", "velocity", "angular_velocity")}, step
    assert b["centre"][1] == float(np.float32(1) + np.float32(3)) and b["velocity"][1] == 0.0


N, H, G = 64, 32, 981.0


def tank(lo, hi, rho, solver=True):
    f = blub_b200.HybridFluid(N, N, N, 8 * N * N * H)
    f.set_gravity_grid((0.0, -G, 0.0))
    seed_around(f, H + 1, lo, (hi[0], min(hi[1], H + 1), hi[2]))  # no particle starts inside the body
    if solver:
        for which in (0, 1):
            f.set_solver_config(which, 1e-5, 4000, 4)
    half = [(h - l) / 2 for l, h in zip(lo, hi)]
    f.set_bodies([body_ref.body("box", half, rho, [(l + h) / 2 for l, h in zip(lo, hi)])])
    return f


def test_a_heavy_box_sinks_and_rests_on_the_floor():
    """It sinks and comes to rest near the floor.  Measured on an H100: from a bottom at y = 20 to 2.4 - 2.7 after 500 steps, on a fluid film of
    about 1.5 cells that the discrete projection does not drain (the composite velocity of a resting body is 0, so the film is not squeezed)."""
    f = tank((29, 20, 29), (35, 28, 35), 2.0, solver=False)
    for _ in range(500):
        f.step(DT)
    bottom = f.body_history(0, 100)["centre"][:, 1] - np.float32(4.0)
    assert bottom.max() < 3.0 and bottom.max() - bottom.min() < 0.5, bottom[::10].tolist()


# ---- 6. Archimedes -------------------------------------------------------------------------------------------------------------
def surface(marker, cx, cz):
    """One cell above the top FLUID cell (discrete hydrostatics), averaged over the columns at least 12 cells from the body's axis."""
    fluid = marker == 1
    ys = np.arange(marker.shape[1])[None, :, None]
    top = np.where(fluid, ys, -1).max(axis=1)  # [z, x]
    z, x = np.meshgrid(np.arange(marker.shape[0]), np.arange(marker.shape[2]), indexing="ij")
    far = (np.maximum(abs(x + 0.5 - cx), abs(z + 0.5 - cz)) > 12) & (top > 0)
    return float(top[far].mean()) + 1.0


@pytest.mark.parametrize("rho", [0.5, 0.75])
def test_a_floating_box_finds_the_discrete_hydrostatic_draft(rho):
    draft = 8 * rho - 1
    bottom = H + 1 - draft
    f = tank((24, int(bottom), 24), (40, int(bottom) + 8, 40), rho)
    drafts, tilts = [], []
    for step in range(400):
        f.step(DT)
        if step >= 300:
            b = f.bodies()[0]
            drafts.append(surface(f.download_grid(F.TAP_MARKER), b["centre"][0], b["centre"][2]) - (b["centre"][1] - 4.0))
            R = body_ref.rotation(b["rotation"])
            tilts.append(np.degrees(np.arccos(min(1.0, float(R[1][1])))))
    assert abs(np.mean(drafts) - draft) < 1.5, (np.mean(drafts), draft, drafts[::10])
    assert max(tilts) < 5.0


# ---- 7. reproducibility --------------------------------------------------------------------------------------------------------
def test_two_runs_and_graph_against_eager_are_bit_identical():
    runs = []
    for graph in (True, True, False):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
        f.set_graph_replay(graph)
        f.set_bodies(DOUBLE_DAM_BODIES)
        for _ in range(100):
            f.step(DT)
        runs.append((snapshot(f), [f.body_history(i) for i in range(2)]))
    for other in runs[1:]:
        assert_same_physics(runs[0][0], other[0], stats=False)
        for ha, hb in zip(runs[0][1], other[1]):
            for name in ha:
                assert np.array_equal(ha[name], hb[name]), name


# ---- 8. checkpoint -------------------------------------------------------------------------------------------------------------
def test_a_saved_fluid_with_bodies_flow_and_tags_resumes_bit_for_bit(tmp_path):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    f.set_bodies([body_ref.body("box", (3, 2, 4), 0.5, (20, 18, 14), S30), body_ref.body("sphere", 3, 1.5, (10, 24, 20))])
    f.paint_tags((1, 1, 1), (16, 31, 31), 7)
    for _ in range(20):
        f.step(DT)
    state = str(tmp_path / "s.blub")
    f.save_state(state)
    assert F.state_info(state).format_version == 8
    g = blub_b200.HybridFluid.from_state(state)
    assert g.bodies() == f.bodies() and len(g.body_history(0)["step"]) == 0
    for _ in range(20):  # past the re-sorts of steps 24 and 32
        f.step(DT)
        g.step(DT)
    a, b = snapshot(f), snapshot(g)
    assert_same_physics(a, b, stats=False)
    assert np.array_equal(bits(a["particles_position"]), bits(b["particles_position"]))
    assert g.bodies() == f.bodies()
    for i in range(2):
        hf, hg = f.body_history(i, 20), g.body_history(i)
        for name in hf:
            assert np.array_equal(hf[name], hg[name]), name


# ---- 9. refusals ---------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    good = [body_ref.body(centre=(16, 20, 16), half_extent=(3, 3, 3))]
    f.set_bodies(good)
    f.step(DT)
    before, hist = f.bodies(), f.body_history(0)
    bad = [[good[0]] * 17, [dict(good[0], shape=2)], [dict(good[0], half_extent=(0.5, 3, 3))], [dict(good[0], relative_density=0.0)],
           [dict(good[0], rotation=(1.01, 0, 0, 0))], [dict(good[0], centre=(3, 20, 16))], [dict(good[0], velocity=(float("nan"), 0, 0))]]
    for b in bad:
        with pytest.raises(F.BlubError):
            f.set_bodies(b)
    f.step_stages(DT, 0, 3)
    with pytest.raises(F.BlubError):
        f.set_bodies(good)
    f.step_stages(DT, 3, 14)
    with pytest.raises(F.BlubError):
        f.body_history(1)
    assert len(f.body_history(0)["step"]) == 2 and f.body_history(0)["step"][0] == hist["step"][0]
    assert f.bodies() != before  # two steps moved it; the refused sets did not replace it
    assert body_ref.normalised((1.0005, 0, 0, 0)) == (1.0, 0.0, 0.0, 0.0)
    f.set_bodies([dict(good[0], rotation=(1.0005, 0, 0, 0))])
    assert f.bodies()[0]["rotation"] == (1.0, 0.0, 0.0, 0.0)


# ---- 10. the runner ------------------------------------------------------------------------------------------------------------
def test_runner_bodies_equal_a_ctypes_run(tmp_path):
    sc = json.load(open(util.scene_path("dam_small")))
    v3 = lambda x, y, z: {"x": x, "y": y, "z": z}  # noqa: E731
    sc["fluid"]["bodies"] = [{"shape": "box", "position": v3(0.1, 0.12, 0.16), "half_extent": v3(0.03, 0.02, 0.04), "relative_density": 0.6,
                              "rotation_angles_deg": v3(0.0, 20.0, 0.0)},
                             {"shape": "sphere", "position": v3(0.24, 0.2, 0.16), "half_extent": 0.03, "relative_density": 1.5}]
    scene = str(tmp_path / "bodies.json")
    json.dump(sc, open(scene, "w"))
    steps = 1100
    out = str(tmp_path / "bodies_out.json")
    r = subprocess.run([RUNNER, scene, "--steps", str(steps), "--bodies", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    state, out2 = str(tmp_path / "s.blub"), str(tmp_path / "bodies2.json")
    r = subprocess.run([RUNNER, scene, "--steps", "600", "--save-state", state], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([RUNNER, scene, "--steps", str(steps - 600), "--load-state", state, "--bodies", out2], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    f = blub_b200.HybridFluid.from_scene(scene)
    got = [[], []]
    for k in range(steps):
        f.step(DT)
        if (k + 1) % 500 == 0 or k + 1 == steps:
            for i in range(2):
                h = f.body_history(i)
                for j in range(len(h["step"])):
                    if not got[i] or h["step"][j] > got[i][-1]["step"]:
                        got[i].append({"step": int(h["step"][j]), "centre": [float(v) for v in h["centre"][j]],
                                       "rotation": [float(v) for v in h["rotation"][j]], "force": h["force"][j].tolist()})
    for run, first in ((json.load(open(out)), 0), (json.load(open(out2)), 600)):
        assert len(run["bodies"]) == 2
        for body, want in zip(run["bodies"], got):
            recs = body["records"]
            assert [r_["step"] for r_ in recs] == list(range(first, steps))
            for r_, w in zip(recs, want[first:]):  # poses written with 9 significant digits: the float32 values round-trip
                assert np.array_equal(np.float32(r_["centre"]), np.float32(w["centre"])) and np.array_equal(np.float32(r_["rotation"]), np.float32(w["rotation"]))
                assert r_["force"] == w["force"]
