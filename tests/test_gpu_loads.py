"""GPU: solid load probes (DESIGN.md §8, "Solid load probes").  Probes change no result of a step; every record agrees bit for bit with the
NumPy restatement (tests/load_ref.py) on the marker and pressure the velocity solve used; a converged hydrostatic tank gives the discrete
hydrostatic wall force and lift; a box pushed into still water feels a force against its motion; the ring keeps the newest 1024 records;
refusals change nothing; probes are not state; and the runner's --loads history equals a ctypes-driven run's."""
import json
import os
import subprocess

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import load_ref, util
from tests.test_gpu_state import snapshot
from tests.test_gpu_tags import assert_same_physics, bits
from tests.util import DT

pytestmark = pytest.mark.gpu

RUNNER = os.path.join(os.path.dirname(F.lib_path()), "blub_run")
INV_DT = np.float32(1.0) / np.float32(DT)  # StepParams::inv_dt
# bench.py's double_dam_box solid: a 24 x 40 x 24-cell box travelling +x about the middle of the basin
BOX = {"world_position": [0.44, 0.20, 0.32], "scale": 1.0, "rotation_angles": [0.0, 0.0, 0.0], "shape": "box", "half_extent": [0.12, 0.20, 0.12],
       "translation": {"target": [0.84, 0.20, 0.32], "curve": "SmoothStep", "duration": 2.0}}


class Solid:
    """Scene::step with one analytic solid: advance the clock, voxelize on the fluid's stream, then the caller steps the fluid."""

    def __init__(self, f, obj, scale=0.01):
        import torch
        self.f, self.obj, self.scale, self.t = f, obj, scale, 0.0
        self.dims = f.grid_dimension()
        self.vol = torch.zeros((self.dims[2], self.dims[1], self.dims[0], 4), dtype=torch.float16, device="cuda:0")
        torch.cuda.synchronize()
        f.set_solid_voxels(self.vol.data_ptr())

    def voxelize(self):
        self.t += DT
        F.solid_voxelize(self.vol.data_ptr(), self.dims, self.obj, self.scale, (0.0, 0.0, 0.0), self.t, DT, cuda_stream=self.f.stream())

    def step(self):
        self.voxelize()
        self.f.step(DT)


def record(h, k=-1):
    return {"wetted_faces": int(h["wetted_faces"][k]), "force_fx": [int(v) for v in h["force_fx"][k]], "torque_fx": [int(v) for v in h["torque_fx"][k]]}


def assert_records_match_the_restatement(f, probes, step):
    """The newest record of every probe against load_ref on the marker and pressure as they are after stage 2 (or 3)."""
    marker, p_vel = f.download_grid(F.TAP_MARKER), f.download_grid(F.TAP_P_VEL)
    dims = f.grid_dimension()
    for k, probe in enumerate(probes):
        h = f.load_history(k, 1)
        assert h["step"].tolist() == [step]
        lo, hi = F.load_probe_cells(dims, probe)
        pivot = probe[2] if len(probe) > 2 else (np.float32(probe[0]) + np.float32(probe[1])) * np.float32(0.5)
        assert record(h) == load_ref.solid_loads(marker, p_vel, INV_DT, lo, hi, pivot), (k, step)


def history_equal(a, b, num_probes):
    for k in range(num_probes):
        ha, hb = a.load_history(k), b.load_history(k)
        for name in ("step", "wetted_faces", "force_fx", "torque_fx"):
            assert np.array_equal(ha[name], hb[name]), (k, name)


def sixteen_probes(dims, seed):
    rng = np.random.default_rng(seed)
    probes = [((0, 0, 0), tuple(dims)), ((0, 0, 0), (1, dims[1], dims[2])), ((0, 0, 0), (dims[0], 1, dims[2]))]
    while len(probes) < 16:
        lo = rng.uniform(-2, np.array(dims) - 2)
        hi = lo + rng.uniform(1, 20, 3)
        probes.append((tuple(lo), tuple(hi), tuple(rng.uniform(-10, 40, 3))))
    return probes


# ---- 1. probes change nothing --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("path", ["scatter", "gather"])
@pytest.mark.parametrize("scene", ["tap_small", "dam_halfhalf"])
def test_probes_change_nothing(tmp_path, scene, path, graph):
    """70 steps with 16 probes against a twin with none: every result and the saved state bit-identical.  Both fluids synchronise after
    every step, so that the solver statistics they keep do not depend on host timing."""
    runs = []
    for probed in (False, True):
        f = blub_b200.HybridFluid.from_scene(util.scene_path(scene))
        f.set_transfer_path(path)
        f.set_graph_replay(graph)
        if probed:
            f.set_load_probes(sixteen_probes(f.grid_dimension(), 3))
        for _ in range(70):
            f.step(DT)
            f.synchronize()
        save = str(tmp_path / f"{int(probed)}.blub")
        f.save_state(save)
        runs.append((f, snapshot(f), open(save, "rb").read()))
    assert_same_physics(runs[0][1], runs[1][1])
    assert np.array_equal(bits(runs[0][1]["particles_position"]), bits(runs[1][1]["particles_position"]))
    assert runs[0][2] == runs[1][2]
    h = runs[1][0].load_history(0)
    assert h["step"].tolist() == list(range(70)) and h["wetted_faces"].min() > 0


# ---- 2. bit for bit against the restatement -------------------------------------------------------------------------------
DOUBLE_DAM_PROBES = [
    ((28, 1, 18), (100, 42, 46)),               # the box's path
    ((0, 0, 0), (1, 64, 64)),                   # the x = 0 tank wall: border cells
    ((4, 30, 4), (20, 50, 20)),                 # no solid inside
    ((28, 1, 18), (64, 42, 46)),                # two overlapping boxes
    ((50, 1, 18), (100, 42, 46)),
    ((28, 1, 18), (100, 42, 46), (0.0, 0.0, 0.0)),  # an off-centre pivot
    ((0, 0, 0), (128, 1, 64)),                  # the floor
    ((-10, -10, -10), (1000, 1000, 1000)),      # the whole grid
]


def test_double_dam_box_records_match_the_restatement_and_a_graph_twin():
    staged = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
    twin = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
    solids = [Solid(staged, BOX), Solid(twin, BOX)]
    for f in (staged, twin):
        f.set_load_probes(DOUBLE_DAM_PROBES)
    chosen = {0, 5, 30, 61}
    for step in range(62):
        solids[1].step()
        if step in chosen:
            solids[0].voxelize()
            staged.step_stages(DT, 0, 3)
            assert_records_match_the_restatement(staged, DOUBLE_DAM_PROBES, step)
            staged.step_stages(DT, 3, 14)
        else:
            solids[0].step()
    history_equal(staged, twin, len(DOUBLE_DAM_PROBES))
    h = [staged.load_history(k) for k in range(len(DOUBLE_DAM_PROBES))]
    assert h[0]["step"].tolist() == list(range(62))
    assert h[0]["wetted_faces"].min() > 0 and h[1]["wetted_faces"].min() > 0 and not h[2]["wetted_faces"].any()
    assert np.array_equal(h[0]["force_fx"], h[5]["force_fx"]) and not np.array_equal(h[0]["torque_fx"], h[5]["torque_fx"])
    assert (h[1]["force_fx"][:, 0] <= 0).all() and (h[1]["force_fx"][:, 1:] == 0).all()  # water pushes the x = 0 wall towards -x
    assert (h[6]["force_fx"][1:, 1] < 0).all()  # and the floor down


def test_tap_small_records_match_the_restatement_on_the_device_count():
    probes = [((0, 0, 0), (32, 1, 32)), ((31, 0, 0), (32, 32, 32), (0.0, 0.0, 0.0)), ((0, 0, 0), (32, 32, 32)), ((10, 0, 10), (20, 3, 20))]
    staged = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    twin = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    assert staged.has_flow
    for f in (staged, twin):
        f.set_load_probes(probes)
    for step in range(12):
        twin.step(DT)
        if step in (0, 3, 9):
            staged.step_stages(DT, 0, 3)
            assert_records_match_the_restatement(staged, probes, step)
            staged.step_stages(DT, 3, 14)
        else:
            staged.step(DT)
    history_equal(staged, twin, len(probes))


# ---- 3. discrete hydrostatics ---------------------------------------------------------------------------------------------
N, H, G = 64, 32, 981.0
BOX_LO, BOX_HI = (24, 8, 24), (40, 16, 40)  # 16 x 8 x 16 solid cells, fully submerged


def seed_around(f, top, lo, hi):
    """Fills cells y in [1, top) except the box [lo, hi): no particle starts inside the solid."""
    n = f.grid_dimension()
    cubes = [((1, 1, 1), (n[0] - 1, lo[1], n[2] - 1)), ((1, hi[1], 1), (n[0] - 1, top, n[2] - 1)),
             ((1, lo[1], 1), (lo[0], hi[1], n[2] - 1)), ((hi[0], lo[1], 1), (n[0] - 1, hi[1], n[2] - 1)),
             ((lo[0], lo[1], 1), (hi[0], hi[1], lo[2])), ((lo[0], lo[1], hi[2]), (hi[0], hi[1], n[2] - 1))]
    for mn, mx in cubes:
        f.add_fluid_cube(mn, mx)


def test_converged_hydrostatic_tank_gives_the_discrete_hydrostatic_loads():
    """64^3 tank filled to H = 32 cells around a static submerged box, both solves converged (1e-5, up to 4000 iterations), step 0.
    Discrete hydrostatics (free surface one cell above the top fluid cell): the +x wall carries |g| (nz - 2) H (H + 1) / 2, the box's lift is
    |g| (V + A).  The 1e-3 tolerances are generous: measured on an H100 80GB HBM3 (196 iterations), the wall force is off by 4.7e-7 and the
    lift by 5.1e-6 (relative), the horizontal box forces are 2.2e-8 of the lift and the torque about the box centre 8.4e-9 of lift x 16 cells."""
    import torch
    f = blub_b200.HybridFluid(N, N, N, 8 * N * N * H)
    f.set_gravity_grid((0.0, -G, 0.0))
    seed_around(f, H + 1, BOX_LO, BOX_HI)
    vol = torch.zeros((N, N, N, 4), dtype=torch.float16, device="cuda:0")
    vol[BOX_LO[2]:BOX_HI[2], BOX_LO[1]:BOX_HI[1], BOX_LO[0]:BOX_HI[0], 3] = 1.0
    torch.cuda.synchronize()
    f.set_solid_voxels(vol.data_ptr())
    util.tight_solver(f, tol=1e-5, max_it=4000)
    centre = tuple(0.5 * (a + b) for a, b in zip(BOX_LO, BOX_HI))
    shift = np.array([3.0, -2.0, 5.0])
    f.set_load_probes([((N - 1, 0, 0), (N, N, N)), ((20, 4, 20), (44, 20, 44), centre), ((20, 4, 20), (44, 20, 44), tuple(np.array(centre) + shift))])
    f.step(DT)
    _, its = f.last_solve(0)
    assert its < 4000
    wall, box, shifted = (f.load_history(k) for k in range(3))
    want_wall = G * (N - 2) * H * (H + 1) / 2
    e_wall = abs(wall["force"][0, 0] - want_wall) / want_wall
    ext = [b - a for a, b in zip(BOX_LO, BOX_HI)]
    want_lift = G * (ext[0] * ext[1] * ext[2] + ext[0] * ext[2])
    force = box["force"][0]
    e_lift = abs(force[1] - want_lift) / want_lift
    e_side = max(abs(force[0]), abs(force[2])) / want_lift
    e_torque = np.abs(box["torque"][0]).max() / (want_lift * max(ext))
    print(f"\nhydrostatics: wall {e_wall:.3e}, lift {e_lift:.3e}, sides {e_side:.3e}, torque {e_torque:.3e}, {its} iterations")
    assert wall["wetted_faces"][0] == (N - 2) * H and e_wall <= 1e-3
    assert e_lift <= 1e-3 and e_side <= 1e-3 and e_torque <= 1e-3
    # about a shifted pivot: tau' = tau - (pivot' - centre) x F
    want = box["torque"][0] - np.cross(shift, force)
    assert np.abs(shifted["torque"][0] - want).max() <= 1e-5 * np.abs(force).max() * (np.abs(shift).max() + max(ext))
    assert np.array_equal(shifted["force_fx"], box["force_fx"])


# ---- 4. sign --------------------------------------------------------------------------------------------------------------
def test_a_box_driven_into_still_water_feels_a_force_against_its_motion():
    """A submerged 12^3-cell box moves +x at 48 cells/s through still water: on average over the push the water pushes it towards -x."""
    f = blub_b200.HybridFluid(N, N, N, 8 * N * N * 40)
    f.set_gravity_grid((0.0, -G, 0.0))
    seed_around(f, 41, (14, 14, 26), (26, 26, 38))
    obj = {"world_position": [0.20, 0.20, 0.32], "shape": "box", "half_extent": [0.06, 0.06, 0.06],
           "translation": {"target": [0.44, 0.20, 0.32], "curve": "Linear", "duration": 0.5}}
    solid = Solid(f, obj)
    f.set_load_probes([((8, 1, 1), (56, 63, 63))])
    for _ in range(60):
        solid.step()
    h = f.load_history(0)
    fx = h["force"][:, 0]
    print(f"\nsign: mean F_x {fx.mean():.4g} (steps 1..59: {fx[1:].mean():.4g}), mean F_y {h['force'][:, 1].mean():.4g}")
    assert h["wetted_faces"].min() > 0 and fx.mean() < 0


# ---- 5. ring ---------------------------------------------------------------------------------------------------------------
def test_the_ring_keeps_the_newest_1024_records():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    probes = [((0, 0, 0), (32, 1, 32)), ((0, 0, 0), (1, 32, 32))]
    f.set_load_probes(probes)
    for _ in range(20):
        f.step(DT)
    h = f.load_history(0)
    assert h["step"].tolist() == list(range(20))
    for _ in range(1080):
        f.step(DT)
    h = f.load_history(1)
    assert len(h["step"]) == F.LOAD_HISTORY_LENGTH and h["step"].tolist() == list(range(1100 - 1024, 1100))
    last = f.load_history(1, 10)
    assert last["step"].tolist() == list(range(1090, 1100)) and np.array_equal(last["force_fx"], h["force_fx"][-10:])
    assert f.load_history(0, 0)["step"].size == 0
    # a refused call leaves the old set recording
    with pytest.raises(blub_b200.BlubError):
        f.set_load_probes([((0, 0, 0), (32, 1, 32)), ((5, 5, 5), (5, 6, 6))])
    f.step(DT)
    assert f.load_history(1)["step"][-1] == 1100 and len(f.load_history(1)["step"]) == 1024
    # a new set starts a new history
    f.set_load_probes(probes[:1])
    assert f.load_history(0)["step"].size == 0
    with pytest.raises(blub_b200.BlubError):
        f.load_history(1)
    f.step(DT)
    assert f.load_history(0)["step"].tolist() == [1101]
    f.set_load_probes([])
    f.step(DT)
    with pytest.raises(blub_b200.BlubError):
        f.load_history(0)


# ---- 6. refusals, save and load -------------------------------------------------------------------------------------------
def test_refusals_change_nothing():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    good = [((0, 0, 0), (32, 1, 32))]
    f.set_load_probes(good)
    f.step(DT)
    nan, inf = float("nan"), float("inf")
    bad = [good * 17, [((0, nan, 0), (4, 4, 4))], [((0, 0, 0), (4, inf, 4))], [((0, 0, 0), (4, 4, 4), (0, 0, nan))],
           [((0, 0, 0), (4, 4, 4), (inf, 0, 0))], [((3, 3, 3), (3, 9, 9))], [((40, 0, 0), (50, 4, 4))], [((-9, 0, 0), (0, 4, 4))]]
    for probes in bad:
        with pytest.raises(blub_b200.BlubError):
            f.set_load_probes(probes)
    with pytest.raises(blub_b200.BlubError):
        f.load_history(1)
    f.step_stages(DT, 0, 3)
    with pytest.raises(blub_b200.BlubError):
        f.set_load_probes(good)
    assert b"inside a step" in F.lib().blub_last_error()
    assert f.load_history(0)["step"].tolist() == [0, 1]  # readable inside a step: stage 2 has recorded step 1
    f.step_stages(DT, 3, 14)
    f.step(DT)
    assert f.load_history(0)["step"].tolist() == [0, 1, 2]
    slab = blub_b200.HybridFluid.create_slab(32, 32, 16, 1000, 0, 2)
    with pytest.raises(blub_b200.BlubError):
        slab.set_load_probes(good)
    assert b"z-slab" in F.lib().blub_last_error()


def test_probes_are_not_state(tmp_path):
    """A save with probes is the save without them; the loaded fluid has none, continues bit for bit and takes new ones."""
    a = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    b = blub_b200.HybridFluid.from_scene(util.scene_path("tap_small"))
    a.set_load_probes([((0, 0, 0), (32, 1, 32))])
    for _ in range(6):
        for f in (a, b):
            f.step(DT)
            f.synchronize()
    pa, pb = str(tmp_path / "a.blub"), str(tmp_path / "b.blub")
    a.save_state(pa)
    b.save_state(pb)
    assert open(pa, "rb").read() == open(pb, "rb").read()
    c = blub_b200.HybridFluid.from_state(pa)
    with pytest.raises(blub_b200.BlubError):
        c.load_history(0)
    for _ in range(4):  # crosses the re-sort at step 8
        for f in (a, c):
            f.step(DT)
            f.synchronize()
    assert_same_physics(snapshot(a), snapshot(c))
    c.set_load_probes([((0, 0, 0), (32, 1, 32))])
    c.step(DT)
    a.step(DT)
    assert c.load_history(0)["step"].tolist() == [10]
    assert record(c.load_history(0)) == record(a.load_history(0))


# ---- 7. runner -------------------------------------------------------------------------------------------------------------
def test_runner_loads_equal_a_ctypes_run(tmp_path):
    sc = json.load(open(util.scene_path("dam_small")))
    v3 = lambda x, y, z: {"x": x, "y": y, "z": z}  # noqa: E731
    sc["fluid"]["load_probes"] = [{"min": v3(0.0, 0.0, 0.0), "max": v3(0.32, 0.01, 0.32)},
                                  {"min": v3(0.31, 0.0, 0.0), "max": v3(0.32, 0.32, 0.32), "pivot": v3(0.32, 0.0, 0.16)}]
    scene = str(tmp_path / "probed.json")
    json.dump(sc, open(scene, "w"))
    steps = 1100
    out = str(tmp_path / "loads.json")
    r = subprocess.run([RUNNER, scene, "--steps", str(steps), "--loads", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # a resumed run sets the scene's probes again
    state, out2 = str(tmp_path / "s.blub"), str(tmp_path / "loads2.json")
    r = subprocess.run([RUNNER, scene, "--steps", "600", "--save-state", state], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([RUNNER, scene, "--steps", str(steps - 600), "--load-state", state, "--loads", out2], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # the ctypes-driven run, reading the history every 500 steps
    f = blub_b200.HybridFluid.from_scene(scene)
    probes = F.scene_load_probes(scene)
    got = [[] for _ in probes]
    for k in range(steps):
        f.step(DT)
        if (k + 1) % 500 == 0 or k + 1 == steps:
            for p in range(len(probes)):
                h = f.load_history(p)
                for i in range(len(h["step"])):
                    if not got[p] or h["step"][i] > got[p][-1]["step"]:
                        got[p].append({"step": int(h["step"][i]), "wetted_faces": int(h["wetted_faces"][i]), "force": h["force"][i].tolist(),
                                       "torque": h["torque"][i].tolist()})
    runner = json.load(open(out))
    assert len(runner["probes"]) == len(probes)
    for p, (probe, want) in enumerate(zip(runner["probes"], got)):
        for key, want_v in zip(("min", "max", "pivot"), probes[p]):  # written with 9 significant digits: the float32 values round-trip
            assert np.array_equal(np.float32(probe[key]), np.float32(want_v)), key
        assert [r_["step"] for r_ in probe["records"]] == list(range(steps))
        assert probe["records"] == want
    resumed = json.load(open(out2))
    for probe, want in zip(resumed["probes"], got):
        assert probe["records"] == want[600:]
