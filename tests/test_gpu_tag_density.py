"""Liquids of different densities on the GPU (DESIGN.md §8 "Liquids of different densities"): a table set and cleared leaves no trace, a table of
ones is solver path 6 bit for bit, stage 0, stage 4 and the weighted solve against the restatement in tests/tag_density_ref.py, the physics
of layered and inverted liquids and of spheres, repeatability, save and load, refusals and the runner."""
import json
import os
import subprocess

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import tag_density_ref as T
from tests import util
from tests.test_gpu_density_fuse import SOLID

pytestmark = pytest.mark.gpu

DT = F.DT_120HZ
RUNNER = os.path.join(os.path.dirname(F.lib_path()), "blub_run")
GRID_TAPS = (F.TAP_UX, F.TAP_UY, F.TAP_UZ, F.TAP_MARKER, F.TAP_P_VEL, F.TAP_P_DEN)
PARTICLE_TAPS = (F.TAP_POS, F.TAP_VX, F.TAP_VY, F.TAP_VZ)
G = float(np.float32(-9.81) / np.float32(0.01))  # the scenes' gravity in cells/s^2


def taps(f):
    f.synchronize()
    return [f.download_grid(t).tobytes() for t in GRID_TAPS] + [f.download_particles(t).tobytes() for t in PARTICLE_TAPS]


def same_taps(a, b, what):
    names = [str(t) for t in GRID_TAPS] + ["p" + str(t) for t in PARTICLE_TAPS]
    bad = [n for n, x, y in zip(names, taps(a), taps(b)) if x != y]
    assert not bad, f"{what}: taps {bad} differ"


def scene_fluid(name, scatter=True, graph=True):
    f = blub_b200.HybridFluid.from_scene(util.scene_path(name))
    f.set_transfer_path(scatter)
    f.set_graph_replay(graph)
    return f


# --- 1. off leaves no trace --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("scatter", [True, False], ids=["scatter", "gather"])
@pytest.mark.parametrize("graph", [True, False], ids=["graph", "eager"])
def test_a_table_set_and_cleared_leaves_no_trace(scatter, graph, tmp_path):
    ref, cleared = scene_fluid("dam_small", scatter, graph), scene_fluid("dam_small", scatter, graph)
    cleared.set_tag_densities({0: 0.5, 3: 2.0})
    cleared.set_tag_densities({})
    assert cleared.tag_densities() == {}
    for k in range(30):
        ref.step(DT)
        cleared.step(DT)
        if k == 12:  # on, one step, off
            cleared.set_tag_densities({0: 1.5})
            cleared.set_tag_densities({})
    same_taps(ref, cleared, "cleared table")
    assert not cleared.download_grid(F.TAP_CELL_DENSITY).any()
    ref.save_state(str(tmp_path / "a.blub"))
    cleared.save_state(str(tmp_path / "b.blub"))
    assert open(tmp_path / "a.blub", "rb").read() == open(tmp_path / "b.blub", "rb").read()


# --- 2. a table of ones against path 6 -----------------------------------------------------------------------------------------------

class DoubleDam:
    """double_dam with its moving box, a flow set and viscosity (floating bodies are refused with a table)."""

    def __init__(self, f):
        import torch

        sc = json.load(open(util.scene_path("double_dam")))
        d = sc["fluid"]["grid_dimension"]
        self.f, self.dims, self.scale = f, (d["x"], d["y"], d["z"]), sc["fluid"]["grid_to_world_scale"]
        self.origin = [sc["fluid"]["world_position"][c] for c in "xyz"]
        self.vol = torch.zeros((d["z"], d["y"], d["x"], 4), dtype=torch.float16, device="cuda:0")
        torch.cuda.synchronize()
        f.set_solid_voxels(self.vol.data_ptr())
        f.set_flow([((60, 40, 30), (64, 44, 34), (0.0, -20.0, 0.0), 7)], [((2, 1, 2), (6, 4, 6))])
        f.set_viscosity(2.0)
        self.k = 0

    def step(self):
        F.solid_voxelize(self.vol.data_ptr(), self.dims, SOLID, self.scale, self.origin, (self.k + 1) * DT, DT, cuda_stream=self.f.stream())
        self.f.step(DT)
        self.k += 1


def test_a_table_of_ones_solves_as_solver_path_6_iteration_by_iteration():
    a, b = scene_fluid("dam_small", graph=False), scene_fluid("dam_small", graph=False)
    for f in (a, b):
        f.set_solver_path(6)
    b.set_tag_densities({0: 1.0, 7: 1.0})
    for f in (a, b):
        f.step_stages(DT, 0, 2)
        f.synchronize()
    rhs = a.download_grid(F.TAP_RESIDUAL)
    assert rhs.tobytes() == b.download_grid(F.TAP_RESIDUAL).tobytes()
    for it in (0, 1, 2, 3, 8, 31):
        out = []
        for f in (a, b):
            f.set_solver_config(0, 1e-12, it, 4)
            f.upload_grid(F.TAP_RESIDUAL, rhs)
            f.upload_grid(F.TAP_P_VEL, np.zeros_like(rhs))
            f.solve_only(0)
            f.synchronize()
            out.append((f.download_grid(F.TAP_P_VEL).tobytes(), f.download_grid(F.TAP_RESIDUAL).tobytes(), f.last_solve_scalars(0)))
        assert out[0] == out[1], f"after iteration {it}"


@pytest.mark.parametrize("name", ["dam_small", "double_dam"])
def test_a_table_of_ones_is_solver_path_6_bit_for_bit(name):
    plain, ones = scene_fluid(name), scene_fluid(name)
    for f in (plain, ones):
        f.set_solver_path(6)
    ones.set_tag_densities({0: 1.0, 7: 1.0})
    if name == "double_dam":
        plain, ones = DoubleDam(plain), DoubleDam(ones)
        steps = [p.step for p in (plain, ones)]
        fluids = (plain.f, ones.f)
    else:
        steps = [lambda f=f: f.step(DT) for f in (plain, ones)]
        fluids = (plain, ones)
    for k in range(24):
        for s_ in steps:
            s_()
        same_taps(fluids[0], fluids[1], f"{name} step {k}")
    if name == "double_dam":
        assert fluids[1].flow_counters["emitted"] > 0


# --- 3. stages against the restatement ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("device_count", [False, True], ids=["host_count", "device_count"])
def test_stage_0_cell_density_is_the_restatement(device_count):
    f = scene_fluid("oil_water_small")
    if device_count:  # a drain far from the liquid puts the count on the device
        f.set_flow([], [((28, 28, 28), (30, 30, 30))])
    table = {1: 0.8, 5: 2.0, 9: 0.5}
    f.set_tag_densities(table)
    for _ in range(5):
        f.step(DT)
    pos = f.download_particles()
    rng = np.random.default_rng(3)
    tags = rng.choice(np.array([0, 1, 5, 9, 11, 0xFFFFFFFF], dtype=np.uint32), size=len(pos))  # 0, 11, 2^32 - 1: not in the table
    pos[:, 3] = tags.view(np.float32)
    f.set_particles(pos, f.download_particles(F.TAP_VX), f.download_particles(F.TAP_VY), f.download_particles(F.TAP_VZ))
    f.step_stages(DT, 0, 1)
    f.synchronize()
    marker = f.download_grid(F.TAP_MARKER)
    got = f.download_grid(F.TAP_CELL_DENSITY)
    want = T.cell_density(pos, tags, table, marker)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert len(np.unique(got[marker == T.FLUID])) > 10  # mixed cells
    f.step_stages(DT, 1, 14)
    # the order of the particles does not matter
    perm = rng.permutation(len(pos))
    shuffled = []
    for order in (np.arange(len(pos)), perm):
        g = scene_fluid("oil_water_small")
        g.set_tag_densities(table)
        g.set_particles(pos[order])
        g.step_stages(DT, 0, 1)
        g.synchronize()
        shuffled.append(g.download_grid(F.TAP_CELL_DENSITY))
        g.step_stages(DT, 1, 14)
    assert np.array_equal(shuffled[0].view(np.uint32), shuffled[1].view(np.uint32))
    assert np.array_equal(shuffled[0].view(np.uint32), want.view(np.uint32))


def test_stage_4_is_the_restatement_given_the_tapped_pressure():
    f = scene_fluid("oil_water_small")
    for _ in range(6):
        f.step(DT)
    f.step_stages(DT, 0, 3)
    f.synchronize()
    marker, p, rho = f.download_grid(F.TAP_MARKER), f.download_grid(F.TAP_P_VEL), f.download_grid(F.TAP_CELL_DENSITY)
    u = [f.download_grid(t) for t in (F.TAP_UX, F.TAP_UY, F.TAP_UZ)]
    beta, _, _ = T.coefficients(marker, rho)
    f.step_stages(DT, 3, 5)
    f.synchronize()
    got = [f.download_grid(t) for t in (F.TAP_UX, F.TAP_UY, F.TAP_UZ)]
    want, live = T.project32(u, marker, beta, p)
    for c in range(3):
        assert live[c].any()
        assert np.array_equal(got[c][live[c]].view(np.uint32), want[c][live[c]].view(np.uint32)), f"component {c}"
    f.step_stages(DT, 5, 14)


def test_the_weighted_solve_follows_the_float64_recurrence_iteration_by_iteration():
    f = scene_fluid("oil_water_small")
    f.set_tag_densities({1: 0.8, 0: 2.0})
    for _ in range(8):
        f.step(DT)
    f.step_stages(DT, 0, 2)
    f.synchronize()
    marker, rho, b = f.download_grid(F.TAP_MARKER), f.download_grid(F.TAP_CELL_DENSITY), f.download_grid(F.TAP_RESIDUAL)
    beta, D, inv = T.coefficients(marker, rho)
    fl = marker == T.FLUID
    ref = T.cg64(beta, D, inv, fl, b, np.zeros(b.shape), 9)
    worst = []
    for k in range(9):
        f.set_solver_config(0, 1e-12, k, 4)
        f.upload_grid(F.TAP_RESIDUAL, b)
        f.upload_grid(F.TAP_P_VEL, np.zeros(b.shape, np.float32))
        f.solve_only(0)
        f.synchronize()
        p = f.download_grid(F.TAP_P_VEL).astype(np.float64)
        alpha, _, sigma = (float(v) for v in f.last_solve_scalars(0))
        p64, alpha64, sigma64 = ref[k]
        err = float(np.abs(p - p64).max() / np.abs(p64).max())
        worst.append(err)
        # float32 against float64: the iterates drift apart by rounding, slowly; a wrong coefficient, diagonal or preconditioner factor
        # is off by O(1) from the first iteration on
        assert err <= 2e-5 * (k + 1), (k, err)
        assert abs(alpha - alpha64) <= 1e-4 * (k + 1) * abs(alpha64), (k, alpha, alpha64)
        assert abs(sigma - sigma64) <= 1e-4 * (k + 1) * abs(sigma64), (k, sigma, sigma64)
    print("MEASURED weighted solve against the float64 recurrence, relative max |p| error per iteration", [f"{e:.2e}" for e in worst])


# --- 4. physics ----------------------------------------------------------------------------------------------------------------------

def layered(lower, upper, table, n=64, depth=40, split=20):
    f = blub_b200.HybridFluid(n, n, n, 8 * (n - 2) * (n - 2) * depth + 1024)
    f.add_fluid_cube((1, 1, 1), (n - 1, split, n - 1), lower)
    f.add_fluid_cube((1, split, 1), (n - 1, depth, n - 1), upper)
    f.set_gravity_grid((0.0, G, 0.0))
    if table:
        f.set_tag_densities(table)
    return f


def gradient_ratio(f, split=20, depth=40):
    """Mean p(y) - p(y + 1) over the inner columns, four cells inside the lower and the upper layer: upper over lower."""
    p = f.download_grid(F.TAP_P_VEL).astype(np.float64)
    inner = p[8:-8, :, 8:-8]
    d = inner[:, :-1, :] - inner[:, 1:, :]
    lo, hi = d[:, 4:split - 4, :].mean(), d[:, split + 4:depth - 6, :].mean()
    return hi / lo


def speeds(f):
    """(largest, 99.9 % quantile) of the particles' |v| (cells/s)."""
    v = np.sqrt(sum(f.download_particles(t)[:, 3].astype(np.float64) ** 2 for t in (F.TAP_VX, F.TAP_VY, F.TAP_VZ)))
    return float(v.max()), float(np.quantile(v, 0.999))


# Measured on an H100 after 120 steps, (gradient ratio, 99.9 % quantile of |v| in cells/s): with the default velocity solve (tolerance 0.1,
# 32 iterations, warm start) the gradient ratio is near the density ratio but the tank sloshes (the same tank of one density does too: its
# largest |v| reached 160.9 cells/s); with a converged solve (tolerance 1e-3, 400 iterations) the layers are at rest and the gradient ratio is
# the density ratio.
LAYERS = {(2.0, 1.0): {"default": (0.498, 18.34), "converged": (0.5, 0.568)}, (1.0, 0.8): {"default": (0.771, 17.52), "converged": (0.8, 0.222)}}


@pytest.mark.parametrize("solve", ["default", "converged"])
@pytest.mark.parametrize("rho_lower, rho_upper", sorted(LAYERS))
def test_stable_layers_stay_at_rest(rho_lower, rho_upper, solve):
    f = layered(1, 2, {1: rho_lower, 2: rho_upper})
    if solve == "converged":
        f.set_solver_config(0, 1e-3, 400, 4)
    top, q = 0.0, 0.0
    for _ in range(120):
        f.step(DT)
        a, b = speeds(f)
        top, q = max(top, a), max(q, b)
    ratio = gradient_ratio(f)
    print(f"MEASURED layers {rho_lower}/{rho_upper} ({solve} solve): largest |v| {top:.4g}, 99.9 % quantile {q:.4g} cells/s, "
          f"gradient ratio {ratio:.5f} (density ratio {rho_upper / rho_lower})")
    want_ratio, want_q = LAYERS[(rho_lower, rho_upper)][solve]
    assert abs(ratio - want_ratio) < (0.01 if solve == "default" else 0.002)
    assert q < 1.1 * want_q


def test_inverted_layers_overturn():
    runs = {}
    for name, table in (("table", {1: 1.0, 2: 2.0}), ("control", None)):
        f = layered(1, 2, table)
        f.paint_tags((1, 20, 1), (20, 40, 63), 2)  # a step in the interface starts the overturn
        f.paint_tags((1, 1, 1), (20, 20, 63), 2)
        f.paint_tags((44, 1, 1), (63, 20, 63), 1)
        f.paint_tags((44, 20, 1), (63, 40, 63), 1)
        f.step(DT)
        c0 = f.tag_census(1, 2)["centroid"][:, 1]
        for _ in range(239):
            f.step(DT)
        c = f.tag_census(1, 2)["centroid"][:, 1]
        runs[name] = (c0, c)
        print(f"MEASURED overturn {name}: light/heavy centroid y {c0} -> {c}")
    (c0, c), (k0, k) = runs["table"], runs["control"]
    assert c[1] < c0[1] - 3.0 and c[0] > c0[0] + 3.0  # the heavy tag sank, the light one rose
    assert abs(k[1] - k0[1]) < 1.5 and abs(k[0] - k0[0]) < 1.5  # one density: no separation


def sphere_pool(rho, table=True, n=48):
    f = blub_b200.HybridFluid(n, n, n, 8 * (n - 2) * (n - 2) * 36)
    f.add_fluid_cube((1, 1, 1), (n - 1, 36, n - 1), 0)
    f.set_gravity_grid((0.0, G, 0.0))
    pos = f.download_particles()
    r = np.linalg.norm(pos[:, :3] - np.array([n / 2, 18.0, n / 2], np.float32), axis=1)
    pos[:, 3] = np.where(r < 7.0, np.uint32(1), np.uint32(0)).view(np.float32)
    f.set_particles(pos)
    if table:
        f.set_tag_densities({1: rho})
    return f


@pytest.mark.parametrize("rho", [0.5, 2.0])
def test_a_light_sphere_rises_and_a_heavy_one_sinks(rho):
    moves = {}
    for name in ("table", "control"):
        f = sphere_pool(rho, name == "table")
        f.step(DT)
        y0 = f.tag_census(1, 1)["centroid"][0, 1]
        for _ in range(100):
            f.step(DT)
        moves[name] = f.tag_census(1, 1)["centroid"][0, 1] - y0
    print(f"MEASURED sphere rho {rho}: centroid moved {moves['table']:.3f} cells (one density: {moves['control']:.3f})")
    assert (moves["table"] > 2.0) if rho < 1 else (moves["table"] < -2.0)
    assert abs(moves["control"]) < 0.5


# --- 5. repeatability ----------------------------------------------------------------------------------------------------------------

def test_runs_repeat_and_graphs_equal_eager():
    fs = [scene_fluid("oil_water_small", graph=g) for g in (True, True, False)]
    for _ in range(30):
        for f in fs:
            f.step(DT)
    same_taps(fs[0], fs[1], "run to run")
    same_taps(fs[0], fs[2], "graph against eager")
    assert fs[0].download_grid(F.TAP_CELL_DENSITY).tobytes() == fs[2].download_grid(F.TAP_CELL_DENSITY).tobytes()


def test_a_new_non_empty_table_replays_the_graph():
    a, b = scene_fluid("oil_water_small"), scene_fluid("oil_water_small", graph=False)
    for k in range(16):
        if k == 8:
            for f in (a, b):
                f.set_tag_densities({1: 0.6, 0: 1.2})
        a.step(DT)
        b.step(DT)
    same_taps(a, b, "table changed between graph replays")


@pytest.mark.parametrize("viscous", [False, True])
def test_save_and_load_resume_bit_for_bit(tmp_path, viscous):
    f = scene_fluid("oil_water_small")
    if viscous:
        f.set_viscosity(3.0)
    for _ in range(10):
        f.step(DT)
    path = str(tmp_path / "s.blub")
    f.save_state(path)
    assert F.state_info(path).format_version == 128
    g = F.HybridFluid.from_state(path)
    assert g.tag_densities() == f.tag_densities()
    for _ in range(10):
        f.step(DT)
        g.step(DT)
    same_taps(f, g, "resumed")


# --- 6. refusals and the runner ---------------------------------------------------------------------------------------------------

def test_refusals_change_nothing():
    f = scene_fluid("dam_small")
    bad = [{k: 1.0 for k in range(17)}, [(1, 1.0), (1, 2.0)], {1: 0.49}, {1: 2.01}, {1: 0.125}, {1: 8.0}, {1: float("nan")}, {1: float("inf")}]
    for t in bad:
        with pytest.raises(F.BlubError):
            f.set_tag_densities(t)
        assert f.tag_densities() == {}
    f.set_surface_tension(5.0)
    with pytest.raises(F.BlubError):
        f.set_tag_densities({1: 2.0})
    f.set_surface_tension(0.0)
    f.set_quirks(precond_mode=1)
    with pytest.raises(F.BlubError):
        f.set_tag_densities({1: 2.0})
    f.set_quirks(precond_mode=0)
    f.set_tag_densities({1: 2.0})
    with pytest.raises(F.BlubError):
        f.set_quirks(precond_mode=1)
    with pytest.raises(F.BlubError):
        f.set_surface_tension(5.0)
    f.step_stages(DT, 0, 5)
    with pytest.raises(F.BlubError):
        f.set_tag_densities({1: 1.5})
    f.step_stages(DT, 5, 14)
    assert f.tag_densities() == {1: 2.0}
    # floating bodies are not supported with a table, either way round
    box = [{"shape": "box", "half_extent": (2.0, 2.0, 2.0), "relative_density": 0.9, "centre": (16.0, 20.0, 16.0)}]
    with pytest.raises(F.BlubError):
        f.set_bodies(box)
    assert f.bodies() == []
    f.set_tag_densities({})
    f.set_bodies(box)
    with pytest.raises(F.BlubError):
        f.set_tag_densities({1: 2.0})
    assert f.tag_densities() == {}
    s = F.HybridFluid.create_slab(32, 32, 16, 1000, 0, 2)
    with pytest.raises(F.BlubError):
        s.set_tag_densities({1: 2.0})


def test_runner_on_the_oil_water_scene(tmp_path):
    scene, stats, dump = util.scene_path("oil_water_small"), str(tmp_path / "stats.json"), str(tmp_path / "p.f32")
    res = subprocess.run([RUNNER, scene, "--steps", "12", "--stats", stats, "--dump", dump], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    f = blub_b200.HybridFluid.from_scene(scene)
    assert f.tag_densities() == {1: float(np.float32(0.8))}
    for _ in range(12):
        f.step(DT)
    assert np.array_equal(np.fromfile(dump, dtype=np.float32).reshape(-1, 4)[:, :3], f.download_particles()[:, :3])
