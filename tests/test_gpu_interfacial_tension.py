"""GPU: interfacial tension (DESIGN.md §8 "Interfacial tension").  A tension that was turned off leaves no trace; a tension without phase-B
particles changes no tap; stages 1 (phi, the curvature, the right-hand side) and 4 (the interface faces) agree bit for bit with the NumPy
restatement tests/interfacial_tension_ref.py inside real steps, with and without a density table, with the free surface's tension and with a
moving solid; runs are reproducible and graph and eager agree; version-512 files resume bit for bit; refusals change nothing; the runner
agrees with a ctypes-driven run; the Laplace pressure of settled drops, a cube rounding up, layers at rest and a rising oil drop are measured,
printed and pinned at the values measured on an H100."""
import json
import os
import subprocess

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import interfacial_tension_ref as I, surface_tension_ref as S, tag_density_ref as T, util
from tests.test_gpu_loads import BOX, Solid
from tests.test_gpu_state import assert_identical, snapshot
from tests.util import DT

pytestmark = pytest.mark.gpu

RUNNER = os.path.join(os.path.dirname(F.lib_path()), "blub_run")
U_TAPS = (F.TAP_UX, F.TAP_UY, F.TAP_UZ)
ROW_TAPS = (F.TAP_VX, F.TAP_VY, F.TAP_VZ)
DT32 = float(np.float32(DT))
SIGMA = 200.0  # cells^3/s^2: a capillary limit of 19.9 ms, above the 1/120 s step


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint8)


# ---- off = never on, and no phase-B particle = no tension ---------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("path", ["scatter", "gather"])
def test_interfacial_tension_turned_off_equals_never_on(tmp_path, path, graph):
    runs = []
    for touched in (False, True):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
        f.set_transfer_path(path)
        f.set_graph_replay(graph)
        if touched:
            f.set_interfacial_tension(SIGMA, [0])
            f.set_interfacial_tension(0.0, [])
            assert f.interfacial_tension() == (0.0, [])
        F.kernel_launch_count(reset=True)
        for _ in range(40):
            f.step(DT)
            f.synchronize()
        launches = F.kernel_launch_count()
        save = str(tmp_path / f"{int(touched)}.blub")
        f.save_state(save)
        runs.append((snapshot(f), launches, open(save, "rb").read()))
        for tap in (F.TAP_INTERFACE_CURVATURE, F.TAP_INTERFACE_FIELD):
            assert not f.download_grid(tap).any()
    assert_identical(runs[0][0], runs[1][0])
    assert runs[0][1] == runs[1][1]
    assert runs[0][2] == runs[1][2]


@pytest.mark.parametrize("graph", [True, False])
def test_a_tension_without_phase_b_particles_changes_no_tap(graph):
    runs = []
    for on in (False, True):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("oil_water_small"))
        f.set_graph_replay(graph)
        if on:
            f.set_interfacial_tension(SIGMA, [99, 7])  # no particle carries either tag
        for _ in range(30):
            f.step(DT)
        f.synchronize()
        runs.append(snapshot(f))
        if on:
            assert not f.download_grid(F.TAP_INTERFACE_CURVATURE).any()
            assert (f.download_grid(F.TAP_INTERFACE_FIELD)[f.download_grid(F.TAP_MARKER) == I.FLUID] <= 0).all()
    assert_identical(runs[0], runs[1])


# ---- stages 1 and 4 against the restatement -----------------------------------------------------------------------------------------
def repaint(f, pos, rows):
    f.set_particles(pos, *rows)


def stage_twins(tmp_path, scene, table, surface=0.0, steps=8, moving=False):
    """(f, plain, splat_all, splat_b): two copies of `scene` after `steps` steps whose particles are repainted in whole 32-particle blocks
    (phase B: tag 1 for the blocks whose mean x lies left of the middle), f with the interfacial tension.  Whole blocks keep every warp's
    peer groups, so the splats of all particles and of the B blocks alone, made by stage 9 of two more copies, are the two splats of stage 1."""
    base = blub_b200.HybridFluid.from_scene(util.scene_path(scene))
    if not table:
        base.set_tag_densities({})
    solid = Solid(base, BOX) if moving else None
    for _ in range(steps):
        if solid:
            solid.voxelize()
        base.step(DT)
    path = str(tmp_path / "base.blub")
    base.save_state(path)
    pos = base.download_particles()
    rows = [base.download_particles(t) for t in ROW_TAPS]
    n = len(pos)
    blocks = np.arange(n) // 32
    mean_x = np.bincount(blocks, weights=pos[:, 0]) / np.bincount(blocks)
    in_b = mean_x[blocks] < base.nx / 2
    tags = pos.view(np.uint32)
    tags[:, 3] = np.where(in_b, 1, 0)
    fluids = [blub_b200.HybridFluid.from_state(path) for _ in range(4)]
    for k, x in enumerate(fluids):
        if k < 3:
            repaint(x, pos, rows)
        else:
            repaint(x, pos[in_b], [r[in_b] for r in rows])
    f, plain, sall, sb = fluids
    splats = []
    for x in (sall, sb):
        x.step_stages(DT, 9, 10)
        splats.append(x.download_grid(F.TAP_DENSITY))
    f.set_interfacial_tension(SIGMA, [1])
    if moving:  # the box where the base's next step would put it; the splats do not read the solid
        for x in (f, plain):
            x.solid = Solid(x, BOX)
            x.solid.t = solid.t
            x.solid.voxelize()
    if surface:
        f.set_surface_tension(surface)
        plain.set_surface_tension(surface)
    return f, plain, splats[0], splats[1]


@pytest.mark.parametrize("scene, table, surface, moving", [("oil_water_small", True, 0.0, False), ("oil_water_small", False, 0.0, False),
                                                            ("oil_water_small", False, 72.8, False), ("double_dam", False, 0.0, True)])
def test_stages_1_and_4_match_the_restatement(tmp_path, scene, table, surface, moving):
    f, plain, splat_all, splat_b = stage_twins(tmp_path, scene, table, surface, steps=30 if moving else 8, moving=moving)
    for x in (f, plain):
        x.step_stages(DT, 0, 2)
    marker = f.download_grid(F.TAP_MARKER)
    assert np.array_equal(marker, plain.download_grid(F.TAP_MARKER))
    phi_ref = I.phase_field(splat_all, splat_b, marker)
    phi = f.download_grid(F.TAP_INTERFACE_FIELD)
    region = S.near_fluid(marker, 2)
    assert np.array_equal(phi[region], phi_ref[region]), "phi"
    kappa = f.download_grid(F.TAP_INTERFACE_CURVATURE)
    b = I.band(phi_ref, marker)
    assert b.sum() > 50
    k64, _ = S.curvature64(phi_ref, b)
    rounded = np.clip(k64[b], -2.0, 2.0).astype(np.float32)
    ulps = np.abs(kappa[b].astype(np.float64) - rounded) / np.spacing(np.maximum(np.abs(rounded), np.float32(2.0 ** -126)))
    print(f"{scene} table={table} surface={surface}: {b.sum()} band cells, max {ulps.max():g} ulps, |kappa| max {np.abs(kappa).max():.3f}")
    assert ulps.max() <= 2 and not kappa[~b].any()
    if moving:
        touching, _ = util.solid_contact(marker, f.download_solid_voxels(), f.download_particles())
        assert touching >= 20, touching
    beta = None
    if table:
        beta, _, _ = T.coefficients(marker, f.download_grid(F.TAP_CELL_DENSITY))
    fl = marker == I.FLUID
    rhs, rhs_plain = f.download_grid(F.TAP_RESIDUAL), plain.download_grid(F.TAP_RESIDUAL)
    want = I.rhs_after(rhs_plain, marker, phi, kappa, DT32, SIGMA, beta)
    assert np.array_equal(bits(rhs)[fl], bits(want)[fl]), "rhs"
    # stage 4 of the plain twin on f's velocity and pressure: only the interface faces differ, by exactly +-beta g
    for x in (f, plain):
        x.step_stages(DT, 2, 4)
    u_before, p = [f.download_grid(t) for t in U_TAPS], f.download_grid(F.TAP_P_VEL)
    for t, u in zip(U_TAPS, u_before):
        plain.upload_grid(t, u)
    plain.upload_grid(F.TAP_P_VEL, p)
    for x in (f, plain):
        x.step_stages(DT, 4, 5)
    changed = 0
    for axis, t in enumerate(U_TAPS):
        got, base = f.download_grid(t), plain.download_grid(t)
        want = I.faces_after(base, marker, phi, kappa, DT32, SIGMA, axis, beta)
        assert np.array_equal(bits(got), bits(want)), axis
        changed += int((bits(got) != bits(base)).sum())
    assert changed > 20
    for x in (f, plain):
        x.step_stages(DT, 5, 14)


# ---- reproducibility, graphs, refusals ----------------------------------------------------------------------------------------------
def run_drop(graph, steps=20, change_at=None):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("oil_drop_zero_g"))
    f.set_graph_replay(graph)
    for k in range(steps):
        if k == change_at:
            f.set_interfacial_tension(2.0 * f.interfacial_tension()[0], [1])
        f.step(DT if k % 2 == 0 else DT / 2)
    f.synchronize()
    return snapshot(f)


def test_runs_are_reproducible_and_graph_equals_eager():
    a, b, c = run_drop(True), run_drop(True), run_drop(False)
    assert_identical(a, b)
    assert_identical(a, c)
    d, e = run_drop(True, change_at=10), run_drop(False, change_at=10)
    assert_identical(d, e)


def test_refusals_change_nothing():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("oil_water_small"))
    f.set_interfacial_tension(SIGMA, [1])
    for sigma, tags in ((-1.0, [1]), (float("nan"), [1]), (float("inf"), [1]), (SIGMA, []), (SIGMA, [1, 1]), (SIGMA, list(range(17)))):
        with pytest.raises(F.BlubError):
            f.set_interfacial_tension(sigma, tags)
        assert f.interfacial_tension() == (SIGMA, [1])
    L = F.lib()
    assert L.blub_fluid_set_interfacial_tension(f.h, None, 2, F.C.c_float(SIGMA)) == 1
    assert f.interfacial_tension() == (SIGMA, [1])
    f.step_stages(DT, 0, 3)
    with pytest.raises(F.BlubError):
        f.set_interfacial_tension(0.0, [])
    f.step_stages(DT, 3, 14)
    with pytest.raises(F.BlubError):  # the existing refusals stay
        f.set_surface_tension(72.8)
    f.set_interfacial_tension(0.0, [])
    assert f.interfacial_tension() == (0.0, [])


def test_version_512_resumes_bit_for_bit(tmp_path):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("oil_drop_zero_g"))
    for _ in range(6):
        f.step(DT)
    path = str(tmp_path / "it.blub")
    f.save_state(path)
    assert F.state_info(path).format_version == 512
    g = blub_b200.HybridFluid.from_state(path)
    assert g.interfacial_tension() == f.interfacial_tension() and g.tag_densities() == f.tag_densities()
    for _ in range(10):
        f.step(DT)
        g.step(DT)
    f.synchronize()
    g.synchronize()
    assert_identical(snapshot(f), snapshot(g))
    f.set_interfacial_tension(0.0, [])
    f.save_state(path)
    assert F.state_info(path).format_version == 128  # without the tension the file is what it was


def test_runner_on_the_oil_drop_equals_a_ctypes_run(tmp_path):
    scene, stats, dump = util.scene_path("oil_drop_zero_g"), str(tmp_path / "stats.json"), str(tmp_path / "p.f32")
    save = str(tmp_path / "run.blub")
    res = subprocess.run([RUNNER, scene, "--steps", "12", "--stats", stats, "--dump", dump, "--save-state", save], capture_output=True, text=True,
                         timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    f = blub_b200.HybridFluid.from_scene(scene)
    for _ in range(12):
        f.step(DT)
    rec = json.load(open(stats))["interfacial_tension"]
    assert np.float32(rec["tension"]) == np.float32(f.interfacial_tension()[0]) > 0 and rec["tags"] == [1]
    assert np.array_equal(np.fromfile(dump, dtype=np.float32).reshape(-1, 4)[:, :3], f.download_particles()[:, :3])
    assert F.state_info(save).format_version == 512


def test_scene_sets_the_tension():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("oil_drop_zero_g"))
    s, tags = f.interfacial_tension()
    assert tags == [1] and s == pytest.approx(3e-5 / 0.01 ** 3, rel=1e-6)


# ---- physics -------------------------------------------------------------------------------------------------------------------------
def cube_extent(f):
    pos = f.download_particles()
    b = pos.view(np.uint32)[:, 3] == 1
    p = pos[b, :3]
    c = p.mean(axis=0)
    r = np.linalg.norm(p - c, axis=1)
    return float(r.max()), float(np.abs(p - c).max(axis=0).min())


def test_a_cube_of_b_rounds_up_and_the_control_stays_a_cube():
    """The cube's farthest particle (a corner) moves in under the tension and not without it."""
    out = {}
    for sigma in (0.0, SIGMA):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("oil_drop_zero_g"))
        f.set_interfacial_tension(sigma, [1] if sigma else [])
        r0, _ = cube_extent(f)
        for _ in range(60):
            f.step(DT)
        r1, _ = cube_extent(f)
        out[sigma] = (r0, r1)
    print(f"cube corner radius: control {out[0.0]}, tension {out[SIGMA]}")
    assert out[SIGMA][1] < out[0.0][1] - 0.3


def lattice(n, keep, tag_of):
    """8 particles per cell on the stratified lattice in the cells 1 .. n - 2 where keep(x, y, z), tagged by tag_of(x, y, z)."""
    g = (np.arange(1, n - 1)[:, None] + np.array([0.25, 0.75])[None, :]).ravel()
    z, y, x = np.meshgrid(g, g, g, indexing="ij")
    x, y, z = x.ravel(), y.ravel(), z.ravel()
    k = keep(x, y, z)
    pos = np.zeros((int(k.sum()), 4), dtype=np.float32)
    pos[:, 0], pos[:, 1], pos[:, 2] = x[k], y[k], z[k]
    pos[:, 3] = np.asarray(tag_of(x[k], y[k], z[k]), dtype=np.uint32).view(np.float32)
    return pos


def test_laplace_pressure_of_settled_b_drops():
    """B drops of R = 8, 12, 16 in A (64^3, zero g, AIR above y = 56 for the solve's Dirichlet boundary), s = 200, 48 steps: the mean p of the
    B cells more than 2 cells inside the interface minus that of the A cells more than 2 cells outside it (and 4 below the free surface),
    against the jump -dt s 2/R of the solve's units."""
    n, out = 64, {}
    for radius in (8, 12, 16):
        c = (32.0, 28.0, 32.0)
        inside = lambda x, y, z: (x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2 < radius ** 2
        pos = lattice(n, lambda x, y, z: y < 56, lambda x, y, z: np.where(inside(x, y, z), 1, 0))
        f = blub_b200.HybridFluid(n, n, n, len(pos) + 1024)
        f.set_particles(pos)
        f.set_interfacial_tension(SIGMA, [1])
        util.tight_solver(f, tol=1e-4, max_it=256)
        for _ in range(48):
            f.step(DT)
        f.step_stages(DT, 0, 3)
        p, m, phi = f.download_grid(F.TAP_P_VEL), f.download_grid(F.TAP_MARKER), f.download_grid(F.TAP_INTERFACE_FIELD)
        f.step_stages(DT, 3, 14)
        pb = f.download_particles()
        b = pb[:, 3].view(np.uint32) == 1
        cc = pb[b, :3].astype(np.float64).mean(axis=0)
        z, y, x = np.indices(m.shape) + 0.5
        r = np.sqrt((x - cc[0]) ** 2 + (y - cc[1]) ** 2 + (z - cc[2]) ** 2)
        fl = m == I.FLUID
        r_eff = (3.0 * (fl & (phi > 0)).sum() / (4.0 * np.pi)) ** (1.0 / 3.0)
        top = max(int(np.nonzero(fl.any(axis=(0, 2)))[0].max()) - 4, 0)
        inner = fl & (r < r_eff - 2.0)
        outer = fl & (r > r_eff + 2.0) & (r < r_eff + 8.0) & (np.indices(m.shape)[1] < top)
        jump = float(p[inner].astype(np.float64).mean() - p[outer].astype(np.float64).mean())
        out[radius] = (jump, -DT32 * SIGMA * 2.0 / radius, r_eff)
    print("interface Laplace pressure (p inside - outside, -dt s 2/R, effective radius): " +
          ", ".join(f"R={k}: {v[0]:.5f} vs {v[1]:.5f} ({v[0] / v[1]:.3f}), {v[2]:.2f}" for k, v in out.items()))
    # Measured on an H100 (DESIGN.md §8 "Interfacial tension"): 1.061, 1.049 and 1.052 of the target for R = 8, 12 and 16 -- not biased low
    # like the free surface's 0.87 / 0.79 / 0.68, as the CPU restatement of a lattice drop predicts (1.035 and 1.073 of 2/R)
    for radius, (jump, target, _) in out.items():
        assert 1.0 <= jump / target <= 1.12, (radius, jump, target)
    assert out[8][0] < out[12][0] < out[16][0] < 0.0


def layered(n=32, oil=(8, 14), drop=None):
    """A 0.8 oil layer (tag 1, y in oil) over water (y below), or with drop = (centre, R) an oil drop in a water pool of depth 20; gravity of
    oil_water_small and its table."""
    if drop is None:
        pos = lattice(n, lambda x, y, z: y < oil[1], lambda x, y, z: np.where(y >= oil[0], 1, 0))
    else:
        c, radius = drop
        pos = lattice(n, lambda x, y, z: y < 20, lambda x, y, z: np.where((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2 < radius ** 2, 1, 0))
    f = blub_b200.HybridFluid(n, n, n, len(pos) + 1024)
    f.set_particles(pos)
    f.set_gravity_grid((0.0, -9.81 / 0.01, 0.0))
    f.set_tag_densities({1: 0.8})
    return f


def test_flat_oil_over_water_stays_at_rest():
    speeds = {}
    for sigma in (0.0, SIGMA):
        f = layered()
        f.set_interfacial_tension(sigma, [1] if sigma else [])
        for _ in range(60):
            f.step(DT)
        v = np.stack([f.download_particles(t)[:, :3] for t in ROW_TAPS])
        speeds[sigma] = float(np.abs(v).max())
    print(f"flat oil over water after 60 steps, largest particle velocity component: control {speeds[0.0]:.4f}, s = {SIGMA:g} {speeds[SIGMA]:.4f}")
    # measured on an H100: 0.0176 against the control's 0.0207 cells/s -- the tension does not stir a flat interface
    assert speeds[SIGMA] <= 1.2 * speeds[0.0]


def test_an_oil_drop_rises_through_water_with_the_tension():
    f = layered(drop=((16.0, 8.0, 16.0), 4.0))
    f.set_interfacial_tension(SIGMA, [1])
    y0 = float(f.download_particles()[f.particle_tags() == 1, 1].mean())
    for _ in range(60):
        f.step(DT)
    y1 = float(f.download_particles()[f.particle_tags() == 1, 1].mean())
    print(f"oil drop centroid y: {y0:.2f} -> {y1:.2f}")
    assert 5.0 <= y1 - y0 <= 8.0  # measured on an H100: 8.00 -> 14.64 with the 0.8 table and the tension
