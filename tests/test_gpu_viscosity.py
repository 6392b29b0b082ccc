"""GPU: viscous liquids (DESIGN.md §8 "Viscous liquids").  Viscosity that was turned off leaves no trace; the solve agrees with the float64
restatement tests/visc_ref.py on uploaded fields and inside real steps (written faces, true residual, distance to the direct solve, reported
error, iterates as prefixes); a sine mode decays by its eigenvalue; a tank at rest stays bit for bit at rest; a moving box drags the liquid;
more viscosity leaves less kinetic energy; runs are reproducible, graph and eager agree and follow dt and the setting; version-32 files resume
bit for bit; refusals change nothing; the runner agrees with a ctypes-driven run."""
import json
import os
import subprocess

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import body_ref, util, visc_ref as V
from tests.test_gpu_loads import BOX, BOX_HI, BOX_LO, G, H, N, Solid, seed_around
from tests.test_gpu_state import assert_identical, snapshot
from tests.util import DT

pytestmark = pytest.mark.gpu

RUNNER = os.path.join(os.path.dirname(F.lib_path()), "blub_run")
U_TAPS = (F.TAP_UX, F.TAP_UY, F.TAP_UZ)
DT32 = float(np.float32(DT))


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint8)


def velocity(f):
    return [f.download_grid(t) for t in U_TAPS]


def check_against_restatement(marker, u_star, result, k, gravity_dt, vox, iterations, max_error, tolerance, cap, need_dirichlet=0):
    """The checks every solve must pass, per component; returns the restatement's systems."""
    systems = []
    for c in range(3):
        s = V.System(marker, c, k, u_star[c], gravity_dt[c], vox)
        systems.append(s)
        changed = bits(result[c]) != bits(u_star[c])
        assert not (changed & ~s.live).any(), f"component {c}: a face that is not live was written"
        if s.n == 0:
            continue
        r = s.residual(result[c])
        rounding = s.rounding_bound(iterations, u_star[c], result[c], vox)
        true_error = float(np.abs(r).max())
        assert abs(true_error - max_error[c]) <= rounding, (c, true_error, max_error[c], rounding)
        if iterations < cap:
            assert true_error <= tolerance + rounding, (c, true_error, tolerance, rounding)
        # |A^-1|_inf <= 1: an iterate is no farther from the solution than its true residual
        x_direct = s.solve()
        distance = float(np.abs(np.asarray(result[c], dtype=np.float64)[s.live] - gravity_dt[c] - x_direct).max())
        assert distance <= true_error + rounding, (c, distance, true_error)
    # live faces that really have a Dirichlet neighbour with a velocity (over the three components: a solid may move along one axis only)
    moving = sum(int(s.dirichlet_nonzero.sum()) for s in systems)
    assert moving >= need_dirichlet, moving
    assert 0 <= iterations <= cap
    return systems


def salt_and_pepper(shape, seed):
    rng = np.random.default_rng(seed)
    m = rng.integers(-1, 2, shape).astype(np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    return m


def uploaded_fluid(dims, marker, u_star, vox, gravity=(0.0, 0.0, 0.0)):
    import torch
    f = blub_b200.HybridFluid(*dims, 1000)
    f.set_gravity_grid(gravity)
    f.upload_grid(F.TAP_MARKER, marker)
    for t, u in zip(U_TAPS, u_star):
        f.upload_grid(t, u)
    vol = None
    if vox is not None:
        vol = torch.from_numpy(vox).to("cuda:0")
        torch.cuda.synchronize()
        f.set_solid_voxels(vol.data_ptr())
    return f, vol


# ---- 1. off = never on -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("path", ["scatter", "gather"])
def test_viscosity_turned_off_equals_never_on(tmp_path, path, graph):
    runs = []
    for touched in (False, True):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
        f.set_transfer_path(path)
        f.set_graph_replay(graph)
        if touched:
            f.set_viscosity(3.0)
            f.set_viscosity(0.0)
            assert f.viscosity()[0] == 0.0
        F.kernel_launch_count(reset=True)
        for _ in range(70):
            f.step(DT)
            f.synchronize()
        launches = F.kernel_launch_count()
        save = str(tmp_path / f"{int(touched)}.blub")
        f.save_state(save)
        runs.append((snapshot(f), launches, open(save, "rb").read()))
    assert_identical(runs[0][0], runs[1][0])
    assert runs[0][1] == runs[1][1]
    assert runs[0][2] == runs[1][2] and F.state_info(str(tmp_path / "1.blub")).format_version == 1


# ---- 2. the solve against the restatement ----------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [0.05, 1.0, 20.0])
@pytest.mark.parametrize("dims", [(32, 32, 32), (40, 24, 24), (1024, 8, 8)])
def test_solve_on_uploaded_fields_matches_the_restatement(dims, k):
    """Salt-and-pepper markers: every neighbour class on every side, on grids at the edges of the tiling (a 40-cell row, nx = 1024 with 8 x 8
    rows), with a solid volume whose every voxel carries a velocity."""
    shape = dims[::-1]
    rng = np.random.default_rng(11)
    marker = salt_and_pepper(shape, 2)
    u_star = [rng.standard_normal(shape).astype(np.float32) for _ in range(3)]
    vox = rng.uniform(-2, 2, shape + (4,)).astype(np.float16)
    gravity = (0.0, -981.0, 0.0)
    f, vol = uploaded_fluid(dims, marker, u_star, vox, gravity)
    nu, tolerance, cap = k / DT32, 1e-4, 400
    f.set_viscosity(nu, tolerance, cap)
    f.viscosity_only(DT)
    iterations, max_error = f.last_viscosity_solve()
    k32 = float(np.float32(nu) * np.float32(DT))
    gdt = [float(np.float32(g) * np.float32(DT)) for g in gravity]
    systems = check_against_restatement(marker, u_star, velocity(f), k32, gdt, vox, iterations, max_error, tolerance, cap, need_dirichlet=50)
    assert iterations >= 1 and all(s.n > 0 for s in systems)
    # iterates with the cap at 1, 2, 3 are the first iterates of the same recurrence: distinct, and each closer in the A-norm sense of
    # the recurrence -- the reported error of cap j equals the error the full solve would report after j iterations only if alpha and beta
    # are formed the same way, which the residual check above pins for every cap
    previous = None
    for cap_j in (1, 2, 3):
        for t, u in zip(U_TAPS, u_star):
            f.upload_grid(t, u)
        f.set_viscosity(nu, 1e-30, cap_j)
        f.viscosity_only(DT)
        it_j, err_j = f.last_viscosity_solve()
        assert it_j == cap_j
        res_j = velocity(f)
        check_against_restatement(marker, u_star, res_j, k32, gdt, vox, it_j, err_j, 1e-30, cap_j)
        if previous is not None:
            assert any((bits(a) != bits(b)).any() for a, b in zip(res_j, previous))
        previous = res_j
    del vol


def test_one_cg_step_on_an_eigenmode_is_exact_and_the_mode_decays_by_its_eigenvalue():
    """32^3 all fluid: u* = a product of three sines is an eigenvector, so r_0 is a multiple of it and one CG step lands on the solution."""
    n, k = 32, 1.0
    marker = np.zeros((n, n, n), dtype=np.int8)
    marker[1:-1, 1:-1, 1:-1] = V.FLUID
    modes = (2, 1, 3)
    z, y, x = np.meshgrid(*[np.arange(n)] * 3, indexing="ij")
    u_star, factor = [], []
    for c in range(3):
        rows = [n - 3 if d == c else n - 2 for d in range(3)]
        vec = np.ones(marker.shape)
        for d, coord in enumerate((x, y, z)):
            vec *= np.sin(np.pi * modes[d] * coord / (rows[d] + 1))
        u_star.append(np.where(V.live_faces(marker, c), vec, 0.0).astype(np.float32))
        factor.append(1.0 / (1.0 + k * sum(2.0 - 2.0 * np.cos(np.pi * modes[d] / (rows[d] + 1)) for d in range(3))))
    f, _ = uploaded_fluid((n, n, n), marker, u_star, None)
    f.set_viscosity(k / DT32, 1e-30, 1)
    f.viscosity_only(DT)
    iterations, max_error = f.last_viscosity_solve()
    assert iterations == 1
    for c, got in enumerate(velocity(f)):
        live = V.live_faces(marker, c)
        assert np.abs(got[live] - factor[c] * u_star[c][live].astype(np.float64)).max() <= 64 * V.EPS32, c
        assert max_error[c] <= 64 * V.EPS32 * (1 + 12 * k)


def twin_without_viscosity(tmp_path, viscous):
    """The same fluid (stale faces included) with viscosity off, through a saved state: its stage 0 gives the solve's input."""
    path = str(tmp_path / "twin.blub")
    viscous.save_state(path)
    twin = blub_b200.HybridFluid.from_state(path)
    twin.set_viscosity(0.0)
    return twin


@pytest.mark.parametrize("k", [0.05, 1.0, 20.0])
def test_stage_0_of_dam_small_matches_the_restatement(tmp_path, k):
    viscous = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    viscous.set_viscosity(k / DT32, 1e-4, 400)
    for _ in range(5):
        viscous.step(DT)
    plain = twin_without_viscosity(tmp_path, viscous)
    for f in (plain, viscous):
        f.step_stages(DT, 0, 1)
    marker = viscous.download_grid(F.TAP_MARKER)
    assert np.array_equal(marker, plain.download_grid(F.TAP_MARKER))
    iterations, max_error = viscous.last_viscosity_solve()
    gdt = [0.0, float(np.float32(-981.0) * np.float32(DT)), 0.0]
    k32 = float(np.float32(k / DT32) * np.float32(DT))
    check_against_restatement(marker, velocity(plain), velocity(viscous), k32, gdt, None, iterations, max_error, 1e-4, 400)
    assert iterations >= 1
    for f in (plain, viscous):
        f.step_stages(DT, 1, 14)


@pytest.mark.parametrize("solid", ["box", "bodies"])
def test_stage_0_of_double_dam_with_moving_solids_matches_the_restatement(tmp_path, solid):
    """Dirichlet values from the borrowed volume (the benchmark's travelling box) and from the composite volume (two floating bodies)."""
    k = 1.0
    viscous = blub_b200.HybridFluid.from_scene(util.scene_path("double_dam"))
    solids = []
    if solid == "box":
        solids.append(Solid(viscous, BOX))
    else:
        viscous.set_bodies([body_ref.body("box", (5, 4, 6), 0.6, (108, 20, 40), velocity=(3, 0, 0), angular_velocity=(0, 0.5, 0)),
                            body_ref.body("sphere", 5, 0.8, (20, 30, 52), velocity=(2, 0, 0))])
    viscous.set_viscosity(k / DT32, 1e-4, 400)
    for _ in range(40 if solid == "box" else 6):
        for s in solids:
            s.voxelize()
        viscous.step(DT)
    plain = twin_without_viscosity(tmp_path, viscous)
    if solid == "box":
        solids.append(Solid(plain, BOX))
        solids[1].t = solids[0].t
    for s in solids:
        s.voxelize()
    for f in (plain, viscous):
        f.step_stages(DT, 0, 1)
    marker = viscous.download_grid(F.TAP_MARKER)
    assert np.array_equal(marker, plain.download_grid(F.TAP_MARKER))
    vox = viscous.download_solid_voxels()
    assert np.array_equal(vox, plain.download_solid_voxels())
    touching, _ = util.solid_contact(marker, vox, viscous.download_particles())
    assert touching >= 20, touching
    iterations, max_error = viscous.last_viscosity_solve()
    gdt = [0.0, float(np.float32(-981.0) * np.float32(DT)), 0.0]
    k32 = float(np.float32(k / DT32) * np.float32(DT))
    check_against_restatement(marker, velocity(plain), velocity(viscous), k32, gdt, vox, iterations, max_error, 1e-4, 400, need_dirichlet=5)


# ---- 3. physics ------------------------------------------------------------------------------------------------------------
def test_a_tank_at_rest_stays_bit_for_bit_at_rest():
    """The 64^3 hydrostatic tank of the load probes' test: grid velocity after stage 0, pressure after stage 2 and the probe records are those
    of the inviscid step, and the solve takes no iteration."""
    import torch
    out = []
    for nu in (0.0, 50.0):
        f = blub_b200.HybridFluid(N, N, N, 8 * N * N * H)
        f.set_gravity_grid((0.0, -G, 0.0))
        seed_around(f, H + 1, BOX_LO, BOX_HI)
        vol = torch.zeros((N, N, N, 4), dtype=torch.float16, device="cuda:0")
        vol[BOX_LO[2]:BOX_HI[2], BOX_LO[1]:BOX_HI[1], BOX_LO[0]:BOX_HI[0], 3] = 1.0
        torch.cuda.synchronize()
        f.set_solid_voxels(vol.data_ptr())
        f.set_load_probes([((N - 1, 0, 0), (N, N, N)), ((20, 4, 20), (44, 20, 44))])
        f.set_viscosity(nu)
        f.step_stages(DT, 0, 1)
        u = velocity(f)
        f.step_stages(DT, 1, 3)
        out.append((u, f.download_grid(F.TAP_P_VEL), [f.load_history(p, 1) for p in range(2)], f.last_viscosity_solve(), vol))
        f.step_stages(DT, 3, 14)
    for a, b in zip(out[0][0], out[1][0]):
        assert np.array_equal(bits(a), bits(b))
    assert np.array_equal(bits(out[0][1]), bits(out[1][1]))
    for ha, hb in zip(out[0][2], out[1][2]):
        for name in ("wetted_faces", "force_fx", "torque_fx"):
            assert np.array_equal(ha[name], hb[name])
    assert out[1][3] == (0, [0.0, 0.0, 0.0])


def test_a_box_driven_along_a_still_surface_drags_the_liquid():
    import torch
    n, h, speed = 64, 16, 20.0
    drag = []
    for nu in (0.0, 100.0):
        f = blub_b200.HybridFluid(n, n, n, 8 * n * n * h)
        f.add_fluid_cube((1, 1, 1), (n - 1, h + 1, n - 1))  # no gravity: the liquid is still, the box lies on its surface
        vol = torch.zeros((n, n, n, 4), dtype=torch.float16, device="cuda:0")
        vol[20:44, h + 1:h + 5, 20:44, 0] = speed
        vol[20:44, h + 1:h + 5, 20:44, 3] = 1.0
        torch.cuda.synchronize()
        f.set_solid_voxels(vol.data_ptr())
        f.set_viscosity(nu)
        f.step_stages(DT, 0, 1)
        marker, ux = f.download_grid(F.TAP_MARKER), f.download_grid(F.TAP_UX)
        near = V.live_faces(marker, 0)
        near[:, :h - 2], near[:, h + 1:] = False, False
        near[:20], near[44:], near[:, :, :20], near[:, :, 44:] = False, False, False, False
        assert near.sum() > 1000
        drag.append(float(ux[near].astype(np.float64).mean()))
        f.step_stages(DT, 1, 14)
        del vol
    assert drag[0] == 0.0 and drag[1] > 1e-3 * speed, drag


def test_more_viscosity_leaves_less_kinetic_energy():
    energy = []
    for nu in (0.0, 0.5, 5.0, 50.0):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
        n0 = f.num_particles
        f.set_viscosity(nu)
        for _ in range(60):
            f.step(DT)
        v = np.stack([f.download_particles(t)[:, 0] for t in (F.TAP_VX, F.TAP_VY, F.TAP_VZ)]).astype(np.float64)
        assert f.num_particles == n0 and np.isfinite(v).all()
        energy.append(float((v * v).sum()))
    assert all(a > b for a, b in zip(energy, energy[1:])), energy


# ---- 4. reproducibility, graphs, settings ------------------------------------------------------------------------------------
def run_viscous(graph, steps=70, nu=5.0, dts=None, change_at=None):
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    f.set_graph_replay(graph)
    f.set_viscosity(nu)
    for s in range(steps):
        if change_at is not None and s == change_at:
            f.set_viscosity(4 * nu, 1e-5, 300)  # no synchronisation in front of it: ordered behind the steps in flight
        f.step(DT if dts is None else dts[s])
        f.synchronize()
    return snapshot(f), f.last_viscosity_solve()


def test_two_runs_and_graph_against_eager_are_bit_identical():
    """70 steps cross the re-sorts every 8 and the rebinning at step 60."""
    a, b, c = run_viscous(True), run_viscous(True), run_viscous(False)
    assert_identical(a[0], b[0])
    assert_identical(a[0], c[0])
    assert a[1] == b[1] == c[1] and a[1][0] >= 1


def test_a_replayed_graph_follows_dt_and_the_setting():
    dts = [DT if s % 3 else 0.5 * DT for s in range(24)]
    assert_identical(run_viscous(True, 24, dts=dts)[0], run_viscous(False, 24, dts=dts)[0])
    a, b = run_viscous(True, 24, change_at=12), run_viscous(False, 24, change_at=12)
    assert_identical(a[0], b[0])
    assert a[1] == b[1]
    plain = run_viscous(True, 24)
    assert (bits(a[0]["grid_velocity_x"]) != bits(plain[0]["grid_velocity_x"])).any()  # the change of the setting was followed


# ---- 5. state, refusals, runner -------------------------------------------------------------------------------------------------
def test_refusals_change_nothing():
    f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    f.set_viscosity(2.0, 1e-3, 50)
    for bad in [(-1.0,), (float("nan"),), (float("inf"),), (1.0, 0.0), (1.0, float("nan")), (1.0, -1e-4), (1.0, 1e-4, 0), (1.0, 1e-4, 10001)]:
        with pytest.raises(blub_b200.BlubError):
            f.set_viscosity(*bad)
    v = F.Viscosity(1.0, 1e-4, 200, 7)
    assert f.L.blub_fluid_set_viscosity(f.h, F.C.byref(v)) == 1
    f.step_stages(DT, 0, 3)
    with pytest.raises(blub_b200.BlubError):
        f.set_viscosity(1.0)
    f.step_stages(DT, 3, 14)
    assert f.viscosity() == (2.0, float(np.float32(1e-3)), 50)
    assert f.L.blub_fluid_set_viscosity(f.h, None) == 0 and f.viscosity()[0] == 0.0
    with pytest.raises(blub_b200.BlubError):
        f.viscosity_only(DT)
    slab = blub_b200.HybridFluid.create_slab(32, 32, 32, 1000, 0, 2)
    with pytest.raises(blub_b200.BlubError):
        slab.set_viscosity(1.0)


@pytest.mark.parametrize("base", ["plain", "flow and tags", "bodies", "mesh body"])
def test_version_32_resumes_bit_for_bit(tmp_path, base):
    scene = {"plain": "dam_small", "flow and tags": "tap_small", "bodies": "double_dam", "mesh body": "double_dam"}[base]
    f = blub_b200.HybridFluid.from_scene(util.scene_path(scene))
    if base == "flow and tags":
        f.paint_tags((1, 1, 1), (16, 16, 16), 5)
    if base == "bodies":
        f.set_bodies([body_ref.body("box", (5, 4, 6), 0.6, (108, 20, 40)), body_ref.body("sphere", 5, 0.8, (20, 30, 52), velocity=(2, 0, 0))])
    if base == "mesh body":
        from tests import mesh_body_ref
        L_POS, L_TRI = mesh_body_ref.l_block()
        f.set_bodies([dict(body_ref.body(centre=(64, 30, 32)), mesh=(L_POS, L_TRI), scale=3.0, relative_density=0.5)])
    f.set_viscosity(4.0, 2e-4, 150)
    for _ in range(12):
        f.step(DT)
        f.synchronize()
    path = str(tmp_path / "viscous.blub")
    f.save_state(path)
    assert F.state_info(path).format_version == 32
    g = blub_b200.HybridFluid.from_state(path)
    assert g.viscosity() == f.viscosity() == (4.0, float(np.float32(2e-4)), 150)
    for _ in range(10):
        for x in (f, g):
            x.step(DT)
            x.synchronize()
    assert_identical(snapshot(f), snapshot(g))
    assert f.last_viscosity_solve() == g.last_viscosity_solve()
    f.set_viscosity(0.0)
    f.save_state(path)
    assert F.state_info(path).format_version in (1, 2, 4, 8, 16)


def test_runner_on_a_viscous_scene_equals_a_ctypes_run_and_resumes(tmp_path):
    scene, stats, state, dump = util.scene_path("dam_viscous"), str(tmp_path / "stats.json"), str(tmp_path / "s.blub"), str(tmp_path / "p.f32")
    res = subprocess.run([RUNNER, scene, "--steps", "8", "--stats", stats, "--save-state", state], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    f = blub_b200.HybridFluid.from_scene(scene)
    nu = F.scene_viscosity(scene)
    assert f.viscosity() == (nu, float(np.float32(1e-4)), 200) and abs(nu - 5.0) < 1e-5
    for _ in range(8):
        f.step(DT)
    record = json.load(open(stats))["viscosity"]
    it, err = f.last_viscosity_solve()
    assert np.float32(record["kinematic_viscosity"]) == np.float32(nu) and record["last_iterations"] == it and np.allclose(record["last_max_error"], err, rtol=1e-6)
    assert F.state_info(state).format_version == 32
    g = blub_b200.HybridFluid.from_state(state)
    a, b = snapshot(f), snapshot(g)
    for name in list(a):
        if isinstance(a[name], np.ndarray):
            assert np.array_equal(bits(a[name]), bits(b[name])), name
    res = subprocess.run([RUNNER, scene, "--steps", "4", "--load-state", state, "--dump", dump], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    for _ in range(4):
        f.step(DT)
    assert np.array_equal(np.fromfile(dump, dtype=np.float32).reshape(-1, 4)[:, :3], f.download_particles()[:, :3])
    plain = subprocess.run([RUNNER, util.scene_path("dam_small"), "--steps", "2", "--stats", stats], capture_output=True, text=True, timeout=300)
    assert plain.returncode == 0 and "viscosity" not in json.load(open(stats))
