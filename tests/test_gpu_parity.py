"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Tolerances are the stated fp32 tolerances of SURVEY.md section 8c; order-dependent quantities (atomics, reductions)
differ in the last bits, never structurally.  Everything here needs an H100: run with `-m gpu`.
"""
import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from oracle import oracle as O
from tests import util
from tests.util import DT, grid_close

pytestmark = pytest.mark.gpu


def make_pair(name, rebin=0, precond=0):
    orc = util.oracle_from_scene(name)
    gpu = blub_b200.HybridFluid.from_scene(util.scene_path(name))
    orc.set_rebin_frequency(rebin)
    gpu.set_rebin_frequency(rebin)
    orc.set_quirks(precond_mode=precond)
    gpu.set_quirks(precond_mode=precond)
    return orc, gpu


def test_scene_seeding_is_bit_exact():
    orc, gpu = make_pair("dam_small")
    assert gpu.num_particles == orc.num_particles > 0
    assert np.array_equal(gpu.download_particles()[:, :3], orc.particles()[:, :3])


def test_hydrostatic_known_answer_on_gpu():
    n = 16 * 2
    gpu = blub_b200.HybridFluid(n, n, n, 8 * n * n * n)
    gpu.add_fluid_cube([1, 1, 1], [n - 1, 9, n - 1])
    gpu.set_gravity_grid([0, -981.0, 0])
    gpu.set_rebin_frequency(0)
    gpu.set_solver_config(0, error_tolerance=1e-6, max_num_iterations=600, error_check_frequency=4)
    gpu.step_stages(DT, 0, 3)
    err, it = gpu.last_solve(0)
    assert 0 < it < 600 and err < 1e-6 / DT
    p = gpu.download_grid(F.TAP_P_VEL)
    gdt = float(np.float32(-981.0) * np.float32(DT))
    for y in range(1, 9):
        assert np.allclose(p[1:n - 1, y, 1:n - 1], gdt * (9 - y), rtol=0, atol=3e-3), y
    gpu.step_stages(DT, 4, 5)
    uy = gpu.download_grid(F.TAP_UY)
    assert np.abs(uy[1:n - 1, 1:8, 1:n - 1]).max() < 3e-3


@pytest.mark.parametrize("precond", [0, 1])
def test_stagewise_parity_one_step(precond):
    """Both implementations walk the 14 stages of one step from identical particles; taps are compared after each (tests/stagewise.py).
    Solver at the reference's defaults (0.1 / 32 / 4): iteration counts must be equal."""
    from tests import stagewise

    orc, gpu = make_pair("dam_small", rebin=0, precond=precond)
    # give the particles a non-trivial velocity / affine state
    rng = np.random.default_rng(5)
    npart = orc.num_particles
    rows = [rng.normal(0, 3.0, (npart, 4)).astype(np.float32) for _ in range(3)]
    pos = orc.particles().copy()
    orc.set_particles(pos, *rows)
    gpu.set_particles(pos, *rows)
    grav = [0.0, -981.0, 0.0]
    orc.set_gravity_grid(grav)
    gpu.set_gravity_grid(grav)
    for f in (orc, gpu):
        f.set_solver_config(0, 0.1, 32, 4)
        f.set_solver_config(1, 0.1, 32, 4)
    stagewise.compare_one_step(orc, gpu)


# a box inside the dam of dam_small at t = 0.3 s, translating toward x = 0.05 and rotating about an axis that is no grid axis, so that the
# solid velocity v + w x r has three non-zero components that differ from cell to cell (also tests/test_gpu_solids.py)
ROTATING_BOX = {"world_position": [0.17, 0.07, 0.15], "scale": 1.0, "rotation_angles": [0.0, 20.0, 0.0], "shape": "box", "half_extent": [0.03, 0.05, 0.05],
                "translation": {"target": [0.05, 0.07, 0.15], "curve": "Linear", "duration": 0.5}, "rotation": {"axis": [0.3, 1.0, 0.2], "deg_per_sec": 90.0}}
ROTATING_BOX_T = 0.3
WIDE = (40, 24, 32)  # x = 32 + 8: one full 32-cell word and an 8-cell tail per row


def moving_rows(orc, gpu, seed=5):
    rng = np.random.default_rng(seed)
    rows = [rng.normal(0, 3.0, (orc.num_particles, 4)).astype(np.float32) for _ in range(3)]
    pos = orc.particles().copy()
    orc.set_particles(pos, *rows)
    gpu.set_particles(pos, *rows)
    for f in (orc, gpu):
        f.set_gravity_grid([0.0, -981.0, 0.0])
        f.set_solver_config(0, 0.1, 32, 4)
        f.set_solver_config(1, 0.1, 32, 4)


def wide_pair():
    orc, gpu = O.OracleFluid(*WIDE, 120000), blub_b200.HybridFluid(*WIDE, 120000)
    for f in (orc, gpu):
        f.add_fluid_cube([1, 1, 1], [39, 12, 31])
        f.set_rebin_frequency(0)
    assert gpu.num_particles == orc.num_particles > 0
    return orc, gpu


def rigid_volume(dims, mask, centre, v, w):
    """RGBA volume of a rigid solid covering `mask`: velocity v + w x (cell centre - centre), rounded to fp16 as the GPU stores it."""
    nx, ny, nz = dims
    z, y, x = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    d = [x + 0.5 - centre[0], y + 0.5 - centre[1], z + 0.5 - centre[2]]
    vol = np.zeros((nz, ny, nx, 4), dtype=np.float16)
    vel = [v[0] + w[1] * d[2] - w[2] * d[1], v[1] + w[2] * d[0] - w[0] * d[2], v[2] + w[0] * d[1] - w[1] * d[0]]
    for k in range(3):
        vol[..., k][mask] = vel[k][mask]
    vol[..., 3][mask] = 1.0
    return vol


@pytest.mark.parametrize("case", ["box_scatter", "box_gather", "sphere_tail", "bodies"])
def test_stagewise_parity_with_solids(case):
    """The stage-by-stage comparison of tests/stagewise.py with a solid volume that the fluid touches: every stage's solid rule (P2G, marker,
    divergence, projection, advection, density rhs, position change, correction) against the oracle, max errors only.
      box_*        dam_small, the rotating and translating analytic box of the CUDA voxelizer, scatter and gather P2G
      sphere_tail  40 x 24 x 32, a rigid sphere across x = 32: solid cells next to fluid in the full 32-cell word and in the 8-cell tail
      bodies       40 x 24 x 32, a rotated box and a sphere as floating bodies (no borrowed volume): the composite the CUDA step builds"""
    import torch
    from tests import body_ref, stagewise

    keep = None
    if case.startswith("box"):
        orc, gpu = make_pair("dam_small", rebin=0)
        gpu.set_transfer_path(case == "box_scatter")
        dims = (32, 32, 32)
        keep = torch.zeros((32, 32, 32, 4), dtype=torch.float16, device="cuda")
        F.solid_voxelize(keep.data_ptr(), dims, ROTATING_BOX, 0.01, (0.0, 0.0, 0.0), ROTATING_BOX_T, DT)
        torch.cuda.synchronize()
        vol = keep.cpu().numpy()
        gpu.set_solid_voxels(keep.data_ptr())
        minimum = (250, 5000)
    elif case == "sphere_tail":
        orc, gpu = wide_pair()
        z, y, x = np.meshgrid(np.arange(32), np.arange(24), np.arange(40), indexing="ij")
        c = (32.3, 7.6, 15.4)
        mask = (x + 0.5 - c[0]) ** 2 + (y + 0.5 - c[1]) ** 2 + (z + 0.5 - c[2]) ** 2 <= 4.6 ** 2
        vol = rigid_volume(WIDE, mask, c, (-6.0, 3.0, 2.0), (0.5, -1.2, 2.0))
        assert (mask[..., :32] & (x[..., :32] >= 26)).any() and mask[..., 32:].any()
        keep = torch.from_numpy(vol).to("cuda").contiguous()
        gpu.set_solid_voxels(keep.data_ptr())
        minimum = (150, 3000)
    else:
        orc, gpu = wide_pair()
        h = np.sin(np.radians(15.0)) / np.sqrt(3.0)
        gpu.set_bodies([body_ref.body("box", (3.0, 2.5, 4.0), 0.7, (12.2, 9.1, 11.7), (np.cos(np.radians(15.0)), h, h, -h), (4.0, -2.0, 1.0), (0.6, 1.1, -0.8)),
                        body_ref.body("sphere", 4.0, 1.2, (28.4, 7.3, 20.6), velocity=(-3.0, 1.0, 2.0), angular_velocity=(-1.0, 0.5, 1.5))])
        vol = body_ref.composite(WIDE, None, gpu.bodies())
        minimum = (150, 3000)
    moving_rows(orc, gpu)
    report = stagewise.compare_one_step(orc, gpu, vox=vol.astype(np.float32), min_contact=minimum)
    print(case, {k: report[k] for k in ("contact0", "contact7", "branches", "advect_flips", "correct_hits", "correct_flips")})
    del keep


def test_binning_is_a_permutation_sorted_by_cell():
    orc, gpu = make_pair("dam_small", rebin=1)
    rng = np.random.default_rng(3)
    pos = orc.particles().copy()
    rng.shuffle(pos)
    gpu.set_particles(pos)
    gpu.step_stages(DT, 3, 4)
    out = gpu.download_particles()[:, :3]
    a, _ = util.sort_rows(pos[:, :3])
    b, _ = util.sort_rows(out)
    assert np.array_equal(a, b)  # same multiset, bit for bit
    c = np.floor(out).astype(np.int64)
    key = (c[:, 2] * gpu.ny + c[:, 1]) * gpu.nx + c[:, 0]
    assert (np.diff(key) >= 0).all()  # x-fastest cell order (particle_binning_prefixsum.comp:18-24)


def test_multi_step_scene_parity():
    """5 steps of a dam break: same particle order (rebin off), tight solver so the iterate is well defined."""
    orc, gpu = make_pair("dam_small", rebin=0)
    for f in (orc, gpu):
        f.set_solver_config(0, 1e-4, 128, 4)
        f.set_solver_config(1, 1e-4, 128, 4)
    for _ in range(5):
        orc.step(DT)
        gpu.step(DT)
    p_o, p_g = orc.particles()[:, :3], gpu.download_particles()[:, :3]
    d = np.abs(p_o - p_g).max(axis=1)
    assert np.isfinite(p_g).all()
    assert np.quantile(d, 0.999) <= 1e-2, (np.quantile(d, 0.999), d.max())
    v_o = np.c_[orc.particles(O.ARR_ROWX)[:, 3], orc.particles(O.ARR_ROWY)[:, 3], orc.particles(O.ARR_ROWZ)[:, 3]].astype(np.float64)
    v_g = np.c_[gpu.download_particles(F.TAP_VX)[:, 3], gpu.download_particles(F.TAP_VY)[:, 3], gpu.download_particles(F.TAP_VZ)[:, 3]].astype(np.float64)
    mom_o, mom_g = v_o.sum(0), v_g.sum(0)
    ke_o, ke_g = (v_o ** 2).sum(), (v_g ** 2).sum()
    assert abs(ke_o - ke_g) <= 1e-3 * ke_o
    assert np.abs(mom_o - mom_g).max() <= 1e-3 * np.abs(v_o).sum(0).max()


def test_single_cell_debug_scene_one_step():
    # configs[0] of BASELINE.json: the reference's own debug scene (8 particles), rebin off (SURVEY B2)
    orc, gpu = make_pair("single_cell_debug", rebin=0)
    orc.step(DT)
    gpu.step(DT)
    assert gpu.num_particles == 8
    assert np.abs(orc.particles()[:, :3] - gpu.download_particles()[:, :3]).max() <= 2e-4
    for to, tg in [(O.ARR_ROWX, F.TAP_VX), (O.ARR_ROWY, F.TAP_VY), (O.ARR_ROWZ, F.TAP_VZ)]:
        assert np.abs(orc.particles(to) - gpu.download_particles(tg)).max() <= 1e-3 * 10


def test_statistics_are_asynchronous_and_scaled_by_dt():
    _, gpu = make_pair("dam_small", rebin=0)
    for _ in range(3):
        gpu.step(DT)
    gpu.synchronize()
    gpu.update_statistics()
    sv, sd = gpu.pressure_solver_stats(0), gpu.pressure_solver_stats(1)
    assert len(sv) == 3 and len(sd) == 3
    e, it = gpu.last_solve(1)
    assert sd[-1][1] == it and abs(sd[-1][0] - e * DT) <= 1e-6 * max(1.0, e * DT)
    assert all(i % 4 == 0 and 4 <= i <= 32 for _, i in sv + sd)


def test_solid_voxels_block_flow():
    """A static solid slab (synthetic analytic solid written straight into the RGBA16F volume) -- config C5's mechanism.  The slab borders the
    dam (fluid in the cells x < 16) over the lower half of its height and carries a velocity with three non-zero components."""
    import torch
    orc, gpu = make_pair("dam_small", rebin=0)
    vox = np.zeros((32, 32, 32, 4), dtype=np.float32)
    vox[4:28, 1:12, 16:19] = (5.0, 1.0, -2.0, 1.0)  # cells/s; fp16-exact
    orc.set_voxels(vox)
    util.tight_solver(orc, gpu)  # trajectory comparison: converged solves (SURVEY 8c)
    tv = torch.from_numpy(vox).to("cuda").to(torch.float16).contiguous()
    gpu.set_solid_voxels(tv.data_ptr())
    for _ in range(2):
        orc.step(DT)
        gpu.step(DT)
        faces, near = util.solid_contact(orc.grid(O.ARR_MARKER), vox, orc.particles())
        assert faces >= 150 and near >= 1500, (faces, near)
    gpu.synchronize()
    util.markers_agree(orc.grid(O.ARR_MARKER), gpu.download_grid(F.TAP_MARKER))
    d = np.abs(orc.particles()[:, :3] - gpu.download_particles()[:, :3]).max(axis=1)
    assert np.quantile(d, 0.999) <= 5e-3, (np.quantile(d, 0.999), d.max())
    inside = vox[..., 3] > 0
    counts = []
    for p in (gpu.download_particles()[:, :3], orc.particles()[:, :3]):
        c = np.floor(p).astype(int)
        counts.append(int(inside[c[:, 2], c[:, 1], c[:, 0]].sum()))
    # the correction may carry a particle across the slab's face (its step is cut to the distance from the face behind it, as written in
    # density_projection_correct_particles.comp:48-70): a few, and the same few in both implementations
    assert counts[0] <= 0.01 * orc.num_particles and abs(counts[0] - counts[1]) <= 0.001 * orc.num_particles, counts


def test_graph_replay_matches_eager_launches():
    """blub_fluid_step replays a captured CUDA graph (persistent PCG inside); the eager three-kernel path must agree.
    Rebinning off so that particles keep their index; the two solver paths group their partial sums differently, so the runs differ in
    the last bits only."""
    a = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    b = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    b.set_graph_replay(False)
    b.set_solver_path(False)
    for f in (a, b):
        f.set_rebin_frequency(0)
        f.set_solver_config(0, 1e-4, 128, 4)
        f.set_solver_config(1, 1e-4, 128, 4)
    dts = [DT, DT, DT * 0.25, DT]  # a changed dt must reach the replayed graph through the device StepParams block
    for dt in dts:
        a.step(dt)
        b.step(dt)
    pa, pb = a.download_particles()[:, :3], b.download_particles()[:, :3]
    d = np.abs(pa - pb).max(axis=1)
    assert np.isfinite(pa).all() and np.quantile(d, 0.999) <= 2e-3 and d.max() <= 5e-2, (np.quantile(d, 0.999), d.max())
    # the same four steps with a constant dt end somewhere else: the dt change really was applied
    c = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
    c.set_rebin_frequency(0)
    for _ in dts:
        c.step(DT)
    assert np.abs(c.download_particles()[:, :3] - pa).max() > 1e-2
    a.synchronize(); b.synchronize()
    a.update_statistics(); b.update_statistics()
    sa, sb = a.pressure_solver_stats(0), b.pressure_solver_stats(0)
    assert len(sa) == len(sb) == 4
    assert all(abs(x[1] - y[1]) <= 4 for x, y in zip(sa, sb))
    ca = blub_b200.kernel_launch_count()
    a.step(DT)
    assert blub_b200.kernel_launch_count() - ca >= 20  # graph replays are counted kernel by kernel


def test_default_step_is_bit_identical_run_to_run():
    """The scatter kernels add into fixed-point integer accumulators: whatever order their atomics arrive in, two fluids built from the
    same scene compute the same steps bit for bit (1.2 M particles, many warps per face; rebinning at step 0 and every 8th step)."""
    runs = []
    for _ in range(2):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_halfhalf"))
        for _ in range(10):
            f.step(DT)
        f.synchronize()
        runs.append([f.download_particles(t) for t in (F.TAP_POS, F.TAP_VX, F.TAP_VY, F.TAP_VZ)]
                    + [f.download_grid(t) for t in (F.TAP_UX, F.TAP_UY, F.TAP_UZ, F.TAP_MARKER, F.TAP_P_VEL, F.TAP_P_DEN)]
                    + [np.array([f.last_solve(w) for w in (0, 1)])])
        f.close()
    for k, (a, b) in enumerate(zip(*runs)):
        assert a.shape == b.shape and np.array_equal(a, b), k


def test_binning_steps_flip_buffers_without_losing_particles():
    """Rebinning every step: graph replay has to follow the position ping-pong buffers."""
    for graph in (True, False):
        f = blub_b200.HybridFluid.from_scene(util.scene_path("dam_small"))
        f.set_graph_replay(graph)
        f.set_rebin_frequency(1)
        n = f.num_particles
        for _ in range(5):
            f.step(DT)
        p = f.download_particles()[:, :3]
        assert p.shape[0] == n and np.isfinite(p).all()
        assert p.min() >= 1.0 and (p.max(axis=0) <= np.array([f.nx, f.ny, f.nz]) - 1.0).all()
        # still 8 particles per cell on average in the bulk of the column: nothing duplicated or dropped
        c = np.floor(p).astype(np.int64)
        counts = np.bincount((c[:, 2] * f.ny + c[:, 1]) * f.nx + c[:, 0], minlength=f.n)
        assert counts.sum() == n and counts.max() < 40


def test_empty_fluid_steps_without_particles():
    """Edge case: no particles at all (every cell AIR / SOLID): the step must run, the solves report 0 error."""
    gpu = blub_b200.HybridFluid(32, 32, 32, 1000)
    gpu.set_gravity_grid([0, -981.0, 0])
    for _ in range(2):
        gpu.step(DT)
    gpu.synchronize()
    gpu.update_statistics()
    assert gpu.num_particles == 0
    m = gpu.download_grid(F.TAP_MARKER)
    assert (m[1:-1, 1:-1, 1:-1] == O.AIR).all() and (m[0] == O.SOLID).all()
    assert all(e == 0.0 for e, _ in gpu.pressure_solver_stats(0))
    assert np.all(gpu.download_grid(F.TAP_P_VEL) == 0)


def test_add_cube_truncates_at_max_num_particles():
    """hybrid_fluid.rs:627-633: more particles than max_num_particles -> log + truncate (here: BLUB_WARN_TRUNCATED)."""
    orc = O.OracleFluid(32, 32, 32, 1000)
    gpu = blub_b200.HybridFluid(32, 32, 32, 1000)
    n_o, trunc_o = orc.add_fluid_cube([1, 1, 1], [9, 9, 9])
    assert gpu.add_fluid_cube([1, 1, 1], [9, 9, 9]) is True and trunc_o
    assert gpu.num_particles == orc.num_particles == 1000
    assert np.array_equal(gpu.download_particles()[:, :3], orc.particles()[:, :3])
    assert gpu.add_fluid_cube([1, 1, 1], [2, 2, 2]) is True and gpu.num_particles == 1000  # full: nothing added
    gpu.step(DT)
    assert np.isfinite(gpu.download_particles()).all()


def test_ragged_grid_full_step_parity():
    """A grid whose x extent is not a multiple of 32 cells (8-cell occupancy segments, 8-lane solver tiles, N % 16384 != 0)."""
    nx, ny, nz = 24, 40, 32
    orc = O.OracleFluid(nx, ny, nz, 30000)
    gpu = blub_b200.HybridFluid(nx, ny, nz, 30000)
    for f in (orc, gpu):
        f.add_fluid_cube([1, 1, 1], [12, 20, 31])
        f.set_gravity_grid([0.0, -981.0, 0.0])
        f.set_rebin_frequency(0)
        f.set_solver_config(0, 1e-4, 200, 4)
        f.set_solver_config(1, 1e-4, 200, 4)
    assert gpu.num_particles == orc.num_particles
    for _ in range(3):
        orc.step(DT)
        gpu.step(DT)
    util.markers_agree(orc.grid(O.ARR_MARKER), gpu.download_grid(F.TAP_MARKER))
    d = np.abs(orc.particles()[:, :3] - gpu.download_particles()[:, :3]).max(axis=1)
    assert np.quantile(d, 0.999) <= 5e-3, (np.quantile(d, 0.999), d.max())


def test_particles_outside_the_domain_do_not_crash():
    """Memory safety for ANY input: particles handed in outside the grid are clamped by the scatter kernels, not written out of bounds."""
    gpu = blub_b200.HybridFluid(32, 32, 32, 64)
    pos = np.array([[-5.0, 3.0, 3.0, 0], [40.0, 3.0, 3.0, 0], [3.0, -1e6, 3.0, 0], [3.0, 3.0, 1e6, 0], [16.2, 16.7, 16.1, 0]], dtype=np.float32)
    gpu.set_particles(pos)
    gpu.step(DT)
    gpu.synchronize()
    p = gpu.download_particles()[:, :3]
    assert np.isfinite(p).all() and p.min() >= 1.0 and p.max() <= 31.0
