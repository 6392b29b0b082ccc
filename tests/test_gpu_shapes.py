"""GPU: every stage on grids at the edges of the kernels' tilings, against the oracle and against the float64 per-face references of
tests/grid_ref.py.

Every kernel on the step path tiles the grid its own way and has a last, partial piece whose size depends on the grid: the 32-cell words of
the FLUID bit mask and of the particle words, the 30-face x blocks of the gather P2G, the 28 x 4 x 4 cell bricks of the scatter schedule,
the scatter tiles' windows, the PCG tiles / quads / 4-plane marches and the TMA boxes (nx % 128 == 0).  SHAPES lists the grids that put
those pieces at their edges; every test below runs on every row (sections 4 and 5b on two rows), and every row's fluid reaches the last
word, the last gather block and the last brick of its rows (assert_edges).

The P2G scatter walks the brick schedule's work items only when they fill several waves of resident blocks (P2G_MIN_ITEM_WAVES, millions of
particles); at these sizes it runs its 256-particle chunks, and test_schedule_steps_on_work_items_match_float64_reference runs the schedule
steps again with BLUB_P2G_ITEM_WAVES=0, which sends P2G through the items here too.  The density scatter walks the items at every size:
the schedule-on steps below check it against the float64 reference."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (nx, ny, nz): what the row exercises
SHAPES = {
    (8, 48, 48): "one partial bit-mask word per row, 2 PCG quads, 8 of 30 gather faces, one partial brick in x; N % 16384 != 0",
    (48, 8, 48): "one PCG tile row and two brick rows in y; the extrapolation's 3 x 3 in-plane neighbourhood at both y walls",
    (48, 48, 8): "two 4-plane PCG marches; gather blocks of exactly 8 z-rows (6 stored + 2 halo)",
    (264, 8, 8): "9 words with an 8-cell tail, 3 PCG tiles (the last 8 cells wide), thin in y and z at once",
    (8, 8, 272): "a 6 x 6 interior column, 68 z-marches, bricks of 8 x 4 x 4",
    (120, 16, 24): "x a multiple of 30 (full last gather block) and of 8 but not of 32 (3 words + 24), bricks 4 x 28 + 8",
    (56, 40, 24): "x = 2 bricks exactly, 1 word + 24-cell tail",
    (128, 24, 16): "the TMA solver path is available; a single 128-wide PCG tile",
}
IDS = [f"{nx}x{ny}x{nz}" for nx, ny, nz in SHAPES]
SHAPE_LIST = list(SHAPES)
PAIR_SHAPES = [(8, 48, 48), (56, 40, 24)]  # the particle-count and body / probe rows
PATHS = [True, False]  # scatter, gather


def shape_params(shapes=SHAPE_LIST):
    return pytest.mark.parametrize("dims", shapes, ids=[f"{a}x{b}x{c}" for a, b, c in shapes])


path_params = pytest.mark.parametrize("scatter", PATHS, ids=["scatter", "gather"])


def fluid_box(dims):
    """A box from the x = 0 wall to the x = nx - 1 wall, on the floor, between both z walls, up to half the height (at most 12 cells)."""
    nx, ny, nz = dims
    return [1, 1, 1], [nx - 1, min(max(4, ny // 2), 12), nz - 1]


def assert_edges(marker):
    """FLUID cells in the last 32-cell word of the rows, in the last gather block (30 faces) and in the last brick (28 cells) along x."""
    from oracle import oracle as O

    nx = marker.shape[2]
    fl = (marker == O.FLUID).any(axis=(0, 1))
    for name, w in (("word", 32), ("gather block", 30), ("brick", 28)):
        assert fl[w * ((nx - 1) // w):].any(), f"no FLUID cell in the last {name} of the rows (nx = {nx})"


def pair(dims, capacity=None):
    import blub_b200
    from oracle import oracle as O

    lo, hi = fluid_box(dims)
    cap = capacity or 8 * int(np.prod(np.subtract(hi, lo))) + 4096
    orc, gpu = O.OracleFluid(*dims, cap), blub_b200.HybridFluid(*dims, cap)
    for f in (orc, gpu):
        f.add_fluid_cube(lo, hi)
        f.set_rebin_frequency(0)
    assert gpu.num_particles == orc.num_particles > 0
    return orc, gpu


def sphere_volume(dims):
    """A rigid sphere (moving and rotating) inside the fluid, across the last 32-cell word of the rows."""
    from tests.test_gpu_parity import rigid_volume

    nx, ny, nz = dims
    lo, hi = fluid_box(dims)
    r = 2.2 if min(dims) == 8 else 3.4
    c = (nx - 1.4 - r, min(hi[1] - 0.6, 1.3 + r), nz / 2 + 0.3)
    z, y, x = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    mask = (x + 0.5 - c[0]) ** 2 + (y + 0.5 - c[1]) ** 2 + (z + 0.5 - c[2]) ** 2 <= r ** 2
    assert mask[..., 32 * ((nx - 1) // 32):].any()
    return rigid_volume(dims, mask, c, (-6.0, 3.0, 2.0), (0.5, -1.2, 2.0))


# ------------------------------------------------------------------------------------------------ 2. every stage against the oracle
@pytest.mark.gpu
@path_params
@pytest.mark.parametrize("solid", [None, "sphere"])
@shape_params()
def test_stagewise_parity_on_shape(dims, solid, scatter):
    """tests/stagewise.py from identical particles with random APIC rows; with a moving sphere in the last x word, max errors only."""
    import torch
    from tests import grid_ref as R
    from tests import stagewise
    from tests.test_gpu_parity import moving_rows

    orc, gpu = pair(dims)
    gpu.set_transfer_path(scatter)
    moving_rows(orc, gpu)
    assert_edges(R.marker(orc.particles(), dims))
    if solid is None:
        stagewise.compare_one_step(orc, gpu)
        return
    vol = sphere_volume(dims)
    keep = torch.from_numpy(vol).to("cuda").contiguous()
    gpu.set_solid_voxels(keep.data_ptr())
    report = stagewise.compare_one_step(orc, gpu, vox=vol.astype(np.float32), min_contact=(10, 100))
    print(dims, {k: report[k] for k in ("contact0", "contact7", "branches", "advect_flips", "correct_hits", "correct_flips")})
    del keep


@pytest.mark.gpu
@shape_params()
def test_pcg_paths_on_shape(dims):
    """Every solver path against the oracle (20 fixed iterations), the tile kernel with the sparse bodies (6) equal to its dense form (4)
    bit for bit, and p = 0 off FLUID on every path."""
    import blub_b200
    from blub_b200 import fluid as F
    from oracle import oracle as O
    from tests.util import DT, grid_close

    nx, ny, nz = dims
    rng = np.random.default_rng(nx * 10000 + ny * 100 + nz)
    m = np.full((nz, ny, nx), O.AIR, dtype=np.int8)
    m[rng.random((nz, ny, nx)) < 0.8] = O.FLUID
    m[rng.random((nz, ny, nx)) < 0.04] = O.SOLID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = rng.uniform(-1, 1, (nz, ny, nx)).astype(np.float32)
    orc = O.OracleFluid(nx, ny, nz, 8)
    orc.set_solver_config(0, 0.0, 20, 4)
    orc.grid(O.ARR_MARKER)[:] = m
    orc.grid(O.ARR_RESIDUAL)[:] = b
    orc.solve(0, DT)
    out = {}
    for path in [1, 6, 4, 0] + ([2] if nx % 128 == 0 else []):
        gpu = blub_b200.HybridFluid(nx, ny, nz, 8)
        gpu.set_solver_path(path)
        gpu.set_solver_config(0, 0.0, 20, 4)
        gpu.upload_grid(F.TAP_MARKER, m)
        gpu.upload_grid(F.TAP_RESIDUAL, b)
        gpu.solve_only(0, DT)
        p = gpu.download_grid(F.TAP_P_VEL)
        assert gpu.last_solve(0)[1] == 20, path
        assert (p[m != O.FLUID] == 0).all(), path
        grid_close(orc.grid(O.ARR_P_VEL), p, f"pressure path={path}", rel=3e-3, abs_=1e-4)
        out[path] = (p, gpu.last_solve(0))
        gpu.close()
    assert out[6][1] == out[4][1] and np.array_equal(out[6][0], out[4][0])


# ------------------------------------------------------------------------------------------------ 3. float64 per-face references
BOUND_RATIOS = {"p2g": [], "rhs": []}  # per-face bound / the grid_close tolerance it replaces, printed by every reference test


def print_bound_ratios(what):
    for k, parts in BOUND_RATIOS.items():
        if parts:
            r = np.concatenate(parts)
            print(f"{what} {k}: {r.size} entries, bound / grid_close tolerance: median {np.median(r):.2e}, max {r.max():.2e}")
        parts.clear()


def reference_particles(dims, order, seed=7):
    """The box fluid's particles, a crowd of 1600 particles in one cell of the last x word, and particles exactly on cell planes and on the
    clamp planes (1.0, 1.001, n - 1.001, n - 1.0); order: "sorted" (x-fastest cell order, as a re-sort leaves it), "shuffled" (random: most
    faces take the scatters' global path) or "decayed" (sorted, then jittered by up to a third of a cell)."""
    from oracle import oracle as O

    nx, ny, nz = dims
    lo, hi = fluid_box(dims)
    f = O.OracleFluid(nx, ny, nz, 8 * int(np.prod(np.subtract(hi, lo))) + 16)
    f.add_fluid_cube(lo, hi)
    p = f.particles()[:, :3].astype(np.float32)
    rng = np.random.default_rng(seed)
    crowd_cell = np.array([nx - 2, 1, nz - 2], dtype=np.float32)
    crowd = (crowd_cell + rng.uniform(0.0, 1.0, (1600, 3))).astype(np.float32)
    planes = []
    for ax, n in enumerate(dims):
        for v in (1.0, np.float32(1.001), np.float32(n) - np.float32(1.001), n - 1.0, 2.0, 3.0, float(n // 2)):
            q = rng.uniform(1.5, 3.5, (6, 3)).astype(np.float32)
            q[:, ax] = v
            planes.append(q)
    p = np.concatenate([p, crowd] + planes).astype(np.float32)
    p = np.minimum(p, (np.array(dims) - 1).astype(np.float32))
    key = lambda q: (lambda c: (c[:, 2] * ny + c[:, 1]) * nx + c[:, 0])(np.floor(q).astype(np.int64))
    p = p[np.argsort(key(p), kind="stable")] if order != "shuffled" else p[rng.permutation(len(p))]
    if order == "decayed":  # the particles drift after the re-sort: many leave the cell their slot was sorted by
        sorted_key = key(p)
        p = np.clip(p + rng.uniform(-0.33, 0.33, p.shape), 1.001, np.array(dims, np.float32) - np.float32(1.001)).astype(np.float32)
        moved = key(p) != sorted_key
        assert moved.mean() > 0.25 and (np.diff(key(p)) < 0).mean() > 0.1, (moved.mean(), (np.diff(key(p)) < 0).mean())
    rows = [rng.normal(0, 3.0, (len(p), 4)).astype(np.float32) for _ in range(3)]
    return np.c_[p, np.zeros(len(p), np.float32)], rows


def check_p2g(gpu, pos, rows, scatter, gdt, what):
    """The P2G stage's marker (exact) and velocities (per-face bound) against the float64 reference of these particles."""
    from blub_b200 import fluid as F
    from tests import grid_ref as R

    dims = (gpu.nx, gpu.ny, gpu.nz)
    m = R.marker(pos, dims)
    assert np.array_equal(gpu.download_grid(F.TAP_MARKER), m), f"{what}: marker"
    sums = R.p2g_sums(pos, rows, dims)
    want = R.p2g_velocity(sums, m, gdt)
    bounds = R.p2g_bound(sums, m, gdt, "scatter" if scatter else "gather")
    for c, tap in enumerate((F.TAP_UX, F.TAP_UY, F.TAP_UZ)):
        got = gpu.download_grid(tap)
        _, b = R.check(got, want[c], bounds[c], f"{what}: P2G u[{c}]")
        sel = ~np.isnan(want[c])
        tol = 1e-4 * max(np.abs(got[sel]).max(), np.abs(want[c][sel]).max()) + 1e-5
        BOUND_RATIOS["p2g"].append(b[np.isfinite(b) & (b > 0)] / tol)
    return m


def check_rhs(gpu, dt, what):
    """The density rhs (stage 9) against the float64 reference of the positions and the marker the density pass saw.  The density pass is
    density_scatter_kernel on both transfer paths: the scatter-form bound."""
    from blub_b200 import fluid as F
    from tests import grid_ref as R

    dims = (gpu.nx, gpu.ny, gpu.nz)
    pos = gpu.download_particles()
    m = gpu.download_grid(F.TAP_MARKER)
    d = R.density_sums(pos, dims)
    got = gpu.download_grid(F.TAP_RESIDUAL)
    _, b = R.check(got, R.density_rhs(d, m, dt), R.rhs_bound(d, m, dt, "scatter"), f"{what}: density rhs")
    tol = 1e-4 * np.abs(got[m == R.FLUID]).max() + 2e-3  # stagewise's rhs2 tolerance
    BOUND_RATIOS["rhs"].append(b / tol)


def gravity_dt(g, dt):
    return [float(np.float32(v) * np.float32(dt)) for v in g]


@pytest.mark.gpu
@path_params
@pytest.mark.parametrize("order", ["sorted", "shuffled", "decayed"])
@shape_params()
def test_p2g_and_density_match_float64_reference(dims, order, scatter):
    """P2G and the density rhs of one set of particles (crowd, plane and clamp-plane particles included) against grid_ref, per face / cell.
    The density pass runs behind a zero velocity grid, so its particles are the P2G's (up to the advection's wall clamp)."""
    import blub_b200
    from blub_b200 import fluid as F
    from tests.util import DT

    pos, rows = reference_particles(dims, order)
    gpu = blub_b200.HybridFluid(*dims, len(pos))
    gpu.set_transfer_path(scatter)
    gpu.set_rebin_frequency(0)
    g = [3.0, -981.0, -2.0]
    gpu.set_gravity_grid(g)
    gpu.set_particles(pos, *rows)
    gpu.step_stages(DT, 0, 1)
    m = check_p2g(gpu, pos, rows, scatter, gravity_dt(g, DT), f"{dims} {order}")
    assert_edges(m)
    for tap in (F.TAP_UX, F.TAP_UY, F.TAP_UZ):
        gpu.upload_grid(tap, np.zeros(m.shape, np.float32))
    gpu.step_stages(DT, 6, 10)  # clear, advect, boundary marker, density rhs
    check_rhs(gpu, DT, f"{dims} {order}")
    print_bound_ratios(f"{dims} {order} {'scatter' if scatter else 'gather'}")


@pytest.mark.gpu
@path_params
@shape_params()
def test_schedule_steps_match_float64_reference(dims, scatter):
    """Ten steps with the default re-sorts (steps 0 and 8): every step's P2G and density rhs against the float64 reference of the particles it
    read.  The density scatter runs the brick schedule's work items from the re-sort of step 0 on; the P2G scatter runs its chunks, or under
    BLUB_P2G_ITEM_WAVES=0 (test_schedule_steps_on_work_items_match_float64_reference) the work items too, whose count is then restated from
    the cell order the re-sort of step 0 left and must be non-zero."""
    import blub_b200
    from blub_b200 import fluid as F
    from tests.util import DT

    lo, hi = fluid_box(dims)
    gpu = blub_b200.HybridFluid(*dims, 8 * int(np.prod(np.subtract(hi, lo))) + 16)
    gpu.set_transfer_path(scatter)
    gpu.add_fluid_cube(lo, hi)
    g = [0.0, -981.0, 0.0]
    gpu.set_gravity_grid(g)
    for k in range(10):
        pos = gpu.download_particles()
        rows = [gpu.download_particles(t) for t in (F.TAP_VX, F.TAP_VY, F.TAP_VZ)]
        gpu.step_stages(DT, 0, 1)
        check_p2g(gpu, pos, rows, scatter, gravity_dt(g, DT), f"{dims} step {k}")
        gpu.step_stages(DT, 1, 4)
        if k == 0 and scatter and os.environ.get("BLUB_P2G_ITEM_WAVES") == "0":  # the items the next steps' P2G walks
            from tests.test_gpu_bench_scale import schedule

            items = int(schedule(gpu.download_particles(), dims)["brick_items"].sum())
            assert items > 0, f"{dims}: no work item after the re-sort of step 0"
            print(f"{dims}: {items} work items for P2G from step 1 on")
        gpu.step_stages(DT, 4, 10)
        check_rhs(gpu, DT, f"{dims} step {k}")
        gpu.step_stages(DT, 10, 14)
    print_bound_ratios(f"{dims} schedule steps {'scatter' if scatter else 'gather'}")


@pytest.mark.gpu
def test_schedule_steps_on_work_items_match_float64_reference():
    """test_schedule_steps_match_float64_reference on every row and path again under BLUB_P2G_ITEM_WAVES=0 (read once per process, hence a
    fresh pytest): the P2G scatter then walks the brick schedule's work items from the re-sort of step 0 on, so that its item path meets the
    brick edges the rows were chosen for."""
    env = dict(os.environ, BLUB_P2G_ITEM_WAVES="0")
    res = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "gpu",
                          f"{os.path.abspath(__file__)}::test_schedule_steps_match_float64_reference"], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=1800)
    assert res.returncode == 0 and f"{2 * len(SHAPES)} passed" in res.stdout, res.stdout[-6000:] + res.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ 4. particle counts at warp and chunk edges
COUNTS = [1, 31, 32, 33, 255, 256, 257, "full"]


def count_pair(dims, count):
    """`count` particles of the box fluid next to the last x word's fluid, in cell order; "full": the whole box in a fluid of exactly that
    capacity."""
    import blub_b200
    from oracle import oracle as O

    if count == "full":
        orc, gpu = pair(dims)
        n = orc.num_particles
        orc, gpu = pair(dims, capacity=n)
        assert gpu.num_particles == n
        return orc, gpu
    orc0, _ = pair(dims)
    p = orc0.particles()[:, :3].copy()
    nx, ny, nz = dims
    near = np.argsort(np.abs(p - np.array([nx - 2.5, 2.0, nz / 2])).sum(axis=1), kind="stable")[:count]
    sel = np.sort(near)
    pos = np.c_[p[sel], np.zeros(count, np.float32)]
    orc, gpu = O.OracleFluid(*dims, 4096), blub_b200.HybridFluid(*dims, 4096)
    for f in (orc, gpu):
        f.set_particles(pos)
        f.set_rebin_frequency(0)
    return orc, gpu


@pytest.mark.gpu
@path_params
@pytest.mark.parametrize("count", COUNTS)
@shape_params(PAIR_SHAPES)
def test_particle_counts_stagewise(dims, count, scatter):
    """P2G, density rhs, advection and correction against the oracle, stage by stage, at counts around a warp (32) and a chunk (256)."""
    from tests import stagewise
    from tests.test_gpu_parity import moving_rows

    orc, gpu = count_pair(dims, count)
    gpu.set_transfer_path(scatter)
    moving_rows(orc, gpu)
    stagewise.compare_one_step(orc, gpu)


def step_digest(f):
    from blub_b200 import fluid as F

    f.synchronize()
    h = hashlib.sha256()
    for t in (F.TAP_POS, F.TAP_VX, F.TAP_VY, F.TAP_VZ):
        h.update(np.ascontiguousarray(f.download_particles(t)).tobytes())
    for t in (F.TAP_UX, F.TAP_UY, F.TAP_UZ, F.TAP_MARKER, F.TAP_P_VEL, F.TAP_P_DEN, F.TAP_RESIDUAL):
        h.update(np.ascontiguousarray(f.download_grid(t)).tobytes())
    h.update(np.array([f.last_solve(w) for w in (0, 1)], dtype=np.float64).tobytes())
    return h.hexdigest()


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [True, False], ids=["graph", "eager"])
@path_params
@shape_params(PAIR_SHAPES)
def test_stale_slots_behind_the_count_are_not_read(dims, scatter, graph):
    """A fluid that held 300 particles (and stepped with them) is given 33 by set_particles: its next three steps equal those of a fresh fluid
    given the same 33, bit for bit.  A kernel that read the slots of a partial warp or chunk behind the count would see the old particles
    there, where a fresh fluid has zeros."""
    import blub_b200
    from blub_b200 import fluid as F
    from tests.util import DT

    orc0, _ = pair(dims)
    p = orc0.particles()[:, :3].copy()
    rng = np.random.default_rng(9)
    pick = np.sort(rng.choice(len(p), 300, replace=False))
    pos300 = np.c_[p[pick], np.zeros(300, np.float32)]
    rows300 = [rng.normal(0, 3.0, (300, 4)).astype(np.float32) for _ in range(3)]
    pos33, rows33 = pos300[150:183].copy(), [r[150:183].copy() for r in rows300]
    used, fresh = blub_b200.HybridFluid(*dims, 512), blub_b200.HybridFluid(*dims, 512)
    for f in (used, fresh):
        f.set_transfer_path(scatter)
        f.set_graph_replay(graph)
        f.set_gravity_grid([0.0, -981.0, 0.0])
        f.set_rebin_frequency(1)  # a re-sort in every step, whatever the step count: both position buffers are read and written
    used.set_particles(pos300, *rows300)
    for _ in range(2):  # every per-particle array holds live data
        used.step(DT)
    used.synchronize()
    for f in (used, fresh):
        f.set_particles(pos33, *rows33)
        # the grids the next step does not rewrite everywhere (faces away from the fluid, the solvers' warm start) start equal
        for tap in (F.TAP_UX, F.TAP_UY, F.TAP_UZ, F.TAP_P_VEL, F.TAP_P_DEN, F.TAP_RESIDUAL):
            f.upload_grid(tap, np.zeros((f.nz, f.ny, f.nx), np.float32))
    for k in range(3):
        used.step(DT)
        fresh.step(DT)
        assert step_digest(used) == step_digest(fresh), k


# ------------------------------------------------------------------------------------------------ 5. trajectories and reproducibility
STEPS = 16


def run_trajectories(dims):
    """Digests of 16 steps of the shape's box fluid (default re-sorts: steps 0 and 8), graph-replayed and eager, per step."""
    import blub_b200

    out = {}
    for graph in (True, False):
        lo, hi = fluid_box(dims)
        f = blub_b200.HybridFluid(*dims, 8 * int(np.prod(np.subtract(hi, lo))) + 16)
        f.set_graph_replay(graph)
        f.add_fluid_cube(lo, hi)
        f.set_gravity_grid([0.0, -981.0, 0.0])
        out["graph" if graph else "eager"] = []
        for _ in range(STEPS):
            f.step()
            out["graph" if graph else "eager"].append(step_digest(f))
        f.close()
    return out


def _subprocess_digests(tmp_path, schedule):
    out = str(tmp_path / f"shapes_{schedule}.npz")
    env = dict(os.environ)
    if schedule == "off":
        env["BLUB_SCATTER_SCHEDULE"] = "off"
    else:
        env.pop("BLUB_SCATTER_SCHEDULE", None)
    res = subprocess.run([sys.executable, "-m", "tests.test_gpu_shapes", out], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout + res.stderr
    return {k: list(v) for k, v in np.load(out).items()}


@pytest.mark.gpu
def test_trajectories_graph_eager_and_schedule_agree_bit_for_bit(tmp_path):
    """On every shape, 16 steps: graph replay equals eager launches, and BLUB_SCATTER_SCHEDULE=off (chunks only) equals the default brick
    schedule, bit for bit, each schedule setting in a fresh process."""
    on, off = _subprocess_digests(tmp_path, "on"), _subprocess_digests(tmp_path, "off")
    assert sorted(on) == sorted(off) == sorted(f"{i}_{m}" for i in IDS for m in ("graph", "eager"))
    for i in IDS:
        assert on[f"{i}_graph"] == on[f"{i}_eager"], f"{i}: graph replay vs eager"
        assert on[f"{i}_graph"] == off[f"{i}_graph"], f"{i}: schedule on vs off"
        assert off[f"{i}_graph"] == off[f"{i}_eager"], f"{i}: graph replay vs eager, schedule off"


@pytest.mark.gpu
@shape_params()
def test_five_steps_against_oracle(dims):
    """5 steps with converged solves: markers agree up to a few surface cells, the 99.9 % quantile of the position error stays within 1e-2."""
    from blub_b200 import fluid as F
    from oracle import oracle as O
    from tests import util
    from tests.util import DT

    orc, gpu = pair(dims)
    for f in (orc, gpu):
        f.set_gravity_grid([0.0, -981.0, 0.0])
    util.tight_solver(orc, gpu)
    for _ in range(5):
        orc.step(DT)
        gpu.step(DT)
    gpu.synchronize()
    util.markers_agree(orc.grid(O.ARR_MARKER), gpu.download_grid(F.TAP_MARKER))
    d = np.abs(orc.particles()[:, :3] - gpu.download_particles()[:, :3]).max(axis=1)
    assert np.isfinite(d).all() and np.quantile(d, 0.999) <= 1e-2, (np.quantile(d, 0.999), d.max())


@pytest.mark.gpu
@shape_params(PAIR_SHAPES)
def test_body_and_probe_records_graph_vs_eager(dims):
    """16 steps with a floating box and a load probe whose box reaches the last x word: the body and probe records of the eager fluid equal
    those of its graph-replayed twin bit for bit, and the probe sees wetted faces."""
    import blub_b200
    from tests import body_ref

    nx, ny, nz = dims
    lo, hi = fluid_box(dims)
    half = (1.5, 1.5, min(3.0, (nz - 4) / 4))
    body = body_ref.body("box", half, 0.6, (nx - 3.2, hi[1] - 1.0, nz / 2 + 0.2), velocity=(-2.0, 0.0, 1.0))
    probe = ([32 * ((nx - 1) // 32), 0, 0], [nx, ny, nz])
    rec = []
    for graph in (True, False):
        f = blub_b200.HybridFluid(*dims, 8 * int(np.prod(np.subtract(hi, lo))) + 16)
        f.set_graph_replay(graph)
        f.add_fluid_cube(lo, hi)
        f.set_gravity_grid([0.0, -981.0, 0.0])
        f.set_bodies([body])
        f.set_load_probes([probe])
        for _ in range(STEPS):
            f.step()
        rec.append((f.body_history(0), f.load_history(0)))
        f.close()
    for which in range(2):
        a, b = rec[0][which], rec[1][which]
        assert sorted(a) == sorted(b) and len(a["step"]) == STEPS
        for k in a:
            assert np.array_equal(a[k], b[k]), (which, k)
    assert rec[0][1]["wetted_faces"].max() > 0


# ------------------------------------------------------------------------------------------------ 6. gravity along every axis
AXES = [(a, s) for a in range(3) for s in (-1, 1)]
AXIS_IDS = [("-" if s < 0 else "+") + "xyz"[a] for a, s in AXES]


@pytest.mark.gpu
@pytest.mark.parametrize("axis,sign", AXES, ids=AXIS_IDS)
def test_hydrostatic_known_answer_along_every_axis(axis, sign):
    """test_hydrostatic_known_answer_on_gpu rotated: a layer 8 cells deep against the wall gravity points into, on 48 x 32 x 40, on the oracle
    and on CUDA: p is g dt times the depth below the free surface, the projected velocity along gravity stays below 3e-3."""
    import blub_b200
    from blub_b200 import fluid as F
    from oracle import oracle as O
    from tests.util import DT

    dims = (48, 32, 40)
    n = dims[axis]
    lo, hi = [1, 1, 1], [d - 1 for d in dims]
    if sign < 0:
        hi[axis] = 9
    else:
        lo[axis] = n - 9
    g = [0.0, 0.0, 0.0]
    g[axis] = sign * 981.0
    gdt = float(np.float32(-981.0) * np.float32(DT))  # p = g dt depth with g the signed acceleration along "down" (negative), as on the y axis
    taps = [(F.TAP_P_VEL, F.TAP_UX, F.TAP_UY, F.TAP_UZ), (O.ARR_P_VEL, O.ARR_UX, O.ARR_UY, O.ARR_UZ)]
    for f, (tp, *tu) in zip((blub_b200.HybridFluid(*dims, 8 * 47 * 31 * 39), O.OracleFluid(*dims, 8 * 47 * 31 * 39)), taps):
        f.add_fluid_cube(lo, hi)
        f.set_gravity_grid(g)
        f.set_rebin_frequency(0)
        f.set_solver_config(0, error_tolerance=1e-6, max_num_iterations=600, error_check_frequency=4)
        f.step_stages(DT, 0, 3)
        err, it = f.last_solve(0)
        assert 0 < it < 600 and err < 1e-6 / DT
        get = f.download_grid if hasattr(f, "download_grid") else f.grid
        p = np.moveaxis(get(tp), 2 - axis, 0)  # [depth axis, ...]
        inner = p[:, 1:-1, 1:-1]
        for k in range(1, 9):
            cell = k if sign < 0 else n - 1 - k
            depth = 9 - k  # cells between this cell's centre and the surface, plus a half cell on each side
            assert np.allclose(inner[cell], gdt * depth, rtol=0, atol=3e-3), (k, inner[cell].min(), inner[cell].max(), gdt * depth)
        f.step_stages(DT, 4, 5)
        u = np.moveaxis(get(tu[axis]), 2 - axis, 0)[:, 1:-1, 1:-1]
        face = slice(1, 8) if sign < 0 else slice(n - 9, n - 2)
        assert np.abs(u[face]).max() < 3e-3


@pytest.mark.gpu
@pytest.mark.parametrize("axis,sign", AXES, ids=AXIS_IDS)
def test_stagewise_with_gravity_into_every_wall(axis, sign):
    """One stagewise step on 40 x 24 x 32 with the fluid pressed against the wall gravity points into (some particles closer to it than the
    clamp plane): the advection clamp and the correction clamp on that wall are each taken by at least 8 particles (classified by
    tests/advect_ref.py), and every stage agrees with the oracle."""
    import torch
    import blub_b200
    from oracle import oracle as O
    from tests import stagewise
    from tests.test_gpu_parity import WIDE

    lo, hi = [1, 1, 1], [d - 1 for d in WIDE]
    depth = 8
    if sign < 0:
        hi[axis] = 1 + depth
    else:
        lo[axis] = WIDE[axis] - 1 - depth
    orc, gpu = O.OracleFluid(*WIDE, 120000), blub_b200.HybridFluid(*WIDE, 120000)
    for f in (orc, gpu):
        f.add_fluid_cube(lo, hi)
        f.set_rebin_frequency(0)
    rng = np.random.default_rng(axis * 2 + (sign > 0))
    n = orc.num_particles
    rows = [rng.normal(0, 3.0, (n, 4)).astype(np.float32) for _ in range(3)]
    for r in rows:
        r[:, 3] *= 0.2
    rows[axis][:, 3] += sign * 20.0  # everything moves into the wall
    # every 8th particle of the layer next to the wall sits between the wall plane and the clamp plane 1.001 cells from it
    pos = orc.particles().copy()
    t = np.float32(1.0 if sign < 0 else WIDE[axis] - 1)
    layer = (np.abs(pos[:, axis] - t) < 1.0) & (np.arange(n) % 8 == 0)
    pos[layer, axis] = (t + (pos[layer, axis] - t) * np.float32(0.001)).astype(np.float32)
    g = [0.0, 0.0, 0.0]
    g[axis] = sign * 981.0
    for f in (orc, gpu):
        f.set_particles(pos, *rows)
        f.set_gravity_grid(g)
        f.set_solver_config(0, 0.1, 32, 4)
        f.set_solver_config(1, 0.1, 32, 4)
    vol = np.zeros((WIDE[2], WIDE[1], WIDE[0], 4), dtype=np.float16)
    keep = torch.from_numpy(vol).to("cuda").contiguous()
    gpu.set_solid_voxels(keep.data_ptr())
    report = stagewise.compare_one_step(orc, gpu, vox=vol.astype(np.float32), min_contact=(0, 0))
    x1, wall = report["advect_ref"]["x1"], report["advect_ref"]["wall"]
    plane = 1.001 if sign < 0 else np.float32(WIDE[axis]) - np.float32(1.001)
    into = wall & ((x1[:, axis] < plane) if sign < 0 else (x1[:, axis] > plane))
    c1, cw = report["correct_ref"]["x1"], report["correct_ref"]["wall"]
    corr = cw & ((c1[:, axis] < plane) if sign < 0 else (c1[:, axis] > plane))
    print(AXIS_IDS[AXES.index((axis, sign))], "advection clamps:", int(into.sum()), "correction clamps:", int(corr.sum()))
    assert into.sum() >= 8 and corr.sum() >= 8, (int(into.sum()), int(corr.sum()))
    del keep


if __name__ == "__main__":
    dst = sys.argv[1]
    res = {}
    for d, i in zip(SHAPE_LIST, IDS):
        for mode, digests in run_trajectories(d).items():
            res[f"{i}_{mode}"] = np.array(digests)
    np.savez(dst, **res)
