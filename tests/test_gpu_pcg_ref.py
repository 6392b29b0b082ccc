"""GPU: the pressure solve iteration by iteration against the float64 restatement of tests/pcg_ref.py, on every solver path and both fields.

Observation protocol (tests/pcg_ref.py): for K = 0, 1, ... the marker, the rhs b and a warm start p_0 (non-zero off FLUID too) are uploaded
(which also makes the solve prepare every tile) and solved with tolerance 0 and max_num_iterations = K.  Run K leaves p_{K+1}, r_{K+1},
the scalars of iteration K (blub_fluid_last_solve_scalars), max|r_{K+1}| and the iteration count; every check is one step from the state
run K - 1 left.  Paths: 1 (column solver), 6 (tile kernel, sparse bodies), 4 (tile kernel, dense bodies), 2 (TMA, when nx % 128 == 0),
0 (three kernels) with precond_mode 0 and 1.  The dot products are bounded with the chain lengths of the walkers: the passes per thread
come from solver_work() and a lower bound on the blocks of every persistent launch (one per SM).

Every system row asserts the feature it exists for and prints, per quantity, the median and the maximum of observed error / bound."""
import time

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from tests import pcg_ref as R
from tests.test_gpu_pcg_setup import tile_geometry
from tests.test_pcg_ref_kat import inputs, neumann_components, salt_and_pepper
from tests.util import DT, scene_path

pytestmark = pytest.mark.gpu

f32 = np.float32
P_TAP = (F.TAP_P_VEL, F.TAP_P_DEN)
PATHS = [(1, 0), (6, 0), (4, 0), (2, 0), (0, 0), (0, 1)]  # (solver path, precond_mode)
PATH_IDS = ["columns", "tiles", "dense", "tma", "three_kernels", "three_kernels_precond1"]


def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def passes(path, work):
    """Most tile and column passes of one thread in a phase: tiles round robin over the blocks, columns 256 per block and pass; at least one
    block per SM on every persistent path.  The three-kernel path runs one tile per block."""
    if path == 0:
        return 1
    nb = sms()
    return -(-work["tiles"] // nb) + -(-work["columns"] // (256 * nb))


def convention(path, mode):
    return "update" if (path, mode) == (0, 0) else "persistent"


def gpu_runs(m, b, p0, K, path, mode, which, freq=4):
    """Runs 0 .. K (tolerance 0) on a fresh fluid; returns (runs, solver_work of the last run)."""
    nz, ny, nx = m.shape
    f = blub_b200.HybridFluid(nx, ny, nz, 8)
    f.set_solver_path(path)
    f.set_quirks(precond_mode=mode)
    f.upload_grid(F.TAP_MARKER, m)
    runs = []
    for k in range(K + 1):
        f.set_solver_config(which, 0.0, k, freq)
        f.upload_grid(P_TAP[which], p0)
        f.upload_grid(F.TAP_RESIDUAL, b)
        f.solve_only(which, DT)
        e, it = f.last_solve(which)
        runs.append(R.Run(f.download_grid(P_TAP[which]), f.download_grid(F.TAP_RESIDUAL), f.last_solve_scalars(which), e, it))
    work = f.solver_work()
    f.close()
    return runs, work


def check_all_paths(label, m, b, p0, K, paths=PATHS, fields=(0, 1)):
    """Every path and field through check_runs; returns {(path, mode, which): runs}."""
    nx = m.shape[2]
    out = {}
    t0 = time.time()
    for path, mode in paths:
        if path == 2 and nx % 128:
            continue
        for which in fields:
            runs, work = gpu_runs(m, b, p0, K, path, mode, which)
            red = R.gpu_reduction(passes(path, work))
            stats = R.check_runs(f"{label} path {path} mode {mode} field {which}", m, b, p0, runs, red, convention(path, mode), mode)
            print(f"\n{label} path {path} mode {mode} field {which} ({red.name}): error / bound median / max: {stats.line()}")
            out[(path, mode, which)] = runs
    print(f"{label}: {time.time() - t0:.1f} s")
    return out


# ---- systems ------------------------------------------------------------------------------------------------------------------------
def units_per_tile(m):
    """[tiles_z, tiles_y, tiles_x]: (thread, plane) quads of the solver tile that hold a FLUID cell (the dense bit: 4 units >= 3 x 1024)."""
    (ez, ey, ex), (tz, ty, tx) = tile_geometry(m.shape)
    nz, ny, nx = m.shape
    fl = np.zeros((tz * ez, ty * ey, tx * ex), dtype=bool)
    fl[:nz, :ny, :nx] = m == R.FLUID
    q = fl.reshape(tz * ez, ty * ey, tx * ex // 4, 4).any(axis=3)
    return q.reshape(tz, ez, ty, ey, tx, ex // 4).sum(axis=(1, 3, 5))


def assert_every_diag(m):
    diag, fl = R.system(m)
    assert set(np.unique(diag[fl])) == set(range(7)), np.unique(diag[fl])
    p = np.pad(m, 1)
    nb_air = sum((np.roll(p, s, a)[1:-1, 1:-1, 1:-1] == R.AIR) for a in range(3) for s in (1, -1))
    assert (fl & (nb_air == 6)).any() and (fl & (diag == 0)).any()  # an isolated FLUID cell and one enclosed by six SOLID cells


def test_salt_and_pepper_every_diag():
    m = salt_and_pepper((16, 24, 64), 11)
    assert_every_diag(m)
    b, p0 = inputs(m, 11)
    diag, fl = R.system(m)
    assert (b[fl & (diag == 0)] != 0).all()  # z = r c_inv_diag2[0] is live in sigma and s
    assert (p0[m != R.FLUID] != 0).all()
    check_all_paths("salt and pepper 64x24x16", m, b, p0, 32)


def seam_system():
    """384 x 24 x 16: the interior tile layer (y 8..15, z 4..7) holds tiles with exactly 767 (x 0..127) and 768 (x 128..255) FLUID units
    next to each other -- a column body beside a tile body -- and a sparse tile (x 256..383) with an x gap of two quads; the tiles around
    them are sparse column tiles bordering the dense one."""
    nx, ny, nz = 384, 24, 16
    rng = np.random.default_rng(21)
    m = np.full((nz, ny, nx), R.AIR, dtype=np.int8)
    interior = np.zeros((nz, ny, nx), dtype=bool)
    interior[1:-1, 1:-1, 1:-1] = True

    def fill_units(zs, ys, x0, count=None, frac=None, gap=None):
        units = [(z, y, q) for z in zs for y in ys for q in range(x0 // 4, x0 // 4 + 32) if not (gap and gap[0] <= q < gap[1])]
        units = [u for u in units if interior[u[0], u[1], 4 * u[2]:4 * u[2] + 4].any()]
        if count is None:
            count = int(frac * len(units))
        pick = rng.choice(len(units), size=count, replace=False)
        for k in pick:
            z, y, q = units[k]
            cells = [x for x in range(4 * q, 4 * q + 4) if interior[z, y, x]]
            for x in rng.choice(cells, size=rng.integers(1, len(cells) + 1), replace=False):
                m[z, y, x] = R.FLUID

    fill_units(range(4, 8), range(8, 16), 0, count=767)
    fill_units(range(4, 8), range(8, 16), 128, count=768)
    fill_units(range(4, 8), range(8, 16), 256, frac=0.4, gap=(64 + 10, 64 + 12))
    for zs, ys in ((range(0, 4), range(8, 16)), (range(8, 12), range(8, 16)), (range(4, 8), range(0, 8)), (range(4, 8), range(16, 24))):
        for x0 in (0, 128, 256):
            fill_units(zs, ys, x0, frac=0.3)
    m[(m == R.AIR) & (rng.random(m.shape) < 0.05)] = R.SOLID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    return m


def test_dense_and_column_bodies_side_by_side():
    m = seam_system()
    u = units_per_tile(m)
    assert u[1, 1, 0] == 767 and u[1, 1, 1] == 768 and 0 < u[1, 1, 2] < 768, u[1, 1]
    assert 4 * u[1, 1, 1] >= 3 * 1024 > 4 * u[1, 1, 0]
    gap = (m[4:8, 8:16, 256 + 40:256 + 48] == R.FLUID)
    assert not gap.any()
    b, p0 = inputs(m, 21)
    check_all_paths("767 / 768 seam", m, b, p0, 32)
    _, work = gpu_runs(m, b, p0, 0, 1, 0, 0)
    assert work["tiles"] >= 1 and work["columns"] >= 1, work  # the column solver runs the tile body and the column body


@pytest.mark.parametrize("dims", [(32, 40, 16), (64, 24, 16), (160, 16, 8)], ids=["bx8", "bx16", "bx32"])
def test_tilemap_widths(dims):
    """Tiles 8, 16 and 32 quads wide; the last tile row only partly inside the grid (by = 32, 16; by = 8 divides every ny, so the bx = 32
    row has a last tile column half outside instead)."""
    nx, ny, nz = dims
    (_, ey, ex), _ = tile_geometry((nz, ny, nx))
    assert ex // 4 in (8, 16, 32) and (ny % ey != 0 or nx % ex != 0), (ex, ey)
    m = salt_and_pepper((nz, ny, nx), nx + ny, fluid=0.7, solid=0.08)
    b, p0 = inputs(m, nx)
    check_all_paths(f"tilemap {nx}x{ny}x{nz}", m, b, p0, 16)


def test_shapes_table():
    from tests.test_gpu_shapes import SHAPE_LIST
    for nx, ny, nz in SHAPE_LIST:
        rng = np.random.default_rng(nx * 10000 + ny * 100 + nz)
        m = np.full((nz, ny, nx), R.AIR, dtype=np.int8)
        m[rng.random((nz, ny, nx)) < 0.8] = R.FLUID
        m[rng.random((nz, ny, nx)) < 0.04] = R.SOLID
        m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
        b, p0 = inputs(m, nx)
        check_all_paths(f"shape {nx}x{ny}x{nz}", m, b, p0, 12)


def test_every_block_has_work():
    """512 x 128 x 64, all FLUID inside: 1024 active tiles, more than the blocks of any launch (at most 4 per SM), so a dropped block
    partial changes every sum."""
    nx, ny, nz = 512, 128, 64
    m = np.full((nz, ny, nx), R.FLUID, dtype=np.int8)
    rng = np.random.default_rng(31)
    m[rng.random(m.shape) < 0.02] = R.SOLID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b, p0 = inputs(m, 31)
    active = int((units_per_tile(m) > 0).sum())
    assert active >= 4 * sms(), (active, sms())
    check_all_paths("every block has work", m, b, p0, 4)


def test_more_passes_than_code_slots():
    """512 x 256 x 256 with FLUID in about 60 % of the quad columns (test_gpu_pcg_setup's column-heavy system): more than 8 column passes
    per thread, beyond the code words kept in shared memory.  The column count is checked against the column solver's launch (three blocks
    per SM, test_gpu_pcg_setup.passes); the bound uses the larger pass count of one block per SM.  This row is the exception to "every path
    and field": with 33.5 M cells it runs K <= 1, the column solver (path 1) on the velocity field and the tile kernel (path 6) on the
    density field -- the two walkers that run many passes; the others share their bodies (4 = 6 bit for bit in test_gpu_shapes.py)."""
    nx, ny, nz = 512, 256, 256
    rng = np.random.default_rng(9)
    on = rng.random((nz // 4, ny, nx // 4)) < 0.6
    m = np.where(on.repeat(4, axis=0).repeat(4, axis=2), R.FLUID, R.AIR).astype(np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = np.where(m == R.FLUID, rng.uniform(-1, 1, m.shape), 0).astype(f32)
    p0 = rng.uniform(-0.5, 0.5, m.shape).astype(f32)
    for path, which in ((1, 0), (6, 1)):
        runs, work = gpu_runs(m, b, p0, 1, path, 0, which)
        n = passes(path, work)
        if path == 1:
            from tests.test_gpu_pcg_setup import passes as column_solver_passes
            assert column_solver_passes(work) > 8, work
        stats = R.check_runs(f"passes path {path}", m, b, p0, runs, R.gpu_reduction(n), "persistent")
        print(f"\nmore passes than slots: path {path} field {which}, {n} passes, {work}: {stats.line()}")


def test_neumann_box_where_the_guard_matters():
    """A closed SOLID box filled with FLUID (singular: no AIR) and a rhs of 1e-6: s.As falls to a few PCG_EPSILON, so the guard's 1e-10
    is a visible part of alpha and beta."""
    nx, ny, nz = 32, 32, 32
    m = np.full((nz, ny, nx), R.FLUID, dtype=np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    assert neumann_components(m)[m == R.FLUID].all()
    rng = np.random.default_rng(41)
    b = np.where(m == R.FLUID, rng.uniform(-1e-6, 1e-6, m.shape), 0).astype(f32)
    p0 = np.where(m == R.FLUID, rng.uniform(-1e-6, 1e-6, m.shape), 1.0).astype(f32)
    out = check_all_paths("neumann box", m, b, p0, 32)
    runs = out[(1, 0, 0)]
    used = [abs(float(r.sigma) / float(r.alpha)) for r in runs if r.alpha != 0]
    print(f"smallest guarded s.As {min(used):.3e}")
    assert min(used) < 100 * float(R.PCG_EPSILON), min(used)


@pytest.mark.parametrize("scene", ["dam_small", "dam_halfhalf"])
def test_in_step_systems(scene):
    """The marker, rhs and warm start of both solves of step 3 of a scene (split by step_stages as audited_step does), K = 0 .. 32."""
    f = blub_b200.HybridFluid.from_scene(scene_path(scene))
    for _ in range(3):
        f.step(DT)
    systems = []
    for first, stage, which in ((0, 2, 0), (3, 10, 1)):
        f.step_stages(DT, first, stage)
        systems.append((which, f.download_grid(F.TAP_MARKER), f.download_grid(F.TAP_RESIDUAL), f.download_grid(P_TAP[which])))
        f.step_stages(DT, stage, stage + 1)
    f.close()
    for which, m, b, p0 in systems:
        assert (m == R.FLUID).sum() > 1000 and np.abs(p0[m == R.FLUID]).max() > 0
        check_all_paths(f"{scene} field {which}", m, b, p0, 32, fields=(which,))


def test_z_slab_ranks():
    """The sharded solve on 2 ranks (z slabs of 16 planes, ghost planes fed by the neighbours, sigma and s.As all-reduced through the
    mailboxes): the owned planes of every rank gathered into the global p and r, checked with a bound whose reduction includes each rank's
    float32 total and the fp64 sum over the ranks.  Every rank must report the same scalars, maximum and count.  Skipped on one GPU."""
    import torch

    from blub_b200 import slab
    from tests.test_gpu_multi import local_view, make_slabs

    world, nx, ny, nz_owned = 2, 64, 24, 16
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    halo = slab.HALO
    m = salt_and_pepper((world * nz_owned, ny, nx), 71)
    assert_every_diag(m)
    b, p0 = inputs(m, 71)
    for which in (0, 1):
        slabs = make_slabs(world, nx, ny, nz_owned)
        for k, s in enumerate(slabs):
            s.upload_grid(F.TAP_MARKER, local_view(m, k, nz_owned))
        runs = []
        for K in range(17):
            for k, s in enumerate(slabs):
                s.set_solver_config(which, 0.0, K, 4)
                s.upload_grid(P_TAP[which], local_view(p0, k, nz_owned))
                s.upload_grid(F.TAP_RESIDUAL, local_view(b, k, nz_owned))
            for s in slabs:  # all ranks enqueue, then all wait: the kernels talk to each other
                s.solve_only(which, DT)
            scal = [tuple(v.tobytes() for v in s.last_solve_scalars(which)) for s in slabs]
            last = [s.last_solve(which) for s in slabs]
            assert all(x == scal[0] for x in scal) and all(x == last[0] for x in last), (K, scal, last)
            p = np.concatenate([s.download_grid(P_TAP[which])[halo:halo + nz_owned] for s in slabs])
            r = np.concatenate([s.download_grid(F.TAP_RESIDUAL)[halo:halo + nz_owned] for s in slabs])
            runs.append(R.Run(p, r, slabs[0].last_solve_scalars(which), *last[0]))
        n = max(passes(1, s.solver_work()) for s in slabs)
        for s in slabs:
            s.close()
        red = R.slab_reduction(n, world)
        stats = R.check_runs(f"z slabs field {which}", m, b, p0, runs, red)
        print(f"\nz slabs field {which} ({red.name}): error / bound median / max: {stats.line()}")


# ---- the prefix property and the stop schedule ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path,mode", PATHS, ids=PATH_IDS)
def test_check_frequency_does_not_change_a_run(path, mode):
    """At tolerance 0 only the stop depends on the schedule: check_frequency 1, 3, 4 and K + 1 (the WITH_ERR variants of the three-kernel
    path) give the same bits."""
    m = salt_and_pepper((16, 16, 128), 51)
    b, p0 = inputs(m, 51)
    K = 9
    want = None
    for freq in (1, 3, 4, K + 1):
        runs, _ = gpu_runs(m, b, p0, K, path, mode, 1, freq=freq)
        got = [(r.p, r.r, (r.alpha, r.beta, r.sigma), r.max_error, r.iterations) for r in runs[K:]]
        if want is None:
            want = got
            continue
        (p, r, sc, e, it), (p2, r2, sc2, e2, it2) = want[0], got[0]
        assert np.array_equal(p, p2) and np.array_equal(r, r2) and sc == sc2 and e == e2 and it == it2, freq


@pytest.mark.parametrize("path,mode", [(1, 0), (6, 0), (0, 0)], ids=["columns", "tiles", "three_kernels"])
def test_stop_schedule_matches_the_prefix_run(path, mode):
    """A converging solve stops where the observed max|r_k| say it must, with the bits of the prefix run that stops there."""
    m = salt_and_pepper((16, 24, 64), 61, fluid=0.7, solid=0.05)
    b, p0 = inputs(m, 61, diag0=0)  # a consistent rhs: max|r| converges
    runs, _ = gpu_runs(m, b, p0, 16, path, mode, 0)
    maxima = [r.max_error for r in runs]
    for freq, lo, hi in ((4, 4, 8), (3, 9, 12)):
        tol = R.tolerance_between(maxima, lo, hi, DT)
        stop = R.predict_stop(maxima, R.tolerance32(tol, DT), freq, 32)
        assert stop == hi
        nz, ny, nx = m.shape
        f = blub_b200.HybridFluid(nx, ny, nz, 8)
        f.set_solver_path(path)
        f.set_quirks(precond_mode=mode)
        f.upload_grid(F.TAP_MARKER, m)
        f.set_solver_config(0, tol, 32, freq)
        f.upload_grid(F.TAP_P_VEL, p0)
        f.upload_grid(F.TAP_RESIDUAL, b)
        f.solve_only(0, DT)
        assert f.last_solve(0) == (float(maxima[hi]), hi)
        assert np.array_equal(f.download_grid(F.TAP_P_VEL), runs[hi].p) and np.array_equal(f.download_grid(F.TAP_RESIDUAL), runs[hi].r)
        f.close()
