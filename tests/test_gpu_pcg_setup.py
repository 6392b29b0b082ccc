"""GPU: the in-step pressure solve's set-up sized by the fluid and its on-chip code words.

The single-GPU column solver prepares only the tiles that hold FLUID now, were active in the previous solve or were active in this field's
previous solve (DESIGN §3.1); every other tile must already be all zeros, so the zero invariant (p, r, s, s1 exactly 0 on every non-FLUID
cell) carries over from one solve to the next.  A stale tile or a wrong code word gives a plausible but wrong pressure, so this file checks:

* along whole trajectories, after every solve: p and r are exactly 0 off the FLUID cells of the marker the solve used, and r equals
  b - A p recomputed in float64 on the FLUID cells;
* the set-up sized by the fluid against the set-up of every tile (``BLUB_PCG_SETUP=dense``) bit for bit, on the default paths, after
  path switches, after ``time_solve`` and after tap uploads (which must make the next solve of each field prepare every tile);
* systems whose threads run more passes than the code words kept in shared memory against ``BLUB_PCG_CODE_SLOTS=0`` (every pass reloads),
  bit for bit.

Both hooks are read when a fluid is created.  Cheapest cases first."""
import json

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from oracle import oracle as O
from tests import util
from tests.test_gpu_state import assert_identical, snapshot
from tests.util import DT

pytestmark = pytest.mark.gpu

P_TAP = (F.TAP_P_VEL, F.TAP_P_DEN)
# float64 check of r = b - A p on the FLUID cells after every solve: |d| <= REL * max|b| + ABS.  Fitted on the set-up of every tile (the
# same bits): the largest |d| / max|b| on these trajectories is 6.6e-5 (dam_halfhalf's velocity solves), 3x below REL; the systems of
# the code-slot tests stay below 1e-5.
REL, ABS = 2e-4, 1e-5


# ---- helpers ------------------------------------------------------------------------------------------------------------------------
def tile_geometry(shape):
    """make_tilemap (pcg.cu): a thread owns a quad of 4 x-cells, a block of bx x by threads (bx = 32 / 16 / 8 quads, by = 256 / bx rows)
    marches 4 z-planes.  Returns the tile extent in cells (z, y, x) and the tile counts."""
    nz, ny, nx = shape
    qx = nx // 4
    bx = 32 if qx > 16 else (16 if qx > 8 else 8)
    by = 256 // bx
    return (4, by, 4 * bx), (nz // 4, -(-ny // by), -(-qx // bx))


def tile_activity(marker):
    """[tiles_z, tiles_y, tiles_x]: the solver tile holds a FLUID cell."""
    (ez, ey, ex), (tz, ty, tx) = tile_geometry(marker.shape)
    nz, ny, nx = marker.shape
    fl = np.zeros((tz * ez, ty * ey, tx * ex), dtype=bool)
    fl[:, :ny, :nx // 4 * 4] = (marker == O.FLUID)[:tz * ez, :, :nx // 4 * 4]
    return fl.reshape(tz, ez, ty, ey, tx, ex).any(axis=(1, 3, 5))


def tile_cells(tiles, shape):
    """Cell mask of the tiles set in `tiles`."""
    (ez, ey, ex), (tz, ty, tx) = tile_geometry(shape)
    big = tiles.repeat(ez, 0).repeat(ey, 1).repeat(ex, 2)
    out = np.zeros(shape, dtype=bool)
    out[:tz * ez] = big[:, :shape[1], :shape[2]]
    return out


def dilate(tiles):
    """Tiles within one tile (26-neighbourhood) of a set tile."""
    p = np.pad(tiles, 1)
    out = np.zeros_like(tiles)
    for dz in range(3):
        for dy in range(3):
            for dx in range(3):
                out |= p[dz:dz + tiles.shape[0], dy:dy + tiles.shape[1], dx:dx + tiles.shape[2]]
    return out


class SkipModel:
    """Which tiles the set-up sized by the fluid leaves alone, restated from the markers of the solves: a solve is sparse when neither the
    scratch flag nor its field's flag is set (both set at creation and by every upload, cleared by the solve); it skips a tile with no
    FLUID cell that was inactive in the previous solve and in this field's previous solve (p_tiles)."""

    def __init__(self):
        self.flags = [True, True, True]
        self.prev = None
        self.p_tiles = [None, None]
        self.sparse_solves = self.skipped = self.left = self.held_by_p = 0
        self.always = None  # tiles skipped by every sparse solve

    def solve(self, which, marker):
        act = tile_activity(marker)
        none = np.zeros_like(act)
        prev = none if self.prev is None else self.prev
        pt = none if self.p_tiles[which] is None else self.p_tiles[which]
        if not self.flags[0] and not self.flags[1 + which]:
            skip = ~act & ~prev & ~pt
            self.sparse_solves += 1
            self.skipped += int(skip.sum())
            self.left += int((pt & ~act).sum())              # went inactive while this field's p_tiles still holds it
            self.held_by_p += int((pt & ~prev & ~act).sum())  # of those: only p_tiles keeps it in the set-up
            self.always = skip if self.always is None else self.always & skip
        self.flags[0] = self.flags[1 + which] = False
        self.prev = act
        self.p_tiles[which] = act

    def report(self):
        always = 0 if self.always is None else int(self.always.sum())
        return (f"{self.sparse_solves} sparse solves, {self.skipped} tile skips, {self.left} tiles left active->inactive while p_tiles held them "
                f"({self.held_by_p} held by p_tiles alone), {always} tiles skipped on every sparse solve")


def check_solve(f, which, b, m):
    """After a solve on marker m with right-hand side b: p and r exactly 0 off FLUID, r = b - A p (float64) on FLUID.  Returns |d| / max|b|."""
    p, r = f.download_grid(P_TAP[which]), f.download_grid(F.TAP_RESIDUAL)
    fl = m == O.FLUID
    assert not p[~fl].any() and not r[~fl].any(), f"field {which}: p or r non-zero off the FLUID cells"
    if not fl.any():
        return 0.0
    want = np.where(fl, b.astype(np.float64), 0.0) - util.apply_A(m, p)
    err = float(np.abs(r[fl] - want[fl]).max())
    bmax = float(np.abs(b[fl]).max())
    assert err <= REL * bmax + ABS, f"field {which}: |r - (b - Ap)| = {err:.3e}, max|b| = {bmax:.3e}"
    return err / max(bmax, 1e-30)


def audited_step(f, model=None):
    """One step split at the two solves (stages 1|2|3 and 9|10|11); downloads write nothing, so they change no decision of the solver."""
    margins = []
    for first, solve_stage, which in ((0, 2, 0), (3, 10, 1)):
        f.step_stages(DT, first, solve_stage)
        b, m = f.download_grid(F.TAP_RESIDUAL), f.download_grid(F.TAP_MARKER)
        f.step_stages(DT, solve_stage, solve_stage + 1)
        if model is not None:
            model.solve(which, m)
        margins.append(check_solve(f, which, b, m))
    f.step_stages(DT, 11, 14)
    return margins


def make(monkeypatch, factory, **env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        return factory()
    finally:
        for k in env:
            monkeypatch.delenv(k)


def twins(monkeypatch, factory):
    """(set-up sized by the fluid, set-up of every tile) on the same scene."""
    return make(monkeypatch, factory), make(monkeypatch, factory, BLUB_PCG_SETUP="dense")


def full_snapshot(f):
    s = snapshot(f)
    s["residual"] = f.download_grid(F.TAP_RESIDUAL)
    return s


def assert_twins_identical(a, b, what):
    sa, sb = full_snapshot(a), full_snapshot(b)
    try:
        assert_identical(sa, sb)
        assert np.array_equal(sa["residual"], sb["residual"]), "residual"
    except AssertionError as e:
        raise AssertionError(f"{what}: {e}") from None


def from_scene(name):
    return lambda: blub_b200.HybridFluid.from_scene(util.scene_path(name))


# ---- (a) zero invariant and float64 residual along trajectories ----------------------------------------------------------------------
def falling_blob():
    """A 32 x 16 x 32-cell block of fluid dropped from y = 60 in a 64 x 96 x 64 box (981 cells/s^2): the tiles it falls through go active,
    then inactive again, and it splashes on the floor after about 42 steps.  Tiles are 64 x 16 x 4 cells here."""
    f = blub_b200.HybridFluid(64, 96, 64, 8 * 32 * 16 * 32)
    f.add_fluid_cube([16.0, 60.0, 16.0], [48.0, 76.0, 48.0])
    f.set_gravity_grid([0.0, -981.0, 0.0])
    return f


@pytest.mark.parametrize("setup", ["fluid", "dense"])
@pytest.mark.parametrize("scene,steps", [("dam_small", 24), ("tap_small", 40), ("dam_halfhalf", 40)])
def test_trajectory_keeps_the_zero_invariant_and_the_residual(monkeypatch, scene, steps, setup):
    """After every solve of the trajectory: p, r exactly 0 off FLUID; r = b - A p in float64 on FLUID.  tap_small's source and drain make
    fluid appear and disappear; dam_halfhalf crosses the re-sorts at 8, 16, 24 and 32.  On an H100 the set-up sized by the fluid skipped
    45 tiles on dam_small and 3744 on dam_halfhalf (48 tiles on every solve); tap_small's tiles (whole 32 x 32 x 4 slabs) all hold fluid."""
    env = {"BLUB_PCG_SETUP": "dense"} if setup == "dense" else {}
    f = make(monkeypatch, from_scene(scene), **env)
    model = SkipModel() if setup == "fluid" else None
    worst = [0.0, 0.0]
    for k in range(steps):
        m = audited_step(f, model)
        worst = [max(w, x) for w, x in zip(worst, m)]
    print(f"\n{scene} ({setup} set-up, {steps} steps): max |r - (b - Ap)| / max|b| = {worst[0]:.2e} (velocity), {worst[1]:.2e} (density)"
          + (f"; {model.report()}" if model else ""))


def test_falling_blob_sparse_setup_equals_dense(monkeypatch):
    """Both set-ups step the falling blob split at the solves, with the checks of the trajectory test after every solve, and agree bit for
    bit after every step.  The markers must show the skip at work: tiles skipped on every solve, and tiles that went inactive while their
    field's p_tiles still held them -- among them tiles that only p_tiles keeps in the set-up (inactive in the previous solve).  On an H100:
    94 sparse solves, 7301 tile skips, 42 tiles skipped on every solve, 98 such transitions, 50 of them held by p_tiles alone."""
    a, b = twins(monkeypatch, falling_blob)
    model = SkipModel()
    for k in range(48):
        audited_step(a, model)
        audited_step(b)
        assert_twins_identical(a, b, f"step {k}")
    print(f"\nfalling blob: {model.report()}")
    assert model.skipped > 0 and model.always is not None and model.always.any(), model.report()
    assert model.left > 0 and model.held_by_p > 0, model.report()


# ---- (c) uploads make the next solve of each field prepare every tile --------------------------------------------------------------
@pytest.mark.parametrize("tap", [F.TAP_P_VEL, F.TAP_P_DEN, F.TAP_RESIDUAL], ids=["p_vel", "p_den", "residual"])
def test_an_upload_makes_both_fields_prepare_every_tile(tap):
    """Junk of order 1 uploaded into tiles that both fields' last solves left inactive (and far from the fluid) must be gone after the next
    solve of the field that owns the volume, and the fluid must go on bit for bit as a twin that uploaded zeros there."""
    a, b = from_scene("dam_halfhalf")(), from_scene("dam_halfhalf")()
    for f in (a, b):
        for _ in range(5):
            f.step(DT)
    markers = []
    for f in (a, b):
        f.step_stages(DT, 0, 2)
        m0 = f.download_grid(F.TAP_MARKER)
        f.step_stages(DT, 2, 14)
        markers.append((m0, f.download_grid(F.TAP_MARKER)))
    assert all(np.array_equal(x, y) for x, y in zip(*markers))
    m0, m1 = markers[0]
    quiet = ~dilate(tile_activity(m0) | tile_activity(m1))
    assert quiet.sum() >= 4, int(quiet.sum())
    cells = tile_cells(quiet, m0.shape)
    cur = a.download_grid(tap)
    assert np.array_equal(cur, b.download_grid(tap)) and not cur[cells].any()
    junk = cur.copy()
    junk[cells] = np.random.default_rng(3).uniform(-1.0, 1.0, int(cells.sum())).astype(np.float32)
    a.upload_grid(tap, junk)
    b.upload_grid(tap, cur)
    owner = 1 if tap == F.TAP_P_DEN else 0  # the residual is scratch of both solves: the velocity solve comes first
    for f in (a, b):
        f.step_stages(DT, 0, 3)
    if owner == 0:
        assert not a.download_grid(tap)[cells].any(), "junk survived the velocity solve"
    for f in (a, b):
        f.step_stages(DT, 3, 11)
    assert not a.download_grid(tap)[cells].any(), "junk survived the density solve"
    for f in (a, b):
        f.step_stages(DT, 11, 14)
    assert_twins_identical(a, b, "step after the upload")
    for k in range(4):
        for f in (a, b):
            f.step(DT)
        assert_twins_identical(a, b, f"step {k + 2} after the upload")
    assert not tile_activity(a.download_grid(F.TAP_MARKER))[quiet].any()  # the junk tiles stayed away from the fluid


# ---- (b) set-up sized by the fluid against the set-up of every tile, bit for bit -----------------------------------------------------
def run_twins(a, b, steps, before_step=lambda f, k: None, step=lambda f, k: f.step(DT)):
    for k in range(steps):
        for f in (a, b):
            before_step(f, k)
            step(f, k)
        assert_twins_identical(a, b, f"step {k}")


@pytest.mark.parametrize("graph", [True, False], ids=["graph", "eager"])
def test_dam_halfhalf_sparse_setup_equals_dense(monkeypatch, graph):
    """Its tile skips are counted by the trajectory test of dam_halfhalf (the same steps, split at the solves)."""
    a, b = twins(monkeypatch, from_scene("dam_halfhalf"))
    for f in (a, b):
        f.set_graph_replay(graph)
    run_twins(a, b, 42)


def test_tap_small_sparse_setup_equals_dense(monkeypatch):
    a, b = twins(monkeypatch, from_scene("tap_small"))
    assert a.has_flow and b.has_flow  # device-count mode
    run_twins(a, b, 40)
    assert a.flow_counters == b.flow_counters and a.flow_counters["emitted"] > 0 and a.flow_counters["drained"] > 0


def test_moving_solid_sparse_setup_equals_dense(monkeypatch):
    """double_dam with the box of tests/test_gpu_state.py moving through the fluid, voxelized before every step."""
    import torch

    sc = json.load(open(util.scene_path("double_dam")))
    d = sc["fluid"]["grid_dimension"]
    dims, scale, origin = (d["x"], d["y"], d["z"]), sc["fluid"]["grid_to_world_scale"], [sc["fluid"]["world_position"][c] for c in "xyz"]
    solid = {"world_position": [0.22, 0.20, 0.32], "scale": 1.0, "rotation_angles": [0.0, 0.0, 0.0], "shape": "box", "half_extent": [0.12, 0.20, 0.12],
             "translation": {"target": [0.84, 0.20, 0.32], "curve": "SmoothStep", "duration": 2.0}}
    a, b = twins(monkeypatch, from_scene("double_dam"))
    vols = {}
    for f in (a, b):  # one volume per fluid: the two streams run concurrently
        vols[id(f)] = torch.zeros((dims[2], dims[1], dims[0], 4), dtype=torch.float16, device="cuda")
    torch.cuda.synchronize()
    for f in (a, b):
        f.set_solid_voxels(vols[id(f)].data_ptr())

    def voxelize(f, k):
        F.solid_voxelize(vols[id(f)].data_ptr(), dims, solid, scale, origin, 0.5 + (k + 1) * DT, DT, cuda_stream=f.stream())

    run_twins(a, b, 24, before_step=voxelize)
    assert (vols[id(a)][..., 3] > 0).sum().item() > 20000


def test_path_switches_and_time_solve_keep_the_sparse_setup_exact(monkeypatch):
    """Column steps, then a few steps on every other path (each leaves the next column solve a full set-up), column steps between them;
    then time_solve of both fields between steps.  dam_halfhalf is 128 cells wide, so the TMA path runs."""
    a, b = twins(monkeypatch, from_scene("dam_halfhalf"))
    run_twins(a, b, 4)
    for path in ("tiles", "dense", False, "precond", "tma"):
        for f in (a, b):
            if path == "precond":
                f.set_quirks(precond_mode=1)
            else:
                f.set_solver_path(path)
        run_twins(a, b, 2)
        for f in (a, b):
            f.set_quirks(precond_mode=0)
            f.set_solver_path(True)
        run_twins(a, b, 3)
    for which in (0, 1):
        for f in (a, b):
            f.time_solve(which, DT, 2)
        assert_twins_identical(a, b, f"time_solve({which})")
        run_twins(a, b, 3)


# ---- (d) passes beyond the code slots, bit for bit against no slots --------------------------------------------------------------------
def blocks_of_the_column_solver():
    import torch
    return min(2048, 3 * torch.cuda.get_device_properties(0).multi_processor_count)


def passes(work):
    """Most tile and column passes of one thread in a phase: tiles go round robin over the blocks, columns 32 per warp and pass."""
    nb = blocks_of_the_column_solver()
    return -(-work["tiles"] // nb) + -(-work["columns"] // (256 * nb))


def solve_twice(monkeypatch, m, b, slots):
    """Two solves (the second warm-starts) with tolerance 0, 32 iterations, check frequency 4."""
    nz, ny, nx = m.shape
    env = {} if slots is None else {"BLUB_PCG_CODE_SLOTS": str(slots)}
    f = make(monkeypatch, lambda: blub_b200.HybridFluid(nx, ny, nz, 8), **env)
    f.set_solver_config(0, 0.0, 32, 4)
    f.upload_grid(F.TAP_MARKER, m)
    for _ in range(2):
        f.upload_grid(F.TAP_RESIDUAL, b)
        f.solve_only(0, DT)
    out = {"p": f.download_grid(F.TAP_P_VEL), "r": f.download_grid(F.TAP_RESIDUAL), "last": f.last_solve(0), "work": f.solver_work()}
    f.close()
    return out


def compare_slots(monkeypatch, m, b, slot_counts, min_passes):
    want = solve_twice(monkeypatch, m, b, 0)
    assert want["last"][1] == 32
    reached = passes(want["work"])
    print(f"\n{m.shape[::-1]}: {want['work']['tiles']} tiles, {want['work']['columns']} columns, {reached} passes per phase "
          f"on {blocks_of_the_column_solver()} blocks")
    assert reached > min_passes, (want["work"], reached)  # otherwise the comparison cannot see a pass beyond the slots
    for slots in slot_counts:
        got = solve_twice(monkeypatch, m, b, slots)
        assert got["work"] == want["work"]
        assert got["last"] == want["last"], slots
        assert np.array_equal(got["p"], want["p"]) and np.array_equal(got["r"], want["r"]), f"slots={slots}"
    fl = m == O.FLUID
    p, r = want["p"], want["r"]
    assert not p[~fl].any() and not r[~fl].any()
    err = np.abs(r[fl] - (b[fl].astype(np.float64) - util.apply_A(m, p)[fl])).max()
    bmax = float(np.abs(b[fl]).max())
    print(f"max |r - (b - Ap)| / max|b| = {err / bmax:.2e}")
    assert err <= REL * bmax + ABS, (err, bmax)
    return reached


def test_mixed_system_slot_boundaries_in_tiles_at_the_seam_and_in_columns(monkeypatch):
    """256 x 256 x 128: dense tiles (1-2 tile passes per block) and one FLUID quad plane in most quad columns of the other tiles (about 3.5
    column passes per warp), so 1, 2 and 3 slots end inside the tile passes, at the tile / column seam and inside the column passes."""
    nx, ny, nz = 256, 256, 128
    rng = np.random.default_rng(5)
    m = np.full((nz, ny, nx), O.AIR, dtype=np.int8)
    m[1:40] = O.FLUID  # ten layers of dense tiles
    plane = rng.integers(0, 4, (nz // 4, ny, nx // 4))
    on = rng.random((nz // 4, ny, nx // 4)) < 0.95
    spray = np.zeros((nz // 4, 4, ny, nx // 4), dtype=bool)
    for k in range(4):
        spray[:, k] = on & (plane == k)
    spray = spray.reshape(nz, ny, nx // 4).repeat(4, axis=2)
    m[40:][spray[40:]] = O.FLUID
    m[rng.random((nz, ny, nx)) < 0.01] = O.SOLID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = rng.uniform(-1, 1, (nz, ny, nx)).astype(np.float32)
    compare_slots(monkeypatch, m, b, (1, 2, 3, None), 3)


def test_all_fluid_roofline_system_beyond_the_slots(monkeypatch):
    """The roofline microbench's system: 256^3, all interior cells FLUID, rhs ~ U[-1, 1) seed 1234 with the mean removed (4096 dense tiles)."""
    n = 256
    m = np.zeros((n, n, n), dtype=np.int8)
    m[1:-1, 1:-1, 1:-1] = O.FLUID
    b = np.random.default_rng(1234).uniform(-1.0, 1.0, (n, n, n)).astype(np.float32)
    b -= b[m == O.FLUID].mean(dtype=np.float64).astype(np.float32)
    b[m != O.FLUID] = 0
    compare_slots(monkeypatch, m, b, (None,), 8)


def test_column_heavy_system_beyond_the_slots(monkeypatch):
    """512 x 256 x 256 with FLUID in about 60 % of the quad columns (whole 4 x 4-cell columns, so no tile reaches 3/4): about 12 column passes."""
    nx, ny, nz = 512, 256, 256
    rng = np.random.default_rng(9)
    on = rng.random((nz // 4, ny, nx // 4)) < 0.6
    m = np.where(on.repeat(4, axis=0).repeat(4, axis=2), O.FLUID, O.AIR).astype(np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = rng.uniform(-1, 1, (nz, ny, nx)).astype(np.float32)
    compare_slots(monkeypatch, m, b, (None,), 8)


def test_dam_256_steps_match_without_slots(monkeypatch):
    """Three steps of the 256^3 dam break (about 2 passes per phase) with the default slots and with none."""
    out = []
    for env in ({}, {"BLUB_PCG_CODE_SLOTS": "0"}):
        f = make(monkeypatch, from_scene("dam_256"), **env)
        for _ in range(3):
            f.step(DT)
        out.append(full_snapshot(f))
        f.close()
    assert_identical(out[0], out[1])
    assert np.array_equal(out[0]["residual"], out[1]["residual"])


# ---- (e) z-slab ranks use the slots too ---------------------------------------------------------------------------------------------
def test_sharded_solve_matches_without_slots(monkeypatch):
    import torch

    from tests.test_gpu_multi import local_view, make_slabs

    world, nx, ny, nz_owned = 2, 64, 48, 16
    if torch.cuda.device_count() < world:
        pytest.skip("needs 2 GPUs")
    NZ = world * nz_owned
    rng = np.random.default_rng(world)
    m = np.full((NZ, ny, nx), O.AIR, dtype=np.int8)
    m[rng.random((NZ, ny, nx)) < 0.75] = O.FLUID
    m[rng.random((NZ, ny, nx)) < 0.03] = O.SOLID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = rng.uniform(-1, 1, (NZ, ny, nx)).astype(np.float32)
    results = []
    for env in ({}, {"BLUB_PCG_CODE_SLOTS": "0"}):
        slabs = make(monkeypatch, lambda: make_slabs(world, nx, ny, nz_owned), **env)
        for k, s in enumerate(slabs):
            s.set_solver_config(0, 0.0, 32, 4)
            s.upload_grid(F.TAP_MARKER, local_view(m, k, nz_owned))
        for _ in range(2):
            for k, s in enumerate(slabs):
                s.upload_grid(F.TAP_RESIDUAL, local_view(b, k, nz_owned))
            for s in slabs:
                s.solve_only(0, DT)
        results.append([(s.download_grid(F.TAP_P_VEL), s.download_grid(F.TAP_RESIDUAL), s.last_solve(0)) for s in slabs])
        for s in slabs:
            s.close()
    for k, (x, y) in enumerate(zip(*results)):
        assert x[2] == y[2] and np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]), f"rank {k}"
