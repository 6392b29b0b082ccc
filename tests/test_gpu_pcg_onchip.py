"""GPU: the column solver's pressure kept on chip through a solve.

The single-GPU column solver keeps the p quads of each thread's first passes in shared memory from init to the end of the solve and writes
them back once (DESIGN §3.1).  That must give the same bits as p in memory, so this file checks:

* systems whose threads run more passes than the p slots against ``BLUB_PCG_P_SLOTS=0`` (p in memory throughout), bit for bit, with the
  slots ending inside the tile passes, at the tile / column seam and inside the column passes;
* three steps of the 256^3 dam break with and without p slots;
* a column system of short, broken rows, against digests of the build that kept p in memory;
* p and r exactly 0 off FLUID after every solve of a short trajectory: the write-back stays inside the planes the solve owns.

The hooks are read when a fluid is created."""
import hashlib

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from oracle import oracle as O
from tests.test_gpu_pcg_setup import audited_step, blocks_of_the_column_solver, from_scene, full_snapshot, make, passes, REL, ABS
from tests.test_gpu_state import assert_identical
from tests import util
from tests.util import DT

pytestmark = pytest.mark.gpu


def solve_twice(monkeypatch, m, b, env):
    """Two solves (the second warm-starts) with tolerance 0, 32 iterations, check frequency 4."""
    nz, ny, nx = m.shape
    f = make(monkeypatch, lambda: blub_b200.HybridFluid(nx, ny, nz, 8), **env)
    f.set_solver_config(0, 0.0, 32, 4)
    f.upload_grid(F.TAP_MARKER, m)
    for _ in range(2):
        f.upload_grid(F.TAP_RESIDUAL, b)
        f.solve_only(0, DT)
    out = {"p": f.download_grid(F.TAP_P_VEL), "r": f.download_grid(F.TAP_RESIDUAL), "last": f.last_solve(0), "work": f.solver_work()}
    f.close()
    return out


def compare_p_slots(monkeypatch, m, b, slot_counts, min_passes):
    want = solve_twice(monkeypatch, m, b, {"BLUB_PCG_P_SLOTS": "0"})
    assert want["last"][1] == 32
    reached = passes(want["work"])
    print(f"\n{m.shape[::-1]}: {want['work']['tiles']} tiles, {want['work']['columns']} columns, {reached} passes per phase "
          f"on {blocks_of_the_column_solver()} blocks")
    assert reached > min_passes, (want["work"], reached)  # otherwise the comparison cannot see a pass beyond the slots
    for slots in slot_counts:
        got = solve_twice(monkeypatch, m, b, {} if slots is None else {"BLUB_PCG_P_SLOTS": str(slots)})
        assert got["work"] == want["work"]
        assert got["last"] == want["last"], slots
        assert np.array_equal(got["p"], want["p"]) and np.array_equal(got["r"], want["r"]), f"p slots={slots}"
    fl = m == O.FLUID
    p, r = want["p"], want["r"]
    assert not p[~fl].any() and not r[~fl].any()
    err = np.abs(r[fl] - (b[fl].astype(np.float64) - util.apply_A(m, p)[fl])).max()
    assert err <= REL * float(np.abs(b[fl]).max()) + ABS


def boundary(m):
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    return m


# ---- passes beyond the p slots, bit for bit against p in memory ---------------------------------------------------------------------
def test_mixed_system_p_slot_boundaries_in_tiles_at_the_seam_and_in_columns(monkeypatch):
    """The mixed system of the code-slot tests (256 x 256 x 128: 1-2 dense tile passes per block, then about 3.5 column passes per warp): 1, 2
    and 3 p slots end inside the tile passes, at the seam and inside the column passes."""
    nx, ny, nz = 256, 256, 128
    rng = np.random.default_rng(5)
    m = np.full((nz, ny, nx), O.AIR, dtype=np.int8)
    m[1:40] = O.FLUID
    plane = rng.integers(0, 4, (nz // 4, ny, nx // 4))
    on = rng.random((nz // 4, ny, nx // 4)) < 0.95
    spray = np.zeros((nz // 4, 4, ny, nx // 4), dtype=bool)
    for k in range(4):
        spray[:, k] = on & (plane == k)
    spray = spray.reshape(nz, ny, nx // 4).repeat(4, axis=2)
    m[40:][spray[40:]] = O.FLUID
    m[rng.random((nz, ny, nx)) < 0.01] = O.SOLID
    b = rng.uniform(-1, 1, (nz, ny, nx)).astype(np.float32)
    compare_p_slots(monkeypatch, boundary(m), b, (1, 2, 3, None), 3)


def test_all_fluid_roofline_system_beyond_the_p_slots(monkeypatch):
    """256^3, all interior cells FLUID (4096 dense tiles, about 11 tile passes per thread)."""
    n = 256
    m = np.zeros((n, n, n), dtype=np.int8)
    m[1:-1, 1:-1, 1:-1] = O.FLUID
    b = np.random.default_rng(1234).uniform(-1.0, 1.0, (n, n, n)).astype(np.float32)
    b -= b[m == O.FLUID].mean(dtype=np.float64).astype(np.float32)
    b[m != O.FLUID] = 0
    compare_p_slots(monkeypatch, m, b, (None,), 8)


def test_column_heavy_system_beyond_the_p_slots(monkeypatch):
    """512 x 256 x 256 with FLUID in about 60 % of the quad columns: about 12 column passes."""
    nx, ny, nz = 512, 256, 256
    rng = np.random.default_rng(9)
    on = rng.random((nz // 4, ny, nx // 4)) < 0.6
    m = boundary(np.where(on.repeat(4, axis=0).repeat(4, axis=2), O.FLUID, O.AIR).astype(np.int8))
    b = rng.uniform(-1, 1, (nz, ny, nx)).astype(np.float32)
    compare_p_slots(monkeypatch, m, b, (None,), 8)


def test_dam_256_steps_match_without_p_slots(monkeypatch):
    out = []
    for env in ({}, {"BLUB_PCG_P_SLOTS": "0"}):
        f = make(monkeypatch, from_scene("dam_256"), **env)
        for _ in range(3):
            f.step(DT)
        out.append(full_snapshot(f))
        f.close()
    assert_identical(out[0], out[1])
    assert np.array_equal(out[0]["residual"], out[1]["residual"])


# ---- short, broken rows of columns, against the build that kept p in memory ---------------------------------------------------------
def broken_rows_system():
    """128 x 64 x 64 (tiles of 32 quads x 8 rows x 4 planes): quad columns switched on at random (about half, so no tile reaches 3/4 and
    everything runs as columns), rows cut every few quads, and every row's first and last quad on: x = 0 of one row follows the last quad of
    the row before it in the column list."""
    nx, ny, nz = 128, 64, 64
    rng = np.random.default_rng(17)
    on = rng.random((nz // 4, ny, nx // 4)) < 0.5
    on[:, :, 0] = on[:, :, -1] = True
    m = boundary(np.where(on.repeat(4, axis=0).repeat(4, axis=2), O.FLUID, O.AIR).astype(np.int8))
    m[rng.random(m.shape) < 0.02] = O.SOLID
    b = rng.uniform(-1, 1, m.shape).astype(np.float32)
    return m, b


def broken_rows_digests(monkeypatch, env):
    m, b = broken_rows_system()
    out = solve_twice(monkeypatch, m, b, env)
    assert out["work"]["columns"] > 0
    return hashlib.sha256(np.ascontiguousarray(out["p"]).tobytes()).hexdigest(), hashlib.sha256(np.ascontiguousarray(out["r"]).tobytes()).hexdigest()


# p and r after the two solves, recorded with the build before p slots (p in memory throughout) on an H100 80GB
# HBM3 (132 SMs).  The column solver runs as many blocks as fit on the GPU, and that sets the grouping of its partial sums.
BROKEN_ROWS_DIGESTS_132_SMS = ("0cda5b399113c5f749248b56c9e3da3a0331dde7823973a1ac0f8b792c32fdfc", "9d13033c9b01815dcd360fa30c58d44050193503f33b645930cf0c39a1960933")


@pytest.mark.parametrize("p_slots", [None, "0"], ids=["default", "no_p_slots"])
def test_broken_rows_match_the_build_without_p_slots(monkeypatch, p_slots):
    import torch

    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("digests recorded with 132 SMs")
    env = {} if p_slots is None else {"BLUB_PCG_P_SLOTS": p_slots}
    assert broken_rows_digests(monkeypatch, env) == BROKEN_ROWS_DIGESTS_132_SMS


# ---- the write-back stays inside the planes the solve owns ------------------------------------------------------------------------------
@pytest.mark.parametrize("p_slots", ["1", "4"])
def test_trajectory_keeps_p_and_r_zero_off_fluid(monkeypatch, p_slots):
    """dam_small split at the solves: after every solve p and r are exactly 0 off FLUID and r = b - A p in float64 on FLUID."""
    f = make(monkeypatch, from_scene("dam_small"), BLUB_PCG_P_SLOTS=p_slots)
    for _ in range(16):
        audited_step(f)
    f.close()
