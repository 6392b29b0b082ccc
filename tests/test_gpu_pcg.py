"""GPU parity of the pressure solve alone: every PCG path of the CUDA library (through the C ABI) against the CPU oracle on the same
markers and right-hand sides.  Collected first among the GPU tests (tests/conftest.py): cheap, local, and everything else builds on it."""
import hashlib

import numpy as np
import pytest

import blub_b200
from blub_b200 import fluid as F
from oracle import oracle as O
from tests import util
from tests.util import DT, grid_close

pytestmark = pytest.mark.gpu


def random_blob(n, seed, fill=0.7):
    rng = np.random.default_rng(seed)
    m = np.full((n, n, n), O.AIR, dtype=np.int8)
    m[rng.random((n, n, n)) < fill] = O.FLUID
    m[rng.random((n, n, n)) < 0.05] = O.SOLID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = rng.uniform(-1, 1, (n, n, n)).astype(np.float32)
    return m, b


@pytest.mark.parametrize("precond,persistent", [(0, True), (0, False), (1, False)])
@pytest.mark.parametrize("max_it,freq", [(32, 4), (7, 3), (2, 4)])
def test_pcg_matches_oracle_on_random_blob(precond, persistent, max_it, freq):
    n = 32
    m, b = random_blob(n, 1234)
    orc = O.OracleFluid(n, n, n, 8)
    gpu = blub_b200.HybridFluid(n, n, n, 8)
    gpu.set_solver_path(persistent)
    for f in (orc, gpu):
        f.set_quirks(precond_mode=precond)
        f.set_solver_config(0, error_tolerance=0.0, max_num_iterations=max_it, error_check_frequency=freq)
    orc.grid(O.ARR_MARKER)[:] = m
    orc.grid(O.ARR_RESIDUAL)[:] = b
    gpu.upload_grid(F.TAP_MARKER, m)
    gpu.upload_grid(F.TAP_RESIDUAL, b)
    orc.solve(0, DT)
    gpu.solve_only(0, DT)
    eo, io = orc.last_solve(0)
    eg, ig = gpu.last_solve(0)
    assert io == ig == max_it  # tolerance 0: never converges, statistics are written at i == max
    fl = m == O.FLUID
    p_o, p_g = orc.grid(O.ARR_P_VEL), gpu.download_grid(F.TAP_P_VEL)
    assert (p_g[~fl] == 0).all()
    grid_close(p_o, p_g, "pressure", rel=2e-3, abs_=1e-5)
    grid_close(orc.grid(O.ARR_RESIDUAL), gpu.download_grid(F.TAP_RESIDUAL), "residual", rel=5e-3, abs_=1e-5, mask=fl)
    assert abs(eo - eg) <= 5e-3 * max(eo, eg) + 1e-6


@pytest.mark.parametrize("persistent", [True, False])
def test_pcg_convergence_schedule_and_warm_start(persistent):
    n = 32
    m, b = random_blob(n, 7, fill=0.9)
    b[m != O.FLUID] = 0
    orc = O.OracleFluid(n, n, n, 8)
    gpu = blub_b200.HybridFluid(n, n, n, 8)
    gpu.set_solver_path(persistent)
    for f in (orc, gpu):
        f.set_solver_config(0, error_tolerance=1e-3, max_num_iterations=128, error_check_frequency=4)
    orc.grid(O.ARR_MARKER)[:] = m
    gpu.upload_grid(F.TAP_MARKER, m)
    for rep in range(2):  # the second solve warm-starts from the first solution
        orc.grid(O.ARR_RESIDUAL)[:] = b
        gpu.upload_grid(F.TAP_RESIDUAL, b)
        orc.solve(0, DT)
        gpu.solve_only(0, DT)
        eo, io = orc.last_solve(0)
        eg, ig = gpu.last_solve(0)
        assert io % 4 == 0 and ig % 4 == 0 and abs(io - ig) <= 4, (rep, io, ig)
        assert eg < 1e-3 / DT
        grid_close(orc.grid(O.ARR_P_VEL), gpu.download_grid(F.TAP_P_VEL), "pressure", rel=2e-3, abs_=2e-3)
    assert ig <= 8  # warm start: already (nearly) converged


def test_pcg_paths_agree_on_nonsquare_grid():
    """Persistent and three-kernel PCG on a grid whose x extent is not a multiple of 32 cells (partial tiles, 8-wide blocks)."""
    nx, ny, nz = 24, 40, 32
    rng = np.random.default_rng(11)
    m = np.full((nz, ny, nx), O.AIR, dtype=np.int8)
    m[rng.random((nz, ny, nx)) < 0.8] = O.FLUID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = rng.uniform(-1, 1, (nz, ny, nx)).astype(np.float32)
    orc = O.OracleFluid(nx, ny, nz, 8)
    orc.set_solver_config(0, 0.0, 20, 4)
    orc.grid(O.ARR_MARKER)[:] = m
    orc.grid(O.ARR_RESIDUAL)[:] = b
    orc.solve(0, DT)
    for persistent in (True, False):
        gpu = blub_b200.HybridFluid(nx, ny, nz, 8)
        gpu.set_solver_path(persistent)
        gpu.set_solver_config(0, 0.0, 20, 4)
        gpu.upload_grid(F.TAP_MARKER, m)
        gpu.upload_grid(F.TAP_RESIDUAL, b)
        gpu.solve_only(0, DT)
        assert gpu.last_solve(0)[1] == 20
        grid_close(orc.grid(O.ARR_P_VEL), gpu.download_grid(F.TAP_P_VEL), f"pressure persistent={persistent}", rel=2e-3, abs_=1e-5)


@pytest.mark.parametrize("max_it,freq,tol", [(32, 4, 0.0), (9, 2, 0.0), (128, 4, 1e-3)])
def test_tma_tiled_pcg_matches_oracle(max_it, freq, tol):
    """The TMA-staged persistent solver (tensor-map box loads, nx % 128 == 0) against the oracle and the register path."""
    nx, ny, nz = 128, 40, 24
    rng = np.random.default_rng(21)
    m = np.full((nz, ny, nx), O.AIR, dtype=np.int8)
    m[rng.random((nz, ny, nx)) < 0.8] = O.FLUID
    m[rng.random((nz, ny, nx)) < 0.04] = O.SOLID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = rng.uniform(-1, 1, (nz, ny, nx)).astype(np.float32)
    orc = O.OracleFluid(nx, ny, nz, 8)
    orc.set_solver_config(0, tol, max_it, freq)
    orc.grid(O.ARR_MARKER)[:] = m
    orc.grid(O.ARR_RESIDUAL)[:] = b
    orc.solve(0, DT)
    results = {}
    for path in ("tma", True):
        gpu = blub_b200.HybridFluid(nx, ny, nz, 8)
        gpu.set_solver_path(path)
        gpu.set_solver_config(0, tol, max_it, freq)
        gpu.upload_grid(F.TAP_MARKER, m)
        gpu.upload_grid(F.TAP_RESIDUAL, b)
        for rep in range(2):  # the second solve warm-starts (and re-arms the mbarrier phases)
            gpu.upload_grid(F.TAP_RESIDUAL, b)
            gpu.solve_only(0, DT)
            if rep == 0:
                e, it = gpu.last_solve(0)
                assert abs(it - orc.last_solve(0)[1]) <= (0 if tol == 0.0 else freq), (path, it, orc.last_solve(0))
                if tol == 0.0:
                    grid_close(orc.grid(O.ARR_P_VEL), gpu.download_grid(F.TAP_P_VEL), f"pressure path={path}", rel=3e-3, abs_=1e-4)
                else:  # converged: the stopping iterate depends on the last bits; check the defining property instead
                    pg = gpu.download_grid(F.TAP_P_VEL)
                    res = np.where(m == O.FLUID, b, 0.0) - util.apply_A(m, pg)
                    assert e < tol / DT and np.abs(res).max() <= 1.02 * tol / DT + 1e-4, (e, np.abs(res).max())
        results[path] = gpu.download_grid(F.TAP_P_VEL)
        assert gpu.last_solve(0)[0] >= 0.0
    if tol == 0.0:  # same arithmetic per cell; only the per-block partial sums are grouped differently (the paths launch different numbers of blocks)
        grid_close(results[True], results["tma"], "tma vs register path", rel=2e-3, abs_=1e-4)


@pytest.mark.parametrize("fill", [0.05, 0.5, 0.97])
def test_sparse_paths_agree_with_the_dense_kernel(fill):
    """The sparse tile bodies only drop work whose result is exactly 0 (zero invariant): the tile kernel (solver path 6) must equal its
    dense form (path 4) bit for bit, on ragged sparse and dense FLUID sets.  The column solver (default, path 1) applies the same bodies
    to a compacted column list: every cell sees the same operands, only the grouping of the per-block partial sums differs."""
    nx, ny, nz = 136, 24, 24  # ragged in x: 34 quads, a partial second tile
    rng = np.random.default_rng(int(fill * 100))
    m = np.full((nz, ny, nx), O.AIR, dtype=np.int8)
    m[rng.random((nz, ny, nx)) < fill] = O.FLUID
    m[rng.random((nz, ny, nx)) < 0.03] = O.SOLID
    m[:, :, 60:70] = O.AIR  # a gap of empty columns inside the rows
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = rng.uniform(-1, 1, (nz, ny, nx)).astype(np.float32)
    orc = O.OracleFluid(nx, ny, nz, 8)
    orc.set_solver_config(0, 0.0, 24, 4)
    orc.grid(O.ARR_MARKER)[:] = m
    orc.grid(O.ARR_RESIDUAL)[:] = b
    orc.solve(0, DT)
    out = {}
    for path in (True, "tiles", "dense"):
        gpu = blub_b200.HybridFluid(nx, ny, nz, 8)
        gpu.set_solver_path(path)
        gpu.set_solver_config(0, 0.0, 24, 4)
        gpu.upload_grid(F.TAP_MARKER, m)
        for rep in range(2):  # second solve: warm start from the first solution
            gpu.upload_grid(F.TAP_RESIDUAL, b)
            gpu.solve_only(0, DT)
            if rep == 0:
                grid_close(orc.grid(O.ARR_P_VEL), gpu.download_grid(F.TAP_P_VEL), f"pressure path={path}", rel=3e-3, abs_=1e-4)
        out[path] = (gpu.download_grid(F.TAP_P_VEL), gpu.last_solve(0))
    assert out["tiles"][1] == out["dense"][1]
    assert np.array_equal(out["tiles"][0], out["dense"][0])
    assert out[True][1][1] == out["dense"][1][1] == 24
    grid_close(out["dense"][0], out[True][0], "column solver vs tile kernel", rel=2e-3, abs_=1e-4)
    assert (out[True][0][m != O.FLUID] == 0).all()


def test_column_solver_is_deterministic_and_handles_mixed_fill():
    """A grid with a dense block (tile body), a sparse sheet and spray (column list): two solves of the same system are bit-identical, and the
    result equals the oracle's."""
    nx, ny, nz = 256, 32, 24
    rng = np.random.default_rng(17)
    m = np.full((nz, ny, nx), O.AIR, dtype=np.int8)
    m[2:20, 2:26, 4:140] = O.FLUID                       # dense body: whole tiles >= 3/4 full
    m[4:8, 10:12, 140:250] = O.FLUID                     # a thin sheet
    m[rng.random((nz, ny, nx)) < 0.01] = O.FLUID         # spray
    m[rng.random((nz, ny, nx)) < 0.01] = O.SOLID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = rng.uniform(-1, 1, (nz, ny, nx)).astype(np.float32)
    orc = O.OracleFluid(nx, ny, nz, 8)
    orc.set_solver_config(0, 0.0, 20, 4)
    orc.grid(O.ARR_MARKER)[:] = m
    orc.grid(O.ARR_RESIDUAL)[:] = b
    orc.solve(0, DT)
    res = []
    for _ in range(2):
        gpu = blub_b200.HybridFluid(nx, ny, nz, 8)
        gpu.set_solver_config(0, 0.0, 20, 4)
        gpu.upload_grid(F.TAP_MARKER, m)
        gpu.upload_grid(F.TAP_RESIDUAL, b)
        gpu.solve_only(0, DT)
        res.append((gpu.download_grid(F.TAP_P_VEL), gpu.download_grid(F.TAP_RESIDUAL), gpu.last_solve(0)))
    assert res[0][2] == res[1][2] and np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
    grid_close(orc.grid(O.ARR_P_VEL), res[0][0], "pressure", rel=2e-3, abs_=1e-4)
    assert (res[0][0][m != O.FLUID] == 0).all()


# ---- every path pinned bit for bit ---------------------------------------------------------------------------------------------------
def mixed_fill_system():
    """Dense block (tile body), thin sheet and spray (column list) on a grid with nx % 128 == 0, so that the TMA solver runs too."""
    nx, ny, nz = 256, 32, 24
    rng = np.random.default_rng(23)
    m = np.full((nz, ny, nx), O.AIR, dtype=np.int8)
    m[2:20, 2:26, 4:140] = O.FLUID
    m[4:8, 10:12, 140:250] = O.FLUID
    m[rng.random((nz, ny, nx)) < 0.01] = O.FLUID
    m[rng.random((nz, ny, nx)) < 0.01] = O.SOLID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    b = rng.uniform(-1, 1, (nz, ny, nx)).astype(np.float32)
    return m, b


def solve_digests(path, precond, tol, max_it, freq):
    """SHA-256 of p and r after two solves of the same system (the second warm-starts from the first), with both solves' statistics."""
    m, b = mixed_fill_system()
    nz, ny, nx = m.shape
    gpu = blub_b200.HybridFluid(nx, ny, nz, 8)
    gpu.set_solver_path(path)
    gpu.set_quirks(precond_mode=precond)
    gpu.set_solver_config(0, tol, max_it, freq)
    gpu.upload_grid(F.TAP_MARKER, m)
    h, stats = hashlib.sha256(), []
    for _ in range(2):
        gpu.upload_grid(F.TAP_RESIDUAL, b)
        gpu.solve_only(0, DT)
        e, it = gpu.last_solve(0)
        stats.append((np.float32(e).view(np.uint32).item(), it))
    h.update(np.ascontiguousarray(gpu.download_grid(F.TAP_P_VEL)).tobytes())
    h.update(np.ascontiguousarray(gpu.download_grid(F.TAP_RESIDUAL)).tobytes())
    return h.hexdigest()[:32], stats


# solver path, precond_mode
DIGEST_PATHS = [(1, 0), (6, 0), (4, 0), (2, 0), (0, 0), (0, 1)]
DIGEST_SCHEDULES = {"fixed": (0.0, 20, 4), "converging": (2e-3, 128, 4)}
# Recorded with the build of commit bcf7894 on an H100 80GB HBM3 (132 SMs, 700 W power limit).  The persistent solvers launch as many
# blocks as fit on the GPU, and that number sets the grouping of their partial sums, so the digests hold for this SM count only.
DIGESTS_132_SMS = {
    (1, 0, "converging"): ("6df751a3414bcc0a1ffdc4d4244dc5b7", [(1045782498, 16), (1044237610, 4)]),
    (1, 0, "fixed"): ("908a50a6a9f52fe7ce427c27b748f858", [(1034478723, 20), (1017826933, 20)]),
    (6, 0, "converging"): ("6eecdc111733ce03e99153441c2bdffe", [(1045782497, 16), (1044237429, 4)]),
    (6, 0, "fixed"): ("91be633f35a0d156be3cde17e0188edc", [(1034478717, 20), (1017834031, 20)]),
    (4, 0, "converging"): ("6eecdc111733ce03e99153441c2bdffe", [(1045782497, 16), (1044237429, 4)]),
    (4, 0, "fixed"): ("91be633f35a0d156be3cde17e0188edc", [(1034478717, 20), (1017834031, 20)]),
    (2, 0, "converging"): ("41d987bfe0f6ef3c05650cd07786bfe6", [(1045782494, 16), (1044237318, 4)]),
    (2, 0, "fixed"): ("0c144d58310804512da86055135fe2b4", [(1034478716, 20), (1017835322, 20)]),
    (0, 0, "converging"): ("9f7ff2941d366b2bb728d17328e82e70", [(1045782502, 16), (1044237736, 4)]),
    (0, 0, "fixed"): ("bea6e61e5d31c7bf0d6329d4ef52fe56", [(1034478716, 20), (1017802166, 20)]),
    (0, 1, "converging"): ("4f097f157a968d33b1b4f8a82943b8a1", [(1068887294, 128), (1068887308, 128)]),
    (0, 1, "fixed"): ("2cfc3874634fdb1984b1a2de06b6cd3d", [(1068886330, 20), (1068887304, 20)]),
}


@pytest.mark.parametrize("schedule", sorted(DIGEST_SCHEDULES))
@pytest.mark.parametrize("path,precond", DIGEST_PATHS)
def test_solver_paths_are_pinned_bit_for_bit(path, precond, schedule):
    """Every solver path's p, r and statistics against digests recorded from an earlier build: a change to the shared solve loop, the
    reductions or a path's walk of its work that moves one bit on any path fails here."""
    import torch

    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("digests recorded with 132 SMs")
    digest, stats = solve_digests(path, precond, *DIGEST_SCHEDULES[schedule])
    if schedule == "converging" and precond == 0:  # stops early (the literal two-pass preconditioner of precond_mode 1 runs to the end)
        assert 0 < stats[0][1] < 128 and stats[0][1] % 4 == 0, stats
    assert (digest, stats) == DIGESTS_132_SMS[(path, precond, schedule)]
