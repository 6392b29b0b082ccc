"""CPU: the float64 restatement of the pressure solve (tests/pcg_ref.py) on closed forms, the oracle within its bounds iteration by
iteration, and planted defects that the per-iteration checks must name."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import pcg_ref as R
from tests.util import DT

f32 = np.float32


# ---- systems ------------------------------------------------------------------------------------------------------------------------
def salt_and_pepper(shape, seed, fluid=0.6, solid=0.15):
    """FLUID / AIR / SOLID at random with a SOLID border, plus a FLUID cell enclosed by six SOLID cells (diag 0) and an isolated FLUID cell
    (all neighbours AIR, diag 6)."""
    rng = np.random.default_rng(seed)
    nz, ny, nx = shape
    u = rng.random(shape)
    m = np.where(u < fluid, R.FLUID, np.where(u < fluid + solid, R.SOLID, R.AIR)).astype(np.int8)
    m[1:4, 1:4, 1:4] = R.SOLID
    m[2, 2, 2] = R.FLUID
    m[nz - 4:nz - 1, ny - 4:ny - 1, nx - 4:nx - 1] = R.AIR
    m[nz - 3, ny - 3, nx - 3] = R.FLUID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = R.SOLID, R.SOLID, R.SOLID, R.SOLID, R.SOLID, R.SOLID
    return m


def neumann_components(m):
    """FLUID cells whose connected FLUID region has no AIR neighbour: A is singular there."""
    from scipy import ndimage
    lab, n = ndimage.label(m == R.FLUID)
    air_next = ndimage.binary_dilation(m == R.AIR) & (lab > 0)
    open_ = np.zeros(n + 1, dtype=bool)
    open_[np.unique(lab[air_next])] = True
    open_[0] = True
    return ~open_[lab]


def inputs(m, seed, diag0=0.05):
    """rhs ~ U[-1, 1) on FLUID (0 elsewhere: the oracle leaves the residual alone off FLUID, and 0 on FLUID regions without an AIR
    neighbour, so that the system is consistent and CG converges) and a warm start that is non-zero everywhere.  A FLUID cell with
    diag 0 (enclosed by six SOLID cells) gets b = diag0 instead: its row of A is 0, so r stays b there and z = r c_inv_diag2[0] enters
    sigma and s in every iteration."""
    rng = np.random.default_rng(seed + 100)
    b = np.where((m == R.FLUID) & ~neumann_components(m), rng.uniform(-1, 1, m.shape), 0.0).astype(f32)
    diag, fl = R.system(m)
    b[fl & (diag == 0)] = diag0
    p0 = rng.uniform(-0.5, 0.5, m.shape).astype(f32)
    return b, p0


def oracle_runs(m, b, p0, K, mode=0, which=0, freq=4):
    """Runs 0 .. K of the oracle (tolerance 0): each one from the same p0 and b.  nx and ny are multiples of 8: the oracle's reductions
    place the cells in 8 x 8 groups and read only the first nx ny nz entries (as the reference does)."""
    nz, ny, nx = m.shape
    assert nx % 8 == 0 and ny % 8 == 0, m.shape
    f = O.OracleFluid(nx, ny, nz, 8)
    f.set_quirks(precond_mode=mode)
    f.grid(O.ARR_MARKER)[:] = m
    f.set_solver_config(which, 0.0, 0, 1)
    f.solve(which, DT)  # the first solve of a field zeroes its pressure: the warm starts below come after it
    parr = O.ARR_P_VEL if which == 0 else O.ARR_P_DEN
    runs = []
    for k in range(K + 1):
        f.grid(parr)[:] = p0
        f.grid(O.ARR_RESIDUAL)[:] = b
        f.set_solver_config(which, 0.0, k, freq)
        f.solve(which, DT)
        e, it = f.last_solve(which)
        runs.append(R.Run(f.grid(parr).copy(), f.grid(O.ARR_RESIDUAL).copy(), f.last_scalars(which), e, it))
    f.close()
    return runs


def check_oracle(label, m, b, p0, runs, mode):
    return R.check_runs(label, m, b, p0, runs, R.oracle_reduction(m.size), mode=mode, z_roundings=3 if mode == 0 else 1)


# ---- closed forms -------------------------------------------------------------------------------------------------------------------
def isolated_cells(shape=(8, 8, 16)):
    """FLUID cells two apart in every direction, all neighbours AIR: A = 6 I on them."""
    m = np.full(shape, R.AIR, dtype=np.int8)
    m[2:-2:2, 2:-2:2, 2:-2:2] = R.FLUID
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    return m


def test_isolated_cells_are_solved_in_one_iteration():
    m = isolated_cells()
    b, p0 = inputs(m, 1)
    diag, fl = R.system(m)
    assert (diag[fl] == 6).all() and fl.sum() >= 8
    p, r, alpha, beta, sigma = R.cg64(m, b, p0, 1)[0]
    den = float(np.sum(np.where(fl, b - 6.0 * p0, 0.0) ** 2)) / 216.0  # s.As; the guard's 1e-10 moves alpha by 1e-10 / den relative
    g = 2e-10 / den
    r0 = float(np.abs(np.where(fl, b - 6.0 * p0, 0.0)).max())
    assert np.abs(p[fl] - b[fl].astype(np.float64) / 6.0).max() <= g * r0 and np.abs(r).max() <= g * r0 and abs(alpha - 1.0 / (6.0 * float(R.C_INV_DIAG2[6]))) <= 6 * g and beta == 0
    runs = oracle_runs(m, b, p0, 2)
    check_oracle("isolated", m, b, p0, runs, 0)
    assert np.abs(runs[0].p[fl] - b[fl] / f32(6)).max() <= 4 * R.U * np.abs(b[fl]).max()
    assert np.abs(runs[0].r).max() <= 16 * R.U * np.abs(b).max()


def test_a_fluid_chain_gives_the_tridiagonal_cg_iterates():
    """A line of n FLUID cells along x in AIR: diag 6, -1 off the diagonal.  Textbook PCG on the dense matrix with M^-1 = c_inv_diag2[6] I
    (the float32 constant)."""
    n = 20
    m = np.full((5, 8, n + 4), R.AIR, dtype=np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    m[2, 2, 2:n + 2] = R.FLUID
    b, p0 = inputs(m, 2)
    ours = R.cg64(m, b, p0, 5)
    A = 6 * np.eye(n) - np.eye(n, k=1) - np.eye(n, k=-1)
    c = float(R.C_INV_DIAG2[6])
    x = p0[2, 2, 2:n + 2].astype(np.float64)
    r = b[2, 2, 2:n + 2].astype(np.float64) - A @ x
    z = r * c
    s, sigma = np.zeros(n), z @ r
    beta = 0.0
    for k in range(5):  # until sigma nears the guard's 1e-10, where the float64 roundings of the two forms stop being negligible
        s = z + beta * s
        alpha = sigma / (s @ A @ s + 1e-10)
        x, r = x + alpha * s, r - alpha * (A @ s)
        p_k, r_k, a_k, b_k, s_k = ours[k]
        assert np.allclose(p_k[2, 2, 2:n + 2], x, rtol=1e-10, atol=1e-12) and np.allclose(r_k[2, 2, 2:n + 2], r, rtol=1e-8, atol=1e-12), k
        assert abs(a_k - alpha) <= 1e-9 * abs(alpha) and abs(s_k - sigma) <= 1e-9 * abs(sigma), k
        z = r * c
        zr = z @ r
        beta, sigma = zr / (sigma + 1e-10), zr
    runs = oracle_runs(m, b, p0, 12)
    check_oracle("chain", m, b, p0, runs, 0)


def test_zero_rhs_gives_zero_scalars_through_the_guard():
    m = salt_and_pepper((8, 8, 16), 3)
    zero = np.zeros(m.shape, dtype=f32)
    runs = oracle_runs(m, zero, zero, 3)
    for k, run in enumerate(runs):
        assert run.alpha == 0 and run.beta == 0 and run.sigma == 0, k
        assert not run.p.any() and not run.r.any() and run.max_error == 0
    check_oracle("zero rhs", m, zero, zero, runs, 0)
    assert R.guarded_div(0, 0) == 0 and R.guarded_div(f32(1e-10), f32(0)) == 1
    assert R.guarded_div(f32(1), f32(-1e-10)) == f32(-0.5e10)


# ---- the oracle within the bounds -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("shape,seed", [((10, 16, 16), 4), ((12, 8, 24), 5)])
def test_oracle_iterates_stay_within_the_bounds(shape, seed, mode):
    m = salt_and_pepper(shape, seed)
    diag, fl = R.system(m)
    assert set(np.unique(diag[fl])) == set(range(7)), np.unique(diag[fl])
    b, p0 = inputs(m, seed)
    runs = oracle_runs(m, b, p0, 32, mode)
    stats = check_oracle(f"oracle {shape} mode {mode}", m, b, p0, runs, mode)
    print(f"\n{shape} mode {mode}: error / bound (median / max): {stats.line()}")
    assert (b[fl & (diag == 0)] != 0).all()  # z = r c_inv_diag2[0] is live in sigma and s
    if mode == 0:  # with a consistent rhs (0 at the diag-0 cell) the same system converges: the checks are not of a stalled iteration
        # (the literal passes of mode 1 are not symmetric)
        b0, _ = inputs(m, seed, diag0=0)
        runs0 = oracle_runs(m, b0, p0, 32, mode)
        check_oracle(f"oracle {shape} mode {mode}, consistent rhs", m, b0, p0, runs0, mode)
        assert runs0[-1].max_error < 1e-2 * runs0[0].max_error


def test_stop_schedule_predicted_from_the_maxima():
    m = salt_and_pepper((10, 16, 16), 6)
    b, p0 = inputs(m, 6, diag0=0)  # max|r| converges
    runs = oracle_runs(m, b, p0, 20)
    maxima = [r.max_error for r in runs]
    for freq, lo, hi in ((4, 4, 8), (3, 6, 9), (1, 5, 6)):
        tol = R.tolerance_between(maxima, lo, hi, DT)
        stop = R.predict_stop(maxima, R.tolerance32(tol, DT), freq, 20)
        assert stop == hi
        nz, ny, nx = m.shape
        f = O.OracleFluid(nx, ny, nz, 8)
        f.grid(O.ARR_MARKER)[:] = m
        f.solve(0, DT)
        f.grid(O.ARR_P_VEL)[:] = p0
        f.grid(O.ARR_RESIDUAL)[:] = b
        f.set_solver_config(0, tol, 20, freq)
        f.solve(0, DT)
        assert f.last_solve(0) == (float(maxima[hi]), hi)
        assert np.array_equal(f.grid(O.ARR_P_VEL), runs[hi].p) and np.array_equal(f.grid(O.ARR_RESIDUAL), runs[hi].r)
        f.close()


# ---- planted defects ----------------------------------------------------------------------------------------------------------------
def emulated_system():
    m = salt_and_pepper((10, 12, 16), 7)
    b, p0 = inputs(m, 7)
    return m, b, p0


def test_float32_emulation_stays_within_the_bounds():
    m, b, p0 = emulated_system()
    for mode in (0, 1):
        runs = R.emulate32(m, b, p0, 24, mode=mode)
        R.check_runs("emulation", m, b, p0, runs, R.Reduction(1, fp64=64), mode=mode)


def _cell_with_fluid_right(m):
    fl = m == R.FLUID
    both = fl.copy()
    both[:, :, :-1] &= fl[:, :, 1:]
    both[:, :, -1] = False
    return int(np.flatnonzero(both)[len(np.flatnonzero(both)) // 2])


@pytest.mark.parametrize("mutation,expect", [
    (("drop_neighbour", 3, None), r"iteration 3, r at cell \(x=\d+, y=\d+, z=\d+\)"),
    (("alpha_scale", 5, 2.0 ** -12), r"iteration 5, s\.As"),
    (("stale_beta", 4, None), r"iteration 5, beta_4"),
    (("c_inv_diag2", 0, 5), r"iteration 0, sigma"),
    (("drop_partial", 6, None), r"iteration 6, sigma"),
    (("max_lanes", 0, None), r"iteration 0, max\|r\|"),
], ids=["dropped_neighbour", "alpha_scaled", "stale_sigma_in_beta", "c_inv_diag2_5", "dropped_partial", "max_over_3_lanes"])
def test_planted_defects_are_named(mutation, expect):
    m, b, p0 = emulated_system()
    if mutation[0] == "drop_neighbour":
        mutation = (mutation[0], mutation[1], _cell_with_fluid_right(m))
    if mutation[0] == "max_lanes":  # leave out the lane that holds the largest |r_1|
        r1 = R.emulate32(m, b, p0, 1)[0].r
        mutation = (mutation[0], mutation[1], int(np.unravel_index(np.abs(r1).argmax(), r1.shape)[2] % 4))
    runs = R.emulate32(m, b, p0, 12, mutation=mutation)
    with pytest.raises(R.Mismatch, match=expect) as info:
        R.check_runs("mutant", m, b, p0, runs, R.Reduction(1, fp64=64))
    print(f"\n{mutation[0]}: {info.value}")


def as_update_convention(runs):
    """The persistent runs relabelled as the three-kernel path with precond_mode 0 leaves them: run K keeps (alpha_K, beta_K, sigma_{K+1})."""
    out = []
    for K in range(len(runs) - 1):
        r, nxt = runs[K], runs[K + 1]
        out.append(R.Run(r.p, r.r, (r.alpha, nxt.beta, nxt.sigma), r.max_error, r.iterations))
    return out


@pytest.mark.parametrize("mutation,expect", [(None, None), (("alpha_scale", 0, 2.0 ** -12), r"iteration 0, alpha"),
                                             (("drop_partial", 0, None), r"iteration (0, alpha|1, beta_0)")],
                         ids=["clean", "alpha0_scaled", "sigma0_without_a_partial"])
def test_update_convention_checks_alpha0_and_beta0_without_sigma0(mutation, expect):
    """sigma_0 is never observed in the "update" convention: alpha_0 and beta_0 are checked against the reference's sigma_0 instead."""
    m, b, p0 = emulated_system()
    runs = as_update_convention(R.emulate32(m, b, p0, 9, mutation=mutation))
    if mutation is None:
        R.check_runs("update", m, b, p0, runs, R.Reduction(1, fp64=64), convention="update")
        return
    with pytest.raises(R.Mismatch, match=expect):
        R.check_runs("update", m, b, p0, runs, R.Reduction(1, fp64=64), convention="update")
