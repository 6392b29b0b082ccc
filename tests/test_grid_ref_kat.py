"""Known-answer tests of the float64 per-face references (tests/grid_ref.py) that the GPU shape tests compare the P2G and density kernels
with: closed-form fields, an exact lattice, and the oracle's float32 sums within their rounding."""
import numpy as np

from oracle import oracle as O
from tests import grid_ref as R
from tests import util
from tests.test_transfer_kat import B_VEC, S_SYM, affine_rows, face_centres, linear_field
from tests.util import DT

N = 32


def test_reference_p2g_reproduces_a_symmetric_affine_field():
    """test_transfer_kat.py's statement: with rows set from v(x) = S x + b (S symmetric) every contribution is w * v_c(q), so the normalised
    sum is v_c(q), whatever the positions."""
    rng = np.random.default_rng(3)
    pos = np.c_[rng.uniform(10.0, 22.0, (20000, 3)), np.zeros(20000)].astype(np.float32)
    dims = (N, N, N)
    sums = R.p2g_sums(pos, affine_rows(pos), dims)
    m = R.marker(pos, dims)
    u = R.p2g_velocity(sums, m, (0.0, 0.0, 0.0))
    checked = 0
    for c in range(3):
        writes, solid = R.written_faces(m, c)
        sel = writes & ~solid
        want = linear_field(S_SYM, face_centres(c))[..., c]
        # the rows hold v_c(x_p) rounded to float32: a weighted mean of values within 2^-24 |v| of the field
        assert np.abs(u[c][sel] - want[sel]).max() <= R.U * np.abs(want).max()
        assert (u[c][solid] == 0).all()
        checked += int(sel.sum())
    assert checked > 3 * 12 ** 3 and np.abs(B_VEC).max() > 0


def lattice(n):
    """8 particles per cell at the cell's quarter points, in every interior cell of an n^3 grid."""
    q = np.arange(1, n - 1, dtype=np.float64)
    q = np.sort(np.r_[q + 0.25, q + 0.75])
    z, y, x = np.meshgrid(q, q, q, indexing="ij")
    return np.c_[x.ravel(), y.ravel(), z.ravel(), np.zeros(x.size)].astype(np.float32)


def test_reference_density_of_a_lattice_is_exact():
    """8 particles per cell at the quarter points: the hat weights of a cell centre add up to 2 per axis, so every cell two or more cells
    away from the walls has density 8 and rhs 0 exactly; the oracle's rhs agrees with the reference everywhere within its rounding."""
    n = 16
    pos = lattice(n)
    dims = (n, n, n)
    m = R.marker(pos, dims)
    d = R.density_sums(pos, dims)
    rhs = R.density_rhs(d, m, DT)
    bulk = np.zeros(m.shape, dtype=bool)
    bulk[2:-2, 2:-2, 2:-2] = True
    assert (d["den"][bulk] == 8.0).all() and (rhs[bulk] == 0.0).all()
    assert (m[1:-1, 1:-1, 1:-1] == R.FLUID).all()
    orc = O.OracleFluid(n, n, n, pos.shape[0])
    orc.set_particles(pos)
    assert np.array_equal(oracle_density(orc), pos[:, :3])
    assert np.array_equal(orc.grid(O.ARR_MARKER), m)
    R.check(orc.grid(O.ARR_RESIDUAL), rhs, R.rhs_bound(d, m, DT, "sequential"), "oracle rhs of the lattice")
    assert (orc.grid(O.ARR_RESIDUAL)[bulk] == 0.0).all()


def oracle_density(orc):
    """The oracle's density rhs: its advection builds the density pass's lists and marker; with a zero velocity grid it moves no particle
    away from the walls.  Returns the positions the density pass saw."""
    for a in (O.ARR_UX, O.ARR_UY, O.ARR_UZ):
        orc.grid(a)[:] = 0.0
    orc.step_stages(DT, 6, 10)  # clear, advect, boundary marker, density
    return orc.particles()[:, :3].copy()


def dam_small_with_rows(seed=5):
    orc = util.oracle_from_scene("dam_small")
    rng = np.random.default_rng(seed)
    rows = [rng.normal(0, 3.0, (orc.num_particles, 4)).astype(np.float32) for _ in range(3)]
    pos = orc.particles().copy()
    orc.set_particles(pos, *rows)
    orc.set_rebin_frequency(0)
    return orc, pos, rows


def gravity_dt(g, dt=DT):
    return [float(np.float32(v) * np.float32(dt)) for v in g]


def test_reference_agrees_with_the_oracle_on_dam_small():
    """The oracle sums each face's list in float32: its P2G velocities and density rhs are within the sequential-form bound of the float64
    reference on every face / cell it writes, and that bound is below grid_close's tolerance."""
    orc, pos, rows = dam_small_with_rows()
    g = [0.0, -981.0, 0.0]
    orc.set_gravity_grid(g)
    dims = (orc.nx, orc.ny, orc.nz)
    orc.step_stages(DT, 0, 1)
    m = R.marker(pos, dims)
    assert np.array_equal(orc.grid(O.ARR_MARKER), m)
    sums = R.p2g_sums(pos, rows, dims)
    want = R.p2g_velocity(sums, m, gravity_dt(g))
    bounds = R.p2g_bound(sums, m, gravity_dt(g), "sequential")
    for c, a in enumerate((O.ARR_UX, O.ARR_UY, O.ARR_UZ)):
        got = orc.grid(a)
        ratio, b = R.check(got, want[c], bounds[c], f"oracle P2G u[{c}]")
        sel = ~np.isnan(want[c])
        tol = 1e-4 * max(np.abs(got[sel]).max(), np.nanmax(np.abs(want[c]))) + 1e-5  # what grid_close allows on the whole field
        # the bound scales with the magnitude of each face's own terms (random rows: about max|u|) and the length of its float32 chain
        assert np.median(b) <= 0.1 * tol, (np.median(b), tol)
    pos = oracle_density(orc)
    m = orc.grid(O.ARR_MARKER)
    d = R.density_sums(pos, dims)
    R.check(orc.grid(O.ARR_RESIDUAL), R.density_rhs(d, m, DT), R.rhs_bound(d, m, DT, "sequential"), "oracle density rhs")


def test_reference_bound_catches_one_lost_particle():
    """The per-face bound sees one particle missing from the sums of slow faces while a fast jet elsewhere sets grid_close's scale: the
    field-wide tolerance lets the same error pass."""
    orc = util.oracle_from_scene("dam_small")
    pos = orc.particles().copy()
    n = len(pos)
    rng = np.random.default_rng(6)
    rows = [np.c_[rng.normal(0, 0.02, (n, 3)), rng.normal(0, 0.05, n)].astype(np.float32) for _ in range(3)]
    rows[0][pos[:, 1] < 3.0, 3] = 300.0  # a fast sheet along the floor
    orc.set_particles(pos, *rows)
    orc.set_rebin_frequency(0)
    g = (0.0, -981.0, 0.0)
    orc.set_gravity_grid(g)
    dims = (orc.nx, orc.ny, orc.nz)
    orc.step_stages(DT, 0, 1)
    m = R.marker(pos, dims)
    gdt = gravity_dt(g)
    k = int(np.argmin(np.abs(pos[:, :3] - np.array([8.3, 10.3, 16.3])).sum(axis=1)))  # in the slow bulk of the dam
    keep = np.ones(n, dtype=bool)
    keep[k] = False
    sums = R.p2g_sums(pos[keep], [r[keep] for r in rows], dims)
    want = R.p2g_velocity(sums, m, gdt)
    bounds = R.p2g_bound(sums, m, gdt, "sequential")
    got = orc.grid(O.ARR_UX)
    try:
        R.check(got, want[0], bounds[0], "P2G u[0] without one particle")
    except AssertionError:
        pass
    else:
        raise AssertionError("a lost particle went unnoticed")
    sel = ~np.isnan(want[0])
    util.grid_close(want[0][sel], got[sel], "grid_close without one particle")
