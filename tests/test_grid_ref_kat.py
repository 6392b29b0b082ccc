"""Known-answer tests of the float64 per-face references (tests/grid_ref.py) that the GPU shape tests compare the P2G and density kernels
with: closed-form fields, an exact lattice, and the oracle's float32 sums within their rounding."""
import numpy as np
import pytest

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


def window_boxes(dims, centre, size=10):
    """One box in the interior (two cells from every wall), one against each of the six walls and one at the high corner, of `size` cells
    per side, centred on `centre` (x, y, z) where the walls allow."""
    dims = np.asarray(dims)
    lo = np.clip(np.asarray(centre, dtype=np.int64) - size // 2, 2, dims - size - 2)
    boxes = {"interior": lo}
    for ax, name in enumerate("xyz"):
        for side, at in (("low", 0), ("high", dims[ax] - size)):
            b = lo.copy()
            b[ax] = at
            boxes[f"{name} {side} wall"] = b
    boxes["high corner"] = dims - size
    return {k: (tuple(int(v) for v in b), tuple(int(v) for v in b + size)) for k, b in boxes.items()}


def surface_centre(m, pos):
    """The FLUID cell next to AIR closest to the particles' median (x, y, z): boxes around it hold fluid and free surface."""
    surf = (m == R.FLUID) & (R._neighbours(m) == R.AIR).any(axis=0)
    zyx = np.argwhere(surf)
    med = np.median(pos[:, :3], axis=0)[::-1]
    return zyx[np.argmin(np.abs(zyx - med).sum(axis=1))][::-1]


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def dam_small_state(steps=60):
    """The oracle's dam_small after `steps` whole steps: positions and APIC rows as the next P2G reads them."""
    orc = util.oracle_from_scene("dam_small")
    for _ in range(steps):
        orc.step(DT)
    return (orc.nx, orc.ny, orc.nz), orc.particles().copy(), [orc.particles(a).copy() for a in (O.ARR_ROWX, O.ARR_ROWY, O.ARR_ROWZ)]


def rough_state():
    """The shape tests' rough inputs on 56 x 40 x 24: the box fluid decayed out of its sorted order, a 1600-particle crowd, particles on cell
    and clamp planes, random APIC rows."""
    from tests.test_gpu_shapes import reference_particles

    dims = (56, 40, 24)
    pos, rows = reference_particles(dims, "decayed")
    return dims, pos, rows


WINDOW_INPUTS = {"dam_small": dam_small_state, "rough": rough_state}


def windowed_p2g(pos, rows, dims, box, gdt, halo=R.REACH, marker_halo=1):
    """P2G velocities, bounds (scatter and gather form) and marker of one box, from the box's own crop of the inputs."""
    frame = R.grow(box, marker_halo, dims)
    sums = R.p2g_sums(pos, rows, dims, box=frame, halo=halo)
    m = R.marker(pos, dims, box=frame)
    core = R.inner(frame, box)
    out = {"marker": m[core]}
    for c, v in enumerate(R.p2g_velocity(sums, m, gdt)):
        out[f"u{c}"] = v[core]
    for form in ("scatter", "gather"):
        for c, b in enumerate(R.p2g_bound(sums, m, gdt, form)):
            out[f"{form} bound {c}"] = b[core]
    return out


def windowed_rhs(pos, dims, box, dt, halo=R.REACH, marker_halo=1):
    frame = R.grow(box, marker_halo, dims)
    d = R.density_sums(pos, dims, box=frame, halo=halo)
    m = R.marker(pos, dims, box=frame)
    core = R.inner(frame, box)
    return {"rhs": R.density_rhs(d, m, dt)[core], "rhs bound": R.rhs_bound(d, m, dt, "scatter")[core]}


@pytest.mark.parametrize("inputs", list(WINDOW_INPUTS))
def test_windowed_reference_equals_the_whole_grid_bit_for_bit(inputs, monkeypatch):
    """A box evaluated from its own crop (the particles of the box grown by the reach, the marker grown by one cell, the grid's own walls)
    gives the P2G velocities, their bounds in both forms, the marker, the density rhs and its bound of the whole-grid evaluation bit for
    bit, on every entry of the box: in the interior, against each of the six walls and at the high corner.  Particles are taken 4096 at a
    time, so that the chunked sums are exercised too."""
    monkeypatch.setattr(R, "CHUNK", 4096)
    dims, pos, rows = WINDOW_INPUTS[inputs]()
    assert len(pos) > 3 * R.CHUNK
    gdt = gravity_dt((3.0, -981.0, -2.0))
    everything = R.whole(dims)
    want = windowed_p2g(pos, rows, dims, everything, gdt)
    want.update(windowed_rhs(pos, dims, everything, DT))
    whole_marker = R.marker(pos, dims)
    boxes = window_boxes(dims, surface_centre(whole_marker, pos))
    with_fluid = 0
    for name, box in boxes.items():
        got = windowed_p2g(pos, rows, dims, box, gdt)
        got.update(windowed_rhs(pos, dims, box, DT))
        with_fluid += int((got["marker"] == R.FLUID).any())
        if name == "interior":
            assert (got["marker"] == R.FLUID).any() and (got["marker"] == R.AIR).any()  # a free surface crosses it
        for k, v in got.items():
            assert same_bits(v, R.crop(want[k], box)), f"{inputs} {name}: {k}"
    assert with_fluid >= len(boxes) - 2, with_fluid  # the rough fluid is 12 cells high: its y high wall and high corner boxes are dry


@pytest.mark.parametrize("inputs", list(WINDOW_INPUTS))
def test_window_one_cell_short_of_the_reach_differs(inputs):
    """The halos are as wide as they must be: particles taken from the box grown by REACH - 1 cells lose contributions to the sums of
    the faces and cells at the box's edges, and a marker crop without its one-cell rim changes the faces P2G writes and the density rhs (the
    six neighbours) at the box's edges."""
    dims, pos, rows = WINDOW_INPUTS[inputs]()
    gdt = gravity_dt((3.0, -981.0, -2.0))
    box = window_boxes(dims, surface_centre(R.marker(pos, dims), pos))["interior"]
    for halo, want in ((R.REACH, True), (R.REACH - 1, False)):
        sums = R.p2g_sums(pos, rows, dims, box=box, halo=halo)
        dens = R.density_sums(pos, dims, box=box, halo=halo)
        whole_sums, whole_dens = R.p2g_sums(pos, rows, dims), R.density_sums(pos, dims)
        for c in range(3):
            assert same_bits(sums[c]["num"], R.crop(whole_sums[c]["num"], box)) == want, (halo, c)
        assert same_bits(dens["den"], R.crop(whole_dens["den"], box)) == want, halo
    good = windowed_p2g(pos, rows, dims, box, gdt)
    good.update(windowed_rhs(pos, dims, box, DT))
    rim = windowed_p2g(pos, rows, dims, box, gdt, marker_halo=0)
    rim.update(windowed_rhs(pos, dims, box, DT, marker_halo=0))
    assert same_bits(good["marker"], rim["marker"])
    assert not same_bits(good["u0"], rim["u0"]) and not same_bits(good["rhs"], rim["rhs"])


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
