"""Known-answer tests of the grid stages (closed forms any correct implementation of the cited shaders must give), evaluated on the
oracle (CPU) and, with the same assertions, on the CUDA path (GPU).

  divergence_compute.comp:28-86          rhs of a linear velocity field u = A x + b inside the fluid  = trace(A)
  divergence_remove.comp:19-49           u_c <- u_c - (p(g) - p(g + e_c)): a linear pressure p = k . x shifts every fluid-fluid face by +k_c
  density_projection_position_change.comp:18-51   D_c = (p(g + e_c) - p(g)) * dt = k_c * dt on fluid-fluid faces, 0 next to SOLID
  extrapolate_velocity.comp:26-90        a constant field on the valid faces is copied to every face of the first ring around them
  density_projection_gather_error.comp:41-199     a regular 2x2x2 lattice (8 particles per cell) has density 8 at every interior cell
                                                   centre: rhs = 0; a missing layer of cells next to it raises the rhs accordingly
"""
import numpy as np
import pytest

from oracle import oracle as O
from tests.util import DT, fluid_adjacent_faces, near_fluid

N = 32
A = np.array([[0.5, -1.0, 2.0], [1.5, 0.25, -0.5], [-2.0, 1.0, -0.75]])
B = np.array([4.0, -6.0, 2.5])
K = np.array([3.0, -2.0, 0.5])  # pressure gradient per cell


def block_marker(lo=8, hi=24):
    m = np.full((N, N, N), O.AIR, dtype=np.int8)
    m[0], m[-1], m[:, 0], m[:, -1], m[:, :, 0], m[:, :, -1] = 0, 0, 0, 0, 0, 0
    m[lo:hi, lo:hi, lo:hi] = O.FLUID
    return m


def face_field(c):
    z, y, x = np.meshgrid(np.arange(N), np.arange(N), np.arange(N), indexing="ij")
    q = np.stack([x, y, z], axis=-1) + 0.5
    q[..., c] += 0.5
    return (q @ A.T + B)[..., c].astype(np.float32)


def cell_pressure():
    z, y, x = np.meshgrid(np.arange(N), np.arange(N), np.arange(N), indexing="ij")
    return ((x + 0.5) * K[0] + (y + 0.5) * K[1] + (z + 0.5) * K[2]).astype(np.float32)


def fluid_fluid_faces(m, c):
    fl = m == O.FLUID
    nb = np.roll(fl, -1, axis=2 - c)
    return fl & nb


def lattice_particles(lo, hi):
    """8 particles per cell at (0.25, 0.75)^3 in the cells [lo, hi)^3."""
    c = np.arange(lo, hi)
    off = np.array([0.25, 0.75])
    ax = (c[:, None] + off[None, :]).ravel()
    z, y, x = np.meshgrid(ax, ax, ax, indexing="ij")
    return np.stack([x.ravel(), y.ravel(), z.ravel(), np.zeros(x.size)], axis=1).astype(np.float32)


class OracleBackend:
    def __init__(self, nparticles=8, dims=(N, N, N)):
        self.f = O.OracleFluid(*dims, nparticles)
        self.f.set_gravity_grid([0.0, 0.0, 0.0])

    def put(self, marker=None, u=None, p=None, which=0, vox=None):
        """vox: the solid volume [nz, ny, nx, 4]; both backends read its fp16 values."""
        if vox is not None:
            self.f.set_voxels(np.asarray(vox, dtype=np.float16).astype(np.float32))
        if marker is not None:
            self.f.grid(O.ARR_MARKER)[:] = marker
        if u is not None:
            for c, a in enumerate((O.ARR_UX, O.ARR_UY, O.ARR_UZ)):
                self.f.grid(a)[:] = u[c]
        if p is not None:
            self.f.grid(O.ARR_P_VEL if which == 0 else O.ARR_P_DEN)[:] = p

    def particles(self, pos, rows=(None, None, None)):
        self.f.set_particles(pos, *rows)

    def run(self, a, b, dt=DT):
        self.f.step_stages(dt, a, b)

    def u(self):
        return [self.f.grid(a).copy() for a in (O.ARR_UX, O.ARR_UY, O.ARR_UZ)]

    def positions(self, row=None):
        return self.f.particles(O.ARR_POS if row is None else (O.ARR_ROWX, O.ARR_ROWY, O.ARR_ROWZ)[row]).copy()

    def set_gravity(self, g):
        self.f.set_gravity_grid(g)

    def marker(self):
        return self.f.grid(O.ARR_MARKER).copy()

    def residual(self):
        return self.f.grid(O.ARR_RESIDUAL).copy()


class CudaBackend:
    SCATTER = True

    def __init__(self, nparticles=8, dims=(N, N, N)):
        import blub_b200
        from blub_b200 import fluid as F
        self.F = F
        self.f = blub_b200.HybridFluid(*dims, nparticles)
        self.f.set_gravity_grid([0.0, 0.0, 0.0])
        self.f.set_transfer_path(self.SCATTER)
        self.vox = None

    def put(self, marker=None, u=None, p=None, which=0, vox=None):
        F = self.F
        if vox is not None:
            import torch
            self.vox = torch.from_numpy(np.ascontiguousarray(vox, dtype=np.float16)).to("cuda")  # kept alive: the fluid borrows it
            torch.cuda.synchronize()
            self.f.set_solid_voxels(self.vox.data_ptr())
        if marker is not None:
            self.f.upload_grid(F.TAP_MARKER, marker)
        if u is not None:
            for c, t in enumerate((F.TAP_UX, F.TAP_UY, F.TAP_UZ)):
                self.f.upload_grid(t, np.ascontiguousarray(u[c], dtype=np.float32))
        if p is not None:
            self.f.upload_grid(F.TAP_P_VEL if which == 0 else F.TAP_P_DEN, p)

    def particles(self, pos, rows=(None, None, None)):
        self.f.set_particles(pos, *rows)

    def run(self, a, b, dt=DT):
        self.f.step_stages(dt, a, b)

    def u(self):
        return [self.f.download_grid(t) for t in (self.F.TAP_UX, self.F.TAP_UY, self.F.TAP_UZ)]

    def positions(self, row=None):
        F = self.F
        return self.f.download_particles(F.TAP_POS if row is None else (F.TAP_VX, F.TAP_VY, F.TAP_VZ)[row])

    def set_gravity(self, g):
        self.f.set_gravity_grid(g)

    def marker(self):
        return self.f.download_grid(self.F.TAP_MARKER)

    def residual(self):
        return self.f.download_grid(self.F.TAP_RESIDUAL)


class CudaGatherBackend(CudaBackend):
    SCATTER = False


BACKENDS = [pytest.param(OracleBackend, id="oracle"), pytest.param(CudaBackend, id="cuda", marks=pytest.mark.gpu)]
# P2G: the oracle's gather and both transfer paths of the CUDA library
P2G_BACKENDS = BACKENDS + [pytest.param(CudaGatherBackend, id="cuda-gather", marks=pytest.mark.gpu)]


@pytest.mark.parametrize("backend", BACKENDS)
def test_divergence_of_a_linear_field_is_its_trace(backend):
    b, m = backend(), block_marker()
    b.put(marker=m, u=[face_field(c) for c in range(3)])
    b.run(1, 2)
    rhs = b.residual()[m == O.FLUID]
    assert np.abs(rhs - np.trace(A)).max() <= 2e-4  # differences of O(100) fp32 numbers


@pytest.mark.parametrize("backend", BACKENDS)
def test_projection_subtracts_the_pressure_gradient(backend):
    b, m = backend(), block_marker()
    b.put(marker=m, u=[np.full((N, N, N), B[c], dtype=np.float32) for c in range(3)], p=cell_pressure(), which=0)
    b.run(4, 5)
    u = b.u()
    for c in range(3):
        ff = fluid_fluid_faces(m, c)
        assert ff.sum() > 3000 and np.abs(u[c][ff] - (B[c] + K[c])).max() <= 1e-4
        # faces between the fluid and the AIR around it see p = 0 outside (free surface); faces touching no FLUID cell are zeroed -- within
        # one cell of the fluid (further away nobody reads them: the CUDA passes do not visit those cells, see tests/util.py:near_fluid)
        fl = m == O.FLUID
        touches = fl | np.roll(fl, -1, axis=2 - c)
        assert (u[c][~touches & near_fluid(m)] == 0).all()


@pytest.mark.parametrize("backend", BACKENDS)
def test_position_change_is_the_pressure_gradient_times_dt(backend):
    b, m = backend(), block_marker(lo=1, hi=24)  # the block touches the SOLID walls at 0
    b.put(marker=m, p=cell_pressure(), which=1)
    b.run(11, 12)
    u = b.u()
    for c in range(3):
        ff = fluid_fluid_faces(m, c)
        assert np.abs(u[c][ff] - np.float32(K[c]) * np.float32(DT)).max() <= 2e-6
        solid = (m == O.SOLID) | (np.roll(m, -1, axis=2 - c) == O.SOLID)
        assert (u[c][solid & near_fluid(m)] == 0).all()  # Neumann: nothing moves through a wall


@pytest.mark.parametrize("backend", BACKENDS)
def test_extrapolation_copies_a_constant_field_into_the_first_ring(backend):
    b, m = backend(), block_marker()
    fl = m == O.FLUID
    rng = np.random.default_rng(0)
    u = []
    for c in range(3):
        valid = fl | np.roll(fl, -1, axis=2 - c)
        f = rng.uniform(50, 60, (N, N, N)).astype(np.float32)  # garbage on the invalid faces
        f[valid] = np.float32(B[c])
        u.append(f)
    garbage = [f.copy() for f in u]
    b.put(marker=m, u=u)
    b.run(8, 9)  # set_boundary_marker: a no-op on this marker; on the CUDA path it also rebuilds the occupancy maps the extrapolation skips by
    b.run(5, 6)
    out = b.u()
    for c in range(3):
        valid = fl | np.roll(fl, -1, axis=2 - c)
        a1, a2 = [ax for ax in range(3) if ax != 2 - c]
        ring = np.zeros_like(valid)
        for d1 in (-1, 0, 1):
            for d2 in (-1, 0, 1):
                if d1 or d2:
                    ring |= np.roll(np.roll(valid, d1, axis=a1), d2, axis=a2)
        ring &= ~valid
        assert ring.sum() > 1000
        assert (out[c][ring] == np.float32(B[c])).all()          # averages of equal numbers
        assert (out[c][valid] == np.float32(B[c])).all()         # valid faces untouched
        rest = ~ring & ~valid
        assert np.array_equal(out[c][rest], garbage[c][rest])    # nothing else is written


@pytest.mark.parametrize("backend", BACKENDS)
def test_density_of_a_regular_lattice(backend):
    lo, hi = 6, 26
    pos = lattice_particles(lo, hi)
    b = backend(nparticles=pos.shape[0])
    b.particles(pos)
    # stages 6..9: clear, advect in a zero velocity field (positions unchanged, cells marked, lists rebuilt), boundary marker, density rhs
    b.put(u=[np.zeros((N, N, N), dtype=np.float32)] * 3)
    b.run(6, 10)
    m = b.marker()
    assert (m[lo:hi, lo:hi, lo:hi] == O.FLUID).all() and (m == O.FLUID).sum() == (hi - lo) ** 3
    rhs = b.residual()
    inner = rhs[lo + 1:hi - 1, lo + 1:hi - 1, lo + 1:hi - 1]
    assert np.abs(inner).max() <= 1e-4  # density exactly 8 up to fp32 rounding of 64 weights, divided by dt
    # a cell on a flat face of the block misses one layer of neighbours: density 8 - 2 (the far layer carries weight 0.25 per axis ->
    # 8 * (1 - 0.25 / 2) = 7), but an AIR neighbour clamps it back up to the rest density: rhs = 0 there as well
    face = rhs[lo + 2:hi - 2, lo + 2:hi - 2, lo]
    assert np.abs(face).max() <= 1e-4


# ---- solids inside the grid ------------------------------------------------------------------------------------------------------
# A FLUID block [10, 22)^3 wrapped in a two-cell SOLID shell [8, 24)^3 away from the border walls (velocity 0): every FLUID cell next to the
# shell has a SOLID neighbour on one, two or three sides.  Every shell cell carries its own solid velocity (fp16 values), so that a pass
# that reads the voxel of the wrong cell of a FLUID/SOLID face is seen.
SHELL_LO, SHELL_HI, FLUID_LO, FLUID_HI = 8, 24, 10, 22


def shell_marker_and_vox():
    m = block_marker(FLUID_LO, FLUID_HI)
    shell = np.zeros((N, N, N), dtype=bool)
    shell[SHELL_LO:SHELL_HI, SHELL_LO:SHELL_HI, SHELL_LO:SHELL_HI] = True
    shell &= m != O.FLUID
    m[shell] = O.SOLID
    rng = np.random.default_rng(11)
    vox = np.zeros((N, N, N, 4), dtype=np.float16)
    vox[shell, :3] = rng.uniform(-8.0, 8.0, (shell.sum(), 3)).astype(np.float16)
    vox[shell, 3] = 1.0
    return m, vox


def face_value_next_to_solid(m, vox, c):
    """The velocity a FLUID/SOLID face of component c must take: the SOLID cell's own voxel, on either side of the face (NaN elsewhere)."""
    v = vox[..., c].astype(np.float32)
    mn = np.roll(m, -1, axis=2 - c)
    vn = np.roll(v, -1, axis=2 - c)
    out = np.full(m.shape, np.nan, dtype=np.float32)
    lo = (m == O.SOLID) & (mn == O.FLUID)
    hi = (m == O.FLUID) & (mn == O.SOLID)
    out[lo] = v[lo]
    out[hi] = vn[hi]
    return out, lo, hi


@pytest.mark.parametrize("backend", BACKENDS)
def test_divergence_next_to_a_moving_solid(backend):
    m, vox = shell_marker_and_vox()
    # (1) a face field equal to the solid's velocity V everywhere: nothing flows through any FLUID cell's faces, rhs = 0 next to the solid too
    V = np.array([3.0, -5.0, 1.5], dtype=np.float32)
    uni = vox.copy()
    uni[m == O.SOLID, :3] = V.astype(np.float16)
    b = backend()
    b.put(marker=m, u=[np.full((N, N, N), V[c], dtype=np.float32) for c in range(3)], vox=uni)
    b.run(1, 2)
    fl = m == O.FLUID
    assert (b.residual()[fl] == 0).all()
    # (2) a linear field and a per-cell solid velocity: every face that has a SOLID cell on its far side counts with the solid's velocity
    # (divergence_compute.comp:28-86): rhs = sum_c (u_c(+face) - u_c(-face)) with a face next to SOLID replaced by that cell's voxel
    b = backend()
    u = [face_field(c) for c in range(3)]
    b.put(marker=m, u=u, vox=vox)
    b.run(1, 2)
    want = np.zeros((N, N, N))
    touching = np.zeros((N, N, N), dtype=bool)
    for c in range(3):
        ax = 2 - c
        v = vox[..., c].astype(np.float64)
        plus = np.where(np.roll(m, -1, axis=ax) == O.SOLID, np.roll(v, -1, axis=ax), u[c])
        minus = np.where(np.roll(m, 1, axis=ax) == O.SOLID, np.roll(v, 1, axis=ax), np.roll(u[c], 1, axis=ax))
        want += plus - minus
        touching |= (np.roll(m, -1, axis=ax) == O.SOLID) | (np.roll(m, 1, axis=ax) == O.SOLID)
    got = b.residual()
    assert (fl & touching).sum() == (FLUID_HI - FLUID_LO) ** 3 - (FLUID_HI - FLUID_LO - 2) ** 3  # the block's surface layer
    assert np.abs(got[fl] - want[fl]).max() <= 2e-4
    assert np.abs(want[fl & touching] - np.trace(A)).min() > 0.1  # the solid terms matter at every such cell


@pytest.mark.parametrize("backend", BACKENDS)
def test_projection_takes_the_velocity_of_the_solid_cell(backend):
    m, vox = shell_marker_and_vox()
    b = backend()
    b.put(marker=m, u=[np.full((N, N, N), B[c], dtype=np.float32) for c in range(3)], p=cell_pressure(), which=0, vox=vox)
    b.run(4, 5)
    u = b.u()
    for c in range(3):
        want, lo, hi = face_value_next_to_solid(m, vox, c)
        assert lo.sum() == hi.sum() == (FLUID_HI - FLUID_LO) ** 2
        assert np.array_equal(u[c][lo], want[lo]), f"solid on the - side, component {c}"
        assert np.array_equal(u[c][hi], want[hi]), f"solid on the + side, component {c}"
        ff = fluid_fluid_faces(m, c)
        assert np.abs(u[c][ff] - (B[c] + K[c])).max() <= 1e-4


@pytest.mark.parametrize("backend", BACKENDS)
def test_position_change_is_zero_next_to_an_interior_solid(backend):
    m, vox = shell_marker_and_vox()
    b = backend()
    b.put(marker=m, p=cell_pressure(), which=1, vox=vox)
    b.run(11, 12)
    u = b.u()
    for c in range(3):
        _, lo, hi = face_value_next_to_solid(m, vox, c)
        assert (u[c][lo | hi] == 0).all()
        ff = fluid_fluid_faces(m, c)
        assert ff.sum() > 1000 and np.abs(u[c][ff] - np.float32(K[c]) * np.float32(DT)).max() <= 2e-6


@pytest.mark.parametrize("backend", BACKENDS)
def test_density_of_a_lattice_against_solid_slabs(backend):
    """The 8-per-cell lattice of [6, 26)^3 with SOLID slabs (from the voxel volume, no particles inside) on its x = 5, y = 5 and z = 5 sides.  Per
    axis a cell collects 2 (both neighbour layers occupied) or 1.75 (one missing); each SOLID neighbour adds 0.5625
    (density_projection_gather_error.comp:99-199); an AIR neighbour clamps the density up to 8.  So a cell on one slab's face has
    rhs = (1 - 7.5625 / 8) / dt, on an edge (1 - (6.125 + 2 * 0.5625) / 8) / dt, in the corner (1 - (5.359375 + 3 * 0.5625) / 8) / dt."""
    lo, hi = 6, 26
    pos = lattice_particles(lo, hi)
    vox = np.zeros((N, N, N, 4), dtype=np.float16)
    s = slice(lo - 1, hi)
    vox[s, s, lo - 1] = (1.0, 2.0, -1.0, 1.0)
    vox[s, lo - 1, s] = (0.0, -3.0, 0.5, 1.0)
    vox[lo - 1, s, s] = (2.0, 0.0, 4.0, 1.0)
    b = backend(nparticles=pos.shape[0])
    b.particles(pos)
    b.put(u=[np.zeros((N, N, N), dtype=np.float32)] * 3, vox=vox)
    b.run(6, 10)
    m = b.marker()
    fl = m == O.FLUID
    assert fl.sum() == (hi - lo) ** 3 and (m[vox[..., 3] != 0] == O.SOLID).all()
    has = np.zeros((N, N, N), dtype=bool)
    has[lo:hi, lo:hi, lo:hi] = True
    dens = np.ones((N, N, N))
    nsolid = np.zeros((N, N, N))
    air = np.zeros((N, N, N), dtype=bool)
    for ax in range(3):
        dens *= 1.5 + 0.25 * np.roll(has, 1, axis=ax) + 0.25 * np.roll(has, -1, axis=ax)
        for sh in (1, -1):
            nsolid += np.roll(m, sh, axis=ax) == O.SOLID
            air |= np.roll(m, sh, axis=ax) == O.AIR
    dens += 0.5625 * nsolid
    dens = np.where(air, np.maximum(8.0, dens), dens)
    want = np.clip(1.0 - dens / 8.0, -0.5, 0.5) / DT
    rhs = b.residual()
    assert np.abs(rhs[fl] - want[fl]).max() <= 1e-4
    k = np.where(fl & ~air, nsolid, 0)
    counts = [int((k == j).sum()) for j in (1, 2, 3)]
    assert counts == [3 * (hi - lo - 2) ** 2, 3 * (hi - lo - 2), 1], counts  # faces, edges and the corner of the three slabs
    for j, d in ((1, 7.5625), (2, 7.25), (3, 7.046875)):
        assert np.abs(rhs[k == j] - (1.0 - d / 8.0) / DT).max() <= 1e-4
    assert np.abs(rhs[fl & (nsolid == 0)]).max() <= 1e-4


@pytest.mark.parametrize("backend", P2G_BACKENDS)
def test_p2g_zeroes_faces_with_a_solid_side(backend):
    """A lattice moving at a constant velocity b, with a SOLID slab from the voxel volume through its middle (particles inside it as well): every
    face the pass writes gets b + g dt -- except those with a SOLID side, which are exactly 0 (transfer_gather_velocity.comp:116-127)."""
    lo, hi = 6, 26
    pos = lattice_particles(lo, hi)
    bvel = np.array([2.5, -1.25, 0.75], dtype=np.float32)
    rows = [np.tile(np.array([0.0, 0.0, 0.0, bvel[c]], dtype=np.float32), (pos.shape[0], 1)) for c in range(3)]
    g = np.array([3.0, -981.0, 1.5], dtype=np.float32)
    vox = np.zeros((N, N, N, 4), dtype=np.float16)
    vox[8:20, 12:15, 10:24] = (4.0, -2.0, 1.0, 1.0)
    b = backend(nparticles=pos.shape[0])
    b.set_gravity(g)
    b.particles(pos, rows)
    b.put(vox=vox)
    b.run(0, 1)
    m = b.marker()
    solid = vox[..., 3] != 0
    has = np.zeros((N, N, N), dtype=bool)
    has[lo:hi, lo:hi, lo:hi] = True
    assert (m[solid] == O.SOLID).all() and np.array_equal(m == O.FLUID, has & ~solid)
    u = b.u()
    gdt = g * np.float32(DT)
    for c in range(3):
        written = fluid_adjacent_faces(m, c)
        side = (m == O.SOLID) | (np.roll(m, -1, axis=2 - c) == O.SOLID)
        assert (written & side).sum() >= 2 * 3 * 12  # both sides of the slab, on every axis
        assert (u[c][written & side] == 0).all(), f"component {c}: a face with a SOLID side is not 0"
        free = written & ~side
        assert free.sum() > 5000
        assert np.abs(u[c][free] - (bvel[c] + gdt[c])).max() <= 1e-5 * (abs(bvel[c]) + abs(gdt[c]))
