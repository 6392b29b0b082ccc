"""Every branch advection and the density correction take at a solid (advect_particles.comp:45-173, density_projection_correct_particles.comp:
25-73), on hand-built inputs of a 40 x 24 x 32 grid: uploaded face velocities, marker and solid volume.  tests/advect_ref.py decides in float64
from the inputs which branch each particle must take; every class below must hold at least 8 particles.  Closed forms are asserted on both
implementations; the CUDA half then compares every particle's position and its four rows with the oracle's (max error 2e-4).

  still field (u = 0), isolated solid cells:  eaten along +-x, +-y, +-z; the exact ties |vx| = |vy| > |vz|, |vx| = |vz| > |vy|, |vy| = |vz| > |vx|
      and all three equal (the tie order of :45-64); a zero solid velocity (sign(0) = 0); a texel with w < 0 (SOLID in the marker, w != 0, but
      no wall for advection, w > 0); the same-cell push inside a thick block, and next to the grid edge where its smooth sample is clamped;
      particles on integer coordinates and on the 1.001 / n - 1.001 clamp planes
  outward field u = 10 (x - centre):  hits on each of the six wall clamps, voxel hits that end in another cell, steps of more than one cell
  correction:  hits on a SOLID marker cell, wall hits, no hit
"""
import numpy as np
import pytest

from oracle import oracle as O
from tests import advect_ref
from tests.test_stage_kat import CudaBackend, OracleBackend
from tests.util import DT

DIMS = (40, 24, 32)
NX, NY, NZ = DIMS
f32 = np.float32
OFFSETS = np.array([[a, b, c] for c in (0.25, 0.75) for b in (0.25, 0.75) for a in (0.25, 0.75)], dtype=f32)
# solid velocity of an isolated cell -> the axis and sign the particle is moved along
EATEN = {"+x": (3.0, 1.0, -0.5), "-x": (-3.0, 1.0, 0.5), "+y": (1.0, 3.0, -2.0), "-y": (0.5, -3.0, 2.0), "+z": (1.0, -2.0, 3.0), "-z": (-1.0, 2.0, -3.0),
         "tie xy": (2.0, -2.0, 1.0), "tie xz": (-2.0, 1.0, 2.0), "tie yz": (1.0, 2.0, -2.0), "tie xyz": (-2.0, 2.0, 2.0)}
EATEN_AXIS = {"+x": (0, 1), "-x": (0, -1), "+y": (1, 1), "-y": (1, -1), "+z": (2, 1), "-z": (2, -1),
              "tie xy": (1, -1), "tie xz": (2, 1), "tie yz": (2, -1), "tie xyz": (2, 1)}
CENTRE = np.array([20.0, 12.0, 16.0])


def cell_particles(cell, offsets=OFFSETS):
    return np.asarray(cell, dtype=f32) + offsets


def face_fields(fn):
    """u_c on the face positions (cell + 0.5, +0.5 on axis c), float32 [nz, ny, nx]."""
    z, y, x = np.meshgrid(np.arange(NZ), np.arange(NY), np.arange(NX), indexing="ij")
    out = []
    for c in range(3):
        q = [x + 0.5, y + 0.5, z + 0.5]
        q[c] = q[c] + 0.5
        out.append(fn(c, q).astype(f32))
    return out


def still_scene():
    """Zero velocity field; isolated eaten cells, a thick block, a block on the x = 0 edge, integer and clamp-plane particles.  Returns
    (u, vox, positions, labels)."""
    vox = np.zeros((NZ, NY, NX, 4), dtype=np.float16)
    pos, labels = [], []
    cells = [(4 + 3 * (k % 5), 4 + 4 * (k // 5), 5) for k in range(len(EATEN) + 2)]
    for (name, v), cell in zip(list(EATEN.items()) + [("zero", (0.0, 0.0, 0.0)), ("w<0", (4.0, 0.0, 0.0))], cells):
        vox[cell[2], cell[1], cell[0]] = v + ((-1.0,) if name == "w<0" else (1.0,))
        pos.append(cell_particles(cell))
        labels += [name] * 8
    vox[8:11, 8:11, 20:23] = (0.0, 0.0, 3.0, 1.0)  # thick block: eaten along +z into another solid cell of the block
    pos.append(cell_particles((21, 9, 9)))
    labels += ["block"] * 8
    vox[14:17, 14:17, 0:3] = (0.0, 3.0, 0.0, 1.0)  # on the x = 0 edge: eaten along +y, stays at x < 1.5
    pos.append(cell_particles((1, 15, 15), OFFSETS * f32([0.4, 1, 1]) + f32([0.0, 0, 0])))
    labels += ["edge"] * 8
    # integer coordinates: on the low x face of the "+x" cell (eaten: floor lands in it) and in free cells
    cx, cy, cz = cells[0]
    on = [(cx, cy + 0.25, cz + 0.5), (cx, cy + 0.75, cz + 0.5), (cx, cy + 0.5, cz + 0.25), (cx, cy + 0.5, cz + 0.75),
          (30.0, 20.0, 25.0), (31.0, 20.0, 25.0), (30.0, 21.0, 26.0), (33.0, 19.0, 27.0)]
    pos.append(np.array(on, dtype=f32))
    labels += ["integer"] * 8
    lo = f32(1.001)
    planes = [(lo, 18.5, 20.5), (f32(NX) - lo, 18.5, 20.5), (25.5, lo, 20.5), (25.5, f32(NY) - lo, 20.5), (25.5, 18.5, lo), (25.5, 18.5, f32(NZ) - lo),
              (lo, lo, 22.5), (f32(NX) - lo, f32(NY) - lo, f32(NZ) - lo)]
    pos.append(np.array(planes, dtype=f32))
    labels += ["plane"] * 8
    u = [np.zeros((NZ, NY, NX), dtype=f32) for _ in range(3)]
    return u, vox, np.concatenate(pos).astype(f32), np.array(labels)


def outward_scene(n=4000):
    """u = 10 (q - centre) per second: every particle moves away from the middle, across the wall clamps near the walls and into a solid slab
    at x = 30..31."""
    vox = np.zeros((NZ, NY, NX, 4), dtype=np.float16)
    vox[6:26, 6:18, 30:32] = (-2.0, 1.0, 0.5, 1.0)
    u = face_fields(lambda c, q: 10.0 * (q[c] - CENTRE[c]))
    rng = np.random.default_rng(21)
    pos = rng.uniform([1.05, 1.05, 1.05], [NX - 1.05, NY - 1.05, NZ - 1.05], (n, 3)).astype(f32)
    return u, vox, pos


def advect(backend_cls, u, vox, pos):
    b = backend_cls(nparticles=pos.shape[0], dims=DIMS)
    b.particles(np.c_[pos, np.zeros(pos.shape[0], f32)])
    b.put(u=u, vox=vox)
    b.run(6, 9)  # clear marker, advect, boundary marker
    return b.positions()[:, :3].copy(), [b.positions(k).copy() for k in range(3)], b.marker()


def compare_with_oracle(backend_cls, got, u, vox, pos):
    if backend_cls is OracleBackend:
        return
    want = advect(OracleBackend, u, vox, pos)
    assert np.abs(got[0].astype(np.float64) - want[0]).max() <= 2e-4
    for k in range(3):
        scale = np.maximum(1.0, np.abs(want[1][k].astype(np.float64)))
        assert (np.abs(got[1][k].astype(np.float64) - want[1][k]) / scale).max() <= 2e-4, f"row {k}"
    assert np.array_equal(got[2], want[2])


@pytest.mark.parametrize("backend", [pytest.param(OracleBackend, id="oracle"), pytest.param(CudaBackend, id="cuda", marks=pytest.mark.gpu)])
def test_advection_in_a_still_field(backend):
    u, vox, pos, labels = still_scene()
    br = advect_ref.advect(u, vox.astype(f32), pos, DT)
    for name, (axis, sign) in EATEN_AXIS.items():
        sel = labels == name
        assert sel.sum() >= 8 and br["eaten"][sel].all() and (br["axis"][sel] == axis).all() and (br["sign"][sel] == sign).all(), name
        assert not br["hit"][sel].any(), name
    sel = labels == "zero"
    assert sel.sum() >= 8 and br["eaten"][sel].all() and (br["sign"][sel] == 0).all() and br["push"][sel].all()
    sel = labels == "w<0"
    assert sel.sum() >= 8 and not br["eaten"][sel].any() and not br["hit"][sel].any() and (br["solid_w"][sel] < 0).all()
    assert (br["push"][labels == "block"]).sum() >= 8 and not br["edge_push"][labels == "block"].any()
    assert (br["edge_push"][labels == "edge"]).sum() >= 8
    assert (np.asarray(pos) == np.round(pos)).any(axis=1)[labels == "integer"].sum() >= 8
    assert br["eaten"][labels == "integer"].sum() >= 4
    assert (labels == "plane").sum() >= 8 and not br["hit"][labels == "plane"].any()
    got = advect(backend, u, vox, pos)
    x1, rows, marker = got
    # closed forms: in a still field an eaten particle whose shifted position is free ends at x0 +- e_k exactly; one that is not eaten stays
    free = ~br["hit"]
    assert np.array_equal(x1[free], br["x0"][free])
    eaten = br["eaten"] & free
    assert eaten.sum() >= 8 * len(EATEN)
    shift = np.zeros_like(pos)
    shift[np.nonzero(eaten)[0], br["axis"][eaten]] = br["sign"][eaten]
    assert np.array_equal(x1[eaten], (pos[eaten] + shift[eaten]).astype(f32))
    for k in range(3):
        assert (rows[k][free] == 0).all()
    # a pushed particle moves along -grad w, and never leaves the clamp box
    pushed = br["push"]
    assert (np.abs(x1[pushed] - br["x0"][pushed]).max(axis=1) > 0).all()
    assert (x1 >= f32(1.001)).all() and (x1 <= np.array([f32(s) - f32(1.001) for s in DIMS])).all()
    # the marker: SOLID wherever w != 0 -- the w < 0 texel as well -- FLUID in the cells the particles end in
    assert (marker[vox[..., 3] != 0] == O.SOLID).all()
    compare_with_oracle(backend, got, u, vox, pos)


@pytest.mark.parametrize("backend", [pytest.param(OracleBackend, id="oracle"), pytest.param(CudaBackend, id="cuda", marks=pytest.mark.gpu)])
def test_advection_in_an_outward_field(backend):
    u, vox, pos = outward_scene()
    br = advect_ref.advect(u, vox.astype(f32), pos, DT)
    lo, hi = advect_ref.clamp_planes(np.array(DIMS))
    x1 = br["x1"]
    for k in range(3):
        assert ((x1[:, k] < lo) & br["wall"]).sum() >= 8, f"low wall {k}"
        assert ((x1[:, k] > hi[k]) & br["wall"]).sum() >= 8, f"high wall {k}"
    into = br["voxel"] & ~br["push"] & ~br["eaten"]  # from a free cell into the slab
    assert into.sum() >= 8
    cfl = (np.abs(br["mv"]) > 1.0).any(axis=1)
    assert (cfl & ~br["hit"]).sum() >= 8 and (cfl & br["wall"]).sum() >= 8
    assert br["eaten"].sum() >= 8
    assert not br["near_plane"].any()  # no particle sits within round-off of a branch
    got = advect(backend, u, vox, pos)
    # closed form: a particle that hits nothing ends at x0 + mv
    free = ~br["hit"]
    assert np.abs(got[0][free] - x1[free]).max() <= 2e-4
    lo_hi = (got[0] >= lo) & (got[0] <= hi)
    assert lo_hi.all()
    compare_with_oracle(backend, got, u, vox, pos)


@pytest.mark.parametrize("backend", [pytest.param(OracleBackend, id="oracle"), pytest.param(CudaBackend, id="cuda", marks=pytest.mark.gpu)])
def test_correction_hits(backend):
    marker = np.full((NZ, NY, NX), O.FLUID, dtype=np.int8)
    marker[0], marker[-1], marker[:, 0], marker[:, -1], marker[:, :, 0], marker[:, :, -1] = 0, 0, 0, 0, 0, 0
    marker[6:26, 6:18, 30:32] = O.SOLID
    u = face_fields(lambda c, q: 0.1 * (q[c] - CENTRE[c]))  # displacements in cells
    rng = np.random.default_rng(22)
    pos = rng.uniform([1.05, 1.05, 1.05], [NX - 1.05, NY - 1.05, NZ - 1.05], (4000, 3)).astype(f32)
    pos = pos[marker[np.floor(pos[:, 2]).astype(int), np.floor(pos[:, 1]).astype(int), np.floor(pos[:, 0]).astype(int)] != O.SOLID]
    br = advect_ref.correct(u, marker, pos)
    assert br["marker"].sum() >= 8 and br["wall"].sum() >= 8 and (~br["hit"]).sum() >= 8
    assert not br["near_plane"].any()

    def run(cls):
        b = cls(nparticles=pos.shape[0], dims=DIMS)
        b.particles(np.c_[pos, np.zeros(pos.shape[0], f32)])
        b.put(marker=marker, u=u)
        b.run(13, 14)
        return b.positions()[:, :3].copy()

    x1 = run(backend)
    free = ~br["hit"]
    assert np.abs(x1[free] - br["x1"][free]).max() <= 2e-5  # no hit: x0 + the trilinear displacement
    # a hit cuts the step short of the restated end point (to the cell-face distance of :48-70, which is measured to the face BEHIND the
    # particle along a positive direction, as written)
    hit = br["hit"]
    assert (np.abs(x1[hit] - pos[hit]).max(axis=1) < np.abs(br["x1"][hit] - pos[hit]).max(axis=1)).all()
    lo, hi = advect_ref.clamp_planes(np.array(DIMS))
    assert ((x1 >= lo) & (x1 <= hi)).all()
    if backend is not OracleBackend:
        assert np.abs(x1.astype(np.float64) - run(OracleBackend)).max() <= 2e-4
