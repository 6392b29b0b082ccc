"""Helpers shared by the parity tests: build identical fluids on the oracle and on the CUDA library."""
import json
import os

import numpy as np

from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
SCENES = os.path.join(HERE, "golden", "scenes")
DT = O.DT_120HZ


def scene_path(name):
    return os.path.join(SCENES, name + ".json")


def oracle_from_scene(name):
    return O.fluid_from_scene(O.load_scene(scene_path(name)))


def grid_close(a, b, what, rel=1e-4, abs_=1e-5, mask=None):
    """SURVEY 8c: max|d| <= rel * max|field| + abs."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    if mask is not None:
        a, b = a[mask], b[mask]
    if a.size == 0:
        return 0.0
    scale = max(np.abs(a).max(), np.abs(b).max())
    err = np.abs(a - b).max()
    assert err <= rel * scale + abs_, f"{what}: max|d|={err:.3e} scale={scale:.3e} (tol {rel * scale + abs_:.3e})"
    return err


def fluid_adjacent_faces(marker, c):
    """Faces a P2G pass writes: face between a cell and its +c neighbour, at least one of them FLUID."""
    fl = marker == O.FLUID
    nb = np.zeros_like(fl)
    sl_src = [slice(None)] * 3
    sl_dst = [slice(None)] * 3
    ax = 2 - c  # arrays are [z, y, x]
    sl_src[ax] = slice(1, None)
    sl_dst[ax] = slice(0, -1)
    nb[tuple(sl_dst)] = fl[tuple(sl_src)]
    return fl | nb


def sort_rows(p):
    """Order-independent particle comparison: lexicographic sort by (cell key, x, y, z)."""
    p = np.asarray(p)
    key = np.lexsort((p[:, 2], p[:, 1], p[:, 0]))
    return p[key], key


def apply_A(m, x):
    """(A x) on FLUID cells of marker volume m (pressure.glsl:34-75), float64, via np.roll (border cells are never FLUID)."""
    fl = m == O.FLUID
    x = np.asarray(x, dtype=np.float64)
    out = np.zeros_like(x)
    diag = np.zeros_like(x)
    for ax in range(3):
        for sh in (1, -1):
            mm = np.roll(m, sh, axis=ax)
            diag += (mm != O.SOLID)
            out -= np.where(mm == O.FLUID, np.roll(x, sh, axis=ax), 0.0)
    return np.where(fl, out + diag * x, 0.0)


def markers_agree(m_o, m_g, what="marker", allowed=8):
    """Marker volumes after SEVERAL steps: a particle within round-off of a cell face may sit in the neighbouring cell in one of the two
    implementations, which flips an AIR/FLUID marker at the free surface.  Structural agreement = at most `allowed` such cells, and never a
    SOLID mismatch (solids do not depend on particles)."""
    bad = m_o != m_g
    assert not (bad & ((m_o == O.SOLID) | (m_g == O.SOLID))).any(), f"{what}: SOLID cells differ"
    assert int(bad.sum()) <= allowed, f"{what}: {int(bad.sum())} cells differ"
    return int(bad.sum())


def tight_solver(*fluids, tol=1e-4, max_it=128):
    """SURVEY 8(c): trajectory comparisons run both solves to convergence so that the iterate is well defined."""
    for f in fluids:
        f.set_solver_config(0, tol, max_it, 4)
        f.set_solver_config(1, tol, max_it, 4)


def dilate(mask):
    """mask dilated by one cell in every direction (Chebyshev), without wrap-around."""
    out = mask.copy()
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                src = [slice(max(0, -d), mask.shape[k] - max(0, d)) for k, d in enumerate((dz, dy, dx))]
                dst = [slice(max(0, d), mask.shape[k] - max(0, -d)) for k, d in enumerate((dz, dy, dx))]
                out[tuple(dst)] |= mask[tuple(src)]
    return out


def solid_contact(marker, vox, positions):
    """How much of a solid test actually reaches the fluid: (FLUID cells with a face neighbour that is SOLID because of the solid volume -- not a
    border wall -- and whose solid velocity is not zero, particles inside or within one cell of a solid voxel).  A solid test asserts a
    minimum of both, so that a geometry that misses the fluid cannot pass quietly.  vox: [nz, ny, nx, 4] (any float type)."""
    marker = np.asarray(marker)
    vox = np.asarray(vox, dtype=np.float32)
    solid = vox[..., 3] != 0
    interior = np.zeros_like(solid)
    interior[1:-1, 1:-1, 1:-1] = True
    moving = (marker == O.SOLID) & solid & interior & (vox[..., :3] != 0).any(axis=-1)
    fl = marker == O.FLUID
    touch = np.zeros_like(fl)
    for ax in range(3):
        for sh in (1, -1):
            nb = np.zeros_like(moving)
            src = [slice(None)] * 3
            dst = [slice(None)] * 3
            src[ax] = slice(max(0, sh), moving.shape[ax] + min(0, sh))
            dst[ax] = slice(max(0, -sh), moving.shape[ax] + min(0, -sh))
            nb[tuple(dst)] = moving[tuple(src)]  # nb[g] = moving[g + sh e_ax]
            touch |= nb
    c = np.floor(np.asarray(positions, dtype=np.float64)[:, :3]).astype(np.int64)
    for k, n in enumerate((marker.shape[2], marker.shape[1], marker.shape[0])):
        c[:, k] = np.clip(c[:, k], 0, n - 1)
    near = dilate(solid)
    return int((fl & touch).sum()), int(near[c[:, 2], c[:, 1], c[:, 0]].sum())


def near_fluid(marker):
    """Cells within one cell (Chebyshev) of a FLUID cell: the region the grid passes of the CUDA path visit.  Further away nothing reads the
    faces (P2G rewrites every face a particle can reach, extrapolation fills the one-cell ring G2P can reach) and the reference's P2G leaves
    them stale too (SURVEY B6), so grid fields are compared inside this region."""
    fl = marker == O.FLUID
    out = fl.copy()
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                sh = np.zeros_like(fl)
                src = [slice(max(0, -d), fl.shape[k] - max(0, d)) for k, d in enumerate((dz, dy, dx))]
                dst = [slice(max(0, d), fl.shape[k] - max(0, -d)) for k, d in enumerate((dz, dy, dx))]
                sh[tuple(dst)] = fl[tuple(src)]
                out |= sh
    return out
